/* Plain-C restatement of DeNovoModel's re-scoring, recalculate_log_probability (core/models/mutation/denovo_model.cpp:199-218), for
 * one alignment given as CIGAR text ('=', 'X', 'I', 'D' runs as make_cigar merges them) and the given haplotype's context model as
 * per-base repeat-table cells with the table logp[cell][k] = logf(calculate_indel_probability) of an indel of length k + 1
 * (indel_mutation_model.cpp:114-123). Compiled by the tests with -ffp-contract=off: every double operation rounds on its own. */
#include <stdint.h>

/* Returns 0 (value in *out) or 5 when an indel starts at pos >= glen (the reference reads past its model). */
int oracle_recalculate(const char* cigar, const int32_t* cell, int64_t glen, const float* logp, int32_t X, double snv_log_prior, double* out)
{
    double result = 0.0;
    int64_t pos = 0;
    uint64_t size = 0;
    for (const char* c = cigar; *c; ++c) {
        if (*c >= '0' && *c <= '9') { size = size * 10u + (uint64_t)(*c - '0'); continue; }
        if (*c == 'X') {
            result += (double)size * snv_log_prior;
            pos += (int64_t)size;
        } else if (*c == 'I' || *c == 'D') {
            if (pos >= glen) return 5;
            const uint64_t k = (size < (uint64_t)X ? size : (uint64_t)X) - 1;
            result += (double)logp[(int64_t)cell[pos] * X + (int64_t)k];
            if (*c == 'D') pos += (int64_t)size;
        } else {
            pos += (int64_t)size;
        }
        size = 0;
    }
    *out = result;
    return 0;
}

/* n alignments: cigar j at cigars + j * stride against given haplotype given[j] of the block (off[], cells over the block). */
void oracle_recalculate_batch(int64_t n, const char* cigars, int32_t stride, const int32_t* given, const int64_t* off, const int32_t* cell,
                              const float* logp, int32_t X, double snv_log_prior, double* out, int32_t* status)
{
    for (int64_t j = 0; j < n; ++j) {
        const int64_t g0 = off[given[j]];
        status[j] = oracle_recalculate(cigars + j * stride, cell + g0, off[given[j] + 1] - g0, logp, X, snv_log_prior, out + j);
    }
}
