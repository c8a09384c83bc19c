/* TEST INFRASTRUCTURE ONLY.
 *
 * Plain-C, scalar restatement of the reference's pair-HMM haplotype-likelihood path (octopus v0.7.4).
 * It exists to CHECK the CUDA engine (tests/, __graft_entry__.smoke(), bench.py's cpu_baseline leg); it is
 * never linked into, imported by, or called from the product path (octopus_b200/).
 *
 * Parity status: PINNED. oracle_align / oracle_align_tb reproduce every known-answer test the reference
 * holds for this path (tests/golden/pair_hmm_kats.json, extracted from test/unit/core/models/pair_hmm_tests.cpp)
 * and agree with the reference's own SIMD kernel compiled here (oracle/_ref, ref_driver.cpp) on seeded fuzz
 * (tests/test_oracle.py). Above the raw kernel the reference has no tests; oracle_evaluate (naive shortcut, window
 * placement, flank discount, lowest()), the single-position align + CIGAR, the band rounding, oracle_kmer_map and
 * oracle_model_evaluate / oracle_model_align (in-range rule, max over mapping positions, fallback shift,
 * ShortHaplotypeError, mapping-quality mixing) are pinned to the reference's OWN code — pair_hmm.hpp,
 * simd_pair_hmm_wrapper.hpp, utils/kmer_mapper.hpp and haplotype_likelihood_model.cpp compiled from /root/reference behind
 * oracle/ref_hmm_driver.cpp — on seeded fuzz (tests/test_oracle.py); oracle_populate equals the compiled
 * HaplotypeLikelihoodArray::populate (haplotype_likelihood_array.cpp, ReadMap and TemplateMap overloads) on random regions.
 *
 * Coordinates: cell (x, y) = x truth-window bases and y target (read) bases consumed; the band is
 * 0 <= x - y <= 2*band - 1; W = truth_len = target_len + 2*band - 1. The reference walks the same cells along
 * anti-diagonals s = x + y with lane i = (x - y) / 2 (simd_pair_hmm.hpp:271-321); this file walks them row by row.
 * State values are kept as the reference keeps them: (score << 2) | label, label = M 0, I 1, D 3
 * (simd_pair_hmm.hpp:57,63-65). In the score-only variant labels are never set (update_traceback is a no-op,
 * :163), so comparisons are on pure scores; in the traceback variant they take part in every min (:147-162).
 */
#include "phmm_oracle.h"

#include <math.h>
#include <stdio.h>
#include <stdlib.h>
#include <string.h>

#define TRACE_BITS 2
#define INF_SCORE (1 << 26)
#define INFP (INF_SCORE << TRACE_BITS)
#define LAB_M 0
#define LAB_I 1
#define LAB_D 3
#define N_SCORE 2 /* simd_pair_hmm.hpp:58 n_score_ = 2 << trace_bits_ */

static const double LN10_DIV_10 = 0.230258509299404568401799145468436420760110148862877297603; /* utils/maths.hpp:41 */

static inline int imin(int a, int b) { return a < b ? a : b; }

static inline int m_gap_open(const oracle_model* m, int x) { return m->gap_open ? m->gap_open[x] : (int8_t)m->gap_open_scalar; }
static inline int m_gap_extend(const oracle_model* m, int x) { return m->gap_extend ? m->gap_extend[x] : (int8_t)m->gap_extend_scalar; }

/* simd_pair_hmm.hpp:121-142 update_match_state, one lane. Returns the substitution cost (phred, unshifted). */
static inline int sub_cost(const char* truth, const char* target, const int8_t* quals, const oracle_model* m, int x, int y)
{
    if (target[y] == truth[x]) return 0;
    int q = quals[y];
    if (m->snv_mask && m->snv_mask[x] == target[y]) q = imin(q, m->snv_prior[x]);
    const int ncost = truth[x] == 'N' ? N_SCORE : INF_SCORE;
    return imin(q, ncost);
}

/* simd_pair_hmm.hpp:240-324 align_helper (both instantiations) + :165-231 set_alignments. */
static int align_impl(int band, const char* truth, const char* target, const int8_t* quals,
                      int truth_len, int target_len, const oracle_model* m,
                      int tb, int* first_pos, char* align1, char* align2)
{
    const int L = target_len, W = truth_len, K = 2 * band;
    if (L <= 0 || W != L + K - 1) { if (tb && first_pos) *first_pos = -1; return -1; }
    const size_t ncell = (size_t)(L + 1) * (size_t)K;
    int* M = (int*)malloc(3 * ncell * sizeof(int));
    int* I = M + ncell;
    int* D = I + ncell;
    unsigned char* bp = tb ? (unsigned char*)calloc(3 * ncell, 1) : NULL; /* [state][cell] predecessor labels */
    for (size_t c = 0; c < ncell; ++c) { M[c] = INFP | (tb ? LAB_M : 0); I[c] = INFP | (tb ? LAB_I : 0); D[c] = INFP | (tb ? LAB_D : 0); }
    const int nuc = m->nuc_prior << TRACE_BITS;
    int best = INFP + (1 << 20), best_x = -1;
    for (int y = 0; y <= L; ++y) {
        for (int k = 0; k < K; ++k) {
            const int x = y + k;
            const size_t c = (size_t)y * K + k;
            int mm = M[c];
            const int ii = I[c], dd = D[c];
            int mg;
            if (y == 0) {
                /* rolling initializer (rolling_initializer.hpp:39-51; simd_pair_hmm.hpp:282-283): the match state of
                 * (x, 0) is the zero score for x < 2*band. The gap transitions out of (x, 0) were computed one half-step
                 * before m1 was initialised when x is even (:317-319 use the un-initialised _m1), so they see infinity there. */
                mm = 0;
                mg = (x & 1) ? 0 : INFP;
            } else {
                mg = mm;
            }
            const int S = imin(mm, imin(ii, dd)); /* :284 / :308 */
            if (y == L) { /* :285-291, :309-315 strict '<' in anti-diagonal order == ascending x on row L */
                if (S < best) { best = S; best_x = x; }
            }
            if (x < W) {
                if (y < L) { /* match / mismatch → (x+1, y+1), same k */
                    const size_t cn = c + K;
                    const int v = S + (sub_cost(truth, target, quals, m, x, y) << TRACE_BITS);
                    if (tb) { bp[0 * ncell + cn] = (unsigned char)(v & 3); M[cn] = (v & ~3) | LAB_M; } else M[cn] = v;
                }
                if (k + 1 < K) { /* deletion → (x+1, y): :293-294 / :317, I→D allowed */
                    const size_t cn = c + 1;
                    const int v = imin(dd + (m_gap_extend(m, x) << TRACE_BITS), imin(mg, ii) + (m_gap_open(m, x) << TRACE_BITS));
                    if (tb) { bp[2 * ncell + cn] = (unsigned char)(v & 3); D[cn] = (v & ~3) | LAB_D; } else D[cn] = v;
                }
            }
            if (k >= 1 && y < L) { /* insertion → (x, y+1): :295 / :318-319, penalties indexed at x-1, no D→I */
                const size_t cn = c + K - 1;
                const int v = imin(ii + (m_gap_extend(m, x - 1) << TRACE_BITS), mg + (m_gap_open(m, x - 1) << TRACE_BITS)) + nuc;
                if (tb) { bp[1 * ncell + cn] = (unsigned char)(v & 3); I[cn] = (v & ~3) | LAB_I; } else I[cn] = v;
            }
        }
    }
    const int score = best >> TRACE_BITS; /* :323 */
    if (tb) {
        /* :165-231 set_alignments, in (x, y) coordinates */
        if (best_x < 0) {
            *first_pos = -1;
        } else {
            int x = best_x, y = L, n = 0;
            int state = best & 3;
            while (y > 0) {
                const size_t c = (size_t)y * K + (x - y);
                int ns;
                if (state == LAB_M) {
                    ns = bp[0 * ncell + c]; align1[n] = truth[--x]; align2[n] = target[--y];
                } else if (state == LAB_I) {
                    ns = bp[1 * ncell + c]; align1[n] = '-'; align2[n] = target[--y];
                } else {
                    ns = bp[2 * ncell + c]; align1[n] = truth[--x]; align2[n] = '-';
                }
                state = ns;
                ++n;
                if (x < y || x - y >= K) { n = -1; break; } /* left the band: overflow in the reference (:195-199) */
            }
            if (n < 0) {
                *first_pos = -1;
            } else {
                align1[n] = 0; align2[n] = 0;
                *first_pos = x;
                for (int a = 0, b = n - 1; a < b; ++a, --b) {
                    char t = align1[a]; align1[a] = align1[b]; align1[b] = t;
                    t = align2[a]; align2[a] = align2[b]; align2[b] = t;
                }
            }
        }
        free(bp);
    }
    free(M);
    return score;
}

int oracle_align(int band, const char* truth, const char* target, const int8_t* quals,
                 int truth_len, int target_len, const oracle_model* m)
{
    return align_impl(band, truth, target, quals, truth_len, target_len, m, 0, NULL, NULL, NULL);
}

int oracle_align_tb(int band, const char* truth, const char* target, const int8_t* quals,
                    int truth_len, int target_len, const oracle_model* m,
                    int* first_pos, char* align1, char* align2)
{
    return align_impl(band, truth, target, quals, truth_len, target_len, m, 1, first_pos, align1, align2);
}

/* simd_pair_hmm.hpp:352-430 calculate_flank_score_helper */
int oracle_flank_score(int truth_len, int lhs_flank, int rhs_flank, const char* target, const int8_t* quals,
                       const oracle_model* m, int first_pos, const char* align1, const char* align2,
                       int* target_mask_size)
{
    enum { ST_M, ST_I, ST_D };
    int prev = ST_M, truth_idx = first_pos, target_idx = 0, result = 0, mask = 0;
    const int rhs_begin = truth_len - rhs_flank;
    for (int a = 0; align1[a]; ++a) {
        int st = ST_M;
        if (align1[a] == '-') st = ST_I; else if (align2[a] == '-') st = ST_D;
        const int in_flank = truth_idx < lhs_flank || truth_idx >= rhs_begin;
        if (st == ST_M) {
            if (in_flank) {
                if (align1[a] != align2[a]) {
                    if (align1[a] != 'N') {
                        /* :326-345 get_mismatch_quality: std::min(int8, int8) */
                        int q = quals[target_idx];
                        if (m->snv_mask && m->snv_mask[truth_idx] == target[target_idx]) q = imin(q, m->snv_prior[truth_idx]);
                        result += q;
                    } else {
                        result += N_SCORE;
                    }
                }
                ++mask;
            }
            ++truth_idx; ++target_idx;
        } else if (st == ST_I) {
            if (in_flank) {
                result += (prev == ST_I ? m_gap_extend(m, truth_idx - 1) : m_gap_open(m, truth_idx - 1)) + m->nuc_prior;
                ++mask;
            }
            ++target_idx;
        } else {
            if (in_flank) result += prev == ST_D ? m_gap_extend(m, truth_idx) : m_gap_open(m, truth_idx);
            ++truth_idx;
        }
        prev = st;
    }
    *target_mask_size = mask;
    return result;
}

/* pair_hmm.hpp:206-214 is_in_flank */
static inline int in_flank_abs(int idx, int truth_len, int lhs, int rhs) { return idx < lhs || idx >= truth_len - rhs; }

/* pair_hmm.hpp:275-319 try_naive_evaluate */
int oracle_try_naive_evaluate(const char* truth, int truth_len, const char* target, const uint8_t* quals, int target_len,
                              int target_offset, const oracle_model* m, int use_flanks, int lhs_flank, int rhs_flank,
                              int* phred)
{
    const char* t = truth + target_offset;
    int i = 0;
    while (i < target_len && target[i] == t[i]) ++i;
    if (i == target_len) { *phred = 0; return 1; }
    int j = i + 1;
    while (j < target_len && target[j] == t[j]) ++j;
    if (j != target_len) return 0; /* two or more mismatches */
    const int tidx = i + target_offset;
    if (use_flanks && in_flank_abs(tidx, truth_len, lhs_flank, rhs_flank)) { *phred = 0; return 1; }
    unsigned mp = quals[i]; /* :240-273 get_mismatch_penalty: std::min(uint8, (uint8)prior) */
    if (m->snv_mask && m->snv_mask[tidx] == target[i]) {
        const unsigned cap = (uint8_t)m->snv_prior[tidx];
        if (cap < mp) mp = cap;
    }
    const int go = m_gap_open(m, tidx);
    if ((int)mp <= go) { *phred = (int)mp; return 1; }
    /* target[i+1..) == truth[tidx..)  : one-base deletion from the read explains it (:305-308) */
    int eq = 1;
    for (int a = i + 1; a < target_len; ++a) if (target[a] != truth[tidx + (a - i - 1)]) { eq = 0; break; }
    if (eq) { *phred = go; return 1; }
    /* target[i..) == truth[tidx+1..)  : one-base insertion (:309-312) */
    eq = 1;
    for (int a = i; a < target_len; ++a) if (target[a] != truth[tidx + 1 + (a - i)]) { eq = 0; break; }
    if (eq) { *phred = go; return 1; }
    if ((int)mp <= go + m_gap_extend(m, tidx)) { *phred = (int)mp; return 1; }
    return 0;
}

static oracle_model offset_model(const oracle_model* m, int a)
{
    oracle_model o = *m;
    if (o.snv_mask) { o.snv_mask += a; o.snv_prior += a; }
    if (o.gap_open) o.gap_open += a;
    if (o.gap_extend) o.gap_extend += a;
    return o;
}

/* pair_hmm.hpp:827-841 evaluate → :275-319 shortcut, :694-782 simd_evaluate_helper */
double oracle_evaluate(int band, const char* truth, int truth_len, const char* target, const uint8_t* quals, int target_len,
                       int target_offset, const oracle_model* m, int use_flanks, int lhs_flank, int rhs_flank,
                       int dp_only, int* used_dp, int* raw_score)
{
    if (used_dp) *used_dp = 0;
    if (raw_score) *raw_score = 0;
    if (!dp_only) {
        int phred;
        if (oracle_try_naive_evaluate(truth, truth_len, target, quals, target_len, target_offset, m, use_flanks, lhs_flank, rhs_flank, &phred)) {
            if (raw_score) *raw_score = phred;
            return -LN10_DIV_10 * (double)phred; /* :286 ln_probability_table[i] = -ln10Div10 * i */
        }
    }
    const int W = target_len + 2 * band - 1;
    const int a = target_offset - band > 0 ? target_offset - band : 0; /* :711 / :735 */
    if (a + W > truth_len) return ORACLE_LOWEST;                       /* :712-714 / :736-738 */
    const oracle_model om = offset_model(m, a);
    const int8_t* q8 = (const int8_t*)quals;                           /* :372 reinterpret_cast */
    /* :123-130 target_overlaps_truth_flank (size_t arithmetic: all operands non-negative here) */
    const int near_flank = use_flanks && (target_offset < lhs_flank + band || target_offset + target_len + band > truth_len - rhs_flank);
    if (!near_flank) {
        const int score = oracle_align(band, truth + a, target, q8, W, target_len, &om);
        if (used_dp) *used_dp = 1;
        if (raw_score) *raw_score = score;
        return -LN10_DIV_10 * (double)score;
    }
    const int n = 2 * (target_len + band) + 1;
    char* a1 = (char*)calloc((size_t)n + 1, 1);
    char* a2 = (char*)calloc((size_t)n + 1, 1);
    int first_pos = 0;
    const int score = oracle_align_tb(band, truth + a, target, q8, W, target_len, &om, &first_pos, a1, a2);
    if (used_dp) *used_dp = 2;
    if (raw_score) *raw_score = score;
    double result;
    if (first_pos == -1) {
        result = ORACLE_LOWEST; /* :750-752 */
    } else {
        /* :573-588 flank sizes in window coordinates */
        int lhs = lhs_flank < a ? 0 : lhs_flank - a;
        int rhs;
        if (a + W < truth_len - rhs_flank) rhs = 0;
        else { rhs = rhs_flank + a + W - truth_len; if (rhs < 0) rhs = 0; }
        int mask_size = 0;
        int flank = oracle_flank_score(W, lhs, rhs, target, q8, &om, first_pos, a1, a2, &mask_size);
        if (target_len - mask_size < 2) flank = 0; /* :757-759 min_explained_bases */
        if (flank <= score) result = -LN10_DIV_10 * (double)(score - flank);
        else result = -LN10_DIV_10 * (double)(flank + score); /* :760-764 "overflow" branch */
    }
    free(a1); free(a2);
    return result;
}

/* haplotype_likelihood_model.cpp:187-201 num_out_of_range_bases (required_pad = band, pair_hmm.hpp:33-38) */
static int num_out_of_range_bases(int64_t pos, int read_len, int hap_len, int band)
{
    if (pos < band) return (int)(band - pos);
    const int64_t end = pos + read_len + band;
    if (end > hap_len) return (int)((int64_t)hap_len - end);
    return 0;
}

/* utils/maths.hpp:294-298 */
static double log_sum_exp2(double a, double b)
{
    const double lo = b < a ? b : a, hi = b < a ? a : b;
    return hi + log1p(exp(lo - hi));
}

/* haplotype_likelihood_model.cpp:211-259 max_score + :261-304 evaluate */
int oracle_model_evaluate(int band, const char* hap, int hap_len, const char* read, const uint8_t* quals, int read_len,
                          const oracle_model* m, int use_flanks, int lhs_flank, int rhs_flank,
                          const int64_t* positions, int n_positions, int64_t original_pos,
                          int use_mapping_quality, int mapping_quality, int mapq_cap, int mapq_cap_trigger,
                          int dp_only, double* out, int* required_extension)
{
    double best = ORACLE_LOWEST;
    int original_mapped = 0, has_in_range = 0;
    for (int p = 0; p < n_positions; ++p) {
        if (positions[p] == original_pos) original_mapped = 1;
        if (num_out_of_range_bases(positions[p], read_len, hap_len, band) == 0) {
            has_in_range = 1;
            const double v = oracle_evaluate(band, hap, hap_len, read, quals, read_len, (int)positions[p], m, use_flanks, lhs_flank, rhs_flank, dp_only, NULL, NULL);
            if (v > best) best = v;
        }
    }
    if (!original_mapped && num_out_of_range_bases(original_pos, read_len, hap_len, band) == 0) {
        has_in_range = 1;
        const double v = oracle_evaluate(band, hap, hap_len, read, quals, read_len, (int)original_pos, m, use_flanks, lhs_flank, rhs_flank, dp_only, NULL, NULL);
        if (v > best) best = v;
    }
    if (!has_in_range) {
        const int min_shift = num_out_of_range_bases(original_pos, read_len, hap_len, band);
        int64_t fin = original_pos;
        if (min_shift > 0) {
            fin += min_shift;
            if (num_out_of_range_bases(fin, read_len, hap_len, band) != 0) { *required_extension = min_shift; return 1; }
        } else {
            const unsigned left = (unsigned)(-min_shift);
            if (original_pos >= (int64_t)left) fin -= left;
            else { *required_extension = (int)(left - original_pos); return 1; }
        }
        best = oracle_evaluate(band, hap, hap_len, read, quals, read_len, (int)fin, m, use_flanks, lhs_flank, rhs_flank, dp_only, NULL, NULL);
    }
    if (use_mapping_quality) {
        int mq = mapping_quality;
        /* set(config) / the constructor drop a trigger that is >= the cap (haplotype_likelihood_model.cpp:49-51, 117-119) */
        if (mapq_cap_trigger >= 0 && mapq_cap_trigger < mapq_cap && mq >= mapq_cap_trigger) mq = mapq_cap;
        const double ln_miss = -LN10_DIV_10 * (double)mq;
        const double ln_mapped = log(1.0 - exp(ln_miss));
        const double r = log_sum_exp2(ln_mapped + best, ln_miss);
        *out = r > -1e-15 ? 0.0 : r;
    } else {
        *out = best > -1e-15 ? 0.0 : best;
    }
    return 0;
}

/* utils/kmer_mapper.hpp:24-41 perfect_hash (A 0, C 1, G 2, T 3, anything else 0), :43-53 perfect_kmer_hash<6> */
static inline unsigned base_hash(char b) { return b == 'C' ? 1u : b == 'G' ? 2u : b == 'T' ? 3u : 0u; }
static inline unsigned kmer6(const char* s)
{
    unsigned h = 0, k = 1;
    for (int i = 0; i < 6; ++i) { h += k * base_hash(s[i]); k *= 4; }
    return h;
}

/* utils/kmer_mapper.hpp:57-69, :85-98, :120-159 */
int oracle_kmer_map(const char* query, int query_len, const char* target, int target_len,
                    int max_positions, int64_t* out_positions)
{
    enum { K = 6, NK = 4096 };
    if (query_len < K || target_len < K || max_positions <= 0) return 0;
    const int nq = query_len - K + 1, nt = target_len - K + 1;
    /* hash table as CSR: bin → ascending target indices (push_back order, :94-96) */
    int* bin_start = (int*)calloc(NK + 1, sizeof(int));
    int* items = (int*)malloc((size_t)nt * sizeof(int));
    unsigned* th = (unsigned*)malloc((size_t)nt * sizeof(unsigned));
    for (int i = 0; i < nt; ++i) { th[i] = kmer6(target + i); ++bin_start[th[i] + 1]; }
    for (int b = 0; b < NK; ++b) bin_start[b + 1] += bin_start[b];
    int* fill = (int*)malloc(NK * sizeof(int));
    memcpy(fill, bin_start, NK * sizeof(int));
    for (int i = 0; i < nt; ++i) items[fill[th[i]]++] = i;
    unsigned* counts = (unsigned*)calloc((size_t)nt, sizeof(unsigned));
    unsigned max_hit = 0, num_max = 0;
    int64_t first_max = 0;
    for (int qi = 0; qi < nq; ++qi) {
        const unsigned h = kmer6(query + qi);
        for (int e = bin_start[h]; e < bin_start[h + 1]; ++e) {
            const int ti = items[e];
            if (ti >= qi) {
                const int mb = ti - qi;
                if (++counts[mb] > max_hit) { max_hit = counts[mb]; first_max = mb; num_max = 1; }
                else if (counts[mb] == max_hit) { ++num_max; if (mb < first_max) first_max = mb; }
            }
        }
    }
    int n = 0;
    if (max_hit > 0) {
        out_positions[n++] = first_max++;
        --num_max; --max_positions;
        while (max_positions > 0 && num_max > 0 && first_max < nt) {
            if (counts[first_max] == max_hit) { out_positions[n++] = first_max; --num_max; --max_positions; }
            ++first_max;
        }
    }
    free(bin_start); free(items); free(th); free(fill); free(counts);
    return n;
}

/* haplotype_likelihood_array.cpp:51-103 populate(ReadMap) for one sample: the H x R loop (haplotype outer, read inner),
 * with the candidate mapping positions supplied as a CSR over [H][R] pairs (pos_off == NULL: none listed) instead of
 * being produced by the k-mer mapper inline (:89-92) — or, with pos_off == NULL and map_positions != 0, by oracle_kmer_map. Writes out[h*R + r]; status[h*R + r] = 0 ok,
 * 2 | ext << 16 for ShortHaplotypeError (the reference throws on the first one; this loop records all and returns 1). */
int oracle_populate(int band, int H, const int64_t* hap_off, const char* seq,
                    const char* mask_f, const int8_t* prior_f, const char* mask_r, const int8_t* prior_r,
                    const int8_t* gap_open, const int8_t* gap_extend, const int64_t* hap_begin,
                    int R, const int64_t* read_off, const char* bases, const uint8_t* quals,
                    const uint8_t* mapq, const uint8_t* reverse, const int64_t* read_begin,
                    const int64_t* pos_off, const int32_t* pos,
                    int use_flanks, int lhs_flank, int rhs_flank,
                    int use_mapping_quality, int mapq_cap, int mapq_cap_trigger, int nuc_prior, int dp_only, int map_positions,
                    double* out, int32_t* status)
{
    int any_short = 0;
    int64_t tmp[64];
    for (int h = 0; h < H; ++h) {
        const int64_t ho = hap_off[h];
        const int hl = (int)(hap_off[h + 1] - ho);
        for (int r = 0; r < R; ++r) {
            const int64_t ro = read_off[r];
            const int rl = (int)(read_off[r + 1] - ro);
            const int rev = reverse ? reverse[r] : 0;
            oracle_model m;
            m.snv_mask = (rev ? mask_r : mask_f) + ho;
            m.snv_prior = (rev ? prior_r : prior_f) + ho;
            m.gap_open = gap_open + ho;
            m.gap_extend = gap_extend + ho;
            m.gap_open_scalar = 0; m.gap_extend_scalar = 0; m.nuc_prior = nuc_prior;
            int np = 0;
            if (pos_off) {
                const int64_t a = pos_off[(int64_t)h * R + r], b = pos_off[(int64_t)h * R + r + 1];
                for (int64_t i = a; i < b && np < 64; ++i) tmp[np++] = pos[i];
            } else if (map_positions) {
                /* :89-92 map_query_to_target(read_hashes, haplotype_hashes, counts, first, maxMappingPositions = 10) */
                np = oracle_kmer_map(bases + ro, rl, seq + ho, hl, 10, tmp);
            }
            const int64_t orig = (read_begin ? read_begin[r] : 0) - (hap_begin ? hap_begin[h] : 0);
            double v = 0; int ext = 0;
            const int st = oracle_model_evaluate(band, seq + ho, hl, bases + ro, quals + ro, rl, &m, use_flanks, lhs_flank, rhs_flank,
                                                 tmp, np, orig, use_mapping_quality, mapq ? mapq[r] : 60, mapq_cap, mapq_cap_trigger,
                                                 dp_only, &v, &ext);
            out[(int64_t)h * R + r] = st ? ORACLE_LOWEST : v;
            if (status) status[(int64_t)h * R + r] = st ? (2 | (ext << 16)) : 0;
            any_short |= st;
        }
    }
    return any_short;
}

/* pair_hmm.hpp:152-188 make_cigar: "=" sequence match, "X" substitution, "I" insertion (align1 == '-'), "D" deletion. */
static int make_cigar_text(const char* a1, const char* a2, char* out, int cap)
{
    int n = (int)strlen(a1), i = 0, w = 0;
    while (i < n) {
        int j = i;
        while (j < n && a1[j] == a2[j]) ++j;
        if (j != i) { w += snprintf(out + w, cap - w, "%d=", j - i); if (j == n) break; }
        i = j;
        if (a1[i] == '-') { j = i + 1; while (j < n && a1[j] == '-') ++j; w += snprintf(out + w, cap - w, "%dI", j - i); i = j; }
        else if (a2[i] == '-') { j = i + 1; while (j < n && a2[j] == '-') ++j; w += snprintf(out + w, cap - w, "%dD", j - i); i = j; }
        else { j = i + 1; while (j < n && a1[j] != a2[j] && a1[j] != '-' && a2[j] != '-') ++j; w += snprintf(out + w, cap - w, "%dX", j - i); i = j; }
    }
    if (w < cap) out[w] = 0;
    return w;
}

/* hmm::align for one mapping position (pair_hmm.hpp:858-874 → :321-340 try_naive_align, :784-823 simd_align, :642-673
 * discount_flank_score). value = integer penalty (likelihood = -ln10/10 * value) or INT_MAX for lowest();
 * target_offset as the reference computes it (size_t arithmetic mirrored in int64). Returns 0, or 1 for HMMOverflow. */
static int align_one_position(int band, const char* hap, int hap_len, const char* read, const uint8_t* quals, int read_len,
                              int offset, const oracle_model* m, int use_flanks, int lhs_flank, int rhs_flank,
                              int* value, int64_t* target_offset, char* cigar, int cigar_cap)
{
    if (memcmp(read, hap + offset, (size_t)read_len) == 0) {   /* :332-336 */
        *value = 0; *target_offset = offset; snprintf(cigar, cigar_cap, "%d=", read_len);
        return 0;
    }
    const int W = read_len + 2 * band - 1;
    const int a = offset - band > 0 ? offset - band : 0;
    if (a + W > hap_len) { *value = 0x7fffffff; *target_offset = 0; cigar[0] = 0; return 0; }   /* :802-807 */
    const oracle_model om = offset_model(m, a);
    const int n = 2 * (read_len + band) + 1;
    char* a1 = (char*)calloc((size_t)n + 1, 1);
    char* a2 = (char*)calloc((size_t)n + 1, 1);
    int first_pos = 0;
    int score = oracle_align_tb(band, hap + a, read, (const int8_t*)quals, W, read_len, &om, &first_pos, a1, a2);
    if (first_pos == -1) { free(a1); free(a2); return 1; }   /* :815-817 HMMOverflow */
    const int near_flank = use_flanks && (offset < lhs_flank + band || offset + read_len + band > hap_len - rhs_flank);
    if (near_flank) {   /* :659-672 */
        int lhs = lhs_flank < a ? 0 : lhs_flank - a, rhs;
        if (a + W < hap_len - rhs_flank) rhs = 0; else { rhs = rhs_flank + a + W - hap_len; if (rhs < 0) rhs = 0; }
        int mask_size = 0;
        int flank = oracle_flank_score(W, lhs, rhs, read, (const int8_t*)quals, &om, first_pos, a1, a2, &mask_size);
        if (read_len - mask_size < 2) flank = 0;
        if (flank <= score) score -= flank; else score += flank;
    }
    *value = score;
    *target_offset = (int64_t)offset - band + first_pos;   /* :820 */
    make_cigar_text(a1, a2, cigar, cigar_cap);
    free(a1); free(a2);
    return 0;
}

/* haplotype_likelihood_model.cpp:335-431 compute_optimal_alignment + HaplotypeLikelihoodModel::align.
 * Returns 0 ok, 1 ShortHaplotypeError (*required_extension), 2 HMMOverflow. */
int oracle_model_align(int band, const char* hap, int hap_len, const char* read, const uint8_t* quals, int read_len,
                       const oracle_model* m, int use_flanks, int lhs_flank, int rhs_flank,
                       const int64_t* positions, int n_positions, int64_t original_pos,
                       int use_mapping_quality, int mapping_quality, int mapq_cap, int mapq_cap_trigger,
                       int64_t* mapping_position, double* likelihood, char* cigar, int cigar_cap, int* required_extension)
{
    int best = 0x7fffffff, have = 0;   /* result.likelihood = lowest() */
    int64_t best_off = 0;
    char* tmp = (char*)malloc((size_t)cigar_cap);
    cigar[0] = 0;
    int original_mapped = 0, has_in_range = 0;
    for (int p = 0; p < n_positions; ++p) {
        if (positions[p] == original_pos) original_mapped = 1;
        if (num_out_of_range_bases(positions[p], read_len, hap_len, band) == 0) {
            has_in_range = 1;
            int v; int64_t off;
            if (align_one_position(band, hap, hap_len, read, quals, read_len, (int)positions[p], m, use_flanks, lhs_flank, rhs_flank, &v, &off, tmp, cigar_cap)) { free(tmp); return 2; }
            if (v < best) { best = v; best_off = off; strcpy(cigar, tmp); have = 1; }   /* :355 likelihood > result.likelihood */
        }
    }
    if (!original_mapped && num_out_of_range_bases(original_pos, read_len, hap_len, band) == 0) {
        has_in_range = 1;
        int v; int64_t off;
        if (align_one_position(band, hap, hap_len, read, quals, read_len, (int)original_pos, m, use_flanks, lhs_flank, rhs_flank, &v, &off, tmp, cigar_cap)) { free(tmp); return 2; }
        if (v <= best) { best = v; best_off = off; strcpy(cigar, tmp); have = 1; }      /* :365 >= */
    }
    if (!has_in_range) {
        const int min_shift = num_out_of_range_bases(original_pos, read_len, hap_len, band);
        int64_t fin = original_pos;
        if (min_shift > 0) {
            fin += min_shift;
            if (num_out_of_range_bases(fin, read_len, hap_len, band) != 0) { *required_extension = min_shift; free(tmp); return 1; }
        } else {
            const unsigned left = (unsigned)(-min_shift);
            if (original_pos >= (int64_t)left) fin -= left; else { *required_extension = (int)(left - original_pos); free(tmp); return 1; }
        }
        int v; int64_t off;
        if (align_one_position(band, hap, hap_len, read, quals, read_len, (int)fin, m, use_flanks, lhs_flank, rhs_flank, &v, &off, tmp, cigar_cap)) { free(tmp); return 2; }
        best = v; best_off = off; strcpy(cigar, tmp); have = 1;
    }
    (void)have;
    free(tmp);
    *mapping_position = best_off;
    const double ln_given = best == 0x7fffffff ? ORACLE_LOWEST : -LN10_DIV_10 * (double)best;
    if (use_mapping_quality) {
        int mq = mapping_quality;
        /* set(config) / the constructor drop a trigger that is >= the cap (haplotype_likelihood_model.cpp:49-51, 117-119) */
        if (mapq_cap_trigger >= 0 && mapq_cap_trigger < mapq_cap && mq >= mapq_cap_trigger) mq = mapq_cap;
        const double ln_miss = -LN10_DIV_10 * (double)mq;
        const double ln_mapped = log(1.0 - exp(ln_miss));
        const double r = log_sum_exp2(ln_mapped + ln_given, ln_miss);
        *likelihood = r > -1e-15 ? 0.0 : r;
    } else {
        *likelihood = ln_given > -1e-15 ? 0.0 : ln_given;
    }
    return 0;
}

/* maths::log_sum_exp (utils/maths.hpp) over n >= 1 terms: the largest term plus ln of the sum, taken in order, of exp(x_k - max).
 * The three-term overload is this with n = 3 (0 + x is exact). */
static double log_sum_exp_n(const double* x, int n)
{
    double mx = x[0];
    for (int k = 1; k < n; ++k) if (x[k] > mx) mx = x[k];
    double s = 0.0;
    for (int k = 0; k < n; ++k) s += exp(x[k] - mx);
    return mx + log(s);
}

/* N1 — ConstantMixtureGenotypeLikelihoodModel::evaluate(const Genotype<IndexedHaplotype<>>&) (core/models/genotype/
 * constant_mixture_genotype_likelihood_model.cpp:66-77, 163-319) over a [H][R] matrix, form by form as the reference dispatches:
 * ln p(reads | g) = sum_r ( ln sum_{h in g} p(r | h) - ln ploidy ), accumulated read by read from 0 like std::accumulate /
 * std::inner_product. A run of m equal adjacent indices enters once, as ln m + its value:
 *   ploidy 0: 0;  1: the plain sum;  2: homozygous the plain sum, else log_sum_exp(a, b) - ln 2 (log1p form);
 *   3: homozygous the plain sum, [a a b] log_sum_exp(ln 2 + a, b), [a b b] log_sum_exp(a, ln 2 + b), else the three-term form,
 *      each - ln 3;
 *   4: homozygous the plain sum, [a a a b] / [a b b b] log_sum_exp(ln 3 + a, b) / (a, ln 3 + b) - ln 4, [a a b b]
 *      log_sum_exp(a, b) - ln 2, [a a b c] / [a b b c] / [a b c c] the three-term form with ln 2 on the doubled one, - ln 4,
 *      else the four-term form - ln 4;
 *   5 and up: the buffer form, log_sum_exp over all ploidy values - ln ploidy, with no homozygous shortcut.
 * The constants ln 2, ln 3, ln 4 are the doubles nearest them, as the reference's lookup table holds them. */
void oracle_genotype_likelihoods(const double* lnl, int H, int R, const int32_t* genotypes, int G, int ploidy, double* out)
{
    static const double LN2 = 0.693147180559945309417232121458176568, LN3 = 1.098612288668109691395245236922525705,
                        LN4 = 1.386294361119890618834464242916353136;
    (void)H;
    for (int g = 0; g < G; ++g) {
        const int32_t* gt = genotypes + (size_t)g * ploidy;
        const double* row[64];
        for (int k = 0; k < ploidy; ++k) row[k] = lnl + (size_t)gt[k] * R;
        double acc = 0.0, x[64];
        if (ploidy == 0) {
            /* the empty genotype: ln 1 */
        } else if (ploidy == 1 || (ploidy <= 4 && gt[0] == gt[1] && (ploidy < 3 || gt[1] == gt[2]) && (ploidy < 4 || gt[2] == gt[3]))) {
            for (int r = 0; r < R; ++r) acc += row[0][r];
        } else if (ploidy == 2) {
            for (int r = 0; r < R; ++r) acc += log_sum_exp2(row[0][r], row[1][r]) - LN2;
        } else if (ploidy == 3) {
            const int e01 = gt[0] == gt[1], e12 = gt[1] == gt[2];
            for (int r = 0; r < R; ++r) {
                double v;
                if (e01) v = log_sum_exp2(LN2 + row[0][r], row[2][r]);
                else if (e12) v = log_sum_exp2(row[0][r], LN2 + row[1][r]);
                else { x[0] = row[0][r]; x[1] = row[1][r]; x[2] = row[2][r]; v = log_sum_exp_n(x, 3); }
                acc += v - LN3;
            }
        } else if (ploidy == 4) {
            const int e01 = gt[0] == gt[1], e12 = gt[1] == gt[2], e23 = gt[2] == gt[3];
            for (int r = 0; r < R; ++r) {
                const double a = row[0][r], b = row[1][r], c = row[2][r], d = row[3][r];
                double v;
                if (e01 && e12) v = log_sum_exp2(LN3 + a, d) - LN4;
                else if (e01 && e23) v = log_sum_exp2(a, c) - LN2;
                else if (e01) { x[0] = LN2 + a; x[1] = c; x[2] = d; v = log_sum_exp_n(x, 3) - LN4; }
                else if (e12 && e23) v = log_sum_exp2(a, LN3 + b) - LN4;
                else if (e12) { x[0] = a; x[1] = LN2 + b; x[2] = d; v = log_sum_exp_n(x, 3) - LN4; }
                else if (e23) { x[0] = a; x[1] = b; x[2] = LN2 + c; v = log_sum_exp_n(x, 3) - LN4; }
                else { x[0] = a; x[1] = b; x[2] = c; x[3] = d; v = log_sum_exp_n(x, 4) - LN4; }
                acc += v;
            }
        } else {
            const double ln_ploidy = log((double)ploidy);
            for (int r = 0; r < R; ++r) {
                for (int k = 0; k < ploidy; ++k) x[k] = row[k][r];
                acc += log_sum_exp_n(x, ploidy) - ln_ploidy;
            }
        }
        out[g] = acc;
    }
}
