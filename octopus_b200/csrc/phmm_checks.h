// Host-side argument checks of the populate, assign, align and mutation-prime entry points, shared by the engine (phmm_engine.cu) and the request batcher
// (phmm_batcher.cpp) so that both report the same error codes and messages. Each check returns PHMM_OK or an error code and
// sets `err`; the callers run them in the order populate reports errors in.
#ifndef PHMM_CHECKS_H
#define PHMM_CHECKS_H

#include "../../include/phmm_b200.h"

#include <algorithm>
#include <string>

namespace phmm_checks {

// config, output pointer and the per-read arrays populate always needs
inline int config_and_output(const phmm_config* cfg, const void* out, const phmm_reads* reads, std::string& err)
{
    if (!cfg || !out) { err = "null config / output"; return PHMM_ERR_INVALID; }
    if (cfg->max_indel_error > 256) { err = "max_indel_error > 256"; return PHMM_ERR_BAND; }
    if (cfg->nuc_prior < 0 || cfg->nuc_prior > 127) { err = "nuc_prior outside [0,127]"; return PHMM_ERR_INVALID; }
    if (!reads || !reads->mapq || !reads->reverse) { err = "reads->mapq / reads->reverse required"; return PHMM_ERR_INVALID; }
    return PHMM_OK;
}

// non-empty blocks with every per-base array present; `derived`: the six penalty arrays are yet to be derived from the sequences
// (a populate call with an error model)
inline int blocks(const phmm_haplotypes* haps, const phmm_reads* reads, std::string& err, bool derived = false)
{
    if (!haps || !reads || haps->n <= 0 || reads->n <= 0 || !haps->off || !reads->off) {
        err = "empty or null haplotype / read block";
        return PHMM_ERR_INVALID;
    }
    if (!haps->seq || (!derived && (!haps->snv_mask_fwd || !haps->snv_prior_fwd || !haps->snv_mask_rev || !haps->snv_prior_rev ||
        !haps->gap_open || !haps->gap_extend)) || !reads->bases || !reads->quals) {
        err = "null per-base array";
        return PHMM_ERR_INVALID;
    }
    return PHMM_OK;
}

// offset arrays, from their first / last entries and the shortest / longest read
inline int offsets(long long hap_first, long long hap_bases, long long read_first, long long read_bases, long long read_len_min,
                   long long read_len_max, std::string& err)
{
    if (hap_first != 0 || read_first != 0 || hap_bases <= 0 || read_bases <= 0) {
        err = "offset arrays must start at 0 and be increasing";
        return PHMM_ERR_INVALID;
    }
    if (read_len_min < 1) { err = "empty read (offsets must be strictly increasing)"; return PHMM_ERR_INVALID; }
    if (read_len_max > (1LL << 30)) { err = "read too long"; return PHMM_ERR_INVALID; }
    return PHMM_OK;
}

// read length range of a host-resident read block
inline void read_length_range(const phmm_reads* reads, long long* len_min, long long* len_max)
{
    long long lo = 1LL << 62, hi = 0;
    for (int r = 0; r < reads->n; ++r) { const long long len = reads->off[r + 1] - reads->off[r]; lo = std::min(lo, len); hi = std::max(hi, len); }
    *len_min = lo; *len_max = hi;
}

// the device k-mer mapper's limits
inline int mapper_haplotypes(long long max_hap_len, long long hap_bases, std::string& err)
{
    if (max_hap_len > 65535) { err = "haplotype longer than 65535 bp: the device k-mer mapper indexes k-mer positions with 16 bits (pass explicit positions)"; return PHMM_ERR_INVALID; }
    if (hap_bases > 65535LL * 65535LL) { err = "haplotype block too large"; return PHMM_ERR_INVALID; }
    return PHMM_OK;
}

// the uncapped pair mapper's read limit (phmm_map_pairs, phmm_realign_reads, phmm_assign_reads): votes are counted in 16 bits
inline int mapper_reads(long long read_len_max, std::string& err)
{
    if (read_len_max > 65540) { err = "read longer than 65540 bp: the device k-mer mapper counts votes in 16 bits"; return PHMM_ERR_INVALID; }
    return PHMM_OK;
}

// the region (group) list of phmm_populate_regions / phmm_assign_reads (host memory): bounds that cover both blocks exactly and at
// least one haplotype and one read per region
inline int regions(const phmm_haplotypes* haps, const phmm_reads* reads, const phmm_regions* regions, std::string& err)
{
    if (!regions || regions->n <= 0 || !regions->hap_first || !regions->read_first || !haps || !reads) { err = "null / empty region list"; return PHMM_ERR_INVALID; }
    if (regions->hap_first[0] != 0 || regions->read_first[0] != 0 || regions->hap_first[regions->n] != haps->n || regions->read_first[regions->n] != reads->n) {
        err = "region ranges must cover the haplotype and read blocks exactly";
        return PHMM_ERR_INVALID;
    }
    for (int g = 0; g < regions->n; ++g) {
        if (regions->hap_first[g + 1] <= regions->hap_first[g] || regions->read_first[g + 1] <= regions->read_first[g]) {
            err = "every region needs at least one haplotype and one read";
            return PHMM_ERR_INVALID;
        }
    }
    return PHMM_OK;
}

// phmm_assign_reads' limits on a checked group list: a read's top set is a 64-bit mask, and the call's result slots are counted in
// 31 bits
inline int assign_groups(const phmm_regions* groups, std::string& err)
{
    long long widest = 0, slots = 0;
    for (int g = 0; g < groups->n; ++g) {
        const long long nH = groups->hap_first[g + 1] - groups->hap_first[g], nR = groups->read_first[g + 1] - groups->read_first[g];
        widest = std::max(widest, nH);
        slots += nH * nR;
    }
    if (widest > 64) { err = "more than 64 haplotypes in one group: a read's top set is a 64-bit mask"; return PHMM_ERR_INVALID; }
    if (slots > 0x7fffffffLL) { err = "more than 2^31 - 1 (read, haplotype) pairs in one call"; return PHMM_ERR_INVALID; }
    return PHMM_OK;
}

// The aligning calls (phmm_align_reads, phmm_realign_reads, phmm_align_pairs): their output pointers, the CIGAR stride, the config
// and the pair count, before anything else; a call of no pairs then returns PHMM_OK without touching anything.
inline int align_arguments(const phmm_config* cfg, const phmm_pair* pairs, int64_t n_pairs, const void* mapping_position, const void* likelihood,
                           const char* cigar, int32_t cigar_stride, const int32_t* status, std::string& err)
{
    if (!cfg || !pairs || !mapping_position || !likelihood || !cigar || !status || cigar_stride < 8) { err = "null argument / cigar_stride < 8"; return PHMM_ERR_INVALID; }
    if (cfg->max_indel_error > 256) { err = "max_indel_error > 256"; return PHMM_ERR_BAND; }
    if (cfg->nuc_prior < 0 || cfg->nuc_prior > 127) { err = "nuc_prior outside [0,127]"; return PHMM_ERR_INVALID; }
    if (n_pairs < 0 || n_pairs > 0x7fffffff) { err = "pair count out of range"; return PHMM_ERR_INVALID; }
    return PHMM_OK;
}

// the per-read arrays the aligning calls need: reverse always, mapping qualities where the config uses them
inline int align_reads(const phmm_config* cfg, const phmm_reads* reads, std::string& err)
{
    if (!reads || !reads->reverse || (!reads->mapq && cfg->use_mapping_quality)) { err = "reads->mapq / reads->reverse required"; return PHMM_ERR_INVALID; }
    return PHMM_OK;
}

// (read, haplotype) indices of a host-resident pair list
inline int pair_indices(const phmm_pair* pairs, long long n, int n_haps, int n_reads, std::string& err)
{
    for (long long i = 0; i < n; ++i) {
        if (pairs[i].read < 0 || pairs[i].read >= n_reads || pairs[i].hap < 0 || pairs[i].hap >= n_haps) { err = "pair index out of range"; return PHMM_ERR_INVALID; }
    }
    return PHMM_OK;
}

// what k_build_tables flags on the device (flags bit 0), scanned on the host: SNV priors and gap penalties in [0,127]
inline int penalties(const phmm_haplotypes* haps, long long hap_bases, std::string& err)
{
    const int8_t* arrays[] = {haps->snv_prior_fwd, haps->snv_prior_rev, haps->gap_open, haps->gap_extend};
    for (const int8_t* a : arrays) {
        for (long long i = 0; i < hap_bases; ++i) {
            if (a[i] < 0) { err = "snv prior / gap penalty outside [0,127]"; return PHMM_ERR_INVALID; }
        }
    }
    return PHMM_OK;
}

// the error-model reset of a populate call with an error model, for host-resident sequences (phmm_engine_reset_haplotypes' checks)
inline int reset_sequences(const void* model, const phmm_haplotype_sequences* seqs, std::string& err)
{
    if (!model || !seqs || seqs->n < 0 || (seqs->n > 0 && (!seqs->off || !seqs->seq))) { err = "null argument"; return PHMM_ERR_INVALID; }
    if (seqs->n > 0 && seqs->off[0] < 0) { err = "bad haplotype offsets"; return PHMM_ERR_INVALID; }
    long long longest = 0;
    for (int32_t h = 0; h < seqs->n; ++h) {
        if (seqs->off[h + 1] < seqs->off[h]) { err = "bad haplotype offsets"; return PHMM_ERR_INVALID; }
        longest = std::max<long long>(longest, seqs->off[h + 1] - seqs->off[h]);
    }
    if (longest > 65535) { err = "haplotype longer than 65535 bases"; return PHMM_ERR_INVALID; }
    return PHMM_OK;
}

// template offsets of a host-resident call
inline int template_offsets(const int64_t* template_off, int32_t n_templates, const phmm_reads* reads, bool host, std::string& err)
{
    if (!template_off || n_templates <= 0 || !reads) { err = "null / empty template offsets"; return PHMM_ERR_INVALID; }
    if (host) {
        if (template_off[0] != 0 || template_off[n_templates] != reads->n) { err = "template offsets must cover the reads exactly"; return PHMM_ERR_INVALID; }
        for (int t = 0; t < n_templates; ++t) if (template_off[t + 1] < template_off[t]) { err = "template offsets must be non-decreasing"; return PHMM_ERR_INVALID; }
    }
    return PHMM_OK;
}

// phmm_assign_templates' templates (host memory) on a checked group list: they cover the reads exactly, each has at least one read,
// and no group boundary falls inside one
inline int assign_templates(const int64_t* template_off, int32_t n_templates, const phmm_reads* reads, const phmm_regions* groups, std::string& err)
{
    if (!template_off || n_templates <= 0) { err = "null / empty template offsets"; return PHMM_ERR_INVALID; }
    if (template_off[0] != 0 || template_off[n_templates] != reads->n) { err = "template offsets must cover the reads exactly"; return PHMM_ERR_INVALID; }
    for (int t = 0; t < n_templates; ++t) {
        if (template_off[t + 1] <= template_off[t]) { err = "template offsets must be strictly increasing (every template needs a read)"; return PHMM_ERR_INVALID; }
    }
    // both lists increase strictly, so one merge pass finds every group boundary among the template boundaries
    int t = 0;
    for (int g = 1; g < groups->n; ++g) {
        while (t < n_templates && template_off[t] < groups->read_first[g]) ++t;
        if (template_off[t] != groups->read_first[g]) { err = "a group boundary falls inside a template"; return PHMM_ERR_INVALID; }
    }
    return PHMM_OK;
}

// phmm_mutation_prime's checks of one haplotype set (host memory), in its order
inline int mutation_haplotype_count(int64_t n, std::string& err)
{
    if (n < 1 || n > PHMM_MUT_MAX_HAPLOTYPES) { err = "haplotype count outside [1, 4096]"; return PHMM_ERR_INVALID; }
    return PHMM_OK;
}

inline int mutation_offsets(int64_t n, const int64_t* off, std::string& err)
{
    if (off[0] != 0) { err = "offset arrays must start at 0"; return PHMM_ERR_INVALID; }
    for (int64_t h = 0; h < n; ++h) {
        const long long len = off[h + 1] - off[h];
        if (len < 1 || len > PHMM_MUT_MAX_LENGTH) { err = "haplotype length outside [1, 65535]"; return PHMM_ERR_INVALID; }
    }
    return PHMM_OK;
}

inline int mutation_set(const void* m, int32_t n, const int64_t* off, const char* seq, const double* out, const int32_t* status, std::string& err)
{
    if (!m || !off || !seq || !out || !status) { err = "null argument"; return PHMM_ERR_INVALID; }
    int rc;
    if ((rc = mutation_haplotype_count(n, err)) != PHMM_OK) return rc;
    return mutation_offsets(n, off, err);
}

// Read-chunk size (in pairs) of phmm_populate's pipelined path for a call of all_pairs pairs; the call is pipelined when it
// has at least twice that many pairs (host space, no position lists). Defined in phmm_engine.cu.
long long populate_chunk_pairs(long long all_pairs);

} // namespace phmm_checks

#endif
