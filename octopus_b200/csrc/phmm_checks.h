// Host-side argument checks of the populate entry points, shared by the engine (phmm_engine.cu) and the request batcher
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

// non-empty blocks with every per-base array present
inline int blocks(const phmm_haplotypes* haps, const phmm_reads* reads, std::string& err)
{
    if (!haps || !reads || haps->n <= 0 || reads->n <= 0 || !haps->off || !reads->off) {
        err = "empty or null haplotype / read block";
        return PHMM_ERR_INVALID;
    }
    if (!haps->seq || !haps->snv_mask_fwd || !haps->snv_prior_fwd || !haps->snv_mask_rev || !haps->snv_prior_rev ||
        !haps->gap_open || !haps->gap_extend || !reads->bases || !reads->quals) {
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

// Read-chunk size (in pairs) of phmm_populate's pipelined path for a call of all_pairs pairs; the call is pipelined when it
// has at least twice that many pairs (host space, no position lists). Defined in phmm_engine.cu.
long long populate_chunk_pairs(long long all_pairs);

} // namespace phmm_checks

#endif
