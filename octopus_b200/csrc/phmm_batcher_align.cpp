// The shared engine's read-assignment and realignment requests (include/phmm_b200.h, phmm_batcher_assign_reads /
// phmm_batcher_realign_reads): the engine's calls, handed to the batcher through phmm_batcher_seam.h.
#include "../../include/phmm_b200.h"
#include "phmm_batcher_seam.h"

namespace {

const phmm_batcher_seam::AlignCalls kEngine {phmm_assign_reads, phmm_realign_reads};

} // namespace

extern "C" {

int phmm_batcher_assign_reads(phmm_batcher* b, const phmm_config* cfg, const phmm_haplotypes* haps, const phmm_reads* reads,
                              const phmm_regions* groups, const double* log_priors, uint64_t* top, double* lnl, int32_t* status)
{
    return phmm_batcher_seam::submit_assign(b, {&kEngine, cfg, haps, reads, groups, log_priors, top, lnl, status});
}

int phmm_batcher_realign_reads(phmm_batcher* b, const phmm_config* cfg, const phmm_haplotypes* haps, const phmm_reads* reads,
                               const phmm_pair* pairs, int64_t n_pairs, const phmm_flank_state* flank,
                               int64_t* mapping_position, double* likelihood, char* cigar, int32_t cigar_stride, int32_t* status)
{
    return phmm_batcher_seam::submit_realign(b, {&kEngine, cfg, haps, reads, pairs, n_pairs, flank, mapping_position, likelihood, cigar,
                                                 cigar_stride, status});
}

} // extern "C"
