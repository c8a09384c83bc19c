// The seam between the request batcher (phmm_batcher.cpp) and its populate requests with an error model (phmm_batcher_reset.cpp),
// its assign / realign requests (phmm_batcher_align.cpp) and its template assign requests (phmm_batcher_templates.cpp).
// phmm_batcher_reset.cpp computes a request's model key; each hands the batcher the engine calls as function pointers, so that phmm_batcher.cpp names no engine symbol beyond the plain populate and
// mutation ones and no error-model internals: a fake engine can stand behind each part.
#ifndef PHMM_BATCHER_SEAM_H
#define PHMM_BATCHER_SEAM_H

#include "../../include/phmm_b200.h"

#include <string>

namespace phmm_batcher_seam {

struct ResetCalls {
    decltype(&phmm_populate_reset) populate;
    decltype(&phmm_populate_regions_reset) populate_regions;
    decltype(&phmm_populate_templates_reset) populate_templates;
};

// One request of phmm_batcher_populate_reset (template_off NULL) or phmm_batcher_populate_templates_reset.
struct ResetRequest {
    const ResetCalls* calls;
    std::string model_key;           // phmm_reset::model_key of m; empty: the request runs alone
    const phmm_config* cfg;
    const phmm_error_model* m;
    const phmm_haplotype_sequences* seqs;
    const phmm_reads* reads;
    const phmm_positions* positions;
    const int64_t* template_off;
    int32_t n_templates;
    const phmm_flank_state* flank;
    double* out;
    int32_t* status;
};

// Checks the request on the calling thread with phmm_populate_reset's checks and messages, then merges it or runs it alone.
int submit_reset(phmm_batcher* b, const ResetRequest& q);

// The engine calls of the assign and realign requests (phmm_batcher_align.cpp).
struct AlignCalls {
    decltype(&phmm_assign_reads) assign;
    decltype(&phmm_realign_reads) realign;
};

// The engine call of the template assign requests (phmm_batcher_templates.cpp).
struct TemplateCalls {
    decltype(&phmm_assign_templates) assign;
};

// One request of phmm_batcher_assign_reads (template_calls NULL) or phmm_batcher_assign_templates (calls NULL): top and lnl are then
// per template.
struct AssignRequest {
    const AlignCalls* calls;
    const phmm_config* cfg; const phmm_haplotypes* haps; const phmm_reads* reads; const phmm_regions* groups;
    const double* log_priors; uint64_t* top; double* lnl; int32_t* status;
    const TemplateCalls* template_calls = nullptr;
    const int64_t* template_off = nullptr; int32_t n_templates = 0;
};

// One request of phmm_batcher_realign_reads.
struct RealignRequest {
    const AlignCalls* calls;
    const phmm_config* cfg; const phmm_haplotypes* haps; const phmm_reads* reads; const phmm_pair* pairs; int64_t n_pairs;
    const phmm_flank_state* flank; int64_t* mapping_position; double* likelihood; char* cigar; int32_t cigar_stride; int32_t* status;
};

// Each checks the request on the calling thread with the plain call's checks and messages, then merges it or runs it alone.
int submit_assign(phmm_batcher* b, const AssignRequest& q);
int submit_realign(phmm_batcher* b, const RealignRequest& q);

} // namespace phmm_batcher_seam

#endif
