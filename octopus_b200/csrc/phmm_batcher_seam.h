// The seam between the request batcher (phmm_batcher.cpp) and its populate requests with an error model (phmm_batcher_reset.cpp).
// phmm_batcher_reset.cpp computes a request's model key and hands the batcher the engine calls as function pointers, so that
// phmm_batcher.cpp names no engine symbol beyond the plain populate ones and no error-model internals: a fake engine can stand
// behind both.
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

} // namespace phmm_batcher_seam

#endif
