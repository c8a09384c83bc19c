// The shared engine's populate requests with an error model (include/phmm_b200.h, phmm_batcher_populate*_reset): the model's
// content key and the engine's _reset calls, handed to the batcher through phmm_batcher_seam.h.
#include "../../include/phmm_b200.h"
#include "phmm_batcher_seam.h"
#include "phmm_reset.cuh"

namespace {

const phmm_batcher_seam::ResetCalls kEngine {phmm_populate_reset, phmm_populate_regions_reset, phmm_populate_templates_reset};

phmm_batcher_seam::ResetRequest request(const phmm_config* cfg, const phmm_error_model* m, const phmm_haplotype_sequences* seqs,
                                        const phmm_reads* reads, const phmm_positions* positions, const int64_t* template_off,
                                        int32_t n_templates, const phmm_flank_state* flank, double* out, int32_t* status)
{
    return {&kEngine, m ? phmm_reset::model_key(m) : std::string(), cfg, m, seqs, reads, positions, template_off, n_templates, flank, out, status};
}

} // namespace

extern "C" {

int phmm_batcher_populate_reset(phmm_batcher* b, const phmm_config* cfg, const phmm_error_model* m, const phmm_haplotype_sequences* seqs,
                                const phmm_reads* reads, const phmm_positions* positions, const phmm_flank_state* flank,
                                double* out, int32_t* status)
{
    return phmm_batcher_seam::submit_reset(b, request(cfg, m, seqs, reads, positions, nullptr, 0, flank, out, status));
}

int phmm_batcher_populate_templates_reset(phmm_batcher* b, const phmm_config* cfg, const phmm_error_model* m,
                                          const phmm_haplotype_sequences* seqs, const phmm_reads* reads, const int64_t* template_off,
                                          int32_t n_templates, const phmm_flank_state* flank, double* out, int32_t* status)
{
    return phmm_batcher_seam::submit_reset(b, request(cfg, m, seqs, reads, nullptr, template_off, n_templates, flank, out, status));
}

} // extern "C"
