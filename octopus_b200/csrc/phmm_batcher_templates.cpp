// The shared engine's template assignment requests (include/phmm_b200.h, phmm_batcher_assign_templates): the engine's call, handed
// to the batcher through phmm_batcher_seam.h. They run as assign requests whose top and lnl are per template.
#include "../../include/phmm_b200.h"
#include "phmm_batcher_seam.h"

namespace {

const phmm_batcher_seam::TemplateCalls kEngine {phmm_assign_templates};

} // namespace

extern "C" {

int phmm_batcher_assign_templates(phmm_batcher* b, const phmm_config* cfg, const phmm_haplotypes* haps, const phmm_reads* reads,
                                  const phmm_regions* groups, const int64_t* template_off, int32_t n_templates,
                                  const double* log_priors, uint64_t* top, double* lnl, int32_t* status)
{
    return phmm_batcher_seam::submit_assign(b, {nullptr, cfg, haps, reads, groups, log_priors, top, lnl, status, &kEngine, template_off, n_templates});
}

} // extern "C"
