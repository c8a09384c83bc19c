// A CPU stand-in for the engine's template assignment (phmm_assign_templates), next to tests/cpp/fake_engine_align.cpp's
// phmm_assign_reads, so that the request batcher's template requests run their whole life cycle without a GPU
// (tests/test_batcher_templates_cpu.py).
//
// It is built as the engine builds it: phmm_assign_reads' checks plus the template checks, in the engine's order, then
// phmm_assign_reads' per-read values (the align fake's: each hashes only its own pair's data), summed per template left to right
// from 0.0, plus the log prior, and find_map_haplotypes' rule per template. So a request gets the same values in a merged call as
// alone exactly when the batcher stages, shifts and slices its groups and templates correctly. The align fake's marker reads and
// short-haplotype statuses carry over. Every call is recorded with its groups, its templates and its return code.
#include "../../include/phmm_b200.h"
#include "../../octopus_b200/csrc/phmm_checks.h"

#include <algorithm>
#include <cmath>
#include <mutex>
#include <string>
#include <vector>

struct phmm_engine {        // fake_engine.cpp's engine, declared identically
    std::string err;
    int64_t dp_cells = 0;
};

namespace fake_templates {

struct Call { int groups; int templates; int rc; };

namespace {
std::mutex g_m;
std::vector<Call> g_calls;

bool almost_equal(double l, double r) { return l == r || std::fabs(l - r) < 2.220446049250313080847263336181640625e-16 * std::fabs(l + r); }
} // namespace

std::vector<Call> calls()
{
    std::lock_guard<std::mutex> lk(g_m);
    return g_calls;
}

void clear_calls()
{
    std::lock_guard<std::mutex> lk(g_m);
    g_calls.clear();
}

} // namespace fake_templates

namespace {

int assign_templates(phmm_engine* e, const phmm_config* cfg, const phmm_haplotypes* haps, const phmm_reads* reads,
                     const phmm_regions* groups, const int64_t* template_off, int32_t n_templates,
                     const double* log_priors, uint64_t* top, double* lnl, int32_t* status, int space)
{
    e->dp_cells = 0;
    e->err.clear();
    int rc;
    if (space != PHMM_SPACE_HOST) { e->err = "bad space"; return PHMM_ERR_INVALID; }
    if ((rc = phmm_checks::regions(haps, reads, groups, e->err)) != PHMM_OK) return rc;
    if ((rc = phmm_checks::config_and_output(cfg, top, reads, e->err)) != PHMM_OK) return rc;
    if ((rc = phmm_checks::assign_groups(groups, e->err)) != PHMM_OK) return rc;
    if ((rc = phmm_checks::assign_templates(template_off, n_templates, reads, groups, e->err)) != PHMM_OK) return rc;
    long long slots = 0;
    for (int g = 0; g < groups->n; ++g)
        slots += (long long)(groups->hap_first[g + 1] - groups->hap_first[g]) * (groups->read_first[g + 1] - groups->read_first[g]);
    std::vector<uint64_t> read_top((size_t)reads->n);
    std::vector<double> v((size_t)slots);
    std::vector<int32_t> st((size_t)slots);
    rc = phmm_assign_reads(e, cfg, haps, reads, groups, log_priors, read_top.data(), v.data(), st.data(), space);
    if (rc != PHMM_OK && rc != PHMM_ERR_SHORT_HAPLOTYPE) return rc;
    if (status) std::copy(st.begin(), st.end(), status);
    long long slot = 0, tout = 0;
    int t = 0;
    for (int g = 0; g < groups->n; ++g) {
        const int h0 = groups->hap_first[g], nH = groups->hap_first[g + 1] - h0, r0 = groups->read_first[g], nR = groups->read_first[g + 1] - r0;
        const int t0 = t;
        while (t < n_templates && template_off[t] < r0 + nR) ++t;
        const int nT = t - t0;
        for (int i = 0; i < nT; ++i) {
            double max_value = -1.7976931348623157e308;
            uint64_t set = 0;
            for (int k = 0; k < nH; ++k) {
                double sum = 0.0;
                for (int64_t r = template_off[t0 + i]; r < template_off[t0 + i + 1]; ++r) sum += v[(size_t)(slot + (long long)k * nR + (r - r0))];
                if (lnl) lnl[tout + (long long)k * nT + i] = sum;
                const double cur = sum + (log_priors ? log_priors[h0 + k] : 0.0);
                if (fake_templates::almost_equal(cur, max_value)) set |= 1ull << k;
                else if (cur > max_value) { set = 1ull << k; max_value = cur; }
            }
            top[t0 + i] = set ? set : (nH == 64 ? ~0ull : (1ull << nH) - 1);
        }
        slot += (long long)nH * nR;
        tout += (long long)nH * nT;
    }
    return rc;
}

} // namespace

extern "C" {

int phmm_assign_templates(phmm_engine* e, const phmm_config* cfg, const phmm_haplotypes* haps, const phmm_reads* reads,
                          const phmm_regions* groups, const int64_t* template_off, int32_t n_templates,
                          const double* log_priors, uint64_t* top, double* lnl, int32_t* status, int space)
{
    const int rc = assign_templates(e, cfg, haps, reads, groups, template_off, n_templates, log_priors, top, lnl, status, space);
    std::lock_guard<std::mutex> lk(fake_templates::g_m);
    fake_templates::g_calls.push_back({groups ? groups->n : 0, n_templates, rc});
    return rc;
}

} // extern "C"
