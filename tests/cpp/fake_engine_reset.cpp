// A CPU stand-in for the engine's _reset populate symbols (phmm_populate_reset, phmm_populate_regions_reset,
// phmm_populate_templates_reset), next to tests/cpp/fake_engine.cpp's plain ones. Each does literally what the engine's contract
// says: the host reset (phmm_reset_haplotypes of octopus_b200/csrc/phmm_error_model.cpp, linked in), then the fake's plain twin on
// the same inputs. The argument checks are the engine's, with its messages. Every call is recorded with its error model's key.
#include "../../include/phmm_b200.h"
#include "../../octopus_b200/csrc/phmm_checks.h"
#include "../../octopus_b200/csrc/phmm_reset.cuh"

#include <mutex>
#include <string>
#include <vector>

struct phmm_engine {        // fake_engine.cpp's engine, declared identically
    std::string err;
    int64_t dp_cells = 0;
};

namespace fake_reset {

struct Call {
    std::string entry;       // "populate_reset", "populate_regions_reset" or "populate_templates_reset"
    int members;             // regions (1 for the one-region calls)
    long long haps;
    std::string model_key;
};

namespace {
std::mutex g_m;
std::vector<Call> g_calls;

// The six arrays of the sequences block, as the engine derives them.
struct Derived {
    std::vector<char> mf, mr;
    std::vector<int8_t> pf, pr, go, ge;
    phmm_haplotypes haps {};
};

int derive(phmm_engine* e, const phmm_error_model* m, const phmm_haplotype_sequences* seqs, int space, Derived& d)
{
    int rc;
    if (space != PHMM_SPACE_HOST) { e->err = "bad memory space"; return PHMM_ERR_INVALID; }
    if ((rc = phmm_checks::reset_sequences(m, seqs, e->err)) != PHMM_OK) return rc;
    const size_t B = seqs->n > 0 ? (size_t)seqs->off[seqs->n] + 1 : 1;
    d.mf.assign(B, 0); d.mr.assign(B, 0); d.pf.assign(B, 0); d.pr.assign(B, 0); d.go.assign(B, 0); d.ge.assign(B, 0);
    if (seqs->n > 0 && phmm_reset_haplotypes(m, seqs->n, seqs->off, seqs->seq, seqs->is_substitution, d.mf.data(), d.pf.data(), d.mr.data(),
                                             d.pr.data(), d.go.data(), d.ge.data(), 1) != PHMM_OK) {
        e->err = phmm_error_model_last_error();
        return PHMM_ERR_INVALID;
    }
    d.haps = {seqs->n, seqs->off, seqs->seq, d.mf.data(), d.pf.data(), d.mr.data(), d.pr.data(), d.go.data(), d.ge.data(), seqs->begin};
    return PHMM_OK;
}

void record(const char* entry, int members, const phmm_haplotype_sequences* seqs, const phmm_error_model* m)
{
    std::lock_guard<std::mutex> lk(g_m);
    g_calls.push_back({entry, members, seqs ? seqs->n : 0, m ? phmm_reset::model_key(m) : std::string()});
}
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

} // namespace fake_reset

extern "C" {

int phmm_populate_reset(phmm_engine* e, const phmm_config* cfg, const phmm_error_model* m, const phmm_haplotype_sequences* seqs,
                        const phmm_reads* reads, const phmm_positions* positions, const phmm_flank_state* flank,
                        double* out, int32_t* status, int space)
{
    fake_reset::record("populate_reset", 1, seqs, m);
    fake_reset::Derived d;
    const int rc = fake_reset::derive(e, m, seqs, space, d);
    return rc != PHMM_OK ? rc : phmm_populate(e, cfg, &d.haps, reads, positions, flank, out, status, space);
}

int phmm_populate_regions_reset(phmm_engine* e, const phmm_config* cfg, const phmm_error_model* m, const phmm_haplotype_sequences* seqs,
                                const phmm_reads* reads, const phmm_regions* regions, double* out, int32_t* status, int space)
{
    fake_reset::record("populate_regions_reset", regions ? regions->n : 0, seqs, m);
    fake_reset::Derived d;
    const int rc = fake_reset::derive(e, m, seqs, space, d);
    return rc != PHMM_OK ? rc : phmm_populate_regions(e, cfg, &d.haps, reads, regions, out, status, space);
}

int phmm_populate_templates_reset(phmm_engine* e, const phmm_config* cfg, const phmm_error_model* m, const phmm_haplotype_sequences* seqs,
                                  const phmm_reads* reads, const int64_t* template_off, int32_t n_templates,
                                  const phmm_positions* positions, const phmm_flank_state* flank, double* out, int32_t* status, int space)
{
    fake_reset::record("populate_templates_reset", 1, seqs, m);
    int rc;
    if (!seqs) { e->err = "null argument"; return PHMM_ERR_INVALID; }
    if ((rc = phmm_checks::template_offsets(template_off, n_templates, reads, true, e->err)) != PHMM_OK) return rc;
    fake_reset::Derived d;
    if ((rc = fake_reset::derive(e, m, seqs, space, d)) != PHMM_OK) return rc;
    return phmm_populate_templates(e, cfg, &d.haps, reads, template_off, n_templates, positions, flank, out, status, space);
}

} // extern "C"
