// A CPU stand-in for the engine symbols the request batcher (octopus_b200/csrc/phmm_batcher.cpp) calls, so that its whole life
// cycle runs without a GPU, under ThreadSanitizer and AddressSanitizer (tests/test_batcher_cpu.py builds it with the batcher and
// tests/cpp/test_batcher_cpu.cpp).
//
// Every value depends only on the data of its own pair: a populate pair's value hashes the pair's haplotype and read bytes, the
// config and the region's flank state; a mutation pair's hashes the model key and the two haplotypes. So a region gets the same
// values in a merged call as in a call of its own, and the batcher stages, offsets and slices correctly exactly when every member
// gets its solo values back. The engine's checks that the batcher relies on are kept, with the engine's messages. Every call is
// recorded, and whatever the real engine would not accept from the batcher (a second call while one runs, region or set bounds
// that do not cover the blocks) is recorded as a violation.
#include "../../include/phmm_b200.h"
#include "../../octopus_b200/csrc/phmm_checks.h"
#include "../../octopus_b200/csrc/phmm_mutation.h"

#include <algorithm>
#include <atomic>
#include <chrono>
#include <cstdlib>
#include <cstring>
#include <mutex>
#include <string>
#include <thread>
#include <vector>

namespace fake {

struct Call {
    std::string entry;       // "populate", "populate_templates", "populate_regions" or "mutation_prime_sets"
    int members;             // regions or sets (1 for populate and populate_templates)
    long long haps;          // haplotypes in the call
    std::string key;         // the config bytes or the model key
};

namespace {
std::mutex g_log_m;
std::vector<Call> g_calls;
std::vector<std::string> g_violations;
std::atomic<int> g_inside {0};
std::atomic<int> g_call_delay_us {0};

void violation(const std::string& what)
{
    std::lock_guard<std::mutex> lk(g_log_m);
    g_violations.push_back(what);
}

// One engine call: counts concurrent entries and records the call.
struct Entry {
    explicit Entry(Call c)
    {
        if (g_inside.fetch_add(1) != 0) violation("a second engine call while one runs (" + c.entry + ")");
        {
            std::lock_guard<std::mutex> lk(g_log_m);
            g_calls.push_back(std::move(c));
        }
        if (const int us = g_call_delay_us.load()) std::this_thread::sleep_for(std::chrono::microseconds(us));
    }
    ~Entry() { g_inside.fetch_sub(1); }
};

struct Hash {
    unsigned long long h = 1469598103934665603ULL;
    Hash& add(const void* p, size_t n)
    {
        const unsigned char* c = static_cast<const unsigned char*>(p);
        for (size_t i = 0; i < n; ++i) { h ^= c[i]; h *= 1099511628211ULL; }
        return *this;
    }
    template <typename T> Hash& value(const T& v) { return add(&v, sizeof(T)); }
    // a finite, negative log-likelihood-like double
    double finish() const { return -1e-3 - (double)(h >> 11) * (100.0 / 9007199254740992.0); }
};

std::string config_key(const phmm_config* cfg) { return std::string(reinterpret_cast<const char*>(cfg), sizeof(phmm_config)); }
} // namespace

std::vector<Call> calls()
{
    std::lock_guard<std::mutex> lk(g_log_m);
    return g_calls;
}

std::vector<std::string> violations()
{
    std::lock_guard<std::mutex> lk(g_log_m);
    return g_violations;
}

void clear_calls()
{
    std::lock_guard<std::mutex> lk(g_log_m);
    g_calls.clear();
}

int calls_inside() { return g_inside.load(); }
void set_call_delay_us(int us) { g_call_delay_us.store(us); }

} // namespace fake

struct phmm_engine {
    std::string err;
    int64_t dp_cells = 0;
};

namespace {

thread_local std::string t_create_error;

// The value and status of pair (h, r); `positions` (optional) is the pair's candidate list.
void score_pair(const phmm_config* cfg, const phmm_haplotypes* haps, int h, const phmm_reads* reads, int r, const phmm_flank_state* flank,
                const int32_t* pos_begin, const int32_t* pos_end, double* out, int32_t* status)
{
    const long long hb = haps->off[h], hl = haps->off[h + 1] - hb, rb = reads->off[r], rl = reads->off[r + 1] - rb;
    fake::Hash x;
    x.add(cfg, sizeof(phmm_config));
    x.add(haps->seq + hb, (size_t)hl).add(haps->snv_mask_fwd + hb, (size_t)hl).add(haps->snv_prior_fwd + hb, (size_t)hl);
    x.add(haps->snv_mask_rev + hb, (size_t)hl).add(haps->snv_prior_rev + hb, (size_t)hl);
    x.add(haps->gap_open + hb, (size_t)hl).add(haps->gap_extend + hb, (size_t)hl);
    x.value(haps->begin ? haps->begin[h] : (int64_t)0);
    x.add(reads->bases + rb, (size_t)rl).add(reads->quals + rb, (size_t)rl).value(reads->mapq[r]).value(reads->reverse[r]);
    x.value(reads->begin ? reads->begin[r] : (int64_t)0);
    const phmm_flank_state none {0, 0, 0};
    const phmm_flank_state& f = flank ? *flank : none;
    x.value(f.has_flank).value(f.lhs_flank).value(f.rhs_flank);
    if (pos_begin) x.add(pos_begin, (size_t)(pos_end - pos_begin) * sizeof(int32_t));
    *out = x.finish();
    *status = hl < rl ? PHMM_STATUS_SHORT_HAP | (int32_t)((rl - hl) << 16) : PHMM_STATUS_OK;
}

// phmm_populate's host checks, in its order
int check_populate(phmm_engine* e, const phmm_config* cfg, const phmm_haplotypes* haps, const phmm_reads* reads, bool positions, const double* out)
{
    int rc;
    if ((rc = phmm_checks::config_and_output(cfg, out, reads, e->err)) != PHMM_OK) return rc;
    if ((rc = phmm_checks::blocks(haps, reads, e->err)) != PHMM_OK) return rc;
    long long len_min, len_max;
    phmm_checks::read_length_range(reads, &len_min, &len_max);
    const long long hap_bases = haps->off[haps->n];
    if ((rc = phmm_checks::offsets(haps->off[0], hap_bases, reads->off[0], reads->off[reads->n], len_min, len_max, e->err)) != PHMM_OK) return rc;
    long long max_hap = 0;
    for (int h = 0; h < haps->n; ++h) max_hap = std::max<long long>(max_hap, haps->off[h + 1] - haps->off[h]);
    if (!positions && cfg->map_positions && (rc = phmm_checks::mapper_haplotypes(max_hap, hap_bases, e->err)) != PHMM_OK) return rc;
    return phmm_checks::penalties(haps, hap_bases, e->err);
}

// Scores haplotypes [h0, h1) x reads [r0, r1) into out / status at `at`, row-major; returns whether a pair was short.
bool score_block(phmm_engine* e, const phmm_config* cfg, const phmm_haplotypes* haps, int h0, int h1, const phmm_reads* reads, int r0, int r1,
                 const phmm_positions* positions, const phmm_flank_state* flank, double* out, int32_t* status)
{
    bool short_hap = false;
    long long i = 0;
    for (int h = h0; h < h1; ++h) {
        for (int r = r0; r < r1; ++r, ++i) {
            const int32_t* pb = nullptr;
            const int32_t* pe = nullptr;
            if (positions) {
                const long long p = (long long)h * reads->n + r;
                pb = positions->pos + positions->off[p];
                pe = positions->pos + positions->off[p + 1];
            }
            int32_t st;
            score_pair(cfg, haps, h, reads, r, flank, pb, pe, &out[i], &st);
            if (status) status[i] = st;
            short_hap |= (st & 0xFFFF) == PHMM_STATUS_SHORT_HAP;
            e->dp_cells += (haps->off[h + 1] - haps->off[h]) * (reads->off[r + 1] - reads->off[r]);
        }
    }
    return short_hap;
}

int finish(phmm_engine* e, bool short_hap)
{
    if (short_hap) { e->err = "Haplotype is too short for alignment"; return PHMM_ERR_SHORT_HAPLOTYPE; }
    e->err.clear();
    return PHMM_OK;
}

bool covers(const int32_t* first, int n, int total)
{
    if (!first || n < 1 || first[0] != 0 || first[n] != total) return false;
    for (int g = 0; g < n; ++g) if (first[g + 1] <= first[g]) return false;
    return true;
}

} // namespace

long long phmm_checks::populate_chunk_pairs(long long all_pairs)
{
    return std::max<long long>(2LL << 20, std::min<long long>(8LL << 20, all_pairs / 8));
}

extern "C" {

int phmm_create(phmm_engine** out, int)
{
    if (!out) { t_create_error = "null output handle"; return PHMM_ERR_INVALID; }
    *out = new phmm_engine();
    return PHMM_OK;
}

void phmm_destroy(phmm_engine* e)
{
    if (fake::calls_inside() != 0) fake::violation("engine destroyed during a call");
    delete e;
}

const char* phmm_last_error(const phmm_engine* e) { return e ? e->err.c_str() : t_create_error.c_str(); }
int64_t phmm_last_dp_cells(const phmm_engine* e) { return e->dp_cells; }
void* phmm_host_alloc(size_t bytes) { return std::malloc(bytes); }
void phmm_host_free(void* p) { std::free(p); }

int phmm_populate(phmm_engine* e, const phmm_config* cfg, const phmm_haplotypes* haps, const phmm_reads* reads,
                  const phmm_positions* positions, const phmm_flank_state* flank, double* out, int32_t* status, int space)
{
    fake::Entry entry({"populate", 1, haps ? haps->n : 0, cfg ? fake::config_key(cfg) : std::string()});
    e->dp_cells = 0;
    if (space != PHMM_SPACE_HOST) fake::violation("populate outside host memory");
    const bool pos = positions && positions->off && positions->pos;
    int rc;
    if ((rc = check_populate(e, cfg, haps, reads, pos, out)) != PHMM_OK) return rc;
    return finish(e, score_block(e, cfg, haps, 0, haps->n, reads, 0, reads->n, pos ? positions : nullptr, flank, out, status));
}

int phmm_populate_templates(phmm_engine* e, const phmm_config* cfg, const phmm_haplotypes* haps, const phmm_reads* reads,
                            const int64_t* template_off, int32_t n_templates, const phmm_positions* positions,
                            const phmm_flank_state* flank, double* out, int32_t* status, int space)
{
    fake::Entry entry({"populate_templates", 1, haps ? haps->n : 0, cfg ? fake::config_key(cfg) : std::string()});
    e->dp_cells = 0;
    if (space != PHMM_SPACE_HOST) fake::violation("populate_templates outside host memory");
    int rc;
    if ((rc = phmm_checks::template_offsets(template_off, n_templates, reads, true, e->err)) != PHMM_OK) return rc;
    const bool pos = positions && positions->off && positions->pos;
    if ((rc = check_populate(e, cfg, haps, reads, pos, out)) != PHMM_OK) return rc;
    const int H = haps->n, R = reads->n;
    std::vector<double> v((size_t)H * R);
    std::vector<int32_t> st((size_t)H * R);
    const bool short_hap = score_block(e, cfg, haps, 0, H, reads, 0, R, pos ? positions : nullptr, flank, v.data(), st.data());
    if (status) std::memcpy(status, st.data(), st.size() * sizeof(int32_t));
    for (int h = 0; h < H; ++h) {
        for (int t = 0; t < n_templates; ++t) {
            double acc = 0.0;
            for (long long r = template_off[t]; r < template_off[t + 1]; ++r) acc += v[(size_t)h * R + r];
            out[(size_t)h * n_templates + t] = acc;
        }
    }
    return finish(e, short_hap);
}

int phmm_populate_regions(phmm_engine* e, const phmm_config* cfg, const phmm_haplotypes* haps, const phmm_reads* reads,
                          const phmm_regions* regions, double* out, int32_t* status, int space)
{
    fake::Entry entry({"populate_regions", regions ? regions->n : 0, haps ? haps->n : 0, cfg ? fake::config_key(cfg) : std::string()});
    e->dp_cells = 0;
    if (space != PHMM_SPACE_HOST) fake::violation("populate_regions outside host memory");
    if (!regions || !covers(regions->hap_first, regions->n, haps->n) || !covers(regions->read_first, regions->n, reads->n)) {
        fake::violation("region bounds do not cover the blocks");
        e->err = "bad regions";
        return PHMM_ERR_INVALID;
    }
    if (haps->n > 65535) fake::violation("more than 65535 haplotypes in one populate_regions call");
    int rc;
    if ((rc = check_populate(e, cfg, haps, reads, false, out)) != PHMM_OK) return rc;
    bool short_hap = false;
    long long at = 0;
    for (int g = 0; g < regions->n; ++g) {
        const int h0 = regions->hap_first[g], h1 = regions->hap_first[g + 1], r0 = regions->read_first[g], r1 = regions->read_first[g + 1];
        const phmm_flank_state* flank = regions->flank ? &regions->flank[g] : nullptr;
        short_hap |= score_block(e, cfg, haps, h0, h1, reads, r0, r1, nullptr, flank, out + at, status ? status + at : nullptr);
        at += (long long)(h1 - h0) * (r1 - r0);
    }
    return finish(e, short_hap);
}

int phmm_mutation_prime_sets(phmm_engine* e, const phmm_mutation_model* m, int32_t n_sets, const int32_t* set_first,
                             const int64_t* off, const char* seq, double* out, int32_t* status)
{
    fake::Entry entry({"mutation_prime_sets", n_sets, set_first && n_sets > 0 ? set_first[n_sets] : 0, m ? m->key : std::string()});
    e->dp_cells = 0;
    if (!m || !set_first || !off || !seq || !out || !status) { e->err = "null argument"; return PHMM_ERR_INVALID; }
    if (n_sets == 0) return PHMM_OK;
    if (!covers(set_first, n_sets, set_first[n_sets])) fake::violation("set bounds do not cover the block");
    int rc;
    if ((rc = phmm_checks::mutation_offsets(set_first[n_sets], off, e->err)) != PHMM_OK) return rc;
    long long pairs = 0;
    for (int s = 0; s < n_sets; ++s) {
        const long long n = set_first[s + 1] - set_first[s];
        if ((rc = phmm_checks::mutation_haplotype_count(n, e->err)) != PHMM_OK) return rc;
        pairs += n * n;
    }
    if (pairs > PHMM_MUT_MAX_PAIRS) fake::violation("more than PHMM_MUT_MAX_PAIRS pairs in one call");
    long long at = 0;
    for (int s = 0; s < n_sets; ++s) {
        const int first = set_first[s], n = set_first[s + 1] - first;
        for (int t = 0; t < n; ++t) {
            for (int g = 0; g < n; ++g, ++at) {
                const long long t0 = off[first + t], tl = off[first + t + 1] - t0, g0 = off[first + g], gl = off[first + g + 1] - g0;
                fake::Hash x;
                x.add(m->key.data(), m->key.size()).value(tl).add(seq + t0, (size_t)tl).value(gl).add(seq + g0, (size_t)gl);
                out[at] = t == g ? 0.0 : x.finish();
                status[at] = t == g ? PHMM_MUT_SELF : std::abs(tl - gl) >= 32 ? PHMM_MUT_APPROX_LENGTH : PHMM_MUT_HMM;
                e->dp_cells += tl * gl;
            }
        }
    }
    e->err.clear();
    return PHMM_OK;
}

} // extern "C"
