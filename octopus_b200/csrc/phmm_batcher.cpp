// Shared engine for many host threads (include/phmm_b200.h, phmm_batcher_*): the populate requests that concurrent threads
// have in flight are merged into one phmm_populate_regions call. Host C++ over the public C ABI; the batch runs the engine's
// existing regions kernel chain. No thread of its own: the first member of a batch (its leader) makes the call.
#include "../../include/phmm_b200.h"
#include "phmm_checks.h"

#include <algorithm>
#include <chrono>
#include <condition_variable>
#include <cstring>
#include <map>
#include <memory>
#include <mutex>
#include <string>
#include <vector>

namespace {

thread_local std::string t_error;

constexpr long long kMaxBatchHaps = 65535;          // the DP task word's 16-bit haplotype field (phmm_engine.cu, task_word_ok)
constexpr long long kMaxBatchPairs = 4LL << 20;     // (haplotype, read) pairs of one merged call
constexpr int kDefaultMaxWaitUs = 500;

using Clock = std::chrono::steady_clock;

// Element counts of a request or a batch.
struct Sizes {
    long long haps = 0, hap_bases = 0, reads = 0, read_bases = 0, pairs = 0;
    Sizes& operator+=(const Sizes& o) { haps += o.haps; hap_bases += o.hap_bases; reads += o.reads; read_bases += o.read_bases; pairs += o.pairs; return *this; }
    bool within(const Sizes& cap) const { return haps <= cap.haps && hap_bases <= cap.hap_bases && reads <= cap.reads && read_bases <= cap.read_bases && pairs <= cap.pairs; }
    static Sizes max(const Sizes& a, const Sizes& b)
    {
        Sizes s;
        s.haps = std::max(a.haps, b.haps); s.hap_bases = std::max(a.hap_bases, b.hap_bases); s.reads = std::max(a.reads, b.reads);
        s.read_bases = std::max(a.read_bases, b.read_bases); s.pairs = std::max(a.pairs, b.pairs);
        return s;
    }
};

// A page-locked array that only grows. Its contents do not survive a growth; it grows only while no batch uses it.
template <typename T>
struct Pinned {
    T* p = nullptr;
    long long cap = 0;
    Pinned() = default;
    Pinned(const Pinned&) = delete;
    Pinned& operator=(const Pinned&) = delete;
    ~Pinned() { phmm_host_free(p); }
    bool ensure(long long n)
    {
        if (n <= cap) return true;
        const long long want = std::max(n, 2 * cap);
        T* q = static_cast<T*>(phmm_host_alloc((size_t)want * sizeof(T)));
        if (!q) return false;
        phmm_host_free(p);
        p = q; cap = want;
        return true;
    }
};

// One batch's page-locked copy of its members' blocks and its results.
struct Staging {
    Pinned<int64_t> hap_off, hap_begin, read_off, read_begin;
    Pinned<char> seq, mask_f, mask_r, bases;
    Pinned<int8_t> prior_f, prior_r, gap_open, gap_extend;
    Pinned<uint8_t> quals, mapq, reverse;
    Pinned<double> out;
    Pinned<int32_t> status;
    Sizes cap;
    bool busy = false;

    bool grow(const Sizes& s)
    {
        if (s.within(cap)) return true;
        const bool ok = hap_off.ensure(s.haps + 1) && hap_begin.ensure(s.haps) && read_off.ensure(s.reads + 1) && read_begin.ensure(s.reads) &&
                        seq.ensure(s.hap_bases) && mask_f.ensure(s.hap_bases) && mask_r.ensure(s.hap_bases) && prior_f.ensure(s.hap_bases) &&
                        prior_r.ensure(s.hap_bases) && gap_open.ensure(s.hap_bases) && gap_extend.ensure(s.hap_bases) &&
                        bases.ensure(s.read_bases) && quals.ensure(s.read_bases) && mapq.ensure(s.reads) && reverse.ensure(s.reads) &&
                        out.ensure(s.pairs) && status.ensure(s.pairs);
        if (!ok) return false;
        cap.haps = std::min(hap_off.cap - 1, hap_begin.cap);
        cap.reads = std::min({read_off.cap - 1, read_begin.cap, mapq.cap, reverse.cap});
        cap.hap_bases = std::min({seq.cap, mask_f.cap, mask_r.cap, prior_f.cap, prior_r.cap, gap_open.cap, gap_extend.cap});
        cap.read_bases = std::min(bases.cap, quals.cap);
        cap.pairs = std::min(out.cap, status.cap);
        return true;
    }
};

struct Batch {
    phmm_config cfg {};
    std::string key;
    Staging* st = nullptr;
    Sizes used;
    std::vector<int32_t> hap_first {0}, read_first {0};
    std::vector<phmm_flank_state> flanks;
    Clock::time_point deadline;
    int members = 0;
    int pending_copies = 0;     // members that reserved space and have not finished copying in
    int readers = 0;            // members that have not finished copying out
    bool open = true;           // accepts members
    bool full = false;          // a request did not fit: send without waiting for company
    bool done = false;          // the call has returned
    int rc = PHMM_OK;
    std::string err;
};

std::string config_key(const phmm_config* cfg) { return std::string(reinterpret_cast<const char*>(cfg), sizeof(phmm_config)); }

} // namespace

struct phmm_batcher {
    phmm_engine* engine = nullptr;
    int clients = 0;
    int max_wait_us = kDefaultMaxWaitUs;
    mutable std::mutex m;
    std::condition_variable cv;
    std::map<std::string, Batch*> open;               // the open batch of each distinct config
    std::vector<std::unique_ptr<Staging>> staging;
    Sizes want;                                       // staging high-water mark: what merged batches have asked for
    bool engine_busy = false;
    int waiting = 0;                                  // requests in batches not yet sent + requests running alone
    int in_flight = 0;                                // requests inside the batcher
    phmm_batcher_stats stats {};
};

namespace {

void count_call(phmm_batcher* b, int requests)
{
    b->stats.requests += requests;
    b->stats.gpu_calls += 1;
    if (requests > 1) b->stats.merged_calls += 1;
    b->stats.max_regions_per_call = std::max<int64_t>(b->stats.max_regions_per_call, requests);
    b->stats.dp_cells += phmm_last_dp_cells(b->engine);
}

// A request phmm_populate_regions cannot merge: one engine call of its own, in turn with the batches.
int run_alone(phmm_batcher* b, const phmm_config* cfg, const phmm_haplotypes* haps, const phmm_reads* reads, const phmm_positions* positions,
              const int64_t* template_off, int32_t n_templates, const phmm_flank_state* flank, double* out, int32_t* status)
{
    std::unique_lock<std::mutex> lk(b->m);
    ++b->waiting;
    b->cv.notify_all();
    b->cv.wait(lk, [&] { return !b->engine_busy; });
    b->engine_busy = true;
    lk.unlock();
    const int rc = template_off ? phmm_populate_templates(b->engine, cfg, haps, reads, template_off, n_templates, positions, flank, out, status, PHMM_SPACE_HOST)
                                : phmm_populate(b->engine, cfg, haps, reads, positions, flank, out, status, PHMM_SPACE_HOST);
    t_error = rc == PHMM_OK ? std::string() : std::string(phmm_last_error(b->engine));
    lk.lock();
    count_call(b, 1);
    b->engine_busy = false;
    --b->waiting;
    b->cv.notify_all();
    return rc;
}

// A batch for `key` with a free staging set large enough for `need` (grown to the high-water mark); nullptr when out of memory.
Batch* open_batch(phmm_batcher* b, const std::string& key, const phmm_config* cfg, const Sizes& need)
{
    Staging* st = nullptr;
    for (auto& s : b->staging) if (!s->busy) { st = s.get(); break; }
    if (!st) { b->staging.emplace_back(new Staging()); st = b->staging.back().get(); }
    if (!st->grow(Sizes::max(need, b->want))) return nullptr;
    st->busy = true;
    Batch* bt = new Batch();
    bt->cfg = *cfg;
    bt->key = key;
    bt->st = st;
    bt->deadline = Clock::now() + std::chrono::microseconds(b->max_wait_us);
    b->open[key] = bt;
    return bt;
}

void close_batch(phmm_batcher* b, Batch* bt)
{
    if (!bt->open) return;
    bt->open = false;
    const auto it = b->open.find(bt->key);
    if (it != b->open.end() && it->second == bt) b->open.erase(it);
}

// Copy one request into its reserved slot of the staging (outside the lock: each member writes its own ranges only).
void copy_in(Staging* st, const Sizes& at, const phmm_haplotypes* haps, const phmm_reads* reads)
{
    const int H = haps->n, R = reads->n;
    const long long hb = haps->off[H], rb = reads->off[R];
    if (at.haps == 0) st->hap_off.p[0] = 0;
    for (int h = 0; h < H; ++h) st->hap_off.p[at.haps + h + 1] = at.hap_bases + haps->off[h + 1];
    if (haps->begin) std::memcpy(st->hap_begin.p + at.haps, haps->begin, (size_t)H * sizeof(int64_t));
    else std::memset(st->hap_begin.p + at.haps, 0, (size_t)H * sizeof(int64_t));
    std::memcpy(st->seq.p + at.hap_bases, haps->seq, (size_t)hb);
    std::memcpy(st->mask_f.p + at.hap_bases, haps->snv_mask_fwd, (size_t)hb);
    std::memcpy(st->prior_f.p + at.hap_bases, haps->snv_prior_fwd, (size_t)hb);
    std::memcpy(st->mask_r.p + at.hap_bases, haps->snv_mask_rev, (size_t)hb);
    std::memcpy(st->prior_r.p + at.hap_bases, haps->snv_prior_rev, (size_t)hb);
    std::memcpy(st->gap_open.p + at.hap_bases, haps->gap_open, (size_t)hb);
    std::memcpy(st->gap_extend.p + at.hap_bases, haps->gap_extend, (size_t)hb);
    if (at.reads == 0) st->read_off.p[0] = 0;
    for (int r = 0; r < R; ++r) st->read_off.p[at.reads + r + 1] = at.read_bases + reads->off[r + 1];
    if (reads->begin) std::memcpy(st->read_begin.p + at.reads, reads->begin, (size_t)R * sizeof(int64_t));
    else std::memset(st->read_begin.p + at.reads, 0, (size_t)R * sizeof(int64_t));
    std::memcpy(st->bases.p + at.read_bases, reads->bases, (size_t)rb);
    std::memcpy(st->quals.p + at.read_bases, reads->quals, (size_t)rb);
    std::memcpy(st->mapq.p + at.reads, reads->mapq, (size_t)R);
    std::memcpy(st->reverse.p + at.reads, reads->reverse, (size_t)R);
}

// The leader's call: the batch's members as the regions of one phmm_populate_regions call.
void run_batch(phmm_batcher* b, Batch* bt)
{
    Staging* st = bt->st;
    const phmm_haplotypes hv {(int32_t)bt->used.haps, st->hap_off.p, st->seq.p, st->mask_f.p, st->prior_f.p, st->mask_r.p, st->prior_r.p,
                              st->gap_open.p, st->gap_extend.p, st->hap_begin.p};
    const phmm_reads rv {(int32_t)bt->used.reads, st->read_off.p, st->bases.p, st->quals.p, st->mapq.p, st->reverse.p, st->read_begin.p};
    const phmm_regions regions {bt->members, bt->hap_first.data(), bt->read_first.data(), bt->flanks.data()};
    bt->rc = phmm_populate_regions(b->engine, &bt->cfg, &hv, &rv, &regions, st->out.p, st->status.p, PHMM_SPACE_HOST);
    if (bt->rc != PHMM_OK) bt->err = phmm_last_error(b->engine);
}

// The host-side checks of phmm_populate, in its order, for a request without position lists. Sets *alone when the request has to
// run on its own (pipelined size, too many haplotypes, a haplotype too long for the task word); the remaining checks are then
// phmm_populate's own.
int check_request(const phmm_config* cfg, const phmm_haplotypes* haps, const phmm_reads* reads, const double* out, bool* alone, Sizes* need)
{
    int rc;
    if ((rc = phmm_checks::config_and_output(cfg, out, reads, t_error)) != PHMM_OK) return rc;
    if ((rc = phmm_checks::blocks(haps, reads, t_error)) != PHMM_OK) return rc;
    const long long pairs = (long long)haps->n * reads->n;
    if (pairs >= 2 * phmm_checks::populate_chunk_pairs(pairs) || haps->n > kMaxBatchHaps) { *alone = true; return PHMM_OK; }
    long long len_min, len_max;
    phmm_checks::read_length_range(reads, &len_min, &len_max);
    const long long hap_bases = haps->off[haps->n], read_bases = reads->off[reads->n];
    if ((rc = phmm_checks::offsets(haps->off[0], hap_bases, reads->off[0], read_bases, len_min, len_max, t_error)) != PHMM_OK) return rc;
    long long max_hap = 0;
    for (int h = 0; h < haps->n; ++h) max_hap = std::max<long long>(max_hap, haps->off[h + 1] - haps->off[h]);
    if (cfg->map_positions && (rc = phmm_checks::mapper_haplotypes(max_hap, hap_bases, t_error)) != PHMM_OK) return rc;
    if (max_hap > 65535) { *alone = true; return PHMM_OK; }
    if ((rc = phmm_checks::penalties(haps, hap_bases, t_error)) != PHMM_OK) return rc;
    need->haps = haps->n; need->hap_bases = hap_bases; need->reads = reads->n; need->read_bases = read_bases; need->pairs = pairs;
    return PHMM_OK;
}

int submit(phmm_batcher* b, const phmm_config* cfg, const phmm_haplotypes* haps, const phmm_reads* reads, const phmm_positions* positions,
           const int64_t* template_off, int32_t n_templates, const phmm_flank_state* flank, double* out, int32_t* status)
{
    bool alone = positions && positions->off && positions->pos;
    Sizes need;
    if (!alone) {
        const int rc = check_request(cfg, haps, reads, out, &alone, &need);
        if (rc != PHMM_OK) return rc;
    }
    if (alone) return run_alone(b, cfg, haps, reads, positions, template_off, n_templates, flank, out, status);

    const std::string key = config_key(cfg);
    std::unique_lock<std::mutex> lk(b->m);
    Batch* bt = nullptr;
    for (;;) {
        const auto it = b->open.find(key);
        if (it == b->open.end()) {
            bt = open_batch(b, key, cfg, need);
            if (!bt) { t_error = "out of page-locked host memory for the batch staging"; return PHMM_ERR_NOMEM; }
            break;
        }
        bt = it->second;
        Sizes total = bt->used;
        total += need;
        if (total.haps <= kMaxBatchHaps && total.pairs <= kMaxBatchPairs && total.within(bt->st->cap)) break;
        if (total.haps <= kMaxBatchHaps && total.pairs <= kMaxBatchPairs) b->want = Sizes::max(b->want, total);   // staging too small
        bt->full = true;
        close_batch(b, bt);
        b->cv.notify_all();
    }
    const Sizes at = bt->used;
    bt->used += need;
    bt->hap_first.push_back((int32_t)bt->used.haps);
    bt->read_first.push_back((int32_t)bt->used.reads);
    bt->flanks.push_back(flank ? *flank : phmm_flank_state {0, 0, 0});
    const bool leader = bt->members == 0;
    ++bt->members; ++bt->pending_copies; ++bt->readers; ++b->waiting;
    b->cv.notify_all();
    lk.unlock();

    copy_in(bt->st, at, haps, reads);

    lk.lock();
    --bt->pending_copies;
    if (leader) {
        for (;;) {
            const bool company = b->clients > 0 && b->waiting >= b->clients;
            const bool go = bt->full || company || Clock::now() >= bt->deadline;
            if (go && !b->engine_busy) break;
            if (go) b->cv.wait(lk);
            else b->cv.wait_until(lk, bt->deadline);
        }
        close_batch(b, bt);
        b->engine_busy = true;
        b->waiting -= bt->members;
        b->cv.wait(lk, [&] { return bt->pending_copies == 0; });
        lk.unlock();
        run_batch(b, bt);
        lk.lock();
        count_call(b, bt->members);
        b->engine_busy = false;
        bt->done = true;
        b->cv.notify_all();
    } else {
        b->cv.notify_all();                       // the leader may be waiting for this copy
        b->cv.wait(lk, [&] { return bt->done; });
    }
    lk.unlock();

    // this member's slice of the result: [H][R] at the pair offset of its region
    int rc = bt->rc;
    const int H = haps->n, R = reads->n;
    const double* res = bt->st->out.p + at.pairs;
    const int32_t* res_status = bt->st->status.p + at.pairs;
    if (rc == PHMM_OK || rc == PHMM_ERR_SHORT_HAPLOTYPE) {
        rc = PHMM_OK;
        for (long long i = 0; i < need.pairs; ++i) if ((res_status[i] & 0xFFFF) == PHMM_STATUS_SHORT_HAP) { rc = PHMM_ERR_SHORT_HAPLOTYPE; break; }
        t_error = rc == PHMM_OK ? std::string() : std::string("Haplotype is too short for alignment");
        if (status) std::memcpy(status, res_status, (size_t)need.pairs * sizeof(int32_t));
        if (template_off) {
            // k_template_sum's order: each template's reads left to right from 0.0
            for (int h = 0; h < H; ++h) {
                for (int t = 0; t < n_templates; ++t) {
                    double acc = 0.0;
                    for (long long r = template_off[t]; r < template_off[t + 1]; ++r) acc += res[(size_t)h * R + r];
                    out[(size_t)h * n_templates + t] = acc;
                }
            }
        } else {
            std::memcpy(out, res, (size_t)need.pairs * sizeof(double));
        }
    } else {
        t_error = bt->err;
    }

    lk.lock();
    if (--bt->readers == 0) {
        bt->st->busy = false;
        delete bt;
    }
    return rc;
}

// Entry and exit of every request: destroy waits until no request is inside.
struct InFlight {
    phmm_batcher* b;
    explicit InFlight(phmm_batcher* batcher) : b(batcher) { std::lock_guard<std::mutex> lk(b->m); ++b->in_flight; }
    ~InFlight() { std::lock_guard<std::mutex> lk(b->m); --b->in_flight; b->cv.notify_all(); }
};

} // namespace

extern "C" {

int phmm_batcher_create(phmm_batcher** out, int device, const phmm_batcher_options* opt)
{
    if (!out) { t_error = "null output handle"; return PHMM_ERR_INVALID; }
    *out = nullptr;
    if (opt && (opt->clients < 0 || opt->max_wait_us < 0)) { t_error = "clients and max_wait_us must be >= 0"; return PHMM_ERR_INVALID; }
    phmm_engine* e = nullptr;
    const int rc = phmm_create(&e, device);
    if (rc != PHMM_OK) { t_error = phmm_last_error(nullptr); return rc; }
    phmm_batcher* b = new phmm_batcher();
    b->engine = e;
    if (opt) { b->clients = opt->clients; b->max_wait_us = opt->max_wait_us; }
    // first staging size: some tens of regions of a few hundred reads; it grows to what merged batches ask for
    b->want.haps = 4096; b->want.hap_bases = 1LL << 20; b->want.reads = 1LL << 16; b->want.read_bases = 8LL << 20; b->want.pairs = 1LL << 20;
    *out = b;
    return PHMM_OK;
}

void phmm_batcher_destroy(phmm_batcher* b)
{
    if (!b) return;
    {
        std::unique_lock<std::mutex> lk(b->m);
        b->cv.wait(lk, [&] { return b->in_flight == 0; });
    }
    phmm_destroy(b->engine);
    delete b;
}

const char* phmm_batcher_last_error(void) { return t_error.c_str(); }

int phmm_batcher_populate(phmm_batcher* b, const phmm_config* cfg, const phmm_haplotypes* haps, const phmm_reads* reads,
                          const phmm_positions* positions, const phmm_flank_state* flank, double* out, int32_t* status)
{
    if (!b) { t_error = "null batcher"; return PHMM_ERR_INVALID; }
    InFlight guard(b);
    return submit(b, cfg, haps, reads, positions, nullptr, 0, flank, out, status);
}

int phmm_batcher_populate_templates(phmm_batcher* b, const phmm_config* cfg, const phmm_haplotypes* haps, const phmm_reads* reads,
                                    const int64_t* template_off, int32_t n_templates, const phmm_flank_state* flank,
                                    double* out, int32_t* status)
{
    if (!b) { t_error = "null batcher"; return PHMM_ERR_INVALID; }
    const int rc = phmm_checks::template_offsets(template_off, n_templates, reads, true, t_error);
    if (rc != PHMM_OK) return rc;
    InFlight guard(b);
    return submit(b, cfg, haps, reads, nullptr, template_off, n_templates, flank, out, status);
}

int phmm_batcher_stats_get(const phmm_batcher* b, phmm_batcher_stats* out)
{
    if (!b || !out) return PHMM_ERR_INVALID;
    std::lock_guard<std::mutex> lk(b->m);
    *out = b->stats;
    return PHMM_OK;
}

} // extern "C"
