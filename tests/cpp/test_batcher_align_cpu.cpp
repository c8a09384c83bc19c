// The request batcher's assign and realign requests (octopus_b200/csrc/phmm_batcher.cpp, phmm_batcher_align.cpp) against the CPU
// fakes of the engine (tests/cpp/fake_engine.cpp for populate and mutation, tests/cpp/fake_engine_align.cpp for assign and realign),
// from many std::threads. Built and run under ThreadSanitizer and under AddressSanitizer + UBSan by tests/test_batcher_align_cpu.py.
// Every request's return code, message and outputs must equal what the fake engine gives it alone, bit for bit: top, lnl and status
// of an assign request (its statuses only when it returns PHMM_ERR_SHORT_HAPLOTYPE), mapping position, likelihood, status and the
// CIGAR text up to its NUL of a realign request. The batcher's DP-cell count must be the sum of its requests' counts alone, and its
// page-locked staging must stay within what its batches need (phmm_host_alloc is wrapped: the build links with
// -Wl,--wrap=phmm_host_alloc). Exits non-zero on any mismatch.
#include "../../include/phmm_b200.h"
#include "../../octopus_b200/csrc/phmm_mutation.h"

#include <algorithm>
#include <atomic>
#include <cstdio>
#include <cstring>
#include <mutex>
#include <random>
#include <string>
#include <thread>
#include <vector>

namespace fake {
struct Call { std::string entry; int members; long long haps; std::string key; };
std::vector<Call> calls();
std::vector<std::string> violations();
void clear_calls();
void set_call_delay_us(int us);
} // namespace fake

namespace fake_align {
struct Call { std::string entry; int members; long long haps; int32_t stride; };
std::vector<Call> calls();
void clear_calls();
} // namespace fake_align

// Every page-locked allocation the batcher makes: the largest one and the total since the last reset.
std::atomic<long long> g_alloc_largest {0}, g_alloc_total {0};

extern "C" void* __real_phmm_host_alloc(size_t bytes);
extern "C" void* __wrap_phmm_host_alloc(size_t bytes)
{
    long long prev = g_alloc_largest.load();
    while ((long long)bytes > prev && !g_alloc_largest.compare_exchange_weak(prev, (long long)bytes)) {}
    g_alloc_total += (long long)bytes;
    return __real_phmm_host_alloc(bytes);
}

namespace {

std::mutex g_report_m;
int g_failures = 0;

void fail(const std::string& what)
{
    std::lock_guard<std::mutex> lk(g_report_m);
    ++g_failures;
    if (g_failures <= 50) std::fprintf(stderr, "FAIL %s\n", what.c_str());
}

void expect(bool ok, const std::string& what) { if (!ok) fail(what); }

const char kAcgt[] = "ACGT";

std::string random_bases(std::mt19937& rng, int n)
{
    std::string s((size_t)n, 'A');
    for (auto& c : s) c = kAcgt[rng() % 4];
    return s;
}

// Two blocks of one request.
struct Blocks {
    std::vector<int64_t> hap_off {0}, hap_begin, read_off {0}, read_begin;
    std::string seq, mask_f, mask_r, bases;
    std::vector<int8_t> prior_f, prior_r, gap_open, gap_extend;
    std::vector<uint8_t> quals, mapq, reverse;
    bool no_mapq = false, no_begin = false;

    void add_haplotype(const std::string& s, int64_t begin, int8_t seed)
    {
        for (size_t i = 0; i < s.size(); ++i) {
            seq += s[i];
            mask_f += s[(i + 1) % s.size()];
            mask_r += s[(i + s.size() - 1) % s.size()];
            prior_f.push_back((int8_t)(1 + (seed + i) % 100)); prior_r.push_back((int8_t)(2 + (seed + i) % 90));
            gap_open.push_back((int8_t)(3 + (seed + i) % 40)); gap_extend.push_back((int8_t)(1 + (seed + i) % 10));
        }
        hap_off.push_back((int64_t)seq.size());
        hap_begin.push_back(begin);
    }
    void add_read(const std::string& b, std::mt19937& rng)
    {
        bases += b;
        for (size_t i = 0; i < b.size(); ++i) quals.push_back((uint8_t)(2 + rng() % 40));
        read_off.push_back((int64_t)bases.size());
        mapq.push_back((uint8_t)(rng() % 2 ? 60 : 20));
        reverse.push_back((uint8_t)(rng() % 2));
        read_begin.push_back((int64_t)(rng() % 1000));
    }
    int n_haps() const { return (int)hap_begin.size(); }
    int n_reads() const { return (int)read_begin.size(); }
    phmm_haplotypes haps() const
    {
        return {n_haps(), hap_off.data(), seq.data(), mask_f.data(), prior_f.data(), mask_r.data(), prior_r.data(), gap_open.data(),
                gap_extend.data(), no_begin ? nullptr : hap_begin.data()};
    }
    phmm_reads reads() const
    {
        return {n_reads(), read_off.data(), bases.data(), quals.data(), no_mapq ? nullptr : mapq.data(), reverse.data(),
                no_begin ? nullptr : read_begin.data()};
    }
};

phmm_config make_config(int band, bool map_positions, bool use_mapq, bool use_flank)
{
    phmm_config c;
    c.max_indel_error = band; c.use_int_scores = 0; c.use_mapping_quality = use_mapq ? 1 : 0; c.mapping_quality_cap = 120;
    c.mapping_quality_cap_trigger = -1; c.use_flank_state = use_flank ? 1 : 0; c.nuc_prior = 2; c.disable_naive_shortcut = 0;
    c.map_positions = map_positions ? 1 : 0;
    return c;
}

enum Kind { ASSIGN, REALIGN, POPULATE, MUTATION };

struct Request {
    Kind kind = ASSIGN;
    phmm_config cfg {};
    Blocks g;
    std::vector<int32_t> hap_first {0}, read_first {0};    // ASSIGN
    std::vector<phmm_flank_state> group_flanks;
    std::vector<double> priors;                             // ASSIGN: empty = NULL
    bool want_lnl = true, want_status = true;
    std::vector<phmm_pair> pairs;                           // REALIGN
    int32_t stride = 64;
    bool has_flank = false;                                 // REALIGN, POPULATE
    phmm_flank_state flank {0, 0, 0};
    bool bad_groups = false;                                // ASSIGN: group bounds that do not cover the blocks
    std::string model_key;                                  // MUTATION
    std::vector<int64_t> mut_off {0};
    std::string mut_seq;
};

struct Result {
    int rc = 0;
    std::string msg;
    std::vector<uint64_t> top;
    std::vector<double> values;
    std::vector<int32_t> status;
    std::vector<int64_t> mapping_position;
    std::vector<std::string> cigar;
};

// An assign request: 1-5 groups of 1-4 haplotypes (a copy of a haplotype ties with it) and 1-30 reads each.
Request assign_request(std::mt19937& rng, const phmm_config& cfg)
{
    Request q;
    q.kind = ASSIGN;
    q.cfg = cfg;
    const int G = 1 + (int)(rng() % 5);
    for (int gi = 0; gi < G; ++gi) {
        const int len = 150 + (int)(rng() % 100);
        const std::string base = random_bases(rng, len);
        const int H = 1 + (int)(rng() % 4), R = 1 + (int)(rng() % 30);
        const int64_t begin = (int64_t)(rng() % 500);
        for (int h = 0; h < H; ++h) {
            std::string s = base;
            if (h != 2) s[rng() % s.size()] = kAcgt[rng() % 4];
            if (h == 2) { s = q.g.seq.substr((size_t)q.g.hap_off[q.g.hap_off.size() - 2]); }    // a copy of the group's previous haplotype
            q.g.add_haplotype(s, h == 2 ? q.g.hap_begin.back() : begin, (int8_t)(h == 2 ? (h - 1) : h));
        }
        for (int r = 0; r < R; ++r) {
            const int rl = 30 + (int)(rng() % 70);
            q.g.add_read(base.substr(rng() % (size_t)(len - rl + 1), (size_t)rl), rng);
        }
        q.hap_first.push_back(q.g.n_haps());
        q.read_first.push_back(q.g.n_reads());
        q.group_flanks.push_back({(int32_t)(rng() % 2), (int64_t)(rng() % 50), (int64_t)(rng() % 50)});
    }
    if (rng() % 2) for (int h = 0; h < q.g.n_haps(); ++h) q.priors.push_back(-(double)(rng() % 5));
    q.want_lnl = rng() % 3 != 0;
    q.want_status = rng() % 3 != 0;
    return q;
}

// A realign request: 1-3 haplotypes, 1-40 reads (one in eight an exact copy of a haplotype's start), every read against one or two
// haplotypes, at a stride from 8 up.
Request realign_request(std::mt19937& rng, const phmm_config& cfg)
{
    Request q;
    q.kind = REALIGN;
    q.cfg = cfg;
    const int H = 1 + (int)(rng() % 3), R = 1 + (int)(rng() % 40);
    const int len = 200 + (int)(rng() % 200);
    const std::string base = random_bases(rng, len);
    for (int h = 0; h < H; ++h) {
        std::string s = base;
        s[rng() % s.size()] = kAcgt[rng() % 4];
        q.g.add_haplotype(s, (int64_t)(rng() % 100), (int8_t)h);
    }
    for (int r = 0; r < R; ++r) {
        const int rl = 20 + (int)(rng() % 150);
        if (rng() % 8 == 0) q.g.add_read(q.g.seq.substr(0, (size_t)rl), rng);
        else q.g.add_read(base.substr(rng() % (size_t)(len - rl + 1), (size_t)rl), rng);
        q.pairs.push_back({r, (int32_t)(rng() % H)});
        if (rng() % 2) q.pairs.push_back({r, (int32_t)(rng() % H)});
    }
    static const int32_t strides[] = {8, 12, 16, 40, 64, 128, 700};
    q.stride = strides[rng() % 7];
    q.has_flank = rng() % 2;
    q.flank = {q.has_flank ? 1 : 0, (int64_t)(rng() % 50), (int64_t)(rng() % 50)};
    q.g.no_mapq = !cfg.use_mapping_quality && rng() % 2;
    q.g.no_begin = rng() % 4 == 0;
    return q;
}

Request populate_request(std::mt19937& rng, const phmm_config& cfg)
{
    Request q;
    q.kind = POPULATE;
    q.cfg = cfg;
    const int len = 150 + (int)(rng() % 80);
    const std::string base = random_bases(rng, len);
    for (int h = 0, H = 1 + (int)(rng() % 8); h < H; ++h) { std::string s = base; s[rng() % s.size()] = 'T'; q.g.add_haplotype(s, 0, (int8_t)h); }
    for (int r = 0, R = 1 + (int)(rng() % 30); r < R; ++r) q.g.add_read(base.substr(rng() % (size_t)(len - 60), 50), rng);
    q.has_flank = rng() % 2;
    q.flank = {q.has_flank ? 1 : 0, 10, 20};
    return q;
}

Request mutation_request(std::mt19937& rng)
{
    Request q;
    q.kind = MUTATION;
    q.model_key = "model A";
    const std::string base = random_bases(rng, 60 + (int)(rng() % 100));
    for (int h = 0, n = 1 + (int)(rng() % 8); h < n; ++h) {
        std::string s = base;
        s[rng() % s.size()] = kAcgt[rng() % 4];
        q.mut_seq += s;
        q.mut_off.push_back((int64_t)q.mut_seq.size());
    }
    return q;
}

std::vector<std::string> texts(const std::vector<char>& cig, size_t n, int32_t stride)
{
    std::vector<std::string> t;
    for (size_t j = 0; j < n; ++j) t.emplace_back(cig.data() + j * (size_t)stride, strnlen(cig.data() + j * (size_t)stride, (size_t)stride));
    return t;
}

// The request through the batcher (b) or alone on an engine of its own (e).
Result run(phmm_batcher* b, phmm_engine* e, const Request& q)
{
    Result res;
    const phmm_haplotypes haps = q.g.haps();
    const phmm_reads reads = q.g.reads();
    if (q.kind == ASSIGN) {
        std::vector<int32_t> hf = q.hap_first;
        if (q.bad_groups) hf.back() += 1;
        const phmm_regions groups {(int32_t)hf.size() - 1, hf.data(), q.read_first.data(), q.group_flanks.data()};
        size_t P = 0;
        for (size_t g = 0; g + 1 < q.hap_first.size(); ++g) P += (size_t)(q.hap_first[g + 1] - q.hap_first[g]) * (size_t)(q.read_first[g + 1] - q.read_first[g]);
        res.top.assign((size_t)reads.n, 0x5a5a5a5aULL);
        if (q.want_lnl) res.values.assign(P, -7.0);
        if (q.want_status) res.status.assign(P, -7);
        const double* pri = q.priors.empty() ? nullptr : q.priors.data();
        double* lnl = q.want_lnl ? res.values.data() : nullptr;
        int32_t* st = q.want_status ? res.status.data() : nullptr;
        res.rc = b ? phmm_batcher_assign_reads(b, &q.cfg, &haps, &reads, &groups, pri, res.top.data(), lnl, st)
                   : phmm_assign_reads(e, &q.cfg, &haps, &reads, &groups, pri, res.top.data(), lnl, st, PHMM_SPACE_HOST);
    } else if (q.kind == REALIGN) {
        const size_t n = q.pairs.size();
        res.mapping_position.assign(n, -7);
        res.values.assign(n, -7.0);
        res.status.assign(n, -7);
        std::vector<char> cig(n * (size_t)q.stride + 1, 'z');
        const phmm_flank_state* flank = q.has_flank ? &q.flank : nullptr;
        res.rc = b ? phmm_batcher_realign_reads(b, &q.cfg, &haps, &reads, q.pairs.data(), (int64_t)n, flank, res.mapping_position.data(),
                                                res.values.data(), cig.data(), q.stride, res.status.data())
                   : phmm_realign_reads(e, &q.cfg, &haps, &reads, q.pairs.data(), (int64_t)n, flank, res.mapping_position.data(),
                                        res.values.data(), cig.data(), q.stride, res.status.data(), PHMM_SPACE_HOST);
        res.cigar = texts(cig, n, q.stride);
    } else if (q.kind == POPULATE) {
        res.values.assign((size_t)haps.n * reads.n, -7.0);
        res.status.assign((size_t)haps.n * reads.n, -7);
        const phmm_flank_state* flank = q.has_flank ? &q.flank : nullptr;
        res.rc = b ? phmm_batcher_populate(b, &q.cfg, &haps, &reads, nullptr, flank, res.values.data(), res.status.data())
                   : phmm_populate(e, &q.cfg, &haps, &reads, nullptr, flank, res.values.data(), res.status.data(), PHMM_SPACE_HOST);
    } else {
        const int n = (int)q.mut_off.size() - 1;
        phmm_mutation_model m;
        m.key = q.model_key;
        res.values.assign((size_t)n * n, -7.0);
        res.status.assign((size_t)n * n, -7);
        const int32_t set_first[2] = {0, n};
        res.rc = b ? phmm_batcher_mutation_prime(b, &m, n, q.mut_off.data(), q.mut_seq.data(), res.values.data(), res.status.data())
                   : phmm_mutation_prime_sets(e, &m, 1, set_first, q.mut_off.data(), q.mut_seq.data(), res.values.data(), res.status.data());
    }
    res.msg = res.rc == PHMM_OK ? "" : (b ? phmm_batcher_last_error() : phmm_last_error(e));
    return res;
}

void compare(const std::string& name, const Request& q, const Result& got, const Result& want)
{
    if (got.rc != want.rc || got.msg != want.msg) {
        fail(name + ": rc " + std::to_string(got.rc) + " '" + got.msg + "', alone " + std::to_string(want.rc) + " '" + want.msg + "'");
        return;
    }
    if (got.rc != PHMM_OK && got.rc != PHMM_ERR_SHORT_HAPLOTYPE) return;
    expect(got.status == want.status, name + ": statuses differ from alone");
    if (q.kind == ASSIGN && got.rc == PHMM_ERR_SHORT_HAPLOTYPE) return;        // top and lnl unspecified
    expect(got.values.size() == want.values.size() &&
           (got.values.empty() || std::memcmp(got.values.data(), want.values.data(), got.values.size() * sizeof(double)) == 0),
           name + ": values differ from alone");
    expect(got.top == want.top, name + ": top sets differ from alone");
    expect(got.mapping_position == want.mapping_position, name + ": mapping positions differ from alone");
    expect(got.cigar == want.cigar, name + ": CIGAR texts differ from alone");
}

struct Stats {
    phmm_batcher_stats s;
    int64_t reruns;
    int64_t solo_cells;          // the requests' DP cells alone, summed
};

// The requests' solo results first (one engine, one thread), then the requests through one batcher from n_threads threads, request i
// on thread i % n_threads; each compared with its solo result. Returns the batcher's stats and rerun count.
Stats check(const std::string& name, const std::vector<Request>& requests, int n_threads, int clients, int max_wait_us)
{
    phmm_engine* e = nullptr;
    phmm_create(&e, 0);
    std::vector<Result> want;
    int64_t solo_cells = 0;
    for (const auto& q : requests) {
        want.push_back(run(nullptr, e, q));
        solo_cells += phmm_last_dp_cells(e);
    }
    phmm_destroy(e);
    fake::clear_calls();
    fake_align::clear_calls();
    phmm_batcher* b = nullptr;
    const phmm_batcher_options opt {clients, max_wait_us};
    if (phmm_batcher_create(&b, 0, &opt) != PHMM_OK) { fail(name + ": batcher creation"); return {}; }
    std::vector<Result> got(requests.size());
    std::atomic<int> ready {0};
    std::vector<std::thread> threads;
    for (int k = 0; k < n_threads; ++k) {
        threads.emplace_back([&, k] {
            ++ready;
            while (ready.load() < n_threads) std::this_thread::yield();
            for (size_t i = (size_t)k; i < requests.size(); i += (size_t)n_threads) got[i] = run(b, nullptr, requests[i]);
        });
    }
    for (auto& t : threads) t.join();
    Stats s {};
    s.solo_cells = solo_cells;
    phmm_batcher_stats_get(b, &s.s);
    s.reruns = phmm_batcher_reruns(b);
    phmm_batcher_destroy(b);
    for (size_t i = 0; i < requests.size(); ++i) compare(name + " request " + std::to_string(i), requests[i], got[i], want[i]);
    return s;
}

int merged_calls_of(const std::string& entry)
{
    int n = 0;
    for (const auto& c : fake_align::calls()) if (c.entry == entry && c.members > 1) ++n;
    return n;
}

// assign, realign, populate and mutation requests interleaved on the same threads; several configs; strides from 8; priors present
// and absent in one batch; short haplotypes; requests that fail their own checks
void mixed(std::mt19937& rng)
{
    const phmm_config cfgs[] = {make_config(8, false, false, false), make_config(16, true, true, true), make_config(8, true, false, true)};
    std::vector<Request> requests;
    for (int i = 0; i < 320; ++i) {
        const phmm_config& cfg = cfgs[rng() % 3];
        switch (i % 8) {
            case 0: case 1: case 2: requests.push_back(assign_request(rng, cfg)); break;
            case 3: case 4: case 5: requests.push_back(realign_request(rng, cfg)); break;
            case 6: requests.push_back(populate_request(rng, cfg)); break;
            default: requests.push_back(mutation_request(rng)); break;
        }
        Request& q = requests.back();
        if (i % 37 == 5 && q.kind == ASSIGN) q.bad_groups = true;                        // fails its own region check
        if (i % 41 == 4 && q.kind == REALIGN) q.pairs.back().hap = 99;                   // fails its own pair check
        if (i % 29 == 3 && q.kind == REALIGN) q.stride = 4;                              // fails its own stride check
        if (i % 23 == 1 && q.kind == ASSIGN) {                                           // a read longer than its group's haplotypes
            q.g.add_read(std::string(400, 'C'), rng);
            q.read_first.back() = q.g.n_reads();
        }
        if (i % 19 == 2 && q.kind == REALIGN) {                                          // likewise
            q.g.add_read(std::string(500, 'G'), rng);
            q.pairs.push_back({q.g.n_reads() - 1, 0});
        }
    }
    fake::set_call_delay_us(200);
    for (int threads : {4, 16}) {
        const Stats s = check("mixed x" + std::to_string(threads), requests, threads, threads, 2000);
        expect(s.s.merged_calls > 0, "mixed: no merged call");
        expect(merged_calls_of("assign_reads") > 0, "mixed: no merged assign call");
        expect(merged_calls_of("realign_reads") > 0, "mixed: no merged realign call");
        expect(s.reruns == 0, "mixed: a rerun without a failing merged call");
        expect(s.s.dp_cells == s.solo_cells, "mixed: DP cells " + std::to_string(s.s.dp_cells) + ", alone " + std::to_string(s.solo_cells));
    }
    fake::set_call_delay_us(0);
}

// One realign request at every stride from 8 to 48 and at 700, merged: each text ends up cut, exactly fitting or whole at its own
// stride, as alone.
void strides(std::mt19937& rng)
{
    const Request base = realign_request(rng, make_config(16, true, true, false));
    std::vector<Request> requests;
    for (int32_t s = 8; s <= 48; ++s) { requests.push_back(base); requests.back().stride = s; }
    requests.push_back(base);
    requests.back().stride = 700;
    fake::set_call_delay_us(200);
    check("strides", requests, 14, 14, 20000);
    fake::set_call_delay_us(0);
    expect(merged_calls_of("realign_reads") > 0, "strides: no merged realign call");
}

// A merged assign or realign call that fails for one member's marker read: the leader reruns every member alone; each gets its solo
// result and message, the rerun is counted, and the DP cells of the reruns count.
void rerun(std::mt19937& rng)
{
    const phmm_config cfg = make_config(8, true, false, false);
    for (const Kind kind : {ASSIGN, REALIGN}) {
        const std::string name = kind == ASSIGN ? "rerun assign" : "rerun realign";
        std::vector<Request> requests;
        for (int i = 0; i < 8; ++i) requests.push_back(kind == ASSIGN ? assign_request(rng, cfg) : realign_request(rng, cfg));
        Request& bad = requests[3];
        bad.g.bases.replace((size_t)bad.g.read_off[0], 4, kind == ASSIGN ? "MMMM" : "RRRR");
        fake::set_call_delay_us(2000);
        const Stats s = check(name, requests, 8, 8, 100000);
        fake::set_call_delay_us(0);
        expect(s.reruns == 1, name + ": reruns " + std::to_string(s.reruns) + ", expected 1");
        expect(fake_align::calls().size() == 9, name + ": " + std::to_string(fake_align::calls().size()) + " calls, expected the merged call and one per member");
        expect(s.s.gpu_calls == 9, name + ": gpu_calls " + std::to_string(s.s.gpu_calls) + ", expected 9");
        expect(s.s.dp_cells == s.solo_cells && s.solo_cells > 0, name + ": DP cells " + std::to_string(s.s.dp_cells) + ", alone " + std::to_string(s.solo_cells));
    }
}

// A realign request of n_reads reads of read_len bases against one haplotype, every read paired with it once, at the C++ adapter's
// stride (4 x the longest read + 64).
Request realign_block(std::mt19937& rng, const phmm_config& cfg, int n_reads, int read_len)
{
    Request q;
    q.kind = REALIGN;
    q.cfg = cfg;
    const std::string hap = random_bases(rng, read_len + 200);
    q.g.add_haplotype(hap, 0, 1);
    for (int r = 0; r < n_reads; ++r) {
        std::string b = hap.substr(1 + rng() % 150, (size_t)read_len);
        b[0] = b[0] == 'A' ? 'C' : 'A';
        q.g.add_read(b, rng);
        q.pairs.push_back({r, 0});
    }
    q.stride = 4 * read_len + 64;
    return q;
}

// The realign staging's page-locked memory follows the CIGAR bytes batches really write (pairs x the batch's largest stride), not the
// largest pair count times the largest stride seen apart: one 15-kb read alone, and a 15-kb read after a merged batch of 16 000
// short-read pairs, each stay within a few MiB of what they need (a merged batch's CIGAR staging is bounded by 128 MiB, and a growing
// set at most doubles it).
void pinned(std::mt19937& rng)
{
    const phmm_config cfg = make_config(8, false, false, false);
    const Request hifi = realign_block(rng, cfg, 1, 15000);            // 60 KB of CIGAR text at its stride
    g_alloc_largest = 0;
    g_alloc_total = 0;
    check("pinned long read", {hifi}, 1, 1, 100);
    expect(g_alloc_largest.load() <= (8LL << 20), "pinned long read: a page-locked allocation of " + std::to_string(g_alloc_largest.load()) + " bytes");
    std::vector<Request> requests;
    for (int i = 0; i < 16; ++i) requests.push_back(realign_block(rng, cfg, 1000, 150));   // 16 000 pairs x 664 bytes: 10.6 MB
    requests.push_back(hifi);                                                              // thread 0's second request
    g_alloc_largest = 0;
    g_alloc_total = 0;
    check("pinned long read after a batch", requests, 16, 16, 100000);
    expect(g_alloc_largest.load() <= (32LL << 20), "pinned long read after a batch: a page-locked allocation of " + std::to_string(g_alloc_largest.load()) + " bytes");
    expect(g_alloc_total.load() <= (128LL << 20), "pinned long read after a batch: " + std::to_string(g_alloc_total.load()) + " page-locked bytes in all");
    expect(merged_calls_of("realign_reads") > 0, "pinned: the short-read requests did not merge");
}

// Requests the limits send alone: more than 65535 haplotypes, a haplotype over 65535 bp, a penalty outside [0,127] (assign); a
// stride too small for the single '=' run of an exact match of its longest read (realign, whose solo text is cut without a status)
void limits(std::mt19937& rng)
{
    const phmm_config cfg = make_config(8, false, false, false);
    std::vector<Request> requests;
    for (int i = 0; i < 6; ++i) requests.push_back(assign_request(rng, cfg));
    for (int i = 0; i < 6; ++i) requests.push_back(realign_request(rng, cfg));
    Request wide;
    wide.kind = ASSIGN;
    wide.cfg = cfg;
    for (int g = 0; g < 1100; ++g) {
        for (int h = 0; h < 60; ++h) wide.g.add_haplotype("ACGTACGTAC", 0, 1);
        wide.g.add_read("ACGTAC", rng);
        wide.hap_first.push_back(wide.g.n_haps());
        wide.read_first.push_back(wide.g.n_reads());
        wide.group_flanks.push_back({0, 0, 0});
    }
    requests.push_back(wide);
    Request longhap = assign_request(rng, cfg);
    longhap.g.seq.append(70000, 'A');
    for (size_t i = longhap.g.prior_f.size(); i < longhap.g.seq.size(); ++i) {
        longhap.g.mask_f += 'A'; longhap.g.mask_r += 'A';
        longhap.g.prior_f.push_back(5); longhap.g.prior_r.push_back(5); longhap.g.gap_open.push_back(5); longhap.g.gap_extend.push_back(1);
    }
    longhap.g.hap_off.back() = (int64_t)longhap.g.seq.size();
    requests.push_back(longhap);
    Request penalty = assign_request(rng, make_config(8, true, false, false));
    penalty.g.gap_open[3] = -4;
    requests.push_back(penalty);
    Request exact;
    exact.kind = REALIGN;
    exact.cfg = cfg;
    const std::string big = random_bases(rng, 1000000);
    exact.g.add_haplotype(big, 0, 1);
    exact.g.add_read(big, rng);                        // "1000000=": 8 characters, which a stride of 9 holds alone but not merged
    exact.pairs.push_back({0, 0});
    exact.stride = 9;
    requests.push_back(exact);
    const size_t n_wide = requests.size() - 4;
    fake::set_call_delay_us(500);
    check("limits", requests, 10, 10, 20000);
    fake::set_call_delay_us(0);
    for (const auto& c : fake_align::calls()) {
        if (c.entry == "assign_reads" && c.haps > 65535) expect(c.members == (int)requests[n_wide].hap_first.size() - 1, "limits: the wide request merged");
        if (c.entry == "realign_reads" && c.stride == 9) expect(c.members == 1, "limits: the exact-match request merged");
    }
}

} // namespace

int main()
{
    std::mt19937 rng(20261017);
    mixed(rng);
    strides(rng);
    rerun(rng);
    pinned(rng);
    limits(rng);
    for (const auto& v : fake::violations()) fail("fake engine: " + v);
    if (g_failures) { std::fprintf(stderr, "%d failures\n", g_failures); return 1; }
    std::printf("BATCHER ALIGN CPU ok\n");
    return 0;
}
