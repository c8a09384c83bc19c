// The request batcher (octopus_b200/csrc/phmm_batcher.cpp) against the CPU fake engine (tests/cpp/fake_engine.cpp): merging,
// staging, slicing, errors, limits, the leader's deadline and destroy, from many std::threads. Built and run under ThreadSanitizer
// and under AddressSanitizer + UBSan by tests/test_batcher_cpu.py. Every request's return code, message, status and values must
// equal what the fake engine gives it alone, bit for bit. Exits non-zero on any mismatch or on any violation the fake recorded.
#include "../../include/phmm_b200.h"
#include "../../octopus_b200/csrc/phmm_mutation.h"

#include <algorithm>
#include <atomic>
#include <chrono>
#include <cstdio>
#include <cstring>
#include <functional>
#include <mutex>
#include <random>
#include <set>
#include <string>
#include <thread>
#include <vector>

namespace fake {
struct Call {
    std::string entry;
    int members;
    long long haps;
    std::string key;
};
std::vector<Call> calls();
std::vector<std::string> violations();
void clear_calls();
int calls_inside();
void set_call_delay_us(int us);
} // namespace fake

namespace {

using Clock = std::chrono::steady_clock;

std::mutex g_report_m;
int g_failures = 0;

void fail(const std::string& what)
{
    std::lock_guard<std::mutex> lk(g_report_m);
    ++g_failures;
    if (g_failures <= 50) std::fprintf(stderr, "FAIL %s\n", what.c_str());
}

void expect(bool ok, const std::string& what)
{
    if (!ok) fail(what);
}

const char kAcgt[] = "ACGT";

struct Region {
    std::vector<int64_t> hap_off {0}, hap_begin, read_off {0}, read_begin;
    std::string seq, mask_f, mask_r, bases;
    std::vector<int8_t> prior_f, prior_r, gap_open, gap_extend;
    std::vector<uint8_t> quals, mapq, reverse;

    void add_haplotype(const std::string& s, std::mt19937& rng)
    {
        for (size_t i = 0; i < s.size(); ++i) {
            seq += s[i];
            mask_f += s[(i + s.size() - 1) % s.size()];
            mask_r += s[(i + 1) % s.size()];
            prior_f.push_back((int8_t)(1 + rng() % 120)); prior_r.push_back((int8_t)(1 + rng() % 120));
            gap_open.push_back((int8_t)(3 + rng() % 40)); gap_extend.push_back((int8_t)(1 + rng() % 10));
        }
        hap_off.push_back((int64_t)seq.size());
        hap_begin.push_back((int64_t)(rng() % 1000));
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
    phmm_haplotypes haps() const
    {
        return {(int32_t)hap_begin.size(), hap_off.data(), seq.data(), mask_f.data(), prior_f.data(), mask_r.data(), prior_r.data(),
                gap_open.data(), gap_extend.data(), hap_begin.data()};
    }
    phmm_reads reads() const { return {(int32_t)read_begin.size(), read_off.data(), bases.data(), quals.data(), mapq.data(), reverse.data(), read_begin.data()}; }
};

std::string random_bases(std::mt19937& rng, int n)
{
    std::string s((size_t)n, 'A');
    for (auto& c : s) c = kAcgt[rng() % 4];
    return s;
}

Region make_region(std::mt19937& rng, int n_haps, int n_reads, int hap_len, int read_len)
{
    Region g;
    const std::string base = random_bases(rng, hap_len);
    for (int h = 0; h < n_haps; ++h) {
        std::string s = base;
        s[rng() % s.size()] = kAcgt[rng() % 4];
        g.add_haplotype(s, rng);
    }
    for (int r = 0; r < n_reads; ++r) {
        const int len = std::max(1, read_len - (int)(rng() % 8));
        g.add_read(base.substr(rng() % (size_t)(hap_len - len + 1), (size_t)len), rng);
    }
    return g;
}

phmm_config make_config(int band, bool map_positions)
{
    phmm_config c;
    c.max_indel_error = band; c.use_int_scores = 0; c.use_mapping_quality = 1; c.mapping_quality_cap = 120;
    c.mapping_quality_cap_trigger = -1; c.use_flank_state = 1; c.nuc_prior = 2; c.disable_naive_shortcut = 0;
    c.map_positions = map_positions ? 1 : 0;
    return c;
}

enum Kind { READS, TEMPLATES, POSITIONS, MUTATION };

struct Request {
    Kind kind = READS;
    phmm_config cfg = make_config(16, true);
    Region g;
    bool has_flank = false;
    phmm_flank_state flank {0, 0, 0};
    bool want_status = true;
    std::vector<int64_t> template_off;                 // TEMPLATES
    std::vector<int64_t> pos_off;                      // POSITIONS
    std::vector<int32_t> pos;
    std::string model_key;                             // MUTATION
    std::vector<int64_t> mut_off {0};
    std::string mut_seq;
};

struct Result {
    int rc = 0;
    std::string msg;
    std::vector<double> out;
    std::vector<int32_t> status;
};

Request populate_request(std::mt19937& rng, Kind kind, const phmm_config& cfg)
{
    Request q;
    q.kind = kind;
    q.cfg = cfg;
    q.g = make_region(rng, 1 + (int)(rng() % 16), 1 + (int)(rng() % 40), 120 + (int)(rng() % 80), 30 + (int)(rng() % 70));
    q.has_flank = rng() % 2;
    q.flank = {q.has_flank ? 1 : 0, (int64_t)(rng() % 80), (int64_t)(rng() % 80)};
    q.want_status = rng() % 4 != 0;
    const int R = (int)q.g.read_begin.size();
    if (kind == TEMPLATES) {
        q.template_off = {0};
        while (q.template_off.back() < R) q.template_off.push_back(std::min<int64_t>(R, q.template_off.back() + 1 + (int64_t)(rng() % 3)));
    }
    if (kind == POSITIONS) {
        q.pos_off = {0};
        for (size_t p = 0; p < q.g.hap_begin.size() * (size_t)R; ++p) {
            for (int k = (int)(rng() % 3); k > 0; --k) q.pos.push_back((int32_t)(rng() % 100));
            q.pos_off.push_back((int64_t)q.pos.size());
        }
    }
    return q;
}

Request mutation_request(std::mt19937& rng, const std::string& key)
{
    Request q;
    q.kind = MUTATION;
    q.model_key = key;
    const int n = 1 + (int)(rng() % 12);
    const std::string base = random_bases(rng, 60 + (int)(rng() % 200));
    for (int h = 0; h < n; ++h) {
        std::string s = base;
        if (h % 3 == 1) s.erase(rng() % s.size(), 1 + rng() % 4);
        if (h % 5 == 4) s += random_bases(rng, 40);          // 32 or more bases longer: an approximate pair
        s[rng() % s.size()] = kAcgt[rng() % 4];
        q.mut_seq += s;
        q.mut_off.push_back((int64_t)q.mut_seq.size());
    }
    return q;
}

int pairs_of(const Request& q) { return (int)(q.g.hap_begin.size() * q.g.read_begin.size()); }

Result batched(phmm_batcher* b, const Request& q)
{
    Result res;
    if (q.kind == MUTATION) {
        const int n = (int)q.mut_off.size() - 1;
        phmm_mutation_model m;                             // a model of its own per request: models merge by their key
        m.key = q.model_key;
        res.out.assign((size_t)n * n, -7.0);
        res.status.assign((size_t)n * n, -7);
        res.rc = phmm_batcher_mutation_prime(b, &m, n, q.mut_off.data(), q.mut_seq.data(), res.out.data(), res.status.data());
    } else {
        const phmm_haplotypes haps = q.g.haps();
        const phmm_reads reads = q.g.reads();
        const int T = (int)q.template_off.size() - 1;
        res.out.assign((size_t)haps.n * (q.kind == TEMPLATES ? T : reads.n), -7.0);
        if (q.want_status) res.status.assign((size_t)pairs_of(q), -7);
        const phmm_flank_state* flank = q.has_flank ? &q.flank : nullptr;
        int32_t* status = q.want_status ? res.status.data() : nullptr;
        const phmm_positions positions {q.pos_off.data(), q.pos.data()};
        if (q.kind == TEMPLATES)
            res.rc = phmm_batcher_populate_templates(b, &q.cfg, &haps, &reads, q.template_off.data(), T, flank, res.out.data(), status);
        else
            res.rc = phmm_batcher_populate(b, &q.cfg, &haps, &reads, q.kind == POSITIONS ? &positions : nullptr, flank, res.out.data(), status);
    }
    res.msg = phmm_batcher_last_error();
    return res;
}

// The request alone on an engine of its own; a template's value is the left-to-right sum of its reads' solo values.
Result solo(phmm_engine* e, const Request& q)
{
    Result res;
    if (q.kind == MUTATION) {
        const int n = (int)q.mut_off.size() - 1;
        phmm_mutation_model m;
        m.key = q.model_key;
        const int32_t set_first[2] = {0, n};
        res.out.assign((size_t)n * n, -7.0);
        res.status.assign((size_t)n * n, -7);
        res.rc = phmm_mutation_prime_sets(e, &m, 1, set_first, q.mut_off.data(), q.mut_seq.data(), res.out.data(), res.status.data());
    } else {
        const phmm_haplotypes haps = q.g.haps();
        const phmm_reads reads = q.g.reads();
        const phmm_positions positions {q.pos_off.data(), q.pos.data()};
        std::vector<double> values((size_t)pairs_of(q), -7.0);
        std::vector<int32_t> status((size_t)pairs_of(q), -7);
        res.rc = phmm_populate(e, &q.cfg, &haps, &reads, q.kind == POSITIONS ? &positions : nullptr, q.has_flank ? &q.flank : nullptr,
                               values.data(), status.data(), PHMM_SPACE_HOST);
        if (q.want_status) res.status = status;
        if (q.kind == TEMPLATES) {
            const int T = (int)q.template_off.size() - 1;
            res.out.assign((size_t)haps.n * T, -7.0);
            if (res.rc == PHMM_OK || res.rc == PHMM_ERR_SHORT_HAPLOTYPE) {
                for (int h = 0; h < haps.n; ++h) {
                    for (int t = 0; t < T; ++t) {
                        double acc = 0.0;
                        for (int64_t r = q.template_off[t]; r < q.template_off[t + 1]; ++r) acc += values[(size_t)h * reads.n + r];
                        res.out[(size_t)h * T + t] = acc;
                    }
                }
            }
        } else {
            res.out = values;
        }
    }
    res.msg = res.rc == PHMM_OK ? "" : phmm_last_error(e);
    return res;
}

void compare(const std::string& name, const Result& got, const Result& want)
{
    if (got.rc != want.rc || got.msg != want.msg) {
        fail(name + ": rc " + std::to_string(got.rc) + " '" + got.msg + "', alone " + std::to_string(want.rc) + " '" + want.msg + "'");
        return;
    }
    if (got.rc != PHMM_OK && got.rc != PHMM_ERR_SHORT_HAPLOTYPE) return;      // out and status unspecified
    expect(got.out.size() == want.out.size() && std::memcmp(got.out.data(), want.out.data(), got.out.size() * sizeof(double)) == 0,
           name + ": values differ from the request's values alone");
    expect(got.status == want.status, name + ": statuses differ from the request's statuses alone");
}

// Runs requests[k] on thread k % n_threads, in order per thread, all threads released at once; returns the results.
std::vector<Result> run_threads(phmm_batcher* b, const std::vector<Request>& requests, int n_threads)
{
    std::vector<Result> got(requests.size());
    std::atomic<int> ready {0};
    std::vector<std::thread> threads;
    for (int k = 0; k < n_threads; ++k) {
        threads.emplace_back([&, k] {
            ++ready;
            while (ready.load() < n_threads) std::this_thread::yield();
            for (size_t i = (size_t)k; i < requests.size(); i += (size_t)n_threads) got[i] = batched(b, requests[i]);
        });
    }
    for (auto& t : threads) t.join();
    return got;
}

phmm_batcher* make_batcher(int clients, int max_wait_us)
{
    phmm_batcher* b = nullptr;
    const phmm_batcher_options opt {clients, max_wait_us};
    if (phmm_batcher_create(&b, 0, &opt) != PHMM_OK) { fail(std::string("batcher creation: ") + phmm_batcher_last_error()); return nullptr; }
    return b;
}

phmm_batcher_stats stats_of(const phmm_batcher* b)
{
    phmm_batcher_stats s {};
    phmm_batcher_stats_get(b, &s);
    return s;
}

std::vector<fake::Call> calls_of(const std::string& entry)
{
    std::vector<fake::Call> out;
    for (const auto& c : fake::calls()) if (c.entry == entry) out.push_back(c);
    return out;
}

// Runs the requests through a batcher from n_threads threads and compares each with its solo result; returns the batcher's stats.
phmm_batcher_stats check_against_solo(phmm_engine* e, const std::string& name, const std::vector<Request>& requests, int n_threads,
                                      int clients, int max_wait_us)
{
    std::vector<Result> want;
    for (const auto& q : requests) want.push_back(solo(e, q));
    fake::clear_calls();
    phmm_batcher* b = make_batcher(clients, max_wait_us);
    if (!b) return {};
    const std::vector<Result> got = run_threads(b, requests, n_threads);
    const phmm_batcher_stats s = stats_of(b);
    phmm_batcher_destroy(b);
    for (size_t i = 0; i < requests.size(); ++i) compare(name + " request " + std::to_string(i), got[i], want[i]);
    return s;
}

// (a) Mixed-config populate requests from many threads.
void scenario_mixed_configs(phmm_engine* e)
{
    std::mt19937 rng {11};
    const phmm_config configs[] = {make_config(8, true), make_config(16, true), make_config(32, false)};
    std::vector<Request> requests;
    for (int i = 0; i < 16 * 12; ++i) requests.push_back(populate_request(rng, i % 5 == 3 ? TEMPLATES : READS, configs[rng() % 3]));
    const phmm_batcher_stats s = check_against_solo(e, "(a)", requests, 16, 16, 20000);
    std::set<std::string> keys;
    for (const auto& c : configs) keys.insert(std::string(reinterpret_cast<const char*>(&c), sizeof(c)));
    long long regions = 0;
    for (const auto& c : calls_of("populate_regions")) {
        regions += c.members;
        expect(keys.count(c.key) == 1, "(a): a call under a config no request had");
    }
    expect(regions == (long long)requests.size(), "(a): every request is one region of one call");
    expect(s.requests == (int64_t)requests.size() && s.gpu_calls < s.requests && s.merged_calls >= 1 && s.dp_cells > 0,
           "(a): stats requests " + std::to_string(s.requests) + " calls " + std::to_string(s.gpu_calls) + " merged " + std::to_string(s.merged_calls));
}

// (b) Populate and mutation requests interleaved on the same threads; every mutation request brings a model of its own.
void scenario_interleaved(phmm_engine* e)
{
    std::mt19937 rng {23};
    const std::string keys[] = {std::string("model A\0\1", 9), std::string("model B\0\2", 9)};
    std::vector<Request> requests;
    for (int i = 0; i < 8 * 16; ++i) {
        if ((i / 8) % 2) requests.push_back(mutation_request(rng, keys[rng() % 2]));
        else requests.push_back(populate_request(rng, i % 3 ? READS : TEMPLATES, make_config(16, true)));
    }
    const phmm_batcher_stats s = check_against_solo(e, "(b)", requests, 8, 8, 20000);
    const auto mutation = calls_of("mutation_prime_sets");
    int sets = 0, merged = 0;
    for (const auto& c : mutation) {
        sets += c.members;
        merged += c.members > 1;
        expect(c.key == keys[0] || c.key == keys[1], "(b): a mutation call under an unknown model key");
    }
    expect(sets == (int)requests.size() / 2, "(b): every mutation request is one set of one call");
    expect(merged >= 1, "(b): no mutation call merged separately built models");
    expect(!calls_of("populate_regions").empty() && s.gpu_calls < s.requests, "(b): populate requests were not merged");
}

// (c) Template requests only: each thread sums its own rows (solo: the left-to-right sums of the solo values).
void scenario_templates(phmm_engine* e)
{
    std::mt19937 rng {31};
    std::vector<Request> requests;
    for (int i = 0; i < 8 * 6; ++i) requests.push_back(populate_request(rng, TEMPLATES, make_config(8, i % 2 == 0)));
    const phmm_batcher_stats s = check_against_solo(e, "(c)", requests, 8, 8, 20000);
    expect(s.merged_calls >= 1, "(c): no template requests merged");
}

// (d) Errors stay with their own request.
void scenario_errors(phmm_engine* e)
{
    std::mt19937 rng {37};
    std::vector<Request> requests;
    for (int k = 0; k < 8; ++k) requests.push_back(populate_request(rng, k == 6 ? POSITIONS : READS, make_config(16, true)));
    requests[2].g.gap_open[3] = -5;                                    // merged path: the batcher's own check
    requests[6].g.prior_r[0] = -1;                                     // with positions: runs alone, the engine's check
    Region& g = requests[5].g;                                         // haplotype 0 shorter than the reads
    g = make_region(rng, 3, 10, 150, 90);
    const int64_t cut = g.hap_off[1] - 80;
    for (std::string* a : {&g.seq, &g.mask_f, &g.mask_r}) a->erase((size_t)cut, 80);
    for (auto* a : {&g.prior_f, &g.prior_r, &g.gap_open, &g.gap_extend}) a->erase(a->begin() + cut, a->begin() + cut + 80);
    for (size_t h = 1; h < g.hap_off.size(); ++h) g.hap_off[h] -= 80;
    requests.push_back(mutation_request(rng, "model"));
    requests.back().mut_off[1] = 0;                                    // an empty first haplotype
    requests.push_back(mutation_request(rng, "model"));

    std::vector<Result> want;
    for (const auto& q : requests) want.push_back(solo(e, q));
    phmm_batcher* b = make_batcher((int)requests.size(), 20000);
    if (!b) return;
    const std::vector<Result> got = run_threads(b, requests, (int)requests.size());
    phmm_batcher_destroy(b);
    const char* bad_penalty = "snv prior / gap penalty outside [0,127]";
    for (size_t i = 0; i < requests.size(); ++i) {
        const int want_rc = i == 2 || i == 6 || i == 8 ? PHMM_ERR_INVALID : i == 5 ? PHMM_ERR_SHORT_HAPLOTYPE : PHMM_OK;
        const std::string want_msg = i == 2 || i == 6 ? bad_penalty : i == 5 ? "Haplotype is too short for alignment"
                                   : i == 8 ? "haplotype length outside [1, 65535]" : "";
        expect(got[i].rc == want_rc && got[i].msg == want_msg, "(d) request " + std::to_string(i) + ": rc " + std::to_string(got[i].rc) + " '" + got[i].msg + "'");
        if (i != 8) compare("(d) request " + std::to_string(i), got[i], want[i]);
    }
}

// (e) Limits: the 65535-haplotype limit of a merged call, requests that run alone, staging growth.
void scenario_limits(phmm_engine* e)
{
    std::mt19937 rng {41};
    // four requests of 20000 haplotypes: the first round outgrows the initial staging (4096 haplotypes) twice; once it has grown,
    // three merge and the fourth, past 65535 haplotypes, goes to a call of its own. The leaders go once all four wait, so the
    // shapes do not depend on timing; a batch left alone by the others' calls goes at its deadline.
    std::vector<Request> big;
    for (int k = 0; k < 4; ++k) {
        Request q;
        q.cfg = make_config(8, true);
        q.g = make_region(rng, 20000, 1, 14, 10);
        big.push_back(q);
    }
    std::vector<Result> want;
    for (const auto& q : big) want.push_back(solo(e, q));
    phmm_batcher* b = make_batcher(4, 1000000);
    if (!b) return;
    for (int round = 0; round < 2; ++round) {
        fake::clear_calls();
        const std::vector<Result> got = run_threads(b, big, 4);
        for (size_t i = 0; i < big.size(); ++i) compare("(e) round " + std::to_string(round) + " request " + std::to_string(i), got[i], want[i]);
        std::vector<int> members;
        for (const auto& c : calls_of("populate_regions")) members.push_back(c.members);
        std::sort(members.begin(), members.end());
        const std::vector<int> expected = round == 0 ? std::vector<int> {1, 1, 2} : std::vector<int> {1, 3};
        expect(members == expected, "(e) round " + std::to_string(round) + ": calls of " + std::to_string(members.size()) + " shapes unexpected");
    }

    // alone: more than 65535 haplotypes; a haplotype longer than 65535 bp without the mapper. With the mapper: an error.
    Request many;
    many.cfg = make_config(8, true);
    many.g = make_region(rng, 70000, 1, 14, 10);
    Request longest;
    longest.cfg = make_config(8, false);
    longest.g = make_region(rng, 2, 3, 70000, 100);
    for (Request* q : {&many, &longest}) {
        const Result want_alone = solo(e, *q);
        fake::clear_calls();
        compare("(e) alone", batched(b, *q), want_alone);
        const auto calls = fake::calls();
        expect(calls.size() == 1 && calls[0].entry == "populate" && calls[0].haps == q->g.haps().n,
               "(e): a request that must run alone made " + std::to_string(calls.size()) + " calls, the first " + (calls.empty() ? "" : calls[0].entry));
    }
    longest.cfg.map_positions = 1;
    fake::clear_calls();
    const Result r = batched(b, longest);
    expect(r.rc == PHMM_ERR_INVALID && r.msg.find("haplotype longer than 65535 bp") == 0 && fake::calls().empty(),
           "(e): a haplotype over 65535 bp under the mapper: rc " + std::to_string(r.rc) + " '" + r.msg + "'");
    phmm_batcher_destroy(b);
}

// (f) A lone thread is never held longer than the deadline by clients that do not come.
void scenario_lone_thread()
{
    std::mt19937 rng {53};
    const int max_wait_us = 50000;
    phmm_batcher* b = make_batcher(4, max_wait_us);
    if (!b) return;
    for (int i = 0; i < 5; ++i) {
        const Request q = populate_request(rng, READS, make_config(16, true));
        const auto t0 = Clock::now();
        const Result r = batched(b, q);
        const long long us = std::chrono::duration_cast<std::chrono::microseconds>(Clock::now() - t0).count();
        expect(r.rc == PHMM_OK || r.rc == PHMM_ERR_SHORT_HAPLOTYPE, "(f): request failed: " + r.msg);
        expect(us < 5LL * max_wait_us, "(f): a lone request took " + std::to_string(us) + " us");
    }
    expect(stats_of(b).gpu_calls == 5, "(f): lone requests were not one call each");
    phmm_batcher_destroy(b);
}

// (g) destroy returns only once the requests in flight have finished: it waits out the merged call that is running, and a
// request that copied its result out of a freed staging or touched the freed batcher would be an AddressSanitizer report.
void scenario_destroy(phmm_engine* e)
{
    std::mt19937 rng {67};
    std::vector<Request> requests;
    for (int k = 0; k < 4; ++k) requests.push_back(populate_request(rng, READS, make_config(16, true)));
    std::vector<Result> want;
    for (const auto& q : requests) want.push_back(solo(e, q));
    phmm_batcher* b = make_batcher(4, 5000000);
    if (!b) return;
    const int delay_us = 300000;
    fake::set_call_delay_us(delay_us);
    std::vector<Result> got(requests.size());
    std::vector<std::thread> threads;
    for (size_t k = 0; k < requests.size(); ++k) threads.emplace_back([&, k] { got[k] = batched(b, requests[k]); });
    const auto t0 = Clock::now();
    while (fake::calls_inside() == 0 && Clock::now() - t0 < std::chrono::seconds(30)) std::this_thread::sleep_for(std::chrono::microseconds(200));
    expect(fake::calls_inside() == 1, "(g): the merged call never started");
    const auto t1 = Clock::now();
    phmm_batcher_destroy(b);
    const long long us = std::chrono::duration_cast<std::chrono::microseconds>(Clock::now() - t1).count();
    expect(fake::calls_inside() == 0 && us >= delay_us / 2, "(g): destroy returned after " + std::to_string(us) + " us, during the call");
    for (auto& t : threads) t.join();
    fake::set_call_delay_us(0);
    for (size_t i = 0; i < requests.size(); ++i) compare("(g) request " + std::to_string(i), got[i], want[i]);
}

} // namespace

int main()
{
    phmm_engine* e = nullptr;
    if (phmm_create(&e, 0) != PHMM_OK) { std::fprintf(stderr, "FAIL engine creation\n"); return 2; }
    const std::pair<const char*, std::function<void()>> scenarios[] = {
        {"(a) mixed configs", [&] { scenario_mixed_configs(e); }},
        {"(b) populate and mutation interleaved", [&] { scenario_interleaved(e); }},
        {"(c) templates", [&] { scenario_templates(e); }},
        {"(d) errors", [&] { scenario_errors(e); }},
        {"(e) limits", [&] { scenario_limits(e); }},
        {"(f) lone thread", [] { scenario_lone_thread(); }},
        {"(g) destroy", [&] { scenario_destroy(e); }},
    };
    for (const auto& s : scenarios) {
        const int before = g_failures;
        const auto t0 = Clock::now();
        s.second();
        std::printf("%-40s %s (%.2f s)\n", s.first, g_failures == before ? "ok" : "FAILED",
                    std::chrono::duration<double>(Clock::now() - t0).count());
    }
    phmm_destroy(e);
    for (const auto& v : fake::violations()) fail("engine: " + v);
    std::printf("BATCHER CPU %s\n", g_failures ? "FAILED" : "ok");
    return g_failures ? 1 : 0;
}
