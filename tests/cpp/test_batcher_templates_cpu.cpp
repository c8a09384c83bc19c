// The request batcher's template assign requests (octopus_b200/csrc/phmm_batcher.cpp, phmm_batcher_templates.cpp) against the CPU
// fakes of the engine (tests/cpp/fake_engine.cpp, fake_engine_align.cpp, fake_engine_templates.cpp), from many std::threads, mixed
// with plain assign requests. Built and run under ThreadSanitizer and under AddressSanitizer + UBSan by
// tests/test_batcher_templates_cpu.py. Every request's return code, message and outputs must equal what the fake engine gives it
// alone, bit for bit: top, lnl and status (its statuses only when it returns PHMM_ERR_SHORT_HAPLOTYPE). Requests cover groups of
// 1-5 haplotypes (duplicates among them, so that templates tie), templates of 1-3 reads, priors present, absent and -inf, bad
// template offsets (checked on the calling thread), short haplotypes and marker reads that fail a whole merged call (rerun member by
// member). Template requests must merge with each other and never with plain assign requests. A last pair of rounds sends only
// requests that cannot fail: there no merged call may be rerun, and merged template calls must return PHMM_OK as they stand (a rerun
// would hide a batch built wrong behind correct solo results). Exits non-zero on any mismatch.
#include "../../include/phmm_b200.h"

#include <algorithm>
#include <atomic>
#include <cmath>
#include <cstdio>
#include <cstring>
#include <limits>
#include <mutex>
#include <random>
#include <string>
#include <thread>
#include <vector>

namespace fake_templates {
struct Call { int groups; int templates; int rc; };
std::vector<Call> calls();
void clear_calls();
} // namespace fake_templates

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

std::string random_bases(std::mt19937& rng, int n)
{
    static const char kAcgt[] = "ACGT";
    std::string s((size_t)n, 'A');
    for (auto& c : s) c = kAcgt[rng() % 4];
    return s;
}

struct Blocks {
    std::vector<int64_t> hap_off {0}, hap_begin, read_off {0}, read_begin;
    std::string seq, mask_f, mask_r, bases;
    std::vector<int8_t> prior_f, prior_r, gap_open, gap_extend;
    std::vector<uint8_t> quals, mapq, reverse;

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
    // a copy of haplotype h (same data: same values, so its group's top sets tie)
    void copy_haplotype(int h)
    {
        const size_t b = (size_t)hap_off[h], n = (size_t)(hap_off[h + 1] - hap_off[h]);
        seq += seq.substr(b, n); mask_f += mask_f.substr(b, n); mask_r += mask_r.substr(b, n);
        for (size_t i = 0; i < n; ++i) {
            prior_f.push_back(prior_f[b + i]); prior_r.push_back(prior_r[b + i]);
            gap_open.push_back(gap_open[b + i]); gap_extend.push_back(gap_extend[b + i]);
        }
        hap_off.push_back((int64_t)seq.size());
        hap_begin.push_back(hap_begin[h]);
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
                gap_extend.data(), hap_begin.data()};
    }
    phmm_reads reads() const { return {n_reads(), read_off.data(), bases.data(), quals.data(), mapq.data(), reverse.data(), read_begin.data()}; }
};

phmm_config make_config(int band, bool map_positions)
{
    phmm_config c;
    c.max_indel_error = band; c.use_int_scores = 0; c.use_mapping_quality = 1; c.mapping_quality_cap = 120;
    c.mapping_quality_cap_trigger = -1; c.use_flank_state = 0; c.nuc_prior = 2; c.disable_naive_shortcut = 0;
    c.map_positions = map_positions ? 1 : 0;
    return c;
}

struct Outputs {
    int rc = PHMM_OK;
    std::string err;
    std::vector<uint64_t> top;
    std::vector<double> lnl;
    std::vector<int32_t> status;
};

struct Request {
    bool templates = true;
    phmm_config cfg {};
    Blocks g;
    std::vector<int32_t> hap_first {0}, read_first {0};
    std::vector<int64_t> template_off {0};
    std::vector<double> priors;                 // empty = NULL
    bool want_lnl = true, want_status = true;
    long long n_values = 0, n_slots = 0;        // lnl / status sizes
    Outputs alone;

    phmm_regions groups() const { return {(int32_t)(hap_first.size() - 1), hap_first.data(), read_first.data(), nullptr}; }
    int32_t n_templates() const { return (int32_t)template_off.size() - 1; }
};

// clean: a request that cannot fail (no short haplotype, no marker read, no bad offsets), so a merged call of clean requests must
// succeed as it stands, without a rerun
Request make_request(std::mt19937& rng, int i, bool clean = false)
{
    Request q;
    q.templates = i % 4 != 3;                   // one request in four is a plain assign request
    q.cfg = make_config(rng() % 2 ? 8 : 16, rng() % 5 != 0);
    const int G = 1 + (int)(rng() % 4);
    for (int g = 0; g < G; ++g) {
        const int nH = 1 + (int)(rng() % 4);
        const int h0 = q.g.n_haps();
        for (int k = 0; k < nH; ++k) {
            if (k > 0 && rng() % 4 == 0) q.g.copy_haplotype(h0 + (int)(rng() % k));
            else q.g.add_haplotype(random_bases(rng, 40 + (int)(rng() % 40)), (int64_t)(rng() % 500), (int8_t)(rng() % 50));
        }
        const int nT = 1 + (int)(rng() % 5);
        for (int t = 0; t < nT; ++t) {
            const int nr = 1 + (int)(rng() % 3);
            for (int r = 0; r < nr; ++r) {
                std::string b = random_bases(rng, 20 + (int)(rng() % 20));
                if (!clean && rng() % 150 == 0) b = std::string(90, 'C');               // longer than every haplotype: SHORT_HAP
                if (!clean && q.cfg.map_positions && rng() % 200 == 0) b.replace(0, 4, "MMMM");   // fails a whole mapping call
                q.g.add_read(b, rng);
            }
            q.template_off.push_back(q.g.n_reads());
        }
        q.hap_first.push_back(q.g.n_haps());
        q.read_first.push_back(q.g.n_reads());
        q.n_values += (long long)nH * (q.templates ? nT : q.read_first[g + 1] - q.read_first[g]);
        q.n_slots += (long long)nH * (q.read_first[g + 1] - q.read_first[g]);
    }
    if (rng() % 3) {
        for (int h = 0; h < q.g.n_haps(); ++h) q.priors.push_back(rng() % 10 == 0 ? -std::numeric_limits<double>::infinity() : -(double)(rng() % 4));
    }
    q.want_lnl = rng() % 4 != 0;
    q.want_status = rng() % 4 != 0;
    if (!clean && q.templates && rng() % 25 == 0) {
        // bad offsets: a group boundary inside a template, an empty template, or offsets past the reads
        const auto boundary = std::find(q.template_off.begin(), q.template_off.end(), (int64_t)q.read_first[1]);
        const int how = (int)(rng() % 3);
        if (how == 0 && q.hap_first.size() > 2) q.template_off.erase(boundary);
        else if (how == 1 && q.n_templates() > 1) q.template_off[1] = q.template_off[0];
        else q.template_off.back() = q.template_off.back() + 1;
    }
    return q;
}

Outputs sized(const Request& q)
{
    Outputs o;
    o.top.assign(q.templates ? (size_t)q.n_templates() : (size_t)q.g.n_reads(), 0xdeadbeefULL);
    if (q.want_lnl) o.lnl.assign((size_t)q.n_values, 7.0);
    if (q.want_status) o.status.assign((size_t)q.n_slots, -7);
    return o;
}

Outputs run_alone(phmm_engine* e, const Request& q)
{
    Outputs o = sized(q);
    const phmm_haplotypes h = q.g.haps();
    const phmm_reads r = q.g.reads();
    const phmm_regions groups = q.groups();
    const double* pri = q.priors.empty() ? nullptr : q.priors.data();
    double* lnl = q.want_lnl ? o.lnl.data() : nullptr;
    int32_t* st = q.want_status ? o.status.data() : nullptr;
    o.rc = q.templates ? phmm_assign_templates(e, &q.cfg, &h, &r, &groups, q.template_off.data(), q.n_templates(), pri, o.top.data(), lnl, st, PHMM_SPACE_HOST)
                       : phmm_assign_reads(e, &q.cfg, &h, &r, &groups, pri, o.top.data(), lnl, st, PHMM_SPACE_HOST);
    o.err = o.rc == PHMM_OK ? std::string() : std::string(phmm_last_error(e));
    return o;
}

Outputs run_batched(phmm_batcher* b, const Request& q)
{
    Outputs o = sized(q);
    const phmm_haplotypes h = q.g.haps();
    const phmm_reads r = q.g.reads();
    const phmm_regions groups = q.groups();
    const double* pri = q.priors.empty() ? nullptr : q.priors.data();
    double* lnl = q.want_lnl ? o.lnl.data() : nullptr;
    int32_t* st = q.want_status ? o.status.data() : nullptr;
    o.rc = q.templates ? phmm_batcher_assign_templates(b, &q.cfg, &h, &r, &groups, q.template_off.data(), q.n_templates(), pri, o.top.data(), lnl, st)
                       : phmm_batcher_assign_reads(b, &q.cfg, &h, &r, &groups, pri, o.top.data(), lnl, st);
    o.err = o.rc == PHMM_OK ? std::string() : std::string(phmm_batcher_last_error());
    return o;
}

template <typename T>
bool same_bits(const std::vector<T>& a, const std::vector<T>& b)
{
    return a.size() == b.size() && (a.empty() || std::memcmp(a.data(), b.data(), a.size() * sizeof(T)) == 0);
}

void compare(const Request& q, const Outputs& got, int i)
{
    const std::string id = "request " + std::to_string(i) + (q.templates ? " (templates)" : " (reads)");
    const Outputs& want = q.alone;
    expect(got.rc == want.rc, id + ": rc " + std::to_string(got.rc) + " != " + std::to_string(want.rc) + " (" + got.err + " / " + want.err + ")");
    expect(got.err == want.err, id + ": message '" + got.err + "' != '" + want.err + "'");
    if (want.rc == PHMM_OK) {
        expect(same_bits(got.top, want.top), id + ": top");
        expect(same_bits(got.lnl, want.lnl), id + ": lnl");
    }
    if (want.rc == PHMM_OK || want.rc == PHMM_ERR_SHORT_HAPLOTYPE) expect(same_bits(got.status, want.status), id + ": status");
}

// One round of requests through a fresh batcher. clean: every request cannot fail, so there must be no rerun, and at least one
// merged template call (more groups than any one template request has) must have returned PHMM_OK.
void round(const std::vector<Request>& reqs, int threads, bool clean = false)
{
    fake_templates::clear_calls();
    phmm_batcher* b = nullptr;
    const phmm_batcher_options opt {threads, 2000};
    if (phmm_batcher_create(&b, 0, &opt) != PHMM_OK) { fail("batcher create"); return; }
    std::atomic<int> next {0};
    std::vector<std::thread> pool;
    for (int k = 0; k < threads; ++k) {
        pool.emplace_back([&] {
            for (int i; (i = next++) < (int)reqs.size();) compare(reqs[(size_t)i], run_batched(b, reqs[(size_t)i]), i);
        });
    }
    for (auto& t : pool) t.join();
    // template requests merged with each other only: a merged call's templates are its members' (every template call holds only
    // template requests, so its group count is a sum of template requests' group counts, checked by the results above); with
    // several threads at least one call carried more than one request
    int widest = 0, widest_alone = 0;
    for (const auto& c : fake_templates::calls()) widest = std::max(widest, c.groups);
    for (const auto& q : reqs) if (q.templates) widest_alone = std::max(widest_alone, (int)q.hap_first.size() - 1);
    if (threads >= 8) expect(widest > widest_alone, "template requests merged (" + std::to_string(threads) + " threads)");
    int merged_ok = 0;
    for (const auto& c : fake_templates::calls()) merged_ok += c.groups > widest_alone && c.rc == PHMM_OK;
    const long long reruns = phmm_batcher_reruns(b);
    if (clean) {
        const std::string id = " (clean, " + std::to_string(threads) + " threads)";
        expect(reruns == 0, "no merged call is rerun" + id + ": " + std::to_string(reruns));
        expect(merged_ok > 0, "a merged template call returned PHMM_OK" + id);
    }
    std::printf("threads %d%s: %zu template calls, widest %d groups, %d merged and ok, %lld reruns\n", threads, clean ? " (clean)" : "",
                fake_templates::calls().size(), widest, merged_ok, reruns);
    phmm_batcher_destroy(b);
}

} // namespace

int main()
{
    std::mt19937 rng(20261017);
    std::vector<Request> reqs;
    for (int i = 0; i < 600; ++i) reqs.push_back(make_request(rng, i));
    phmm_engine* e = nullptr;
    if (phmm_create(&e, 0) != PHMM_OK) { std::fprintf(stderr, "FAIL engine create\n"); return 1; }
    int n_ok = 0, n_short = 0, n_invalid = 0, n_marker = 0;
    for (auto& q : reqs) {
        q.alone = run_alone(e, q);
        n_ok += q.alone.rc == PHMM_OK;
        n_short += q.alone.rc == PHMM_ERR_SHORT_HAPLOTYPE;
        n_invalid += q.alone.rc == PHMM_ERR_INVALID;
        n_marker += q.alone.err.find("4096") != std::string::npos;
    }
    phmm_destroy(e);
    std::printf("alone: %d ok, %d short, %d invalid (%d marker)\n", n_ok, n_short, n_invalid, n_marker);
    expect(n_ok > 400 && n_short > 0 && n_invalid > n_marker && n_marker > 0, "the request mix covers every outcome");

    // ties: some template request has an ambiguous template whose set is not every haplotype of its group
    bool tie = false;
    for (const auto& q : reqs) {
        if (!q.templates || q.alone.rc != PHMM_OK) continue;
        for (uint64_t t : q.alone.top) tie |= (t & (t - 1)) != 0;
    }
    expect(tie, "ambiguous templates");

    for (int threads : {1, 8, 32}) round(reqs, threads);

    // requests that cannot fail: merged template calls must succeed as they stand
    std::vector<Request> clean;
    for (int i = 0; i < 400; ++i) clean.push_back(make_request(rng, i, true));
    e = nullptr;
    if (phmm_create(&e, 0) != PHMM_OK) { std::fprintf(stderr, "FAIL engine create\n"); return 1; }
    for (auto& q : clean) {
        q.alone = run_alone(e, q);
        expect(q.alone.rc == PHMM_OK, "a clean request succeeds alone: " + q.alone.err);
    }
    phmm_destroy(e);
    for (int threads : {8, 32}) round(clean, threads, true);
    if (g_failures) { std::fprintf(stderr, "%d failures\n", g_failures); return 1; }
    std::printf("BATCHER TEMPLATES CPU ok\n");
    return 0;
}
