// Plain C++14 client of the C++ adapter's SharedEngine (no torch, no Python): built by tests/test_gpu_batcher.py with g++ and run
// on the GPU box. Eight std::threads share one SharedEngine; every thread's arrays must equal those of an Engine of its own, and
// ShortHaplotypeError must be thrown in the thread whose region has the short haplotype only.
#include <atomic>
#include <cstdio>
#include <cstring>
#include <random>
#include <string>
#include <thread>
#include <vector>
#include "phmm_b200.hpp"

using namespace octopus_b200;

namespace {

struct Region {
    HaplotypeBlock haps;
    HaplotypeLikelihoodArray::ReadMap samples;
    TemplateBlock templates;
};

Region make_region(unsigned seed, bool short_haplotype)
{
    std::mt19937 rng {seed};
    const char* acgt = "ACGT";
    const int hap_len = 300, n_haps = 4 + (int)(rng() % 12);
    std::string base(hap_len, 'A');
    for (auto& c : base) c = acgt[rng() % 4];
    Region g;
    std::vector<std::string> seqs;
    for (int h = 0; h < n_haps; ++h) {
        std::string s = base;
        for (int k = 0; k < 3; ++k) s[rng() % hap_len] = acgt[rng() % 4];
        if (short_haplotype && h == 1) s = s.substr(0, 120);   // shorter than the reads need
        seqs.push_back(s);
        const std::size_t n = s.size();
        std::vector<char> mf(n), mr(n);
        std::vector<std::int8_t> pf(n), pr(n), go(n), ge(n);
        for (std::size_t i = 0; i < n; ++i) {
            mf[i] = s[(i + n - 1) % n]; mr[i] = s[(i + 1) % n];
            pf[i] = (std::int8_t)(1 + rng() % 125); pr[i] = (std::int8_t)(1 + rng() % 125);
            go[i] = (std::int8_t)(3 + rng() % 43); ge[i] = (std::int8_t)(1 + rng() % 10);
        }
        g.haps.add(s, mf, pf, mr, pr, go, ge, 0);
    }
    for (int sample = 0; sample < 2; ++sample) {
        ReadBlock rb;
        const int n_reads = 20 + (int)(rng() % 60);
        for (int r = 0; r < n_reads; ++r) {
            const int L = (r % 3 == 0) ? 150 : 100;
            const int p = 16 + (int)(rng() % (hap_len - L - 32));
            std::string b = base.substr((std::size_t)p, (std::size_t)L);
            for (int k = 0; k < 2; ++k) b[rng() % L] = acgt[rng() % 4];
            std::vector<std::uint8_t> q((std::size_t)L);
            for (auto& x : q) x = (std::uint8_t)(2 + rng() % 40);
            rb.add(b, q, (std::uint8_t)(rng() % 2 ? 60 : 20), rng() % 2 == 0, p);
        }
        g.samples.emplace_back(sample ? "S2" : "S1", rb);
        g.templates.add(rb);
    }
    return g;
}

bool same(const HaplotypeLikelihoodArray& a, const HaplotypeLikelihoodArray& b)
{
    std::size_t width = 0;
    for (const auto& s : a.samples()) width += a.num_likelihoods(s);
    return a.num_haplotypes() == b.num_haplotypes() && a.samples() == b.samples() &&
           std::memcmp(a.data(), b.data(), a.num_haplotypes() * width * sizeof(double)) == 0;
}

} // namespace

int main()
{
    const int kThreads = 8, kRequests = 6, kShortThread = 3;
    try {
        SharedEngine shared {0, kThreads, 2000};
        auto cfg = HaplotypeLikelihoodArray::default_config();
        cfg.max_indel_error = 16;
        std::vector<int> mismatches(kThreads, 0), shared_threw(kThreads, 0), own_threw(kThreads, 0), errors(kThreads, 0);
        std::vector<std::thread> threads;
        for (int k = 0; k < kThreads; ++k) {
            threads.emplace_back([&, k] {
                try {
                    Engine own {0};
                    for (int i = 0; i < kRequests; ++i) {
                        const Region g = make_region(1000u * (unsigned)k + (unsigned)i, k == kShortThread && i == 2);
                        const bool templates = i % 3 == 1;
                        HaplotypeLikelihoodArray a {cfg, own}, s {cfg, shared};
                        bool a_threw = false, s_threw = false;
                        try {
                            if (templates) a.populate(HaplotypeLikelihoodArray::TemplateMap {{"T", g.templates}}, g.haps); else a.populate(g.samples, g.haps);
                        } catch (const ShortHaplotypeError&) { a_threw = true; }
                        try {
                            if (templates) s.populate(HaplotypeLikelihoodArray::TemplateMap {{"T", g.templates}}, g.haps); else s.populate(g.samples, g.haps);
                        } catch (const ShortHaplotypeError&) { s_threw = true; }
                        own_threw[k] += a_threw; shared_threw[k] += s_threw;
                        if (!a_threw && !s_threw && !same(a, s)) ++mismatches[k];
                        if (!a_threw && !s_threw) {
                            const auto merged = s.merge_samples();
                            if (merged.num_haplotypes() != s.num_haplotypes()) ++mismatches[k];
                        }
                    }
                } catch (const std::exception& ex) {
                    std::printf("ERROR thread %d: %s\n", k, ex.what());
                    errors[k] = 1;
                }
            });
        }
        for (auto& t : threads) t.join();
        bool ok = true;
        for (int k = 0; k < kThreads; ++k) {
            const int want_throw = k == kShortThread ? 1 : 0;
            ok = ok && !errors[k] && mismatches[k] == 0 && shared_threw[k] == want_throw && own_threw[k] == want_throw;
            std::printf("THREAD %d mismatches=%d shared_threw=%d own_threw=%d\n", k, mismatches[k], shared_threw[k], own_threw[k]);
        }
        const auto st = shared.stats();
        std::printf("STATS requests=%lld gpu_calls=%lld merged_calls=%lld max_regions=%lld\n", (long long)st.requests, (long long)st.gpu_calls,
                    (long long)st.merged_calls, (long long)st.max_regions_per_call);
        std::printf("BATCHER %s\n", ok ? "ok" : "FAILED");
        return ok ? 0 : 1;
    } catch (const std::exception& ex) {
        std::printf("ERROR %s\n", ex.what());
        return 2;
    }
}
