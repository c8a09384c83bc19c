// Plain C++14 client of the C++ adapter's compute_haplotype_support and realign on a SharedEngine (no torch, no Python): built by
// tests/test_gpu_batcher_align.py with g++ and run on the GPU. Eight std::threads share one SharedEngine; every thread's supports
// and realignments must equal those of an Engine of its own, and the ShortHaplotypeError of a region with a short haplotype must be
// the Engine's (same haplotype index, same required extension), in that thread only.
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
    ReadBlock reads;
    std::vector<std::int32_t> hap_first {0}, read_first {0};
    std::vector<double> priors;
};

// Two or three genotypes of 2-3 haplotypes of 300-700 bp with reads of 150 bp; short_haplotype: the last genotype's second
// haplotype is cut to 120 bp.
Region make_region(unsigned seed, bool short_haplotype)
{
    std::mt19937 rng {seed};
    const char* acgt = "ACGT";
    Region g;
    const int G = 2 + (int)(rng() % 2);
    for (int gi = 0; gi < G; ++gi) {
        const int hap_len = 300 + (int)(rng() % 400), n_haps = 2 + (int)(rng() % 2);
        std::string base((std::size_t)hap_len, 'A');
        for (auto& c : base) c = acgt[rng() % 4];
        for (int h = 0; h < n_haps; ++h) {
            std::string s = base;
            for (int k = 0; k < 3; ++k) s[rng() % (std::size_t)hap_len] = acgt[rng() % 4];
            if (short_haplotype && gi == G - 1 && h == 1) s = s.substr(0, 120);
            const std::size_t n = s.size();
            std::vector<char> mf(n), mr(n);
            std::vector<std::int8_t> pf(n), pr(n), go(n), ge(n);
            for (std::size_t i = 0; i < n; ++i) {
                mf[i] = s[(i + n - 1) % n]; mr[i] = s[(i + 1) % n];
                pf[i] = (std::int8_t)(1 + rng() % 125); pr[i] = (std::int8_t)(1 + rng() % 125);
                go[i] = (std::int8_t)(3 + rng() % 43); ge[i] = (std::int8_t)(1 + rng() % 10);
            }
            g.haps.add(s, mf, pf, mr, pr, go, ge, 0);
            g.priors.push_back(-(double)(rng() % 3));
        }
        for (int r = 0, n_reads = 20 + (int)(rng() % 60); r < n_reads; ++r) {
            const int L = 150;
            const int p = (int)(rng() % (std::size_t)(hap_len - L));
            std::string b = base.substr((std::size_t)p, (std::size_t)L);
            for (int k = 0; k < 2; ++k) b[rng() % L] = acgt[rng() % 4];
            std::vector<std::uint8_t> q((std::size_t)L);
            for (auto& x : q) x = (std::uint8_t)(2 + rng() % 40);
            g.reads.add(b, q, (std::uint8_t)(rng() % 2 ? 60 : 20), rng() % 2 == 0, p);
        }
        g.hap_first.push_back((std::int32_t)g.haps.size());
        g.read_first.push_back((std::int32_t)g.reads.size());
    }
    return g;
}

bool same(const std::vector<HaplotypeSupport>& a, const std::vector<HaplotypeSupport>& b)
{
    if (a.size() != b.size()) return false;
    for (std::size_t g = 0; g < a.size(); ++g) if (a[g].reads != b[g].reads || a[g].ambiguous != b[g].ambiguous) return false;
    return true;
}

bool same(const std::vector<Realignment>& a, const std::vector<Realignment>& b)
{
    if (a.size() != b.size()) return false;
    for (std::size_t i = 0; i < a.size(); ++i) {
        if (a[i].mapping_position != b[i].mapping_position || a[i].cigar != b[i].cigar ||
            std::memcmp(&a[i].likelihood, &b[i].likelihood, sizeof(double)) != 0) return false;
    }
    return true;
}

// what a call threw: "" (nothing), or the ShortHaplotypeError's index and extension
template <typename F>
std::string thrown(F&& f)
{
    try { f(); } catch (const ShortHaplotypeError& e) { return "short " + std::to_string(e.haplotype_index()) + " " + std::to_string(e.required_extension()); }
    return "";
}

} // namespace

int main()
{
    const int kThreads = 8, kRequests = 6, kShortThread = 5;
    try {
        SharedEngine shared {0, kThreads, 2000};
        phmm_config cfg;
        phmm_default_config(&cfg);
        cfg.max_indel_error = 8; cfg.use_mapping_quality = 0; cfg.use_flank_state = 0;
        const AmbiguousAction actions[] = {AmbiguousAction::drop, AmbiguousAction::first, AmbiguousAction::all};
        std::vector<int> mismatches(kThreads, 0), threw(kThreads, 0), errors(kThreads, 0);
        std::vector<std::thread> threads;
        for (int k = 0; k < kThreads; ++k) {
            threads.emplace_back([&, k] {
                try {
                    Engine own {0};
                    for (int i = 0; i < kRequests; ++i) {
                        const Region g = make_region(7919u * (unsigned)k + (unsigned)i, k == kShortThread && i == 3);
                        const AmbiguousAction action = actions[(k + i) % 3];
                        const std::vector<double>* priors = i % 2 ? &g.priors : nullptr;
                        std::vector<HaplotypeSupport> a, s;
                        const std::string a_threw = thrown([&] { a = compute_haplotype_support(g.reads, g.haps, g.hap_first, g.read_first, priors, action, cfg, own); });
                        const std::string s_threw = thrown([&] { s = compute_haplotype_support(g.reads, g.haps, g.hap_first, g.read_first, priors, action, cfg, shared); });
                        if (a_threw != s_threw || !same(a, s)) ++mismatches[k];
                        threw[k] += !s_threw.empty();
                        // realign every read of the region against haplotype i % H (ReadRealigner::realign)
                        const std::size_t hap = (std::size_t)i % g.haps.size();
                        std::vector<Realignment> ra, rs;
                        const std::string ra_threw = thrown([&] { ra = realign(g.reads, g.haps, hap, cfg, own); });
                        const std::string rs_threw = thrown([&] { rs = realign(g.reads, g.haps, hap, cfg, shared); });
                        if (ra_threw != rs_threw || !same(ra, rs)) ++mismatches[k];
                        threw[k] += !rs_threw.empty();
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
            ok = ok && !errors[k] && mismatches[k] == 0 && (k == kShortThread ? threw[k] >= 1 : threw[k] == 0);
            std::printf("THREAD %d mismatches=%d threw=%d\n", k, mismatches[k], threw[k]);
        }
        const auto st = shared.stats();
        std::printf("STATS requests=%lld gpu_calls=%lld merged_calls=%lld\n", (long long)st.requests, (long long)st.gpu_calls, (long long)st.merged_calls);
        ok = ok && st.merged_calls > 0;
        std::printf("BATCHER ALIGN %s\n", ok ? "ok" : "FAILED");
        return ok ? 0 : 1;
    } catch (const std::exception& ex) {
        std::printf("ERROR %s\n", ex.what());
        return 2;
    }
}
