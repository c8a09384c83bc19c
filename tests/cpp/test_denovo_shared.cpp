// Plain C++14 client of octopus_b200::DeNovoModel over one SharedEngine: N threads each build a new model per region (as
// trio_caller.cpp:406 does), prime it through the shared engine at the same time as the others, and compare every evaluate / status
// with a model over an Engine of the thread's own. Threads 0 .. N-2 use one pair of priors (their models are equal by content and
// merge); the last thread uses other priors (its requests never share a call with the others'). Built and run by
// tests/test_gpu_mutation_sets.py. Prints "SHARED ok <requests> <gpu_calls> <merged_calls> <max_regions_per_call>" on success.
#include <cstdio>
#include <cstdint>
#include <cstring>
#include <string>
#include <thread>
#include <vector>
#include "phmm_b200.hpp"

namespace {

using namespace octopus_b200;

constexpr int kThreads = 6, kRegions = 4;

struct Rng {
    std::uint64_t s;
    std::uint32_t next() { s = s * 6364136223846793005ULL + 1442695040888963407ULL; return static_cast<std::uint32_t>(s >> 33); }
    int below(int n) { return static_cast<int>(next() % static_cast<std::uint32_t>(n)); }
};

// one region's haplotypes: a base of 200-300 bp with a short tandem repeat, and copies of it with SNVs and 1-10 bp indels
std::vector<std::string> region(Rng& rng, int n)
{
    const char* acgt = "ACGT";
    std::string base;
    const int len = 200 + rng.below(100);
    for (int i = 0; i < len; ++i) base += acgt[rng.below(4)];
    const std::string unit = base.substr(0, 1 + rng.below(4));
    std::string str;
    for (int k = 0; k < 4 + rng.below(10); ++k) str += unit;
    base.insert(static_cast<std::size_t>(rng.below(len)), str);
    std::vector<std::string> haps {base};
    for (int h = 1; h < n; ++h) {
        std::string s = base;
        for (int e = rng.below(6); e > 0; --e) {
            const std::size_t at = static_cast<std::size_t>(rng.below(static_cast<int>(s.size()) - 12));
            const int kind = rng.below(3), k = 1 + rng.below(10);
            if (kind == 0) s[at] = acgt[(std::string {acgt}.find(s[at]) + 1 + rng.below(3)) % 4];
            else if (kind == 1) s.insert(at, s.substr(at, static_cast<std::size_t>(k)));
            else s.erase(at, static_cast<std::size_t>(k));
        }
        haps.push_back(s);
    }
    return haps;
}

MutationRepeatTable table()
{
    MutationRepeatTable t;
    const int cells = (t.max_period + 1) * (t.max_periodicity + 1);
    for (int c = 0; c < cells; ++c) {
        const int periods = c % (t.max_periodicity + 1);
        t.open.push_back(periods < 2 ? 1e-9f : 1e-9f * static_cast<float>(periods * periods));
        for (int k = 0; k < t.max_indel_length; ++k) t.extend.push_back(periods < 2 ? 0.5f : 0.8f);
    }
    return t;
}

} // namespace

int main(int argc, char** argv)
{
    if (argc > 1 && std::string {argv[1]} == "--compile-only") return 0;
    try {
        const MutationRepeatTable t = table();
        SharedEngine shared {0, kThreads, 200000};
        std::vector<std::string> failures(kThreads);
        std::vector<std::thread> pool;
        for (int k = 0; k < kThreads; ++k) {
            pool.emplace_back([&, k] {
                try {
                    Rng rng {1234567ULL + 7919ULL * static_cast<std::uint64_t>(k)};
                    const DeNovoModel::Parameters priors = k == kThreads - 1 ? DeNovoModel::Parameters {1e-4, 1e-6} : DeNovoModel::Parameters {1.3e-8, 1e-9};
                    auto approx = [] (std::size_t target, std::size_t given) { return -1000.0 - static_cast<double>(target * 1000 + given); };
                    std::vector<std::vector<std::string>> sets;
                    for (int r = 0; r < kRegions; ++r) sets.push_back(region(rng, 2 + rng.below(40)));
                    std::vector<DeNovoModel> on_shared;
                    for (const auto& haps : sets) {
                        on_shared.emplace_back(priors, t, shared, approx);
                        on_shared.back().prime(haps);
                    }
                    Engine own {0};
                    for (std::size_t r = 0; r < sets.size(); ++r) {
                        DeNovoModel alone {priors, t, own, approx};
                        alone.prime(sets[r]);
                        const std::size_t n = sets[r].size();
                        for (std::size_t a = 0; a < n; ++a) {
                            for (std::size_t b = 0; b < n; ++b) {
                                const double x = on_shared[r].evaluate(a, b), y = alone.evaluate(a, b);
                                if (on_shared[r].status(a, b) != alone.status(a, b) || std::memcmp(&x, &y, sizeof x) != 0) {
                                    char msg[200];
                                    std::snprintf(msg, sizeof msg, "thread %d region %zu pair (%zu, %zu): %a status %d vs %a status %d", k, r, a, b, x,
                                                  on_shared[r].status(a, b), y, alone.status(a, b));
                                    failures[k] = msg;
                                    return;
                                }
                            }
                        }
                    }
                } catch (const std::exception& ex) {
                    failures[k] = ex.what();
                }
            });
        }
        for (auto& th : pool) th.join();
        for (int k = 0; k < kThreads; ++k) {
            if (!failures[k].empty()) { std::printf("ERROR %s\n", failures[k].c_str()); return 1; }
        }
        const phmm_batcher_stats s = shared.stats();
        std::printf("SHARED ok %lld %lld %lld %lld\n", static_cast<long long>(s.requests), static_cast<long long>(s.gpu_calls),
                    static_cast<long long>(s.merged_calls), static_cast<long long>(s.max_regions_per_call));
    } catch (const std::exception& ex) {
        std::printf("ERROR %s\n", ex.what());
        return 1;
    }
    return 0;
}
