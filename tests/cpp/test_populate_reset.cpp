// Plain C++14 client of octopus_b200::HaplotypeLikelihoodArray with an error model: N std::threads, each with its own array over one
// SharedEngine, populate from haplotype sequences only (the GPU runs the model's reset() in the call). Every result is compared,
// byte for byte, with HaplotypeBlock::reset(model) + an array over an Engine of the thread's own, for a two-sample ReadMap and a
// TemplateMap; a region with a haplotype shorter than its reads throws the same ShortHaplotypeError both ways; merge_samples keeps the
// model. Built and run by tests/test_gpu_populate_reset.py. Prints "RESET ok <requests> <gpu_calls> <merged_calls>" on success.
#include <cstdio>
#include <cstdint>
#include <cstring>
#include <functional>
#include <mutex>
#include <string>
#include <thread>
#include <vector>
#include "phmm_b200.hpp"

namespace {

using namespace octopus_b200;

constexpr int kThreads = 6, kRegions = 3;

struct Rng {
    std::uint64_t s;
    std::uint32_t next() { s = s * 6364136223846793005ULL + 1442695040888963407ULL; return static_cast<std::uint32_t>(s >> 33); }
    int below(int n) { return static_cast<int>(next() % static_cast<std::uint32_t>(n)); }
};

struct Region {
    std::vector<std::string> haps;
    std::vector<std::vector<bool>> subs;
    HaplotypeLikelihoodArray::ReadMap reads;
    HaplotypeLikelihoodArray::TemplateMap templates;
};

// 8 haplotypes of 300 bp with a tandem repeat and a few SNVs (some flagged as substitutions); two samples of reads drawn from them
Region region(Rng& rng, int hap_len)
{
    const char* acgt = "ACGT";
    std::string base;
    for (int i = 0; i < hap_len; ++i) base += acgt[rng.below(4)];
    const std::string unit = base.substr(0, 1 + rng.below(3));
    std::string str;
    for (int k = 0; k < 6 + rng.below(8); ++k) str += unit;
    base.replace(static_cast<std::size_t>(rng.below(hap_len - static_cast<int>(str.size()))), str.size(), str);
    Region g;
    for (int h = 0; h < 8; ++h) {
        std::string s = base;
        std::vector<bool> sub(s.size(), false);
        for (int e = rng.below(4); e > 0; --e) { const auto at = static_cast<std::size_t>(rng.below(hap_len)); s[at] = acgt[rng.below(4)]; sub[at] = true; }
        g.haps.push_back(s);
        g.subs.push_back(sub);
    }
    for (int sample = 0; sample < 2; ++sample) {
        ReadBlock rb;
        TemplateBlock tb;
        for (int r = 0; r < 40; ++r) {
            const int len = 60 + rng.below(60);
            const int at = hap_len > len ? rng.below(hap_len - len) : 0;
            std::string bases = g.haps[static_cast<std::size_t>(rng.below(8))].substr(static_cast<std::size_t>(at), static_cast<std::size_t>(len));
            bases.resize(static_cast<std::size_t>(len), 'A');
            if (rng.below(3) == 0) bases[static_cast<std::size_t>(rng.below(len))] = acgt[rng.below(4)];
            std::vector<std::uint8_t> quals;
            for (int i = 0; i < len; ++i) quals.push_back(static_cast<std::uint8_t>(10 + rng.below(30)));
            const auto mapq = static_cast<std::uint8_t>(rng.below(61));
            rb.add(bases, quals, mapq, rng.below(2) == 1, 1000 + at);
            ReadBlock one;
            one.add(bases, quals, mapq, rng.below(2) == 1, 1000 + at);
            tb.add(one);
        }
        g.reads.emplace_back("S" + std::to_string(sample), rb);
        g.templates.emplace_back("S" + std::to_string(sample), tb);
    }
    return g;
}

HaplotypeBlock sequences(const Region& g)
{
    HaplotypeBlock hb;
    for (std::size_t h = 0; h < g.haps.size(); ++h) hb.add(g.haps[h], 1000, &g.subs[h]);
    return hb;
}

bool same(const HaplotypeLikelihoodArray& a, const HaplotypeLikelihoodArray& b)
{
    if (a.num_haplotypes() != b.num_haplotypes() || a.samples() != b.samples()) return false;
    for (const auto& s : a.samples()) {
        if (a.num_likelihoods(s) != b.num_likelihoods(s)) return false;
        for (std::size_t h = 0; h < a.num_haplotypes(); ++h) {
            const auto x = a(s, h), y = b(s, h);
            if (std::memcmp(x.begin(), y.begin(), x.size() * sizeof(double)) != 0) return false;
        }
    }
    return true;
}

std::string short_error(const std::function<void()>& f)
{
    try { f(); } catch (const ShortHaplotypeError& e) { return e.what(); }
    return "";
}

} // namespace

int main(int argc, char** argv)
{
    if (argc > 1 && std::string {argv[1]} == "--compile-only") return 0;
    phmm_config cfg = HaplotypeLikelihoodArray::default_config();
    cfg.max_indel_error = 16;
    const ErrorModel model {"PCR.NovaSeq"};
    SharedEngine shared {0, kThreads, 2000};
    FlankState flank {20, 30};
    std::mutex m;
    std::vector<std::string> failures;
    auto fail = [&](const std::string& what) { std::lock_guard<std::mutex> lk(m); failures.push_back(what); };

    std::vector<std::thread> threads;
    for (int t = 0; t < kThreads; ++t) {
        threads.emplace_back([&, t] {
            Rng rng {0x5EED0000ULL + static_cast<std::uint64_t>(t)};
            Engine own;
            for (int k = 0; k < kRegions; ++k) {
                const Region g = region(rng, 300);
                const HaplotypeBlock seqs = sequences(g);
                HaplotypeBlock full = sequences(g);
                full.reset(model);
                HaplotypeLikelihoodArray got {cfg, model, shared}, want {cfg, own};
                got.populate(g.reads, seqs, &flank);
                want.populate(g.reads, full, &flank);
                if (!same(got, want)) fail("ReadMap thread " + std::to_string(t));
                HaplotypeLikelihoodArray merged = got.merge_samples();
                merged.populate(g.reads[0].second, seqs, &flank);     // still runs the model: the block has no penalty arrays
                HaplotypeLikelihoodArray want_one {cfg, own};
                want_one.populate(g.reads[0].second, full, &flank);
                if (!same(merged, want_one)) fail("merge_samples thread " + std::to_string(t));
                got.populate(g.templates, seqs, &flank);
                want.populate(g.templates, full, &flank);
                if (!same(got, want)) fail("TemplateMap thread " + std::to_string(t));
                HaplotypeLikelihoodArray on_engine {cfg, model, own};
                on_engine.populate(g.reads, seqs, &flank);
                want.populate(g.reads, full, &flank);
                if (!same(on_engine, want)) fail("Engine array thread " + std::to_string(t));
            }
            if (t == 0) {                                         // 50-base haplotypes under reads of 60-119 bases
                const Region g = region(rng, 50);
                HaplotypeBlock full = sequences(g);
                full.reset(model);
                HaplotypeLikelihoodArray got {cfg, model, shared}, want {cfg, own};
                const std::string a = short_error([&] { got.populate(g.reads, sequences(g)); });
                const std::string b = short_error([&] { want.populate(g.reads, full); });
                if (a.empty() || a != b) fail("ShortHaplotypeError '" + a + "' vs '" + b + "'");
            }
        });
    }
    for (auto& th : threads) th.join();
    for (const auto& f : failures) std::printf("FAIL %s\n", f.c_str());
    if (!failures.empty()) return 1;
    const phmm_batcher_stats st = shared.stats();
    std::printf("RESET ok %lld %lld %lld\n", static_cast<long long>(st.requests), static_cast<long long>(st.gpu_calls),
                static_cast<long long>(st.merged_calls));
    return 0;
}
