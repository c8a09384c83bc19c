// The per-call seam, literally: the reference's OWN hmm::evaluate / hmm::align templates (src/core/models/pairhmm/pair_hmm.hpp:827-874,
// compiled from the reference checkout, Boost-free through oracle/ref_shim/) instantiated over octopus_b200::GpuPairHMM<Band>
// and over the reference's SIMD kernel, on the same seeded inputs. Every value must be identical: the GPU type is a drop-in
// for the duck-typed PairHMM concept (band_size, name, 4 x align, calculate_flank_score).
//
// Built only where the reference checkout is given (tests/test_gpu_cpp.py), into oracle/_ref/ beside the other reference builds.
#include <cstdint>
#include <cstdio>
#include <string>
#include <vector>

#include "core/models/pairhmm/pair_hmm.hpp"
#include "phmm_b200.hpp"

namespace {

struct Rng   // splitmix64: the test must not depend on a library's distribution implementations
{
    std::uint64_t s;
    std::uint64_t next() { std::uint64_t z = (s += 0x9E3779B97F4A7C15ull); z = (z ^ (z >> 30)) * 0xBF58476D1CE4E5B9ull; z = (z ^ (z >> 27)) * 0x94D049BB133111EBull; return z ^ (z >> 31); }
    int below(int n) { return static_cast<int>(next() % static_cast<std::uint64_t>(n)); }
    int range(int lo, int hi) { return lo + below(hi - lo + 1); }
    char base() { return "ACGT"[below(4)]; }
};

std::string cigar_text(const octopus::CigarString& cigar)
{
    std::string text;
    for (const auto& op : cigar) { text += std::to_string(op.size()); text += static_cast<char>(op.flag()); }
    return text;
}

template <int Band>
int run(Rng& rng, int n_cases, int& n_traceback)
{
    using namespace octopus::hmm;
    const octopus_b200::GpuPairHMM<Band> gpu;
    const auto cpu = simd::make_simd_pair_hmm<Band>();
    int bad = 0;
    for (int it = 0; it < n_cases; ++it) {
        const int L = rng.range(8, 70), hap_len = L + 2 * Band + rng.range(2, 70);
        std::string truth(hap_len, 'A');
        for (auto& b : truth) b = rng.base();
        if (rng.below(5) == 0) truth[rng.below(hap_len)] = 'N';
        const int start = rng.below(hap_len - L + 1);
        std::string target = truth.substr(start, L);
        for (auto& b : target) if (b == 'N') b = 'A';
        const int kind = rng.below(10);
        if (kind >= 2) { const int n_sub = kind < 5 ? 1 : rng.range(1, 4); for (int i = 0; i < n_sub; ++i) target[rng.below(L)] = rng.base(); }
        if (kind >= 8 && L > 12) { const int p = rng.range(3, L - 6); target = target.substr(0, p) + target.substr(p + 2) + std::string {rng.base(), rng.base()}; }
        std::vector<std::uint8_t> quals(L);
        for (auto& q : quals) q = static_cast<std::uint8_t>(rng.range(2, 41));
        PenaltyVector go(hap_len), ge(hap_len), pr(hap_len);
        NucleotideVector mask(hap_len);
        for (int i = 0; i < hap_len; ++i) { go[i] = rng.range(3, 45); ge[i] = rng.range(1, 10); pr[i] = rng.range(1, 125); mask[i] = "ACGTN"[rng.below(5)]; }
        const std::size_t lhs = rng.below(3) ? rng.below(hap_len / 2) : 0, rhs = rng.below(3) ? rng.below(hap_len / 2) : 0;
        const MutationModel params {go, ge, mask, pr, {}, lhs, rhs, 2};
        // near the true position, or anywhere (including windows that leave the haplotype → lowest())
        int offset = rng.below(5) ? start + rng.range(-3, 3) : rng.below(hap_len);
        if (offset < 0) offset = 0;
        const double eg = evaluate(truth, target, quals, static_cast<std::size_t>(offset), gpu, params);
        const double ec = evaluate(truth, target, quals, static_cast<std::size_t>(offset), cpu, params);
        bool ok = eg == ec;
        if (detail::target_overlaps_truth_flank(truth, target, static_cast<std::size_t>(offset), cpu, params)) ++n_traceback;
        if (offset >= Band && offset + L + Band <= hap_len) {   // align() asserts an in-range window
            Alignment ag, ac;
            align(truth, target, quals, static_cast<std::size_t>(offset), gpu, params, ag);
            align(truth, target, quals, static_cast<std::size_t>(offset), cpu, params, ac);
            ok = ok && ag.target_offset == ac.target_offset && ag.likelihood == ac.likelihood && cigar_text(ag.cigar) == cigar_text(ac.cigar);
        }
        if (!ok) { if (++bad <= 5) std::printf("MISMATCH band=%d case=%d L=%d hap=%d offset=%d gpu=%.17g cpu=%.17g\n", Band, it, L, hap_len, offset, eg, ec); }
    }
    return bad;
}

} // namespace

// octopus_b200::PairHMM<Parameters> against octopus::hmm::PairHMM<Parameters> (pair_hmm.hpp:892-1032): same constructor, set(), band_size(),
// evaluate() and align() — the class HaplotypeLikelihoodModel holds (haplotype_likelihood_model.hpp:106), runtime band 8..256.
int run_class(Rng& rng, int n_cases)
{
    using namespace octopus::hmm;
    int bad = 0;
    for (int it = 0; it < n_cases; ++it) {
        const unsigned request = static_cast<unsigned>(rng.range(1, 70));
        const int L = rng.range(8, 60);
        octopus::hmm::PairHMM<MutationModel> cpu {request};
        octopus_b200::PairHMM<MutationModel> gpu {request};
        if (cpu.band_size() != gpu.band_size()) { ++bad; continue; }
        const int band = cpu.band_size(), hap_len = L + 2 * band + rng.range(2, 40);
        std::string truth(hap_len, 'A');
        for (auto& b : truth) b = rng.base();
        const int start = rng.range(band, hap_len - L - band);
        std::string target = truth.substr(start, L);
        for (int i = 0; i < rng.range(0, 3); ++i) target[rng.below(L)] = rng.base();
        std::vector<std::uint8_t> quals(L);
        for (auto& q : quals) q = static_cast<std::uint8_t>(rng.range(2, 41));
        PenaltyVector go(hap_len), ge(hap_len), pr(hap_len);
        NucleotideVector mask(hap_len);
        for (int i = 0; i < hap_len; ++i) { go[i] = rng.range(3, 45); ge[i] = rng.range(1, 10); pr[i] = rng.range(1, 125); mask[i] = "ACGTN"[rng.below(5)]; }
        const MutationModel params {go, ge, mask, pr, {}, static_cast<std::size_t>(rng.below(hap_len / 3)), static_cast<std::size_t>(rng.below(hap_len / 3)), 2};
        cpu.set(params); gpu.set(params);
        const std::size_t offset = static_cast<std::size_t>(start);
        bool ok = cpu.evaluate(target, truth, quals, offset) == gpu.evaluate(target, truth, quals, offset);
        const Alignment ac = cpu.align(target, truth, quals, offset), ag = gpu.align(target, truth, quals, offset);
        ok = ok && ag.target_offset == ac.target_offset && ag.likelihood == ac.likelihood && cigar_text(ag.cigar) == cigar_text(ac.cigar);
        if (!ok && ++bad <= 5) std::printf("CLASS MISMATCH case=%d band=%d L=%d\n", it, band, L);
    }
    bool threw = false;
    try { octopus_b200::PairHMM<MutationModel> too_wide {300u}; } catch (const octopus_b200::TooLargeBandSizeError&) { threw = true; }
    return bad + (threw ? 0 : 1);
}

int main()
{
    try {
        Rng rng {20240923};
        int n_traceback = 0;
        const int bad = run<8>(rng, 250, n_traceback) + run<16>(rng, 250, n_traceback) + run<32>(rng, 120, n_traceback) + run_class(rng, 60);
        std::printf("DROPIN %s mismatches=%d traceback_cases=%d\n", bad == 0 ? "ok" : "FAILED", bad, n_traceback);
        return bad == 0 ? 0 : 1;
    } catch (const std::exception& e) {
        std::printf("EXCEPTION %s\n", e.what());
        return 2;
    }
}
