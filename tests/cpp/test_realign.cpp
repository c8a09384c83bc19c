// Plain C++14 client of the realignment entry points through the C++ adapter: octopus_b200::realign (ReadRealigner::realign
// for one haplotype), Engine::map_pairs and the ShortHaplotypeError the helper throws. Built and run by tests/test_gpu_realign.py,
// which checks the printed results against the reference composition (k-mer mapper uncapped, then HaplotypeLikelihoodModel::align).
#include <cstdio>
#include <string>
#include <vector>
#include "phmm_b200.hpp"

namespace {

void add_haplotype(octopus_b200::HaplotypeBlock& haps, const std::string& h)
{
    std::vector<char> mask(h.begin(), h.end());
    std::vector<std::int8_t> prior(h.size(), 50), go(h.size(), 40), ge(h.size(), 3);
    haps.add(h, mask, prior, mask, prior, go, ge, 0);
}

} // namespace

int main()
{
    using namespace octopus_b200;
    try {
        const std::string h0 = "ACGTTGCAAGCTTAGGCTAACGTTAGCATCGATCGGATCTAGCTAGGATCGATACGATCGATCGTAGCTAGCTAGTCGATCGATTTAGCGCGATATCGCGAT";
        std::string rep;
        for (int i = 0; i < 60; ++i) rep += "AC";
        const std::string h1 = "GGCT" + rep + "TTGA";
        HaplotypeBlock haps;
        add_haplotype(haps, h0);
        add_haplotype(haps, h1);
        ReadBlock reads;
        std::string r1 = h0.substr(35, 40);
        r1[12] = r1[12] == 'A' ? 'C' : 'A';
        reads.add(h0.substr(30, 40), std::vector<std::uint8_t>(40, 30), 60, false, 30);
        reads.add(r1, std::vector<std::uint8_t>(40, 25), 60, true, 35);
        reads.add(rep.substr(0, 40), std::vector<std::uint8_t>(40, 35), 60, false, 10);
        auto cfg = HaplotypeLikelihoodArray::default_config();
        cfg.max_indel_error = 8;          // the realigner's default model
        cfg.use_mapping_quality = 0;      // likelihoods are -ln10/10 times an integer penalty: compared bit for bit
        Engine engine;
        for (std::size_t h = 0; h < haps.size(); ++h) {
            const auto result = realign(reads, haps, h, cfg, engine);
            for (std::size_t r = 0; r < result.size(); ++r)
                std::printf("RA %zu %zu %lld %s %.17g\n", h, r, (long long)result[r].mapping_position, result[r].cigar.c_str(), result[r].likelihood);
        }
        const std::vector<phmm_pair> pairs {{0, 0}, {1, 0}, {2, 1}, {0, 1}};
        const auto m = engine.map_pairs(haps.view(), reads.view(), pairs);
        for (std::size_t j = 0; j < pairs.size(); ++j) {
            std::printf("MAP %d %d", pairs[j].read, pairs[j].hap);
            for (auto k = m.offsets[j]; k < m.offsets[j + 1]; ++k) std::printf(" %d", m.positions[(std::size_t)k]);
            std::printf("\n");
        }
        // a haplotype too short for the reads: the helper throws for the first such read in read order
        HaplotypeBlock short_haps;
        add_haplotype(short_haps, h0.substr(25, 45));
        try {
            realign(reads, short_haps, 0, cfg, engine);
            std::printf("SHORT none\n");
        } catch (const ShortHaplotypeError& e) {
            std::printf("SHORT hap=%zu ext=%u\n", e.haplotype_index(), e.required_extension());
        }
    } catch (const std::exception& e) {
        std::printf("EXCEPTION %s\n", e.what());
        return 1;
    }
    return 0;
}
