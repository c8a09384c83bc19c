// Plain C++14 client of octopus_b200::compute_haplotype_support (read assignment for many genotypes in one GPU call) with the drop,
// first and all ambiguity actions, and the ShortHaplotypeError it throws. Built and run by tests/test_gpu_assign.py, which writes the
// groups to a file (argv[1]) and checks the printed support against the reference composition and find_map_haplotypes.
//   line 1: H R G; then H haplotype lines "seq mask_fwd prior_fwd mask_rev prior_rev gap_open gap_extend log_prior" (lists
//   comma-separated), R read lines "bases quals mapq reverse begin", and the lines hap_first[G+1], read_first[G+1].
#include <cstdio>
#include <fstream>
#include <sstream>
#include <string>
#include <vector>
#include "phmm_b200.hpp"

namespace {

template <typename T>
std::vector<T> list(const std::string& s)
{
    std::vector<T> out;
    std::stringstream ss {s};
    std::string item;
    while (std::getline(ss, item, ',')) out.push_back(static_cast<T>(std::stol(item)));
    return out;
}

const char* name(octopus_b200::AmbiguousAction a)
{
    return a == octopus_b200::AmbiguousAction::drop ? "drop" : a == octopus_b200::AmbiguousAction::first ? "first" : "all";
}

} // namespace

int main(int argc, char** argv)
{
    using namespace octopus_b200;
    if (argc < 2) return 2;
    try {
        std::ifstream in {argv[1]};
        std::size_t H = 0, R = 0, G = 0;
        in >> H >> R >> G;
        HaplotypeBlock haps;
        std::vector<double> priors;
        for (std::size_t h = 0; h < H; ++h) {
            std::string seq, mf, pf, mr, pr, go, ge;
            double prior;
            in >> seq >> mf >> pf >> mr >> pr >> go >> ge >> prior;
            haps.add(seq, std::vector<char>(mf.begin(), mf.end()), list<std::int8_t>(pf), std::vector<char>(mr.begin(), mr.end()),
                     list<std::int8_t>(pr), list<std::int8_t>(go), list<std::int8_t>(ge), 0);
            priors.push_back(prior);
        }
        ReadBlock reads;
        for (std::size_t r = 0; r < R; ++r) {
            std::string bases, quals;
            int mapq, reverse;
            long long begin;
            in >> bases >> quals >> mapq >> reverse >> begin;
            reads.add(bases, list<std::uint8_t>(quals), static_cast<std::uint8_t>(mapq), reverse != 0, begin);
        }
        std::vector<std::int32_t> hap_first(G + 1), read_first(G + 1);
        for (auto& x : hap_first) in >> x;
        for (auto& x : read_first) in >> x;
        auto cfg = HaplotypeLikelihoodArray::default_config();
        cfg.max_indel_error = 16;
        cfg.use_mapping_quality = 0;
        Engine engine;
        for (const auto action : {AmbiguousAction::drop, AmbiguousAction::first, AmbiguousAction::all}) {
            const auto support = compute_haplotype_support(reads, haps, hap_first, read_first, &priors, action, cfg, engine);
            for (std::size_t g = 0; g < support.size(); ++g) {
                for (std::size_t k = 0; k < support[g].reads.size(); ++k)
                    for (const auto r : support[g].reads[k]) std::printf("SUP %s %zu %zu %zu\n", name(action), g, k, r);
                for (const auto& a : support[g].ambiguous) {
                    std::printf("AMB %s %zu %zu", name(action), g, a.first);
                    for (const auto k : a.second) std::printf(" %u", k);
                    std::printf("\n");
                }
            }
        }
        // one more group: haplotype 0's first 60 bases against group 0's reads, too short for them
        HaplotypeBlock more = haps;
        const std::string seq0(haps.seq.begin(), haps.seq.begin() + 60);
        more.add(seq0, std::vector<char>(haps.snv_mask_fwd.begin(), haps.snv_mask_fwd.begin() + 60),
                 std::vector<std::int8_t>(haps.snv_prior_fwd.begin(), haps.snv_prior_fwd.begin() + 60),
                 std::vector<char>(haps.snv_mask_rev.begin(), haps.snv_mask_rev.begin() + 60),
                 std::vector<std::int8_t>(haps.snv_prior_rev.begin(), haps.snv_prior_rev.begin() + 60),
                 std::vector<std::int8_t>(haps.gap_open.begin(), haps.gap_open.begin() + 60),
                 std::vector<std::int8_t>(haps.gap_extend.begin(), haps.gap_extend.begin() + 60), 0);
        ReadBlock more_reads = reads;
        for (std::int32_t r = read_first[0]; r < read_first[1]; ++r) {
            const auto b = static_cast<std::size_t>(reads.off[r]), e = static_cast<std::size_t>(reads.off[r + 1]);
            more_reads.add(std::string(reads.bases.begin() + b, reads.bases.begin() + e),
                           std::vector<std::uint8_t>(reads.quals.begin() + b, reads.quals.begin() + e), reads.mapq[r], reads.reverse[r] != 0, reads.begin[r]);
        }
        auto hf = hap_first, rf = read_first;
        hf.push_back(hf.back() + 1);
        rf.push_back(rf.back() + (read_first[1] - read_first[0]));
        priors.push_back(0.0);
        try {
            compute_haplotype_support(more_reads, more, hf, rf, &priors, AmbiguousAction::drop, cfg, engine);
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
