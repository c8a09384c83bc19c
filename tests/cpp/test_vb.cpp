// The C++ adapter octopus_b200::run_variational_bayes over a populated two-sample HaplotypeLikelihoodArray. Prints the matrix
// (MATRIX H R, then H*R values), the sample widths (WIDTHS) and the result (POST, LPOST, WEIGHTED, ALPHA per sample, EVIDENCE),
// every value as %.17g, for tests/test_gpu_variational_bayes.py to hold against the Python API on the same matrix.
#include <cstdio>
#include <string>
#include <vector>
#include "phmm_b200.hpp"

using namespace octopus_b200;

int main()
{
    try {
        HaplotypeBlock haps;
        const std::string h0 = "ACGTTGCAAGCTTAGGCTAACGTTAGCATCGATCGGATCTAGCTAGGATCGATACGATCGATCGTAGCTAGCTAGTCGATCGATTTAGCGCGATATCGCGAT";
        std::string h1 = h0, h2 = h0; h1[50] = h1[50] == 'A' ? 'C' : 'A'; h2[40] = h2[40] == 'G' ? 'T' : 'G';
        for (const auto& h : {h0, h1, h2}) {
            std::vector<char> mf(h.begin(), h.end()), mr(h.begin(), h.end());
            std::vector<std::int8_t> p(h.size(), 50), go(h.size(), 40), ge(h.size(), 3);
            haps.add(h, mf, p, mr, p, go, ge, 0);
        }
        ReadBlock normal, tumour;
        for (int i = 0; i < 6; ++i) normal.add(h0.substr(20 + 5 * i, 40), std::vector<std::uint8_t>(40, 30), 60, i % 2, 20 + 5 * i);
        for (int i = 0; i < 5; ++i) tumour.add((i < 2 ? h1 : h0).substr(25 + 6 * i, 40), std::vector<std::uint8_t>(40, 28), 60, i % 2, 25 + 6 * i);
        auto cfg = HaplotypeLikelihoodArray::default_config();
        cfg.max_indel_error = 16;
        HaplotypeLikelihoodArray arr {cfg};
        arr.populate(HaplotypeLikelihoodArray::ReadMap {{"normal", normal}, {"tumour", tumour}}, haps);
        const std::vector<SampleName> samples {"normal", "tumour"};
        std::printf("MATRIX %zu %zu", arr.num_haplotypes(), arr.num_likelihoods("normal") + arr.num_likelihoods("tumour"));
        for (std::size_t h = 0; h < arr.num_haplotypes(); ++h)
            for (const auto& s : samples) for (double v : arr(s, h)) std::printf(" %.17g", v);
        std::printf("\nWIDTHS %zu %zu\n", arr.num_likelihoods("normal"), arr.num_likelihoods("tumour"));
        const std::vector<std::vector<std::int32_t>> genotypes {{0, 0}, {0, 1}, {0, 2}, {1, 2}, {1, 1}};
        const std::unordered_map<SampleName, std::vector<double>> prior_alphas {{"normal", {1.0, 0.5}}, {"tumour", {1.0, 0.8}}};
        const std::vector<double> log_priors(genotypes.size(), -1.6094379124341003);
        std::vector<std::vector<double>> seeds;
        for (std::size_t i = 0; i < genotypes.size(); ++i) {
            seeds.emplace_back(genotypes.size(), -13.815510557964274);
            seeds.back()[i] = -4e-6;
        }
        Engine engine;
        const auto r = run_variational_bayes(engine, arr, samples, genotypes, prior_alphas, log_priors, VariationalBayesParameters {}, seeds);
        auto row = [] (const char* name, const std::vector<double>& v) { std::printf("%s", name); for (double x : v) std::printf(" %.17g", x); std::printf("\n"); };
        row("POST", r.max_evidence_params.genotype_probabilities);
        row("LPOST", r.max_evidence_params.genotype_log_probabilities);
        row("WEIGHTED", r.weighted_genotype_posteriors);
        row("ALPHA_normal", r.max_evidence_params.alphas.at("normal"));
        row("ALPHA_tumour", r.max_evidence_params.alphas.at("tumour"));
        std::printf("EVIDENCE %.17g\n", r.approx_log_evidence);
        try {   // refused input surfaces as Error
            run_variational_bayes(engine, arr, samples, genotypes, prior_alphas, log_priors, VariationalBayesParameters {0.05, 0}, seeds);
            std::printf("REFUSED no\n");
        } catch (const Error&) { std::printf("REFUSED yes\n"); }
    } catch (const std::exception& e) {
        std::printf("ERROR %s\n", e.what());
        return 1;
    }
    return 0;
}
