// The C++ adapter octopus_b200::VariationalBayesMixtureMixtureModel over a populated four-cell HaplotypeLikelihoodArray, one
// haploid and one diploid group. Prints the matrix (MATRIX H R, then H*R values), the cell widths (WIDTHS) and the result of
// the scalar overload with group priors on cell 1 (POST, LPOST, GCONC, MCONC, SIGMA, WEIGHTED, WSIGMA, EVIDENCE), every value as
// %.17g, for tests/test_gpu_variational_bayes_mixture_mixture.py to hold against the Python API on the same matrix. Also checks
// that the scalar overloads give the bits of the general one with the expanded concentrations (EXPANSION), and that refused
// input surfaces as Error (REFUSED).
#include <cstdio>
#include <string>
#include <vector>
#include "phmm_b200.hpp"

using namespace octopus_b200;
using Model = VariationalBayesMixtureMixtureModel;

namespace {

bool same(const Model::Inferences& a, const Model::Inferences& b)
{
    const auto& x = a.map.latents;
    const auto& y = b.map.latents;
    return x.genotype_posteriors == y.genotype_posteriors && x.genotype_log_posteriors == y.genotype_log_posteriors &&
           x.group_concentrations == y.group_concentrations && x.mixture_concentrations == y.mixture_concentrations &&
           x.group_responsibilities == y.group_responsibilities && a.map.approx_log_evidence == b.map.approx_log_evidence &&
           a.weighted_genotype_posteriors == b.weighted_genotype_posteriors &&
           a.weighted_group_responsibilities == b.weighted_group_responsibilities;
}

} // namespace

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
        const std::vector<SampleName> cells {"c0", "c1", "c2", "c3"};
        HaplotypeLikelihoodArray::ReadMap reads;
        const int n_reads[4] = {4, 1, 2, 5};
        for (int c = 0; c < 4; ++c) {
            ReadBlock b;
            for (int i = 0; i < n_reads[c]; ++i) {
                const auto& src = (c + i) % 3 == 0 ? h1 : ((c + i) % 3 == 1 ? h2 : h0);
                b.add(src.substr(20 + 6 * i, 40), std::vector<std::uint8_t>(40, 30), 60, i % 2, 20 + 6 * i);
            }
            reads.emplace_back(cells[c], b);
        }
        auto cfg = HaplotypeLikelihoodArray::default_config();
        cfg.max_indel_error = 16;
        HaplotypeLikelihoodArray arr {cfg};
        arr.populate(reads, haps);
        std::size_t R = 0;
        for (const auto& c : cells) R += arr.num_likelihoods(c);
        std::printf("MATRIX %zu %zu", arr.num_haplotypes(), R);
        for (std::size_t h = 0; h < arr.num_haplotypes(); ++h)
            for (const auto& c : cells) for (double v : arr(c, h)) std::printf(" %.17g", v);
        std::printf("\nWIDTHS");
        for (const auto& c : cells) std::printf(" %zu", arr.num_likelihoods(c));
        std::printf("\n");
        const Model::GenotypeVector genotypes {{0}, {1}, {2}, {0, 0}, {0, 1}, {0, 2}, {1, 2}};
        Model::GenotypeCombinationVector combos;
        for (std::size_t a = 0; a < 3; ++a) for (std::size_t b = 3; b < 7; ++b) combos.push_back({a, b});
        const std::vector<double> log_priors(combos.size(), -2.4849066497880004);
        std::vector<std::vector<double>> seeds {std::vector<double>(combos.size(), -2.4849066497880004)};
        for (std::size_t i = 0; i < 3; ++i) {
            seeds.emplace_back(combos.size(), -11.608235644774552);
            seeds.back()[i] = -0.00010000500033334732;
        }
        Model::GroupOptionalPriorArray priors(cells.size());
        priors[1] = {0.7, 0.3};
        Engine engine;
        const Model model {Model::Options {}, engine};
        const auto r = model.evaluate(log_priors, arr, cells, genotypes, combos, priors, 1.0, 0.8, seeds);
        auto row = [] (const char* name, const std::vector<double>& v) { std::printf("%s", name); for (double x : v) std::printf(" %.17g", x); std::printf("\n"); };
        auto flat = [] (const std::vector<std::vector<double>>& v) { std::vector<double> f; for (const auto& x : v) f.insert(f.end(), x.begin(), x.end()); return f; };
        row("POST", r.map.latents.genotype_posteriors);
        row("LPOST", r.map.latents.genotype_log_posteriors);
        row("GCONC", r.map.latents.group_concentrations);
        std::vector<double> mc;
        for (const auto& s : r.map.latents.mixture_concentrations) { const auto f = flat(s); mc.insert(mc.end(), f.begin(), f.end()); }
        row("MCONC", mc);
        row("SIGMA", flat(r.map.latents.group_responsibilities));
        row("WEIGHTED", r.weighted_genotype_posteriors);
        row("WSIGMA", flat(r.weighted_group_responsibilities));
        std::printf("EVIDENCE %.17g\n", r.map.approx_log_evidence);
        const Model::MixtureConcentrationArray full(cells.size(), Model::MixtureConcentrationVector {{0.8}, {0.8, 0.8}});
        const bool expansion = same(r, model.evaluate(log_priors, arr, cells, genotypes, combos, priors, {1.0, 1.0}, full, seeds)) &&
                               same(r, model.evaluate(log_priors, arr, cells, genotypes, combos, priors, 1.0, std::vector<double>(4, 0.8), seeds)) &&
                               same(model.evaluate(log_priors, arr, cells, genotypes, combos, 1.0, 0.8, seeds),
                                    model.evaluate(log_priors, arr, cells, genotypes, combos, Model::GroupOptionalPriorArray(4), 1.0, 0.8, seeds)) &&
                               same(model.evaluate(log_priors, arr, cells, genotypes, combos, 1.0, std::vector<double>(4, 0.8), seeds),
                                    model.evaluate(log_priors, arr, cells, genotypes, combos, {1.0, 1.0}, full, seeds));
        std::printf("EXPANSION %s\n", expansion ? "yes" : "no");
        try {
            Model {Model::Options {0.05, 0}, engine}.evaluate(log_priors, arr, cells, genotypes, combos, 1.0, 0.8, seeds);
            std::printf("REFUSED no\n");
        } catch (const Error&) { std::printf("REFUSED yes\n"); }
    } catch (const std::exception& e) {
        std::printf("ERROR %s\n", e.what());
        return 1;
    }
    return 0;
}
