// TEST INFRASTRUCTURE ONLY. A C entry point over the UNMODIFIED reference VariationalBayesMixtureMixtureModel
// (core/models/genotype/variational_bayes_mixture_mixture_model.cpp, compiled alongside), built by vbmm.mk into
// _ref/libref_vbmm.so. It builds the reference's HaplotypeLikelihoodMatrix from per-sample copies of the matrix columns and calls
// its most general evaluate overload.
#include <cstdint>
#include <vector>

#include "core/models/genotype/variational_bayes_mixture_mixture_model.hpp"

using namespace octopus;
using Model = octopus::model::VariationalBayesMixtureMixtureModel;

namespace {

bool same_latents(const Model::Latents& a, const Model::Latents& b)
{
    return a.genotype_log_posteriors == b.genotype_log_posteriors && a.group_concentrations == b.group_concentrations &&
           a.mixture_concentrations == b.mixture_concentrations && a.group_responsibilities == b.group_responsibilities &&
           a.component_responsibilities == b.component_responsibilities;
}

} // namespace

// Outputs as phmm_variational_bayes_mixture_mixture's; with seed_iters also every seed's evidence (its own one-seed evaluate)
// and iteration count: the smallest max_iterations whose run ends in the same latents as the full run (a seed that stops at trip
// i gives the same result for every max_iterations >= i).
extern "C" int ref_vbmm_run(const double* lnl, int H, int R, const int64_t* soff, int S, const int32_t* sizes, int T,
                            const int32_t* gt, int C, const double* lp, const double* gprior, const int32_t* mask, const double* gc0,
                            const double* mc0, const double* seeds, int n_seeds, double eps, int max_it, double* post, double* lpost,
                            double* gconc, double* mconc, double* sigma, double* weighted, double* wsigma, double* max_ev,
                            int32_t* max_seed, double* seed_ev, int32_t* seed_iters)
{
    std::vector<std::vector<std::vector<double>>> cols(S, std::vector<std::vector<double>>(H));
    for (int s = 0; s < S; ++s)
        for (int h = 0; h < H; ++h) cols[s][h].assign(lnl + (std::size_t)h * R + soff[s], lnl + (std::size_t)h * R + soff[s + 1]);
    int K = 0;
    std::vector<int> koff(T + 1, 0);
    for (int t = 0; t < T; ++t) { koff[t] = K; K += sizes[t]; }
    koff[T] = K;
    Model::HaplotypeLikelihoodMatrix m(S, Model::GenotypeCombinationLikelihoodVector(C, Model::GenotypeLikelihoodVector(T)));
    for (int s = 0; s < S; ++s)
        for (int c = 0; c < C; ++c)
            for (int t = 0; t < T; ++t) {
                auto& g = m[s][c][t];
                g.resize(sizes[t]);
                for (int k = 0; k < sizes[t]; ++k) g[k] = cols[s][gt[(std::size_t)c * K + koff[t] + k]];
            }
    const Model::LogProbabilityVector log_priors(lp, lp + C);
    Model::GroupOptionalPriorArray priors(S);
    if (gprior)
        for (int s = 0; s < S; ++s) if (!mask || mask[s]) priors[s] = Model::ProbabilityVector(gprior + (std::size_t)s * T, gprior + (std::size_t)(s + 1) * T);
    const Model::GroupConcentrationVector gcv(gc0, gc0 + T);
    Model::MixtureConcentrationArray mca(S, Model::MixtureConcentrationVector(T));
    for (int s = 0; s < S; ++s)
        for (int t = 0; t < T; ++t) mca[s][t].assign(mc0 + (std::size_t)s * K + koff[t], mc0 + (std::size_t)s * K + koff[t + 1]);
    std::vector<Model::LogProbabilityVector> sv(n_seeds);
    for (int i = 0; i < n_seeds; ++i) sv[i].assign(seeds + (std::size_t)i * C, seeds + (std::size_t)(i + 1) * C);
    Model::Options opt {};
    opt.epsilon = eps;
    opt.max_iterations = static_cast<unsigned>(max_it);
    const auto r = Model {opt}.evaluate(log_priors, m, priors, gcv, mca, sv);
    const auto& L = r.map.latents;
    std::copy(L.genotype_posteriors.begin(), L.genotype_posteriors.end(), post);
    std::copy(L.genotype_log_posteriors.begin(), L.genotype_log_posteriors.end(), lpost);
    std::copy(L.group_concentrations.begin(), L.group_concentrations.end(), gconc);
    for (int s = 0; s < S; ++s) {
        for (int t = 0; t < T; ++t) {
            std::copy(L.mixture_concentrations[s][t].begin(), L.mixture_concentrations[s][t].end(), mconc + (std::size_t)s * K + koff[t]);
            sigma[(std::size_t)s * T + t] = L.group_responsibilities[s][t];
            wsigma[(std::size_t)s * T + t] = r.weighted_group_responsibilities[s][t];
        }
    }
    std::copy(r.weighted_genotype_posteriors.begin(), r.weighted_genotype_posteriors.end(), weighted);
    *max_ev = r.map.approx_log_evidence;
    if (!seed_iters) return 0;      // the Inferences alone (what SingleCellModel computes), e.g. for timing
    int best = 0;
    for (int i = 0; i < n_seeds; ++i) {
        const std::vector<Model::LogProbabilityVector> one {sv[i]};
        const auto full = Model {opt}.evaluate(log_priors, m, priors, gcv, mca, one);
        unsigned lo = 1, hi = opt.max_iterations;
        while (lo < hi) {
            const unsigned mid = lo + (hi - lo) / 2;
            Model::Options pm = opt;
            pm.max_iterations = mid;
            if (same_latents(Model {pm}.evaluate(log_priors, m, priors, gcv, mca, one).map.latents, full.map.latents)) hi = mid;
            else lo = mid + 1;
        }
        seed_iters[i] = static_cast<int32_t>(lo);
        seed_ev[i] = full.map.approx_log_evidence;
        if (seed_ev[i] > seed_ev[best]) best = i;
    }
    *max_seed = best;
    return 0;
}
