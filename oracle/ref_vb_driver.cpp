// TEST INFRASTRUCTURE ONLY. C entry points over the UNMODIFIED reference variational Bayes header
// (core/models/genotype/variational_bayes_mixture_model.hpp), built by vb.mk into _ref/libref_vb.so. Instantiated for the K the
// tests use: 1, 2, 3, 4, 8, 100.
#include <cstdint>
#include <cstring>
#include <vector>

#include "core/models/genotype/variational_bayes_mixture_model.hpp"

using namespace octopus;
using namespace octopus::model;

namespace {

struct Problem {
    // per sample, per haplotype: that sample's columns of the matrix (the reference's per-sample likelihood vectors)
    std::vector<std::vector<std::vector<double>>> cols;
};

template <std::size_t K>
struct Inputs {
    VBAlphaVector<K> prior;
    VBReadLikelihoodMatrix<K> lnl;
};

template <std::size_t K>
Inputs<K> make(const Problem& p, const int* gt, int G, const double* prior, int S)
{
    Inputs<K> in;
    in.prior.resize(S);
    for (int s = 0; s < S; ++s) for (std::size_t k = 0; k < K; ++k) in.prior[s][k] = static_cast<float>(prior[s * K + k]);
    in.lnl.resize(S);
    for (int s = 0; s < S; ++s) {
        in.lnl[s].resize(G);
        for (int g = 0; g < G; ++g) for (std::size_t k = 0; k < K; ++k) in.lnl[s][g][k] = p.cols[s][gt[(std::size_t)g * K + k]];
    }
    return in;
}

template <std::size_t K>
bool same_latents(const VBLatents<K>& a, const VBLatents<K>& b)
{
    if (a.genotype_log_posteriors != b.genotype_log_posteriors || a.alphas != b.alphas) return false;
    for (std::size_t s = 0; s < a.responsibilities.size(); ++s)
        for (std::size_t k = 0; k < K; ++k) if (a.responsibilities[s][k] != b.responsibilities[s][k]) return false;
    return true;
}

template <std::size_t K>
int run(const Problem& p, const int* gt, int G, const double* prior, int S, const double* lp, const double* seeds, int n_seeds,
        double eps, int max_it, double* post, double* lpost, double* alphas, double* weighted, double* max_ev, int32_t* max_seed,
        double* seed_ev, int32_t* seed_iters)
{
    const auto in = make<K>(p, gt, G, prior, S);
    const LogProbabilityVector log_priors(lp, lp + G);
    std::vector<LogProbabilityVector> sv(n_seeds);
    for (int i = 0; i < n_seeds; ++i) sv[i].assign(seeds + (std::size_t)i * G, seeds + (std::size_t)(i + 1) * G);
    VariationalBayesParameters params {};
    params.epsilon = eps;
    params.max_iterations = static_cast<unsigned>(max_it);
    const auto packet = run_variational_bayes(in.prior, log_priors, in.lnl, params, sv);
    std::copy(packet.map_latents.genotype_posteriors.begin(), packet.map_latents.genotype_posteriors.end(), post);
    std::copy(packet.map_latents.genotype_log_posteriors.begin(), packet.map_latents.genotype_log_posteriors.end(), lpost);
    for (int s = 0; s < S; ++s) for (std::size_t k = 0; k < K; ++k) alphas[s * K + k] = packet.map_latents.alphas[s][k];
    std::copy(packet.evidence_weighted_genotype_posteriors.begin(), packet.evidence_weighted_genotype_posteriors.end(), weighted);
    *max_ev = packet.max_log_evidence;
    if (!seed_iters) return 0;      // the packet alone (what SubcloneModel::evaluate computes), e.g. for timing
    // per seed: the reference's own single-seed run, its final evidence, and its iteration count — the smallest max_iterations
    // whose run ends in the same latents (a seed that stops at trip i gives the same result for every max_iterations >= i)
    const auto inverted = model::detail::invert(in.lnl);
    std::vector<VBLatents<K>> latents;
    for (int i = 0; i < n_seeds; ++i) {
        auto full = model::detail::run_variational_bayes(in.prior, log_priors, in.lnl, inverted, sv[i], params);
        unsigned lo = 1, hi = params.max_iterations;
        while (lo < hi) {
            const unsigned mid = lo + (hi - lo) / 2;
            VariationalBayesParameters pm = params;
            pm.max_iterations = mid;
            if (same_latents(model::detail::run_variational_bayes(in.prior, log_priors, in.lnl, inverted, sv[i], pm), full)) hi = mid;
            else lo = mid + 1;
        }
        seed_iters[i] = static_cast<int32_t>(lo);
        latents.push_back(std::move(full));
    }
    const auto ev = model::detail::calculate_log_evidences(latents, in.prior, log_priors, in.lnl);
    std::copy(ev.begin(), ev.end(), seed_ev);
    *max_seed = static_cast<int32_t>(model::detail::max_element_index(ev));
    return 0;
}

} // namespace

extern "C" int ref_vb_run(int K, const double* lnl, int H, int R, const int64_t* soff, int S, const int32_t* gt, int G,
                          const double* prior, const double* lp, const double* seeds, int n_seeds, double eps, int max_it,
                          double* post, double* lpost, double* alphas, double* weighted, double* max_ev, int32_t* max_seed,
                          double* seed_ev, int32_t* seed_iters)
{
    Problem p;
    p.cols.resize(S);
    for (int s = 0; s < S; ++s) {
        p.cols[s].resize(H);
        for (int h = 0; h < H; ++h) p.cols[s][h].assign(lnl + (std::size_t)h * R + soff[s], lnl + (std::size_t)h * R + soff[s + 1]);
    }
#define VB_CASE(k) case k: return run<k>(p, gt, G, prior, S, lp, seeds, n_seeds, eps, max_it, post, lpost, alphas, weighted, max_ev, max_seed, seed_ev, seed_iters);
    switch (K) {
        VB_CASE(1) VB_CASE(2) VB_CASE(3) VB_CASE(4) VB_CASE(8) VB_CASE(100)
        default: return -1;
    }
#undef VB_CASE
}
