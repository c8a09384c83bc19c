// TEST HELPER (not part of the product library): the mixture-of-mixtures variational Bayes loop of
// phmm_variational_bayes_mixture_mixture on the CPU, one seed, built from the same __host__ __device__ functions the kernel executes
// (octopus_b200/csrc/phmm_vb_mm.cuh: component_responsibilities, init_group_term, group_update, combination_term,
// sample_evidence, normalise_exp, dirichlet_expectation_log), in the device's haplotype-grouped form with sequential sums, so that
// `pytest -m "not gpu"` can hold that arithmetic to tests/vbmm_exact.py.
#include <vector>
#include "../../octopus_b200/csrc/phmm_vb_mm.cuh"

using namespace phmm::vbmm;

extern "C" {

// One seed: writes lpost[C], gconc[T], mconc[S*K], sigma[S*T] and returns its last evidence; *iterations the loop trips.
// gprior may be null; has_prior[s] selects the samples that have group priors.
double emul_vbmm_seed(const double* lnl, int H, int R, const int* soff, int S, const int* gsz, int T, const int* gt, int C,
                      const double* lp, const double* gprior, const int* has_prior, const double* gc0, const double* mc0,
                      const double* seed, double epsilon, int max_iterations, double* lpost, double* gconc, double* mconc,
                      double* sigma, int* iterations)
{
    std::vector<int> koff(T + 1, 0);
    int maxK = 0;
    for (int t = 0; t < T; ++t) { koff[t + 1] = koff[t] + gsz[t]; if (gsz[t] > maxK) maxK = gsz[t]; }
    const int K = koff[T];
    std::vector<int> slot_t(K), pofs(K + 1, 0), ph;
    for (int t = 0; t < T; ++t) for (int k = 0; k < gsz[t]; ++k) slot_t[koff[t] + k] = t;
    for (int j = 0; j < K; ++j) {           // the occurring haplotypes of each slot, in haplotype order (k_vb_index's kh)
        std::vector<char> used(H, 0);
        for (int c = 0; c < C; ++c) used[gt[(long long)c * K + j]] = 1;
        for (int h = 0; h < H; ++h) if (used[h]) ph.push_back(h);
        pofs[j + 1] = (int)ph.size();
    }
    const int P = pofs[K];
    std::vector<double> post(C), W((size_t)K * H), E((size_t)K * H), tau((size_t)K * R), pad((size_t)T * R), en((size_t)T * R),
        q((size_t)T * R), D((size_t)S * P), A((size_t)S * K), X((size_t)S * T), lnEpi((size_t)S * K), lnEpsi(T);
    auto gp = [&](int s) { return gprior && has_prior[s] ? gprior + (long long)s * T : nullptr; };
    int cmax = 0;
    for (int c = 0; c < C; ++c) { lpost[c] = seed[c]; post[c] = exp(seed[c]); if (post[c] > post[cmax]) cmax = c; }
    for (int t = 0; t < T; ++t) gconc[t] = gc0[t];
    for (int i = 0; i < S * K; ++i) mconc[i] = mc0[i];
    auto expectations = [&]() {
        dirichlet_expectation_log(gconc, T, lnEpsi.data());
        for (int s = 0; s < S; ++s) for (int t = 0; t < T; ++t) dirichlet_expectation_log(mconc + s * K + koff[t], gsz[t], lnEpi.data() + s * K + koff[t]);
    };
    auto rebuild_w = [&]() {
        std::fill(W.begin(), W.end(), 0.0);
        for (int j = 0; j < K; ++j) for (int c = 0; c < C; ++c) W[(size_t)j * H + gt[(long long)c * K + j]] += post[c];
    };
    auto component_update = [&](bool init) {    // then D, A, X per sample, sums in read order
        for (int s = 0; s < S; ++s)
            for (int n = soff[s]; n < soff[s + 1]; ++n)
                for (int t = 0; t < T; ++t) {
                    const int o = koff[t];
                    for (int k = 0; k < gsz[t]; ++k) {
                        const int j = o + k;
                        double m = 0.0;
                        for (int p = pofs[j]; p < pofs[j + 1]; ++p) m += W[(size_t)j * H + ph[p]] * lnl[(size_t)ph[p] * R + n];
                        double& x = tau[(size_t)j * R + n];
                        x = init ? m : (t > 0 ? x : 0.0) + (lnEpi[s * K + j] + m);
                    }
                    if (init) {
                        q[(size_t)t * R + n] = init_group_term(lnEpi.data() + s * K + o, gt + (long long)cmax * K + o, lnl, R, n,
                                                               tau.data() + (size_t)o * R + n, R, gsz[t]);
                        for (int k = 0; k < gsz[t]; ++k) { double& x = tau[(size_t)(o + k) * R + n]; x = 0.0 + (lnEpi[s * K + o + k] + x); }
                    }
                    en[(size_t)t * R + n] = component_responsibilities(tau.data() + (size_t)o * R + n, gsz[t], maxK, R, pad.data() + (size_t)t * R + n);
                }
        for (int s = 0; s < S; ++s) {
            for (int j = 0; j < K; ++j) {
                const int t = slot_t[j];
                double a = 0.0;
                for (int n = soff[s]; n < soff[s + 1]; ++n) a += tau[(size_t)j * R + n];
                A[s * K + j] = a;
                for (int p = pofs[j]; p < pofs[j + 1]; ++p) {
                    double v = 0.0;
                    for (int n = soff[s]; n < soff[s + 1]; ++n)
                        v += (tau[(size_t)j * R + n] + (j == koff[t] ? pad[(size_t)t * R + n] : 0.0)) * lnl[(size_t)ph[p] * R + n];
                    D[(size_t)s * P + p] = v;
                }
            }
            for (int t = 0; t < T; ++t) {
                double x = 0.0;
                for (int n = soff[s]; n < soff[s + 1]; ++n) x += en[(size_t)t * R + n];
                X[s * T + t] = x;
            }
        }
    };
    auto fold_sigma = [&]() {
        for (int j = 0; j < K; ++j)
            for (int p = pofs[j]; p < pofs[j + 1]; ++p) {
                double v = 0.0;
                for (int s = 0; s < S; ++s) v += sigma[s * T + slot_t[j]] * D[(size_t)s * P + p];
                E[(size_t)j * H + ph[p]] = v;
            }
    };
    auto evidence = [&]() {
        double acc = 0.0;
        for (int c = 0; c < C; ++c) acc += post[c] * ((lp[c] - lpost[c]) + combination_term(E.data(), gt + (long long)c * K, K, H));
        for (int s = 0; s < S; ++s) acc += sample_evidence(sigma + s * T, X.data() + s * T, mconc + s * K, mc0 + s * K, gsz, T, gp(s));
        return acc + (phmm::vb::log_beta(gconc, T) - phmm::vb::log_beta(gc0, T));
    };
    expectations();
    rebuild_w();
    component_update(true);
    for (int s = 0; s < S; ++s) {
        for (int t = 0; t < T; ++t) {
            double v = lnEpsi[t];
            if (gp(s)) v += group_log_prior(gp(s)[t]);
            double qs = 0.0;
            for (int n = soff[s]; n < soff[s + 1]; ++n) qs += q[(size_t)t * R + n];
            sigma[s * T + t] = v + qs;
        }
        normalise_exp(sigma + s * T, T);
    }
    fold_sigma();
    double prev = -1.7976931348623157e308, curr = prev;
    int it = 0;
    while (it < max_iterations) {
        ++it;
        for (int c = 0; c < C; ++c) lpost[c] = lp[c] + combination_term(E.data(), gt + (long long)c * K, K, H);
        double mx = lpost[0];
        for (int c = 1; c < C; ++c) if (lpost[c] > mx) mx = lpost[c];
        double sum = 0.0;
        for (int c = 0; c < C; ++c) sum += exp(lpost[c] - mx);
        const double norm = mx + log(sum);
        for (int c = 0; c < C; ++c) { lpost[c] -= norm; post[c] = exp(lpost[c]); }
        for (int t = 0; t < T; ++t) { double v = gc0[t]; for (int s = 0; s < S; ++s) v += sigma[s * T + t]; gconc[t] = v; }
        for (int i = 0; i < S * K; ++i) mconc[i] = mc0[i] + A[i];
        curr = evidence();
        if (phmm::vb::converged(curr, prev, epsilon)) break;
        prev = curr;
        expectations();
        rebuild_w();
        for (int s = 0; s < S; ++s) {
            for (int t = 0; t < T; ++t)
                sigma[s * T + t] = group_update(lnEpsi[t], gp(s) ? gp(s) + t : nullptr, lnEpi.data() + s * K, W.data(),
                                                D.data() + (size_t)s * P, pofs.data(), ph.data(), koff[t], gsz[t], H);
            normalise_exp(sigma + s * T, T);
        }
        component_update(false);
        fold_sigma();
    }
    *iterations = it;
    return curr;
}

}
