// TEST HELPER (not part of the product library): the variational Bayes loop of phmm_variational_bayes on the CPU, built from the
// same __host__ __device__ digamma, responsibility and ELBO functions the kernels execute (octopus_b200/csrc/phmm_vb.cuh), in the
// device's haplotype-grouped form with sequential sums, so that `pytest -m "not gpu"` can hold that arithmetic to tests/vb_exact.py.
#include <vector>
#include "../../octopus_b200/csrc/phmm_vb.cuh"

using namespace phmm::vb;

extern "C" {

// One seed: writes lpost[G], alpha[S*K] and returns its final evidence; *iterations the loop trips.
double emul_vb_seed(const double* lnl, int H, int R, const int* soff, int S, const int* gt, int G, int K, const double* prior,
                    const double* lp, const double* seed, double epsilon, int max_iterations, double* lpost, double* alpha, int* iterations)
{
    const int KH = K * H;
    std::vector<double> W(KH), M((size_t)S * KH), tau((size_t)K * R), post(G), al((size_t)S * K), A((size_t)S * K), X(S);
    for (int g = 0; g < G; ++g) { lpost[g] = seed[g]; post[g] = exp(seed[g]); }
    for (int i = 0; i < S * K; ++i) alpha[i] = prior[i];
    auto sweep = [&](const double* alpha_src) {
        std::fill(W.begin(), W.end(), 0.0);
        for (int k = 0; k < K; ++k) for (int g = 0; g < G; ++g) W[k * H + gt[g * K + k]] += post[g];
        std::vector<char> used(KH, 0);
        for (int k = 0; k < K; ++k) for (int g = 0; g < G; ++g) used[k * H + gt[g * K + k]] = 1;
        for (int s = 0; s < S; ++s) {
            digamma_diffs(alpha_src + s * K, K, al.data() + s * K);
            X[s] = 0.0;
            for (int n = soff[s]; n < soff[s + 1]; ++n) {
                for (int k = 0; k < K; ++k) {
                    double m = 0.0;
                    for (int h = 0; h < H; ++h) if (used[k * H + h]) m += W[k * H + h] * lnl[(size_t)h * R + n];
                    tau[(size_t)k * R + n] = al[s * K + k] + m;
                }
                X[s] += responsibilities(tau.data() + n, K, R);
            }
            for (int k = 0; k < K; ++k) {
                double a = 0.0;
                for (int n = soff[s]; n < soff[s + 1]; ++n) a += tau[(size_t)k * R + n];
                A[s * K + k] = a;
                for (int h = 0; h < H; ++h) {
                    double v = 0.0;
                    for (int n = soff[s]; n < soff[s + 1]; ++n) v += tau[(size_t)k * R + n] * lnl[(size_t)h * R + n];
                    M[(size_t)s * KH + k * H + h] = v;
                }
            }
        }
    };
    auto elbo = [&](bool skip) {
        double acc = 0.0;
        for (int g = 0; g < G; ++g)
            if (!skip || post[g] >= kPosteriorSkip) acc += elbo_genotype_term(post[g], lp[g], lpost[g], M.data(), S, gt + g * K, K, H);
        return elbo_add_samples(acc, prior, alpha, X.data(), S, K);
    };
    sweep(prior);
    double prev = -1.7976931348623157e308;
    int it = 0;
    while (it < max_iterations) {
        ++it;
        double mx = -INFINITY;
        for (int g = 0; g < G; ++g) { lpost[g] = genotype_update(lp[g], M.data(), S, gt + g * K, K, H); if (lpost[g] > mx) mx = lpost[g]; }
        double sum = 0.0;
        for (int g = 0; g < G; ++g) sum += exp(lpost[g] - mx);
        const double norm = mx + log(sum);
        for (int g = 0; g < G; ++g) { lpost[g] -= norm; post[g] = exp(lpost[g]); }
        for (int i = 0; i < S * K; ++i) alpha[i] = prior[i] + A[i];
        const double curr = elbo(true);
        if (converged(curr, prev, epsilon)) break;
        prev = curr;
        sweep(alpha);
    }
    *iterations = it;
    return elbo(false);
}

double emul_vb_digamma(double x) { return digamma(x); }

}
