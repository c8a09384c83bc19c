// Variational Bayes mixture-of-mixtures inference of SingleCellModel::evaluate_model
// (core/models/genotype/variational_bayes_mixture_mixture_model.cpp, VariationalBayesMixtureMixtureModel::evaluate over every
// seed) on the resident [H][R] likelihood matrix, in double throughout (phmm_variational_bayes_mixture_mixture).
//
// Shapes: S samples (cells), sample s owning the columns [soff[s], soff[s+1]); T groups (clones), group t with K_t components.
// The real components are slots j = koff[t] + k, k < K_t, K = sum_t K_t <= 100 of them; maxK = max_t K_t. Combination c gives
// slot j the haplotype gt[c][j]. The reference's O(S T K N C) products are taken over haplotypes instead:
//   W[j][h]    = sum_{c: gt[c][j] = h} p_c                       (k_vb_index's per-slot index, rebuilt as phmm_vb.cuh rebuilds it)
//   D[s][j][h] = sum_{n in s} tau'[j][n] lnl[h][n]               over slot j's occurring haplotypes only
//   E[j][h]    = sum_s sigma[s][t] D[s][j][h]                    so a combination's term is sum_j E[j][gt[c][j]], O(K)
// where tau'[j] is slot j's responsibility, plus, for a group's first slot, its padded components' (they reuse hap(c, t, 0)).
// An iteration of one seed costs O(R sum_j nk_j + C K): nk_j is the number of haplotypes that occur at slot j.
//
// Reference behaviours this reproduces (each pinned by a test):
//  * tau is not reset for groups t > 0 (:465): ln rho[s][t][k][n] = the previous iteration's tau + ln E[pi_k] + sum_c p_c lnl.
//    At initialisation the previous tau is 0. This is a quirk of the reference, not of the model.
//  * Padded components (t, k >= K_t, only when the groups' ploidies differ) get ln rho = -10000 (Options::null_log_probability);
//    each read is normalised over all maxK components of a group. Sigma's update, the genotype update and the evidence use
//    hap(c, t, 0) for them (:389-393, :526-531). A padded tau is 0 in practice, 1 when every real ln rho lies below -10000.
//  * Sigma's update adds sum_{k < K_t} ln E[pi_k] (:386); its initialisation (:316-364) does not, and takes approximate tau over
//    the real components from the first combination of largest exp(seed).
//  * dirichlet_expectation_log of a single concentration is 0 (:231): T = 1 and K_t = 1 give 0.
//  * Group priors p enter as ln p, or ln DBL_MIN for p <= 0 (:148-151); the evidence adds log_sum_exp_t(ln sigma + ln prior)
//    for the samples that have them, where ln sigma may be -inf.
//  * A seed's evidence is the last ELBO the loop computed. A seed that runs out of iterations ends with sigma one update ahead.
//  * Seeds combine as compute_evidence_weighted_latents (:644-691) does; the weighted posteriors and each sample's weighted sigma
//    get check_normalisation, the MAP seed's posteriors do not.
// Precision: the reference keeps its expanded likelihoods and the component update's sum_c p_c lnl in float, which turns a
// lowest() entry into -inf; this computes in double throughout.
//
// Every reduction runs in a fixed order and no floating-point atomic is used: the same inputs give the same bits. The
// __host__ __device__ functions below are the per-read, per-sample and per-combination arithmetic the kernel executes.
#pragma once

#include "phmm_vb.cuh"

namespace phmm {
namespace vbmm {

using vb::digamma_diffs;
using vb::log_beta;
using vb::xlogx;

constexpr int kMaxGroups = 32;
constexpr int kMaxSlots = 100;                          // sum_t K_t: k_vb_index's K
constexpr double kNullLogProbability = -10000.0;        // VariationalBayesMixtureMixtureModel::Options::null_log_probability
constexpr double kMinLogPrior = -708.3964185322641;     // ln DBL_MIN (to_logs, :148-151)

// to_logs of one group prior.
VB_HD double group_log_prior(double p) { return p > 0.0 ? log(p) : kMinLogPrior; }

// dirichlet_expectation_log (:227-238): psi(a_k) - psi(sum a), and 0 for a single concentration.
VB_HD void dirichlet_expectation_log(const double* a, int K, double* out)
{
    if (K > 1) digamma_diffs(a, K, out);
    else for (int k = 0; k < K; ++k) out[k] = 0.0;
}

// maths::normalise_exp of n values in place: the first maximum, the sum in order.
VB_HD void normalise_exp(double* x, int n)
{
    double mx = x[0];
    for (int i = 1; i < n; ++i) if (x[i] > mx) mx = x[i];
    double sum = 0.0;
    for (int i = 0; i < n; ++i) sum += exp(x[i] - mx);
    const double norm = mx + log(sum);
    for (int i = 0; i < n; ++i) x[i] = exp(x[i] - norm);
}

// One read's component responsibilities of one group (:474-483): x[k * stride], k < Kt, holds ln rho_k on entry and tau_k on
// return; the padded components k in [Kt, maxK) have ln rho = -10000. *pad receives the padded components' tau summed in k order.
// Returns sum_{k < maxK} tau_k ln tau_k.
VB_HD double component_responsibilities(double* x, int Kt, int maxK, long long stride, double* pad)
{
    double mx = x[0];
    for (int k = 1; k < maxK; ++k) {
        const double v = k < Kt ? x[k * stride] : kNullLogProbability;
        if (v > mx) mx = v;
    }
    double sum = 0.0;
    for (int k = 0; k < maxK; ++k) sum += exp((k < Kt ? x[k * stride] : kNullLogProbability) - mx);
    const double norm = mx + log(sum);
    double ent = 0.0, ps = 0.0;
    for (int k = 0; k < maxK; ++k) {
        const double t = exp((k < Kt ? x[k * stride] : kNullLogProbability) - norm);
        if (k < Kt) x[k * stride] = t;
        else ps += t;
        ent += xlogx(t);
    }
    *pad = ps;
    return ent;
}

// One read's part of init_responsibilities' group term (:345-358): the approximate tau over the group's Kt components, from
// ln E[pi_k] + lnl[hmax[k]][n] (hmax: the combination of largest prior's haplotypes), times m[k * stride] = sum_c p_c lnl[hap(c,t,k)][n].
VB_HD double init_group_term(const double* lnEpi, const int* hmax, const double* lnl, long long R, int n, const double* m,
                             long long stride, int Kt)
{
    double mx = lnEpi[0] + lnl[(long long)hmax[0] * R + n];
    for (int k = 1; k < Kt; ++k) {
        const double a = lnEpi[k] + lnl[(long long)hmax[k] * R + n];
        if (a > mx) mx = a;
    }
    double sum = 0.0;
    for (int k = 0; k < Kt; ++k) sum += exp(lnEpi[k] + lnl[(long long)hmax[k] * R + n] - mx);
    const double norm = mx + log(sum);
    double q = 0.0;
    for (int k = 0; k < Kt; ++k) q += exp(lnEpi[k] + lnl[(long long)hmax[k] * R + n] - norm) * m[k * stride];
    return q;
}

// A combination's marginal (marginalise, :501-534, summed over samples and groups): sum_j E[j][gt[j]].
VB_HD double combination_term(const double* E, const int* gt, int K, int H)
{
    double r = 0.0;
    for (int j = 0; j < K; ++j) r += E[(long long)j * H + gt[j]];
    return r;
}

// One sample's terms of calculate_evidence (:615-628): the entropy of sigma; per group sigma_t times the entropy of its
// responsibilities (X[t] = sum tau ln tau) and times (log_beta(posterior) - log_beta(prior)) of its mixture concentrations; and,
// where the sample has group priors (gprior not null), log_sum_exp_t(ln sigma_t + ln prior_t).
VB_HD double sample_evidence(const double* sigma, const double* X, const double* mconc, const double* mc0, const int* gsz, int T,
                             const double* gprior)
{
    double ent = 0.0;
    for (int t = 0; t < T; ++t) ent += xlogx(sigma[t]);
    double r = -ent;
    for (int t = 0, o = 0; t < T; o += gsz[t], ++t) {
        r += sigma[t] * -X[t];
        r += sigma[t] * (log_beta(mconc + o, gsz[t]) - log_beta(mc0 + o, gsz[t]));
    }
    if (gprior) {
        double mx = log(sigma[0]) + group_log_prior(gprior[0]);
        for (int t = 1; t < T; ++t) { const double v = log(sigma[t]) + group_log_prior(gprior[t]); if (v > mx) mx = v; }
        double sum = 0.0;
        for (int t = 0; t < T; ++t) sum += exp(log(sigma[t]) + group_log_prior(gprior[t]) - mx);
        r += mx + log(sum);
    }
    return r;
}

// One sample's ln sigma_t before normalisation in update_responsibilities (:379-396): ln E[psi_t] (+ ln prior_t) +
// sum_{k < K_t} ln E[pi_k] + sum over the group's slots j and their occurring haplotypes of W[j][h] D[j][h] (Ds: the sample's
// D by pair; pofs, ph: the pairs of each slot).
VB_HD double group_update(double lnEpsi, const double* gprior_t, const double* lnEpi, const double* W, const double* Ds,
                          const int* pofs, const int* ph, int o, int Kt, int H)
{
    double r = lnEpsi;
    if (gprior_t) r += group_log_prior(*gprior_t);
    double se = 0.0;
    for (int k = 0; k < Kt; ++k) se += lnEpi[o + k];
    r += se;
    for (int k = 0; k < Kt; ++k) {
        const int j = o + k;
        for (int p = pofs[j]; p < pofs[j + 1]; ++p) r += W[(long long)j * H + ph[p]] * Ds[p];
    }
    return r;
}

} // namespace vbmm
} // namespace phmm

#if defined(__CUDACC__)
namespace phmm {
namespace vbmm {

using vb::kThreads;
using vb::kFinishThreads;
using vb::block_sum;
using vb::block_max;
using vb::block_argmax;
using vb::converged;

constexpr int kChunk = 32;     // reads per partial sum of the per-sample reductions

struct Args {
    const double* lnl; int H, R, S, G, K, T, maxK, n_seeds;   // G: combinations; K: slots, sum_t K_t
    const int* soff; const int* rsamp;                        // [S + 1] read offsets of the samples; [R] each read's sample
    const int *gsz, *koff, *slot_t;                           // [T] K_t; [T + 1] first slot of each group; [K] group of each slot
    const int* gt;                                            // [G][K]
    const double* lp;                                         // [G] combination log priors
    const double* seeds;                                      // [n_seeds][G]
    const double* gprior; const int* has_prior;               // [S][T] group priors (null: none); [S] which samples have them
    const double *gc0, *mc0;                                  // [T] prior group concentrations; [S][K] prior mixture concentrations
    double epsilon; int max_iterations;
    const int *cnt, *start, *kh, *nk, *L, *sid;               // k_vb_index's per-slot index (see phmm_vb.cuh)
    const int* bad;
    const int *pofs, *pj, *ph;                                // occurring (slot, haplotype) pairs: slot j's are [pofs[j], pofs[j+1])
    int P, Pmax;                                              // their count (pofs[K], set by k_vbmm_seeds) and its bound K min(H, G), which lays out the workspace
    const int *chunk_s, *chunk_n0, *schunk; int NC;           // read chunks (at most kChunk reads of one sample); sample s's chunks [schunk[s], schunk[s+1])
    double* ws; long long ws_stride;                          // per-block workspace
    double* lpost; double* ev; int* iters; int* map;          // [n_seeds][G], [n_seeds] x 3
    double *gconc, *mconc, *sigma;                            // [n_seeds][T], [n_seeds][S][K], [n_seeds][S][T]
};

struct Workspace {
    double *W, *E, *post, *tau, *pad, *en, *q, *part, *D, *A, *X, *mconc, *lnEpi, *sigma;
    __device__ Workspace(const Args& a, double* p)
    {
        const long long KH = (long long)a.K * a.H, KR = (long long)a.K * a.R, TR = (long long)a.T * a.R;
        W = p; E = W + KH; post = E + KH; tau = post + a.G; pad = tau + KR; en = pad + TR; q = en + TR; part = q + TR;
        D = part + (long long)a.NC * (a.Pmax + a.K + a.T); A = D + (long long)a.S * a.Pmax; X = A + (long long)a.S * a.K;
        mconc = X + (long long)a.S * a.T; lnEpi = mconc + (long long)a.S * a.K; sigma = lnEpi + (long long)a.S * a.K;
    }
    static long long doubles(int H, int R, int S, int G, int K, int T, int P, int NC)
    {
        return 2LL * K * H + G + (long long)K * R + 3LL * T * R + (long long)NC * (P + K + T) + (long long)S * P + 3LL * S * K + 2LL * S * T;
    }
};

struct Shared {
    vb::Shared vb;
    double gconc[kMaxGroups], lnEpsi[kMaxGroups];
};

// The occurring (slot, haplotype) pairs from k_vb_index's nk and kh, slot by slot; one block.
__global__ void k_vbmm_pairs(const int* __restrict__ bad, const int* __restrict__ nk, const int* __restrict__ kh, const int K, const int H,
                             int* __restrict__ pofs, int* __restrict__ pj, int* __restrict__ ph)
{
    __shared__ int o[kMaxSlots + 1];
    if (*bad) return;
    if (threadIdx.x == 0) { int run = 0; for (int j = 0; j < K; ++j) { o[j] = run; run += nk[j]; } o[K] = run; }
    __syncthreads();
    for (int j = threadIdx.x; j <= K; j += blockDim.x) pofs[j] = o[j];
    for (int j = 0; j < K; ++j)
        for (int i = threadIdx.x; i < nk[j]; i += blockDim.x) { pj[o[j] + i] = j; ph[o[j] + i] = kh[(long long)j * H + i]; }
}

// The concentrations' digamma differences: ln E[psi] into shared memory, ln E[pi] per sample.
__device__ void expectations(const Args& a, const Workspace& w, Shared& sh)
{
    if (threadIdx.x == 0) dirichlet_expectation_log(sh.gconc, a.T, sh.lnEpsi);
    for (int s = threadIdx.x; s < a.S; s += blockDim.x)
        for (int t = 0; t < a.T; ++t) {
            const long long o = (long long)s * a.K + a.koff[t];
            dirichlet_expectation_log(w.mconc + o, a.gsz[t], w.lnEpi + o);
        }
}

// The component update (update_responsibilities, :446-486) for every read, one thread per read across the samples. With
// `init` (>= 0: the combination of largest prior) it is init_responsibilities: the previous tau counts 0, and each read's part of
// sigma's initial group term goes to q[t][n].
__device__ void component_update(const Args& a, const Workspace& w, int init)
{
    const int H = a.H, R = a.R, K = a.K;
    for (int n = threadIdx.x; n < R; n += blockDim.x) {
        const int s = a.rsamp[n];
        const double* lnEpi = w.lnEpi + (long long)s * K;
        for (int t = 0; t < a.T; ++t) {
            const int o = a.koff[t], Kt = a.gsz[t];
            for (int k = 0; k < Kt; ++k) {
                const int j = o + k;
                double m = 0.0;
                const int* hs = a.kh + (long long)j * H;
                for (int i = 0, e = a.nk[j]; i < e; ++i) {
                    const int h = hs[i];
                    m += w.W[(long long)j * H + h] * a.lnl[(long long)h * R + n];
                }
                double* x = w.tau + (long long)j * R + n;
                if (init >= 0) *x = m;
                else *x = (t > 0 ? *x : 0.0) + (lnEpi[j] + m);
            }
            if (init >= 0) {
                w.q[(long long)t * R + n] = init_group_term(lnEpi + o, a.gt + (long long)init * K + o, a.lnl, R, n, w.tau + (long long)o * R + n, R, Kt);
                for (int k = 0; k < Kt; ++k) { double* x = w.tau + (long long)(o + k) * R + n; *x = 0.0 + (lnEpi[o + k] + *x); }
            }
            w.en[(long long)t * R + n] = component_responsibilities(w.tau + (long long)o * R + n, Kt, a.maxK, R, w.pad + (long long)t * R + n);
        }
    }
}

// Per sample: D[s][p] = sum_n tau'[j][n] lnl[h][n] for every occurring pair p = (j, h), A[s][j] = sum_n tau[j][n] and
// X[s][t] = sum_n (the read's sum_k tau ln tau). Each thread sums one quantity over one chunk of at most kChunk reads of one
// sample, in read order; then the chunks of each sample are added in order.
__device__ void reduce_samples(const Args& a, const Workspace& w)
{
    const int R = a.R, P = a.P, K = a.K, T = a.T, Q = P + K + T;
    for (long long item = threadIdx.x; item < (long long)a.NC * Q; item += blockDim.x) {
        const int c = (int)(item / Q), i = (int)(item % Q);
        const int n0 = a.chunk_n0[c], s = a.chunk_s[c], n1 = min(n0 + kChunk, a.soff[s + 1]);
        double v = 0.0;
        if (i < P) {
            const int j = a.pj[i], t = a.slot_t[j];
            const double* lh = a.lnl + (long long)a.ph[i] * R;
            const double* tj = w.tau + (long long)j * R;
            if (j == a.koff[t]) {
                const double* pt = w.pad + (long long)t * R;
                for (int n = n0; n < n1; ++n) v += (tj[n] + pt[n]) * lh[n];
            } else {
                for (int n = n0; n < n1; ++n) v += tj[n] * lh[n];
            }
        } else {
            const double* x = i < P + K ? w.tau + (long long)(i - P) * R : w.en + (long long)(i - P - K) * R;
            for (int n = n0; n < n1; ++n) v += x[n];
        }
        w.part[item] = v;
    }
    __syncthreads();
    for (long long item = threadIdx.x; item < (long long)a.S * Q; item += blockDim.x) {
        const int s = (int)(item / Q), i = (int)(item % Q);
        double v = 0.0;
        for (int c = a.schunk[s]; c < a.schunk[s + 1]; ++c) v += w.part[(long long)c * Q + i];
        if (i < P) w.D[(long long)s * P + i] = v;
        else if (i < P + K) w.A[(long long)s * K + (i - P)] = v;
        else w.X[(long long)s * T + (i - P - K)] = v;
    }
    __syncthreads();
}

// E[j][h] = sum_s sigma[s][t_j] D[s][p], in sample order, for every occurring pair p = (j, h).
__device__ void fold_sigma(const Args& a, const Workspace& w)
{
    for (int p = threadIdx.x; p < a.P; p += blockDim.x) {
        const int j = a.pj[p], t = a.slot_t[j];
        double v = 0.0;
        for (int s = 0; s < a.S; ++s) v += w.sigma[(long long)s * a.T + t] * w.D[(long long)s * a.P + p];
        w.E[(long long)j * a.H + a.ph[p]] = v;
    }
    __syncthreads();
}

// calculate_evidence (:587-631) of the current state.
__device__ double evidence(const Args& a, const Workspace& w, const double* lpost, Shared& sh)
{
    double acc = 0.0;
    for (int c = threadIdx.x; c < a.G; c += blockDim.x)
        acc += w.post[c] * ((a.lp[c] - lpost[c]) + combination_term(w.E, a.gt + (long long)c * a.K, a.K, a.H));
    acc = block_sum(acc, sh.vb.red);
    double sv = 0.0;
    for (int s = threadIdx.x; s < a.S; s += blockDim.x)
        sv += sample_evidence(w.sigma + (long long)s * a.T, w.X + (long long)s * a.T, w.mconc + (long long)s * a.K,
                              a.mc0 + (long long)s * a.K, a.gsz, a.T, a.gprior && a.has_prior[s] ? a.gprior + (long long)s * a.T : nullptr);
    sv = block_sum(sv, sh.vb.red);
    return acc + sv + (log_beta(sh.gconc, a.T) - log_beta(a.gc0, a.T));
}

// Every seed's run of the loop (evaluate, :254-298), one block per seed at a time, its last evidence and the first index of its
// maximum posterior.
__global__ void __launch_bounds__(kThreads)
k_vbmm_seeds(Args a)
{
    __shared__ Shared sh;
    if (*a.bad) return;
    a.P = a.pofs[a.K];
    const Workspace w(a, a.ws + blockIdx.x * a.ws_stride);
    const int G = a.G, T = a.T, SK = a.S * a.K, ST = a.S * a.T;
    for (int seed = blockIdx.x; seed < a.n_seeds; seed += gridDim.x) {
        double* lpost = a.lpost + (long long)seed * G;
        const double* sd = a.seeds + (long long)seed * G;
        double best = 0.0; int bi = -1;
        for (int c = threadIdx.x; c < G; c += blockDim.x) {
            lpost[c] = sd[c];
            w.post[c] = exp(sd[c]);
            if (bi < 0 || w.post[c] > best) { best = w.post[c]; bi = c; }
        }
        for (int i = threadIdx.x; i < SK; i += blockDim.x) w.mconc[i] = a.mc0[i];
        for (int t = threadIdx.x; t < T; t += blockDim.x) sh.gconc[t] = a.gc0[t];
        const int cmax = block_argmax(best, bi, sh.vb.red, sh.vb.redi);   // also orders the writes above
        expectations(a, w, sh);
        vb::rebuild_w(a, w, sh.vb);
        __syncthreads();
        component_update(a, w, cmax);
        __syncthreads();
        reduce_samples(a, w);
        for (int s = threadIdx.x; s < a.S; s += blockDim.x) {     // init_responsibilities (:316-364)
            double* sg = w.sigma + (long long)s * T;
            for (int t = 0; t < T; ++t) {
                double v = sh.lnEpsi[t];
                if (a.gprior && a.has_prior[s]) v += group_log_prior(a.gprior[(long long)s * T + t]);
                double qs = 0.0;
                for (int n = a.soff[s]; n < a.soff[s + 1]; ++n) qs += w.q[(long long)t * a.R + n];
                sg[t] = v + qs;
            }
            normalise_exp(sg, T);
        }
        __syncthreads();
        fold_sigma(a, w);
        double prev = -1.7976931348623157e308, curr = prev;   // std::numeric_limits<double>::lowest()
        int it = 0;
        while (it < a.max_iterations) {
            ++it;
            double mx = -INFINITY;
            for (int c = threadIdx.x; c < G; c += blockDim.x) {
                const double v = a.lp[c] + combination_term(w.E, a.gt + (long long)c * a.K, a.K, a.H);
                lpost[c] = v;
                if (v > mx) mx = v;
            }
            mx = block_max(mx, sh.vb.red);
            double sum = 0.0;
            for (int c = threadIdx.x; c < G; c += blockDim.x) sum += exp(lpost[c] - mx);
            const double norm = mx + log(block_sum(sum, sh.vb.red));
            for (int c = threadIdx.x; c < G; c += blockDim.x) { const double v = lpost[c] - norm; lpost[c] = v; w.post[c] = exp(v); }
            for (int t = threadIdx.x; t < T; t += blockDim.x) {
                double v = a.gc0[t];
                for (int s = 0; s < a.S; ++s) v += w.sigma[(long long)s * T + t];
                sh.gconc[t] = v;
            }
            for (int i = threadIdx.x; i < SK; i += blockDim.x) w.mconc[i] = a.mc0[i] + w.A[i];
            __syncthreads();
            curr = evidence(a, w, lpost, sh);
            if (converged(curr, prev, a.epsilon)) break;
            prev = curr;
            expectations(a, w, sh);
            vb::rebuild_w(a, w, sh.vb);
            __syncthreads();
            for (int s = threadIdx.x; s < a.S; s += blockDim.x) {     // sigma from the previous tau (:366-399)
                double* sg = w.sigma + (long long)s * T;
                for (int t = 0; t < T; ++t)
                    sg[t] = group_update(sh.lnEpsi[t], a.gprior && a.has_prior[s] ? a.gprior + (long long)s * T + t : nullptr,
                                         w.lnEpi + (long long)s * a.K, w.W, w.D + (long long)s * a.P, a.pofs, a.ph, a.koff[t], a.gsz[t], a.H);
                normalise_exp(sg, T);
            }
            __syncthreads();
            component_update(a, w, -1);
            __syncthreads();
            reduce_samples(a, w);
            fold_sigma(a, w);
        }
        best = 0.0; bi = -1;
        for (int c = threadIdx.x; c < G; c += blockDim.x) if (bi < 0 || w.post[c] > best) { best = w.post[c]; bi = c; }
        bi = block_argmax(best, bi, sh.vb.red, sh.vb.redi);
        if (threadIdx.x == 0) { a.ev[seed] = curr; a.iters[seed] = it; a.map[seed] = bi; }
        for (int t = threadIdx.x; t < T; t += blockDim.x) a.gconc[(long long)seed * T + t] = sh.gconc[t];
        for (int i = threadIdx.x; i < SK; i += blockDim.x) a.mconc[(long long)seed * SK + i] = w.mconc[i];
        for (int i = threadIdx.x; i < ST; i += blockDim.x) a.sigma[(long long)seed * ST + i] = w.sigma[i];
        __syncthreads();
    }
}

// compute_evidence_weighted_latents' remainder (:670-690) and the MAP seed's latents: check_normalisation of the weighted
// posteriors; each sample's weighted sigma, summed over the modes in order, then check_normalisation; one block.
__global__ void __launch_bounds__(kFinishThreads)
k_vbmm_finish(const int* __restrict__ bad, const int G, const int S, const int T, const int K, double* __restrict__ weighted,
              const int* __restrict__ modes, const double* __restrict__ weights, const int* __restrict__ n_modes,
              const int* __restrict__ max_seed, const double* __restrict__ ev, const double* __restrict__ seed_gconc,
              const double* __restrict__ seed_mconc, const double* __restrict__ seed_sigma, double* __restrict__ gconc,
              double* __restrict__ mconc, double* __restrict__ sigma, double* __restrict__ wsigma, double* __restrict__ max_ev,
              int* __restrict__ max_seed_out)
{
    if (*bad) return;   // k_vb_index found an index outside [0, H): nothing below was computed
    __shared__ double red[kFinishThreads];
    const int tid = threadIdx.x, nt = blockDim.x;
    double m = 0.0;
    for (int c = tid; c < G; c += nt) m += weighted[c];
    m = block_sum(m, red);
    if (m > 1.0) for (int c = tid; c < G; c += nt) weighted[c] /= m;
    const int nm = *n_modes, ms = *max_seed;
    const long long ST = (long long)S * T, SK = (long long)S * K;
    for (int s = tid; s < S; s += nt) {
        double* o = wsigma + (long long)s * T;
        double mass = 0.0;
        for (int t = 0; t < T; ++t) {
            double v = 0.0;
            for (int i = 0; i < nm; ++i) v = v + weights[i] * seed_sigma[modes[i] * ST + (long long)s * T + t];
            o[t] = v;
            mass += v;
        }
        if (mass > 1.0) for (int t = 0; t < T; ++t) o[t] /= mass;
    }
    for (long long i = tid; i < ST; i += nt) sigma[i] = seed_sigma[ms * ST + i];
    for (long long i = tid; i < SK; i += nt) mconc[i] = seed_mconc[ms * SK + i];
    for (int t = tid; t < T; t += nt) gconc[t] = seed_gconc[(long long)ms * T + t];
    if (tid == 0) { *max_ev = ev[ms]; *max_seed_out = ms; }
}

} // namespace vbmm
} // namespace phmm
#endif
