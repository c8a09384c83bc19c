// Variational Bayes mixture inference of SubcloneModel / SomaticSubcloneModel::evaluate
// (core/models/genotype/variational_bayes_mixture_model.hpp:653-669, run_variational_bayes over every seed) on the resident
// [H][R] likelihood matrix, in double throughout (phmm_variational_bayes).
//
// The reference's two G*K*N inner products are taken over haplotypes instead of genotypes:
//   responsibilities  sum_g p_g lnl[gt[g][k]][n]        = sum_h W[k][h] lnl[h][n],   W[k][h] = sum_{g: gt[g][k] = h} p_g
//   genotype update   sum_{n in s} tau[s][k][n] lnl[gt[g][k]][n] = M[s][k][gt[g][k]], M[s][k][h] = sum_{n in s} tau[k][n] lnl[h][n]
// so an iteration of one seed costs O(K*H*N + G*K). Only the haplotypes that occur at slot k enter slot k's sums, so a zero
// weight never multiplies a lowest() entry. W is rebuilt in a fixed order (the per-slot index of genotypes by haplotype that
// k_vb_index builds once per call), every reduction runs in a fixed tree and no floating-point atomic is used: the same inputs
// give the same bits.
//
// The __host__ __device__ functions below are the per-read and per-genotype arithmetic the kernels execute; the CPU emulation
// (tests/cpu_emul/vb_emul.cu) runs the same functions.
#pragma once

#include <cstdint>
#include <cmath>
#include <cuda_runtime.h>

namespace phmm {
namespace vb {

#if defined(__CUDACC__)
#define VB_HD __host__ __device__ __forceinline__
#else
#define VB_HD inline
#endif

constexpr int kMaxK = 100;                  // the reference's max_ploidy (subclone_model.hpp:32)
constexpr double kPosteriorSkip = 1e-10;    // the ELBO's max_posterior_skip inside the loop (:479)

// digamma in double: the recurrence psi(x) = psi(x + 1) - 1/x up to x >= 10, then the asymptotic series
// ln x - 1/(2x) - sum_k B_2k / (2k x^2k) to x^-14 (its truncation error below 5e-17 at x >= 10). x <= 0 uses the reflection
// psi(1 - x) - pi / tan(pi x); the non-positive integers give NaN.
VB_HD double digamma(double x)
{
    double r = 0.0;
    if (!(x == x)) return x;
    if (x <= 0.0) {
        if (x == floor(x)) return NAN;
        const double pi = 3.14159265358979323846;
        r = -pi / tan(pi * x);
        x = 1.0 - x;
    }
    while (x < 10.0) { r -= 1.0 / x; x += 1.0; }
    const double f = 1.0 / (x * x);
    const double t = f * (-1.0 / 12 + f * (1.0 / 120 + f * (-1.0 / 252 + f * (1.0 / 240 + f * (-1.0 / 132 + f * (691.0 / 32760 + f * (-1.0 / 12)))))));
    return r + log(x) - 0.5 / x + t;
}

// compute_digamma_diffs (:173-183): al[k] = psi(alpha[k]) - psi(sum_k alpha[k]), the sum taken in k order.
VB_HD void digamma_diffs(const double* alpha, int K, double* al)
{
    double a0 = 0.0;
    for (int k = 0; k < K; ++k) a0 += alpha[k];
    const double d0 = digamma(a0);
    for (int k = 0; k < K; ++k) al[k] = digamma(alpha[k]) - d0;
}

// maths::log_beta: sum_k lgamma(a_k) - lgamma(sum_k a_k), both sums in k order.
VB_HD double log_beta(const double* a, int K)
{
    double s = 0.0, a0 = 0.0;
    for (int k = 0; k < K; ++k) { s += lgamma(a[k]); a0 += a[k]; }
    return s - lgamma(a0);
}

// t ln t, with its limit 0 at t = 0 (a responsibility that underflows to 0 carries no entropy).
VB_HD double xlogx(double t) { return t > 0.0 ? t * log(t) : 0.0; }

// One read's responsibilities (update_responsibilities_helper, :232-243): x[k * stride] holds ln rho_k = al[k] + sum_h W lnl on
// entry and tau_k = exp(ln rho_k - ln sum_k' exp(ln rho_k')) on return; the maximum is the first maximum, the sum in k order.
// Returns sum_k tau_k ln tau_k.
VB_HD double responsibilities(double* x, int K, long long stride)
{
    double mx = x[0];
    for (int k = 1; k < K; ++k) if (x[k * stride] > mx) mx = x[k * stride];
    double sum = 0.0;
    for (int k = 0; k < K; ++k) sum += exp(x[k * stride] - mx);
    const double norm = mx + log(sum);
    double ent = 0.0;
    for (int k = 0; k < K; ++k) {
        const double t = exp(x[k * stride] - norm);
        x[k * stride] = t;
        ent += xlogx(t);
    }
    return ent;
}

// sum_k M[s][k][gt[k]] for one sample (marginalise over a genotype's slots, :366-375); Ms = M + s * K * H.
VB_HD double genotype_marginal(const double* Ms, const int* gt, int K, int H)
{
    double r = 0.0;
    for (int k = 0; k < K; ++k) r += Ms[(long long)k * H + gt[k]];
    return r;
}

// The genotype log posterior before normalisation (update_genotype_log_posteriors, :391-402): lp + sum_s (sum_k M[s][k][gt[k]]).
VB_HD double genotype_update(double lp, const double* M, int S, const int* gt, int K, int H)
{
    double r = 0.0;
    for (int s = 0; s < S; ++s) r += genotype_marginal(M + (long long)s * K * H, gt, K, H);
    return lp + r;
}

// A genotype's ELBO term (calculate_evidence_lower_bound, :433-441): p * ((lp - lpost) + sum_s sum_k M[s][k][gt[k]]).
VB_HD double elbo_genotype_term(double p, double lp, double lpost, const double* M, int S, const int* gt, int K, int H)
{
    double w = lp - lpost;
    for (int s = 0; s < S; ++s) w += genotype_marginal(M + (long long)s * K * H, gt, K, H);
    return p * w;
}

// The samples' ELBO terms added after the genotype sum (:442-445): for each s, (log_beta(alpha_s) - log_beta(prior_s)), then the
// entropy -sum tau ln tau (xlogx_sum[s]).
VB_HD double elbo_add_samples(double acc, const double* prior, const double* alpha, const double* xlogx_sum, int S, int K)
{
    for (int s = 0; s < S; ++s) {
        acc += log_beta(alpha + (long long)s * K, K) - log_beta(prior + (long long)s * K, K);
        acc += -xlogx_sum[s];
    }
    return acc;
}

// The loop's stopping rule (:480).
VB_HD bool converged(double curr, double prev, double epsilon) { return curr <= prev || (curr - prev) < epsilon; }

} // namespace vb
} // namespace phmm

#if defined(__CUDACC__)
namespace phmm {
namespace vb {

constexpr int kThreads = 512;        // k_vb_seeds: one block per seed at a time
constexpr int kFinishThreads = 1024; // k_vb_modes_compact, k_vb_normalise

struct Args {
    const double* lnl; int H, R, S, G, K, n_seeds;
    const int* soff;                   // [S + 1] read offsets of the samples
    const int* gt;                     // [G][K]
    const double* prior;               // [S][K]
    const double* lp;                  // [G] genotype log priors
    const double* seeds;               // [n_seeds][G]
    double epsilon; int max_iterations;
    // k_vb_index's output: per (k, h) the count and first position of slot k's genotypes with haplotype h in L's slot-k block;
    // slot k's occurring haplotypes kh[k * H + i], i < nk[k]; L[k * G + i] the genotypes ordered by (haplotype, genotype) and
    // sid[k * G + i] = k * H + their haplotype
    const int *cnt, *start, *kh, *nk, *L, *sid;
    const int* bad;                    // set by k_vb_index: an index outside [0, H)
    double* ws; long long ws_stride;   // per-block workspace
    double* lpost;                     // [n_seeds][G] each seed's log posteriors
    double* ev; int* iters; int* map;  // [n_seeds]
    double* alpha;                     // [n_seeds][S][K]
};

__device__ __forceinline__ double block_sum(double v, double* red)
{
    red[threadIdx.x] = v;
    __syncthreads();
    for (int s = blockDim.x / 2; s > 0; s >>= 1) {
        if ((int)threadIdx.x < s) red[threadIdx.x] += red[threadIdx.x + s];
        __syncthreads();
    }
    const double r = red[0];
    __syncthreads();
    return r;
}

__device__ __forceinline__ double block_max(double v, double* red)
{
    red[threadIdx.x] = v;
    __syncthreads();
    for (int s = blockDim.x / 2; s > 0; s >>= 1) {
        if ((int)threadIdx.x < s && red[threadIdx.x + s] > red[threadIdx.x]) red[threadIdx.x] = red[threadIdx.x + s];
        __syncthreads();
    }
    const double r = red[0];
    __syncthreads();
    return r;
}

// The first index of the maximum (std::max_element): each thread's candidate is the first maximum of its strided values.
__device__ __forceinline__ int block_argmax(double v, int i, double* red, int* redi)
{
    red[threadIdx.x] = v; redi[threadIdx.x] = i;
    __syncthreads();
    for (int s = blockDim.x / 2; s > 0; s >>= 1) {
        if ((int)threadIdx.x < s) {
            const double o = red[threadIdx.x + s]; const int oi = redi[threadIdx.x + s];
            if (oi >= 0 && (redi[threadIdx.x] < 0 || o > red[threadIdx.x] || (o == red[threadIdx.x] && oi < redi[threadIdx.x]))) {
                red[threadIdx.x] = o; redi[threadIdx.x] = oi;
            }
        }
        __syncthreads();
    }
    const int r = redi[0];
    __syncthreads();
    return r;
}

__device__ __forceinline__ double warp_sum(double v)
{
    for (int o = 16; o > 0; o >>= 1) v += __shfl_down_sync(0xffffffffu, v, o);
    return v;
}

// The per-slot index of genotypes by haplotype, one block per slot k: counts, offsets and occurring haplotypes, then a stable
// placement of the genotypes in haplotype order by one warp (integer atomics only). An index outside [0, H) sets *bad.
__global__ void __launch_bounds__(256)
k_vb_index(const int* __restrict__ gt, const int G, const int K, const int H, int* __restrict__ cnt, int* __restrict__ start,
           int* __restrict__ kh, int* __restrict__ nk, int* __restrict__ L, int* __restrict__ sid, int* __restrict__ bad)
{
    extern __shared__ int cur[];
    __shared__ int out_of_range;
    const int k = blockIdx.x;
    if (threadIdx.x == 0) out_of_range = 0;
    for (int h = threadIdx.x; h < H; h += blockDim.x) cur[h] = 0;
    __syncthreads();
    for (int g = threadIdx.x; g < G; g += blockDim.x) {
        const int h = gt[(long long)g * K + k];
        if (h < 0 || h >= H) out_of_range = 1;
        else atomicAdd(&cur[h], 1);
    }
    __syncthreads();
    if (out_of_range) {
        if (threadIdx.x == 0) atomicOr(bad, 1);
        return;
    }
    if (threadIdx.x == 0) {
        int run = 0, n = 0;
        for (int h = 0; h < H; ++h) {
            const int c = cur[h];
            cnt[k * H + h] = c;
            start[k * H + h] = run;
            if (c) kh[k * H + n++] = h;
            cur[h] = run;
            run += c;
        }
        nk[k] = n;
    }
    __syncthreads();
    if (threadIdx.x >= 32) return;
    const int lane = threadIdx.x;
    for (int base = 0; base < G; base += 32) {
        const int g = base + lane;
        const unsigned active = __ballot_sync(0xffffffffu, g < G);
        if (g < G) {
            const int h = gt[(long long)g * K + k];
            const unsigned peers = __match_any_sync(active, h);
            const int pos = cur[h] + __popc(peers & ((1u << lane) - 1u));
            L[(long long)k * G + pos] = g;
            sid[(long long)k * G + pos] = k * H + h;
            __syncwarp(active);
            if (lane == __ffs(peers) - 1) cur[h] += __popc(peers);
        }
        __syncwarp();
    }
}

struct Workspace {
    double *W, *M, *tau, *en, *post, *alpha, *al, *A, *X;
    __device__ Workspace(const Args& a, double* p)
    {
        const long long KH = (long long)a.K * a.H;
        W = p; M = W + KH; tau = M + a.S * KH; en = tau + (long long)a.K * a.R; post = en + a.R;
        alpha = post + a.G; al = alpha + a.S * a.K; A = al + a.S * a.K; X = A + a.S * a.K;
    }
    static long long doubles(int H, int R, int S, int G, int K)
    {
        const long long KH = (long long)K * H;
        return KH + S * KH + (long long)K * R + R + G + 3LL * S * K + S;
    }
};

struct Shared {
    double red[kThreads];
    int redi[kThreads];
    double head[kThreads], tail[kThreads];
    long long tail_end[kThreads];
    int tail_seg[kThreads];
    double scalar;
    int stop;
};

// W[k][h] = sum of post over slot k's genotypes with haplotype h, in L's order: each thread sums a contiguous chunk of L; a
// segment that crosses chunks is finished by the thread where it starts, adding the later chunks' heads in order. Also used by
// phmm_vb_mm.cuh, whose arguments carry the same index fields (K slots, G genotypes) and whose workspace the same W and post.
template <typename A, typename WS>
__device__ void rebuild_w(const A& a, const WS& w, Shared& sh)
{
    const long long NL = (long long)a.K * a.G;
    const long long chunk = (NL + blockDim.x - 1) / blockDim.x;
    const long long lo = (long long)threadIdx.x * chunk, hi = min(lo + chunk, NL);
    sh.tail_seg[threadIdx.x] = -1;
    sh.head[threadIdx.x] = 0.0;
    int cur = -1; long long sb = 0, se = 0; double acc = 0.0;
    auto flush = [&]() {
        if (sb >= lo && se <= hi) w.W[cur] = acc;
        else if (sb < lo) sh.head[threadIdx.x] = acc;
        else { sh.tail[threadIdx.x] = acc; sh.tail_seg[threadIdx.x] = cur; sh.tail_end[threadIdx.x] = se; }
    };
    for (long long i = lo; i < hi; ++i) {
        const int sg = a.sid[i];
        if (sg != cur) {
            if (cur >= 0) flush();
            cur = sg;
            sb = (long long)(sg / a.H) * a.G + a.start[sg];
            se = sb + a.cnt[sg];
            acc = 0.0;
        }
        acc += w.post[a.L[i]];
    }
    if (cur >= 0) flush();
    __syncthreads();
    const int seg = sh.tail_seg[threadIdx.x];
    if (seg >= 0) {
        double sum = sh.tail[threadIdx.x];
        const long long end = sh.tail_end[threadIdx.x];
        for (int t = threadIdx.x + 1; t < (int)blockDim.x; ++t) {
            sum += sh.head[t];
            if (min((long long)(t + 1) * chunk, NL) >= end) break;
        }
        w.W[seg] = sum;
    }
}

// The responsibility update (update_responsibilities, :284-304) from the posterior alphas `alpha_src` and w.post, followed by
// what the rest of the iteration needs from it: M, the alpha sums A[s][k] = sum tau and X[s] = sum tau ln tau.
__device__ void sweep(const Args& a, const Workspace& w, const double* alpha_src, Shared& sh)
{
    rebuild_w(a, w, sh);
    for (int s = threadIdx.x; s < a.S; s += blockDim.x) digamma_diffs(alpha_src + s * a.K, a.K, w.al + s * a.K);
    __syncthreads();
    const int H = a.H, R = a.R, K = a.K;
    for (int s = 0; s < a.S; ++s) {
        for (int n = a.soff[s] + threadIdx.x; n < a.soff[s + 1]; n += blockDim.x) {
            for (int k = 0; k < K; ++k) {
                double m = 0.0;
                const int* hs = a.kh + k * H;
                for (int i = 0, e = a.nk[k]; i < e; ++i) {
                    const int h = hs[i];
                    m += w.W[k * H + h] * a.lnl[(long long)h * R + n];
                }
                w.tau[(long long)k * R + n] = w.al[s * K + k] + m;
            }
            w.en[n] = responsibilities(w.tau + n, K, R);
        }
    }
    __syncthreads();
    const int KH = K * H;
    const long long per = (long long)KH + K + 1;
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, nwarps = blockDim.x >> 5;
    for (long long t = warp; t < a.S * per; t += nwarps) {
        const int s = (int)(t / per), j = (int)(t % per);
        const int n0 = a.soff[s], n1 = a.soff[s + 1];
        double v = 0.0;
        if (j < KH) {
            if (a.cnt[j] == 0) continue;
            const double* tk = w.tau + (long long)(j / H) * R;
            const double* lh = a.lnl + (long long)(j % H) * R;
            for (int n = n0 + lane; n < n1; n += 32) v += tk[n] * lh[n];
        } else if (j < KH + K) {
            const double* tk = w.tau + (long long)(j - KH) * R;
            for (int n = n0 + lane; n < n1; n += 32) v += tk[n];
        } else {
            for (int n = n0 + lane; n < n1; n += 32) v += w.en[n];
        }
        v = warp_sum(v);
        if (lane == 0) {
            if (j < KH) w.M[(long long)s * KH + j] = v;
            else if (j < KH + K) w.A[s * K + (j - KH)] = v;
            else w.X[s] = v;
        }
    }
    __syncthreads();
}

// The ELBO (calculate_evidence_lower_bound) of the current state: genotypes below kPosteriorSkip left out when `skip`.
__device__ double elbo(const Args& a, const Workspace& w, const double* lpost, bool skip, Shared& sh)
{
    double acc = 0.0;
    for (int g = threadIdx.x; g < a.G; g += blockDim.x) {
        const double p = w.post[g];
        if (!skip || p >= kPosteriorSkip)
            acc += elbo_genotype_term(p, a.lp[g], lpost[g], w.M, a.S, a.gt + (long long)g * a.K, a.K, a.H);
    }
    acc = block_sum(acc, sh.red);
    return elbo_add_samples(acc, a.prior, w.alpha, w.X, a.S, a.K);
}

// Every seed's run of the loop (detail::run_variational_bayes, :452-488), one block per seed at a time, then its final evidence
// (calculate_log_evidences, no posterior skip) and the first index of its maximum posterior.
__global__ void __launch_bounds__(kThreads)
k_vb_seeds(const Args a)
{
    __shared__ Shared sh;
    if (*a.bad) return;
    const Workspace w(a, a.ws + blockIdx.x * a.ws_stride);
    const int G = a.G, SK = a.S * a.K;
    for (int seed = blockIdx.x; seed < a.n_seeds; seed += gridDim.x) {
        double* lpost = a.lpost + (long long)seed * G;
        const double* sd = a.seeds + (long long)seed * G;
        for (int g = threadIdx.x; g < G; g += blockDim.x) { lpost[g] = sd[g]; w.post[g] = exp(sd[g]); }
        for (int i = threadIdx.x; i < SK; i += blockDim.x) w.alpha[i] = a.prior[i];
        __syncthreads();
        sweep(a, w, a.prior, sh);
        double prev = -1.7976931348623157e308;   // std::numeric_limits<double>::lowest()
        int it = 0;
        while (it < a.max_iterations) {
            ++it;
            double mx = -INFINITY;
            for (int g = threadIdx.x; g < G; g += blockDim.x) {
                const double v = genotype_update(a.lp[g], w.M, a.S, a.gt + (long long)g * a.K, a.K, a.H);
                lpost[g] = v;
                if (v > mx) mx = v;
            }
            mx = block_max(mx, sh.red);
            double sum = 0.0;
            for (int g = threadIdx.x; g < G; g += blockDim.x) sum += exp(lpost[g] - mx);
            const double norm = mx + log(block_sum(sum, sh.red));
            for (int g = threadIdx.x; g < G; g += blockDim.x) { const double v = lpost[g] - norm; lpost[g] = v; w.post[g] = exp(v); }
            for (int i = threadIdx.x; i < SK; i += blockDim.x) w.alpha[i] = a.prior[i] + w.A[i];
            __syncthreads();
            const double curr = elbo(a, w, lpost, true, sh);
            if (converged(curr, prev, a.epsilon)) break;
            prev = curr;
            sweep(a, w, w.alpha, sh);
        }
        const double ev = elbo(a, w, lpost, false, sh);
        double best = 0.0; int bi = -1;
        for (int g = threadIdx.x; g < G; g += blockDim.x) if (bi < 0 || w.post[g] > best) { best = w.post[g]; bi = g; }
        bi = block_argmax(best, bi, sh.red, sh.redi);
        if (threadIdx.x == 0) { a.ev[seed] = ev; a.iters[seed] = it; a.map[seed] = bi; }
        for (int i = threadIdx.x; i < SK; i += blockDim.x) a.alpha[(long long)seed * SK + i] = w.alpha[i];
        __syncthreads();
    }
}

// A double's bits as an unsigned key with the same order (for the integer atomicMax of find_map_modes).
__device__ __forceinline__ unsigned long long order_key(double x)
{
    const unsigned long long b = (unsigned long long)__double_as_longlong(x);
    return (b >> 63) ? ~b : (b | 0x8000000000000000ULL);
}

// find_map_modes (:578-599), first pass: the largest evidence among the seeds whose MAP genotype is g.
__global__ void k_vb_mode_max(const int* __restrict__ bad, const double* __restrict__ ev, const int* __restrict__ map, const int n, unsigned long long* __restrict__ key)
{
    if (*bad) return;   // k_vb_index found an index outside [0, H): nothing below was computed
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i < n) atomicMax(&key[map[i]], order_key(ev[i]));
}

// Second pass: the first seed with that evidence (a later seed replaces an earlier one only when strictly larger).
__global__ void k_vb_mode_first(const int* __restrict__ bad, const double* __restrict__ ev, const int* __restrict__ map, const int n,
                                const unsigned long long* __restrict__ key, int* __restrict__ first)
{
    if (*bad) return;   // k_vb_index found an index outside [0, H): nothing below was computed
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i < n && order_key(ev[i]) == key[map[i]]) atomicMin(&first[map[i]], i);
}

// The modes in genotype order, their weights (maths::normalise_exp of their evidences) and the max-evidence seed (the first
// maximum, std::max_element); one block.
__global__ void __launch_bounds__(kFinishThreads)
k_vb_modes_compact(const int* __restrict__ bad, const double* __restrict__ ev, const int n_seeds, const int* __restrict__ first, const int G,
                   int* __restrict__ modes, double* __restrict__ weights, int* __restrict__ n_modes, int* __restrict__ max_seed)
{
    if (*bad) return;   // k_vb_index found an index outside [0, H): nothing below was computed
    __shared__ double red[kFinishThreads];
    __shared__ int redi[kFinishThreads];
    __shared__ int base[kFinishThreads];
    const int T = blockDim.x, t = threadIdx.x;
    const int chunk = (G + T - 1) / T, lo = min(t * chunk, G), hi = min(lo + chunk, G);
    int c = 0;
    for (int g = lo; g < hi; ++g) c += first[g] < n_seeds;
    base[t] = c;
    __syncthreads();
    if (t == 0) { int run = 0; for (int i = 0; i < T; ++i) { const int v = base[i]; base[i] = run; run += v; } *n_modes = run; }
    __syncthreads();
    int o = base[t];
    for (int g = lo; g < hi; ++g) if (first[g] < n_seeds) modes[o++] = first[g];
    __syncthreads();
    const int nm = *n_modes;
    double best = 0.0; int bi = -1;
    for (int i = t; i < n_seeds; i += T) if (bi < 0 || ev[i] > best) { best = ev[i]; bi = i; }
    bi = block_argmax(best, bi, red, redi);
    if (t == 0) *max_seed = bi;
    double mx = -INFINITY;
    for (int i = t; i < nm; i += T) mx = fmax(mx, ev[modes[i]]);
    mx = block_max(mx, red);
    double sum = 0.0;
    for (int i = t; i < nm; i += T) sum += exp(ev[modes[i]] - mx);
    const double norm = mx + log(block_sum(sum, red));
    for (int i = t; i < nm; i += T) weights[i] = exp(ev[modes[i]] - norm);
}

// compute_evidence_weighted_genotype_posteriors' sum over the modes in order, and the max-evidence seed's posteriors.
__global__ void k_vb_weighted(const int* __restrict__ bad, const double* __restrict__ lpost, const int G, const int* __restrict__ modes, const double* __restrict__ weights,
                              const int* __restrict__ n_modes, const int* __restrict__ max_seed, double* __restrict__ weighted,
                              double* __restrict__ post, double* __restrict__ log_post)
{
    if (*bad) return;   // k_vb_index found an index outside [0, H): nothing below was computed
    const int g = blockIdx.x * blockDim.x + threadIdx.x;
    if (g >= G) return;
    double r = 0.0;
    for (int i = 0, e = *n_modes; i < e; ++i) r = r + weights[i] * exp(lpost[(long long)modes[i] * G + g]);
    weighted[g] = r;
    const double lp = lpost[(long long)*max_seed * G + g];
    log_post[g] = lp;
    post[g] = exp(lp);
}

// check_normalisation (:561-565) of both posterior vectors, and the max-evidence seed's scalars and alphas; one block.
__global__ void __launch_bounds__(kFinishThreads)
k_vb_normalise(const int* __restrict__ bad, const int G, double* __restrict__ weighted, double* __restrict__ post, const double* __restrict__ ev,
               const double* __restrict__ seed_alpha, const int SK, const int* __restrict__ max_seed, double* __restrict__ alpha,
               double* __restrict__ max_ev, int* __restrict__ max_seed_out)
{
    if (*bad) return;   // k_vb_index found an index outside [0, H): nothing below was computed
    __shared__ double red[kFinishThreads];
    const int t = threadIdx.x, T = blockDim.x;
    for (int v = 0; v < 2; ++v) {
        double* p = v ? post : weighted;
        double m = 0.0;
        for (int g = t; g < G; g += T) m += p[g];
        m = block_sum(m, red);
        if (m > 1.0) for (int g = t; g < G; g += T) p[g] /= m;
    }
    const int ms = *max_seed;
    for (int i = t; i < SK; i += T) alpha[i] = seed_alpha[(long long)ms * SK + i];
    if (t == 0) { *max_ev = ev[ms]; *max_seed_out = ms; }
}

} // namespace vb
} // namespace phmm
#endif
