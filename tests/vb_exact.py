"""High-precision restatement of the variational Bayes mixture inference (run_variational_bayes,
core/models/genotype/variational_bayes_mixture_model.hpp:452-669, its save_memory = false path) that phmm_variational_bayes
computes, in numpy.longdouble (64-bit mantissa) with mpmath for the digamma and lgamma values.

Per seed (detail::run_variational_bayes, :452-488):
  * genotype_posteriors = exp(seed), not normalised; the responsibilities start from the prior alphas (:468-470);
  * each iteration: the log posteriors lp + sum_s sum_k sum_n tau[s][k][n] lnl[gt[g][k]][n], normalised (normalise_logs); their
    exp; alpha = prior + sum_n tau; the ELBO with genotypes of posterior < 1e-10 left out; stop if curr <= prev or
    curr - prev < epsilon; otherwise the responsibility update. A seed that runs out of iterations ends with its
    responsibilities one update ahead of its posteriors.
  * its final evidence is the ELBO with no posterior skip (calculate_log_evidences, :627-641).
Seeds are combined as the reference does (:573-669): find_map_modes keeps per MAP genotype the first seed of largest evidence;
the modes' evidences are normalise_exp'd into weights; the weighted sum and the max-evidence seed's (the first maximum)
posteriors get check_normalisation (divide only when the mass exceeds 1).

The inner products over genotypes are taken in one of two forms that are equal in real arithmetic: `direct` sums over genotypes
as the reference writes it (O(G K N) per iteration, for small cases); otherwise they are grouped by haplotype first,
W[k][h] = sum_{g: gt[g][k] = h} p_g and M[s][k][h] = sum_n tau lnl[h][n] (the device's form). A CPU test holds the two to each
other. A responsibility of 0 contributes 0 to the entropy (the limit of t ln t).

`run` reports, for each seed, the ELBO pair (curr, prev) of every stopping decision, so that a test can tell a decision that lies
within rounding of the threshold (`near_threshold`) from a wrong one; `forced` runs every seed for exactly that many iterations."""

import mpmath
import numpy as np

LD = np.longdouble
assert np.finfo(LD).nmant >= 63, "vb_exact needs an 80-bit long double (64-bit mantissa)"
LOWEST = -1.7976931348623157e308
SKIP = 1e-10


def _digamma(x):
    return LD(str(mpmath.digamma(mpmath.mpf(str(x)))))


def _lgamma(x):
    return LD(str(mpmath.loggamma(mpmath.mpf(str(x)))))


def _log_beta(a):
    return sum((_lgamma(v) for v in a), LD(0)) - _lgamma(sum(a, LD(0)))


def _lse(x, axis=None):
    mx = np.max(x, axis=axis, keepdims=True)
    return (mx + np.log(np.sum(np.exp(x - mx), axis=axis, keepdims=True))).squeeze(axis) if axis is not None else \
        LD(mx.ravel()[0] + np.log(np.sum(np.exp(x - mx))))


def _xlogx(t):
    with np.errstate(divide="ignore", invalid="ignore"):
        return np.where(t > 0, t * np.log(np.where(t > 0, t, 1)), LD(0))


class _Problem:
    def __init__(self, lnl, sample_off, gt, prior, lp, direct):
        self.L = np.asarray(lnl, dtype=np.float64).astype(LD)
        self.off = [int(v) for v in sample_off]
        self.gt = np.asarray(gt, dtype=np.int64)
        self.prior = np.asarray(prior, dtype=np.float64).astype(LD)
        self.lp = np.asarray(lp, dtype=np.float64).astype(LD)
        self.G, self.K = self.gt.shape
        self.S = len(self.off) - 1
        self.H = self.L.shape[0]
        self.direct = direct
        # per slot: the haplotypes that occur there, and each genotype's position among them (sums over the others are never read)
        self.used = [np.unique(self.gt[:, k], return_inverse=True) for k in range(self.K)]

    def cols(self, s):
        return self.L[:, self.off[s]:self.off[s + 1]]

    def marginal_reads(self, post, s):
        """[K][N_s]: sum_g p_g lnl[gt[g][k]][n]."""
        Ls = self.cols(s)
        out = np.zeros((self.K, Ls.shape[1]), dtype=LD)
        for k in range(self.K):
            if self.direct:
                for g in range(self.G):
                    out[k] += post[g] * Ls[self.gt[g, k]]
            else:
                W = np.zeros(self.H, dtype=LD)
                np.add.at(W, self.gt[:, k], post)
                used = np.nonzero(np.bincount(self.gt[:, k], minlength=self.H))[0]
                out[k] = W[used] @ Ls[used] if len(used) else 0
        return out

    def marginal_genotypes(self, tau, s):
        """[G]: sum_k sum_n tau[k][n] lnl[gt[g][k]][n] for sample s."""
        Ls = self.cols(s)
        r = np.zeros(self.G, dtype=LD)
        for k in range(self.K):
            if Ls.shape[1] == 0:
                continue
            if self.direct:
                r += np.array([np.sum(tau[k] * Ls[self.gt[g, k]]) for g in range(self.G)], dtype=LD)
            else:
                used, at = self.used[k]
                r += (Ls[used] @ tau[k])[at]
        return r

    def responsibilities(self, alphas, post):
        taus, ent = [], []
        for s in range(self.S):
            a = alphas[s]
            d0 = _digamma(sum(a, LD(0)))
            al = np.array([_digamma(v) - d0 for v in a], dtype=LD)
            rho = al[:, None] + self.marginal_reads(post, s)
            if rho.shape[1]:
                rho = rho - _lse(rho, axis=0)[None, :]
            t = np.exp(rho)
            taus.append(t)
            ent.append(np.sum(_xlogx(t)))
        return taus, ent

    def elbo(self, alphas, lpost, post, taus, ent, skip):
        w = self.lp - lpost
        for s in range(self.S):
            w = w + self.marginal_genotypes(taus[s], s)
        keep = post >= SKIP if skip else np.ones(self.G, dtype=bool)
        r = np.sum(post[keep] * w[keep])
        for s in range(self.S):
            r += _log_beta(alphas[s]) - _log_beta(self.prior[s])
            r += -ent[s]
        return LD(r)


def run_seed(problem, seed, epsilon, max_iterations, forced=None):
    P = problem
    lpost = np.asarray(seed, dtype=np.float64).astype(LD)
    post = np.exp(lpost)
    alphas = P.prior.copy()
    taus, ent = P.responsibilities(alphas, post)
    prev = LD(LOWEST)
    decisions = []
    n = min(forced, max_iterations) if forced is not None else max_iterations
    it = 0
    for _ in range(n):
        it += 1
        u = P.lp.copy()
        marg = np.zeros(P.G, dtype=LD)
        for s in range(P.S):
            marg = marg + P.marginal_genotypes(taus[s], s)
        lpost = u + marg
        lpost = lpost - _lse(lpost)
        post = np.exp(lpost)
        alphas = np.array([P.prior[s] + np.sum(taus[s], axis=1) for s in range(P.S)], dtype=LD)
        curr = P.elbo(alphas, lpost, post, taus, ent, True)
        decisions.append((float(curr), float(prev)))
        stop = bool(curr <= prev or curr - prev < epsilon)
        if forced is not None and it < forced:
            stop = False
        elif forced is not None and it == forced < max_iterations:
            stop = True      # the device stopped here; at max_iterations its own decision says whether tau moved on
        if stop:
            break
        prev = curr
        taus, ent = P.responsibilities(alphas, post)
    ev = P.elbo(alphas, lpost, post, taus, ent, False)
    return dict(lpost=lpost, post=post, alphas=alphas, evidence=ev, iterations=it, decisions=decisions)


def near_threshold(decisions, epsilon, rel=1e-9):
    """Whether any stopping decision of a seed lies within rounding of epsilon or of 0: the device may decide it either way."""
    for curr, prev in decisions:
        if prev == LOWEST:
            continue
        d = curr - prev
        margin = rel * (1.0 + abs(curr))
        if abs(d) <= margin or abs(d - epsilon) <= margin:
            return True
    return False


def combine(seed_results):
    """compute_evidence_weighted_genotype_posteriors, the max-evidence seed and check_normalisation (:561-669)."""
    ev = [r["evidence"] for r in seed_results]
    G = len(seed_results[0]["post"])
    map_of = [int(np.argmax(r["post"])) for r in seed_results]
    best = {}
    for i, g in enumerate(map_of):
        if g not in best or ev[i] > ev[best[g]]:
            best[g] = i
    modes = [best[g] for g in sorted(best)]
    me = np.array([ev[i] for i in modes], dtype=LD)
    w = np.exp(me - _lse(me))
    weighted = np.zeros(G, dtype=LD)
    for wi, i in zip(w, modes):
        weighted = weighted + wi * seed_results[i]["post"]
    mass = np.sum(weighted)
    if mass > 1:
        weighted = weighted / mass
    ms = int(np.argmax(np.array(ev, dtype=LD)))
    post = seed_results[ms]["post"].copy()
    mass = np.sum(post)
    if mass > 1:
        post = post / mass
    return dict(posteriors=post, log_posteriors=seed_results[ms]["lpost"], alphas=seed_results[ms]["alphas"],
                weighted=weighted, max_log_evidence=ev[ms], max_seed=ms, modes=modes)


def _reuse(free, forced, i):
    """A seed's run without `forced` when it ran for exactly forced[i] iterations: forcing that count then changes no decision."""
    if free is None or forced is None or free["seeds"][i]["iterations"] != int(forced[i]):
        return None
    return free["seeds"][i]


def run(lnl, sample_off, genotypes, prior_alphas, genotype_log_priors, seeds, epsilon=0.05, max_iterations=1000, forced=None,
        direct=False, free=None):
    """The whole call. forced: None, or one iteration count per seed (e.g. the device's) to run each seed for exactly that long.
    free: this call's result without `forced`, whose seeds are reused where they ran for their forced count."""
    P = _Problem(lnl, sample_off, genotypes, prior_alphas, genotype_log_priors, direct)
    seeds = np.asarray(seeds, dtype=np.float64)
    res = [_reuse(free, forced, i) or run_seed(P, seeds[i], epsilon, max_iterations, None if forced is None else int(forced[i]))
           for i in range(len(seeds))]
    out = combine(res)
    out["seeds"] = res
    return out


# -- forward-error bound of one iteration -----------------------------------------------------------------------------------------
# The first-order error of a double evaluation of a one-seed call with max_iterations = 1: the initial responsibility sweep from
# exp(seed) and the prior alphas, one genotype update (its ELBO decision always continues: prev is lowest()), the second sweep, and
# the final evidence. u = 2^-53 is the unit roundoff; CUDA's double exp, log and lgamma are within 2 ulp (2u relative), the project's
# digamma within 32u (|psi(x)| + sum of its recurrence terms 1/(x+j) + 1). A sum of n terms in any order adds at most (n - 1) u
# times the sum of their magnitudes (first order). Step by step, with d. the absolute error bound of a quantity:
#   W[k][h] = sum over the c_kh genotypes of p:            dW = sum dp + c_kh u W
#   m[k][n] = sum_h W lnl[h][n] over slot k's nk terms:    dm = sum_h dW |lnl| + (nk + 1) u sum_h W |lnl|
#   al_k = psi(alpha_k) - psi(alpha_0):                    dal = dpsi(alpha_k) + dpsi(alpha_0) + psi'(alpha_k) dalpha_k
#                                                               + psi'(alpha_0) (sum dalpha + K u alpha_0) + u |al_k|
#   x = al + m:                                            dx = dal + dm + u |x|
#   tau = exp(x - (mx + ln sum exp(x - mx))): relative     e_n = 2 max_k dx + 2u (max_k |x| + |norm|) + (K + 4) u
#   M[s][k][h] = sum_n tau lnl:                            dM = sum_n tau |lnl| (e_n + (N_s + 1) u)
#   A[s][k] = sum_n tau:                                   dA = sum_n tau (e_n + N_s u);   alpha = prior + A: dalpha = dA + u alpha
#   X[s] = sum tau ln tau:                                 dX = sum tau (|1 + ln tau| e_n + (K + N_s + 3) u |ln tau|)
#   v_g = lp + sum_s sum_k M:                              dv = sum dM + (S K + 1) u (|lp| + sum |M|)
#   norm = ln sum_g exp(v):                                dnorm = max dv + (G + 3) u (|norm| + 1)
#   lpost = v - norm:                                      dlpost = dv + dnorm + u |lpost|;   post = exp(lpost): dpost = post (dlpost + 2u)
#   ELBO = sum_g p w + sum_s (logB(alpha) - logB(prior) - X'), w = lp - lpost + sum M' (M', X' of the second sweep):
#       dw = dlpost + sum dM' + (S K + 2) u (|lp| + |lpost| + sum |M'|);  the genotype sum: sum (dp |w| + p dw) + (G + 1) u sum |p w|;
#       dlogB(a) = sum_k |psi(a_k)| da_k + |psi(a_0)| sum da + 2u (sum |lgamma(a_k)| + |lgamma(a_0)|) + (K + 1) u sum |lgamma|;
#       and (2 S + 1) u times the magnitudes of the terms added last.
#   With one seed the weights are exactly 1, so the weighted posteriors are the posteriors; check_normalisation's division adds
#   (G + 1) u post.
# The tests allow BOUND_UNITS times this, for the second-order terms left out.
U = 2.0 ** -53
BOUND_UNITS = 2.0


def _psi_terms(x):
    x = float(x)
    rec = 0.0
    while x < 10.0:
        rec += 1.0 / abs(x)
        x += 1.0
    return rec


def _dpsi(x, dx):
    x = float(x)
    return 32 * U * (abs(float(mpmath.digamma(x))) + _psi_terms(x) + 1) + float(mpmath.psi(1, x)) * dx


def _dlogbeta(a, da, K):
    a = [float(v) for v in a]
    lg = [abs(float(mpmath.loggamma(v))) for v in a]
    a0 = sum(a)
    lg0 = abs(float(mpmath.loggamma(a0)))
    return (sum(abs(float(mpmath.digamma(v))) * d for v, d in zip(a, da)) + abs(float(mpmath.digamma(a0))) * sum(da)
            + 2 * U * (sum(lg) + lg0) + (K + 1) * U * (sum(lg) + lg0))


def _sweep_bound(P, post, dpost, alphas, dalpha):
    """Responsibilities from (post, alphas) with absolute errors (dpost, dalpha): exact tau and the bounds of M, A, X."""
    L = np.asarray(P.L, dtype=np.float64)
    aL = np.abs(L)
    p, dp = np.asarray(post, float), np.asarray(dpost, float)
    taus, _ = P.responsibilities(alphas, post)
    dM, dA, dX = [], [], []
    for s in range(P.S):
        cols = slice(P.off[s], P.off[s + 1])
        Ns = P.off[s + 1] - P.off[s]
        a = [float(v) for v in alphas[s]]
        a0 = sum(a)
        dx = np.zeros((P.K, Ns))
        absx = np.zeros((P.K, Ns))
        for k in range(P.K):
            c = np.bincount(P.gt[:, k], minlength=P.H)
            W = np.bincount(P.gt[:, k], weights=p, minlength=P.H)
            dW = np.bincount(P.gt[:, k], weights=dp, minlength=P.H) + c * U * W
            used = c > 0
            nk = int(used.sum())
            m_mag = W[used] @ aL[used][:, cols]
            dm = dW[used] @ aL[used][:, cols] + (nk + 1) * U * m_mag
            al = float(mpmath.digamma(a[k]) - mpmath.digamma(a0))
            dal = (_dpsi(a[k], dalpha[s][k]) + _dpsi(a0, sum(dalpha[s]) + P.K * U * a0) + U * abs(al))
            m = W[used] @ L[used][:, cols]
            absx[k] = np.abs(al + m)
            dx[k] = dal + dm + U * absx[k]
        t = np.asarray(taus[s], float)
        with np.errstate(divide="ignore"):
            lt = np.where(t > 0, np.log(np.where(t > 0, t, 1)), 0.0)
        norm = np.abs(np.max(absx, axis=0)) + 1.0 if Ns else np.zeros(0)
        e = 2 * np.max(dx, axis=0) + 2 * U * (np.max(absx, axis=0) + norm) + (P.K + 4) * U if Ns else np.zeros(0)
        dM.append(np.stack([(t[k] * (e + (Ns + 1) * U)) @ aL[:, cols].T for k in range(P.K)]) if Ns else np.zeros((P.K, P.H)))
        dA.append(np.array([np.sum(t[k] * (e + Ns * U)) for k in range(P.K)]))
        dX.append(float(np.sum(t * (np.abs(1 + lt) * e[None, :] + (P.K + Ns + 3) * U * np.abs(lt)))) if Ns else 0.0)
    return taus, dM, dA, dX


def one_iteration_bound(lnl, sample_off, genotypes, prior_alphas, genotype_log_priors, seed):
    """Absolute error bounds (times BOUND_UNITS) of a one-seed, max_iterations = 1 call's outputs, derived above: dict of
    log_posteriors[G], posteriors[G], weighted[G], alphas[S][K], evidence."""
    P = _Problem(lnl, sample_off, genotypes, prior_alphas, genotype_log_priors, False)
    lp = np.asarray(P.lp, float)
    p0 = np.exp(np.asarray(seed, dtype=np.float64).astype(LD))
    taus, dM, dA, _ = _sweep_bound(P, p0, 2 * U * np.asarray(p0, float), P.prior, np.zeros((P.S, P.K)))
    Ms = [np.asarray(P.cols(s), float) @ np.asarray(taus[s], float).T for s in range(P.S)]       # [H][K] per sample
    alphas = np.array([P.prior[s] + np.sum(taus[s], axis=1) for s in range(P.S)], dtype=LD)
    dalpha = np.array(dA) + U * np.asarray(alphas, float)
    dv = np.zeros(P.G)
    magM = np.zeros(P.G)
    v = lp.copy()
    for s in range(P.S):
        for k in range(P.K):
            dv += dM[s][k][P.gt[:, k]]
            magM += np.abs(Ms[s][P.gt[:, k], k])
            v += Ms[s][P.gt[:, k], k]
    dv += (P.S * P.K + 1) * U * (np.abs(lp) + magM)
    norm = float(_lse(v.astype(LD)))
    lpost = v - norm
    dlpost = dv + np.max(dv) + (P.G + 3) * U * (abs(norm) + 1) + U * np.abs(lpost)
    post = np.exp(lpost)
    dpost = post * (dlpost + 2 * U)
    postL = np.exp(lpost.astype(LD))
    taus2, dM2, _, dX2 = _sweep_bound(P, postL, dpost, alphas, dalpha)
    Ms2 = [np.asarray(P.cols(s), float) @ np.asarray(taus2[s], float).T for s in range(P.S)]
    w = lp - lpost
    dw = dlpost.copy()
    magw = np.abs(lp) + np.abs(lpost)
    for s in range(P.S):
        for k in range(P.K):
            w = w + Ms2[s][P.gt[:, k], k]
            dw += dM2[s][k][P.gt[:, k]]
            magw += np.abs(Ms2[s][P.gt[:, k], k])
    dw += (P.S * P.K + 2) * U * magw
    dE = float(np.sum(dpost * np.abs(w) + post * dw) + (P.G + 1) * U * np.sum(np.abs(post * w)))
    mag = float(np.sum(np.abs(post * w)))
    for s in range(P.S):
        dE += _dlogbeta(alphas[s], dalpha[s], P.K) + _dlogbeta(P.prior[s], np.zeros(P.K), P.K) + dX2[s]
        mag += abs(float(_log_beta(alphas[s]))) + abs(float(_log_beta(P.prior[s]))) + abs(float(np.sum(_xlogx(taus2[s]))))
    dE += (2 * P.S + 1) * U * mag
    dpost_n = dpost + (P.G + 1) * U * post
    return dict(log_posteriors=BOUND_UNITS * dlpost, posteriors=BOUND_UNITS * dpost_n, weighted=BOUND_UNITS * dpost_n,
                alphas=BOUND_UNITS * dalpha, evidence=BOUND_UNITS * dE)
