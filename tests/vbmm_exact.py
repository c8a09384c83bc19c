"""High-precision restatement of the mixture-of-mixtures variational Bayes inference (VariationalBayesMixtureMixtureModel::evaluate,
core/models/genotype/variational_bayes_mixture_mixture_model.cpp) that phmm_variational_bayes_mixture_mixture computes, in
numpy.longdouble (64-bit mantissa) with mpmath for the digamma and lgamma values.

Notation: S samples, sample s owning columns [off[s], off[s+1]); T groups, group t with K_t components at slots
j = koff[t] + k; maxK = max K_t; combination c gives slot j the haplotype gt[c][j]; m[j][n] = sum_c p_c lnl[gt[c][j]][n].
Per seed (evaluate, :254-298):
  * p = exp(seed), not normalised; the concentrations start at the priors.
  * sigma starts from init_responsibilities (:316-364): ln E[psi_t] (+ ln prior) + sum_{k < K_t} sum_n atau_k[n] m[j][n],
    atau the approximate tau of the first combination of largest p, normalise_exp'd over t.
  * tau starts from the component update (:446-486) with previous tau 0.
  * each iteration: the log posteriors lp + sum_s sum_t sigma sum_{k < maxK} <tau_k, lnl[gt[c][j(k)]]>, j(k) = koff + k for a
    real component and koff for a padded one, normalised; p = exp; group concentrations prior + sum_s sigma; mixture
    concentrations prior + sum_n tau for k < K_t; the evidence (:587-631); stop if curr <= prev or curr - prev < epsilon;
    otherwise sigma's update (:366-399, with sum_{k < K_t} ln E[pi_k]), then tau's.
  * the component update: ln rho = (tau of the previous iteration if t > 0 and `quirk`) + ln E[pi_k] + m[j][n] for a real
    component, -10000 for a padded one; normalised over the group's maxK components.
  * its evidence is the last ELBO computed.
Seeds are combined as compute_evidence_weighted_latents (:644-691) does.

The combination sums are taken in one of two forms equal in real arithmetic: `direct` sums over combinations as the reference
writes them (for small cases); otherwise grouped by haplotype, W[j][h] = sum_{c: gt[c][j] = h} p_c and
D[s][t][k][h] = sum_n tau lnl[h][n] (the device's form). `quirk=False` resets tau for every group, as the model would; a test
shows the reference differs from that.

`run` reports, for each seed, the evidence pair (curr, prev) of every stopping decision (see vb_exact.near_threshold);
`forced` runs every seed for exactly that many iterations."""

import functools

import mpmath
import numpy as np

from vb_exact import LD, LOWEST, _lse, _reuse, _xlogx, near_threshold  # noqa: F401  (near_threshold: re-exported for the tests)

NULL = LD(-10000)
MIN_LOG_PRIOR = LD(np.log(np.finfo(np.float64).tiny))


@functools.lru_cache(maxsize=1 << 16)
def _digamma(x):
    return LD(str(mpmath.digamma(mpmath.mpf(str(x)))))


@functools.lru_cache(maxsize=1 << 16)
def _lgamma(x):
    return LD(str(mpmath.loggamma(mpmath.mpf(str(x)))))


def _log_beta(a):
    return sum((_lgamma(v) for v in a), LD(0)) - _lgamma(sum(a, LD(0)))


def _dexp(a):
    """dirichlet_expectation_log: 0 for a single concentration."""
    if len(a) <= 1:
        return np.zeros(len(a), dtype=LD)
    d0 = _digamma(sum(a, LD(0)))
    return np.array([_digamma(v) - d0 for v in a], dtype=LD)


def _normalise_exp(x):
    return np.exp(x - _lse(x))


class _Problem:
    def __init__(self, lnl, sample_off, sizes, gt, lp, gc0, mc0, gprior, mask, direct, quirk):
        self.L = np.asarray(lnl, dtype=np.float64).astype(LD)
        self.off = [int(v) for v in sample_off]
        self.sizes = [int(k) for k in sizes]
        self.koff = np.concatenate([[0], np.cumsum(self.sizes)]).astype(int)
        self.T, self.K, self.maxK = len(self.sizes), int(self.koff[-1]), max(self.sizes)
        self.gt = np.asarray(gt, dtype=np.int64)
        self.lp = np.asarray(lp, dtype=np.float64).astype(LD)
        self.gc0 = np.asarray(gc0, dtype=np.float64).astype(LD)
        self.mc0 = np.asarray(mc0, dtype=np.float64).astype(LD)
        self.S, self.H, self.C = len(self.off) - 1, self.L.shape[0], self.gt.shape[0]
        self.lprior = [None] * self.S
        if gprior is not None:
            gp = np.asarray(gprior, dtype=np.float64)
            for s in range(self.S):
                if mask is None or mask[s]:
                    with np.errstate(divide="ignore"):
                        self.lprior[s] = np.where(gp[s] > 0, np.log(np.where(gp[s] > 0, gp[s], 1)).astype(LD), MIN_LOG_PRIOR).astype(LD)
        self.direct, self.quirk = direct, quirk
        # per slot: the haplotypes that occur there, and each combination's position among them (as vb_exact._Problem.used)
        self.used = [np.unique(self.gt[:, j], return_inverse=True) for j in range(self.K)]

    def cols(self, s):
        return self.L[:, self.off[s]:self.off[s + 1]]

    def slot_t_of(self):
        """The group of every slot."""
        return np.repeat(np.arange(self.T), self.sizes)

    def slot(self, t, k):
        return self.koff[t] + (k if k < self.sizes[t] else 0)

    def lnEpi(self, mconc, s, t):
        return _dexp(mconc[s][self.koff[t]:self.koff[t + 1]])

    def m_reads(self, post, s):
        """[K][N_s]: sum_c p_c lnl[gt[c][j]][n]."""
        Ls = self.cols(s)
        out = np.zeros((self.K, Ls.shape[1]), dtype=LD)
        for j in range(self.K):
            if self.direct:
                for c in range(self.C):
                    out[j] += post[c] * Ls[self.gt[c, j]]
            else:
                W = np.zeros(self.H, dtype=LD)
                np.add.at(W, self.gt[:, j], post)
                used = np.nonzero(np.bincount(self.gt[:, j], minlength=self.H))[0]
                out[j] = W[used] @ Ls[used] if len(used) else 0
        return out

    def marginal(self, sigma, taus):
        """[C]: sum_s sum_t sigma[s][t] sum_{k < maxK} <tau[s][t][k], lnl[gt[c][j(k)]]>."""
        r = np.zeros(self.C, dtype=LD)
        for s in range(self.S):
            Ls = self.cols(s)
            if Ls.shape[1] == 0:
                continue
            for t in range(self.T):
                acc = np.zeros(self.C, dtype=LD)
                for k in range(self.maxK):
                    j = self.slot(t, k)
                    if self.direct:
                        acc += np.array([np.sum(taus[s][t][k] * Ls[self.gt[c, j]]) for c in range(self.C)], dtype=LD)
                    else:
                        used, at = self.used[j]
                        acc += (Ls[used] @ taus[s][t][k])[at]
                r += sigma[s][t] * acc
        return r

    def init_sigma(self, gc, mconc, post):
        lnEpsi = _dexp(gc)
        cmax = int(np.argmax(post))
        sig = []
        for s in range(self.S):
            Ls = self.cols(s)
            m = self.m_reads(post, s)
            v = np.zeros(self.T, dtype=LD)
            for t in range(self.T):
                v[t] = lnEpsi[t] + (self.lprior[s][t] if self.lprior[s] is not None else 0)
                lnEpi = self.lnEpi(mconc, s, t)
                js = range(self.koff[t], self.koff[t + 1])
                if Ls.shape[1]:
                    a = np.array([lnEpi[k] + Ls[self.gt[cmax, j]] for k, j in enumerate(js)], dtype=LD)
                    at = np.exp(a - _lse(a, axis=0)[None, :])
                    v[t] += sum((np.sum(at[k] * m[j]) for k, j in enumerate(js)), LD(0))
            sig.append(_normalise_exp(v))
        return np.array(sig, dtype=LD)

    def components(self, mconc, post, prev):
        """tau[s][t][k][n] from the component update; prev: the previous taus (None at initialisation)."""
        taus = []
        for s in range(self.S):
            m = self.m_reads(post, s)
            N = m.shape[1]
            ts = np.zeros((self.T, self.maxK, N), dtype=LD)
            for t in range(self.T):
                lnEpi = self.lnEpi(mconc, s, t)
                x = np.full((self.maxK, N), NULL, dtype=LD)
                for k in range(self.sizes[t]):
                    before = prev[s][t][k] if (prev is not None and t > 0 and self.quirk) else LD(0)
                    x[k] = before + (lnEpi[k] + m[self.koff[t] + k])
                if N:
                    ts[t] = np.exp(x - _lse(x, axis=0)[None, :])
            taus.append(ts)
        return taus

    def update_sigma(self, gc, mconc, post, taus):
        lnEpsi = _dexp(gc)
        sig = []
        for s in range(self.S):
            m = self.m_reads(post, s)
            v = np.zeros(self.T, dtype=LD)
            for t in range(self.T):
                lnEpi = self.lnEpi(mconc, s, t)
                v[t] = lnEpsi[t] + (self.lprior[s][t] if self.lprior[s] is not None else 0) + np.sum(lnEpi)
                for k in range(self.maxK):
                    v[t] += np.sum(taus[s][t][k] * m[self.slot(t, k)])
            sig.append(_normalise_exp(v))
        return np.array(sig, dtype=LD)

    def evidence(self, gc, mconc, lpost, post, sigma, taus):
        r = np.sum(post * ((self.lp - lpost) + self.marginal(sigma, taus)))
        for s in range(self.S):
            r += -np.sum(_xlogx(sigma[s]))
            for t in range(self.T):
                r += sigma[s][t] * -np.sum(_xlogx(taus[s][t]))
                sl = slice(self.koff[t], self.koff[t + 1])
                r += sigma[s][t] * (_log_beta(mconc[s][sl]) - _log_beta(self.mc0[s][sl]))
            if self.lprior[s] is not None:
                with np.errstate(divide="ignore"):
                    r += _lse(np.log(sigma[s]) + self.lprior[s])
        r += _log_beta(gc) - _log_beta(self.gc0)
        return LD(r)


def run_seed(P, seed, epsilon, max_iterations, forced=None):
    lpost = np.asarray(seed, dtype=np.float64).astype(LD)
    post = np.exp(lpost)
    gc, mconc = P.gc0.copy(), P.mc0.copy()
    sigma = P.init_sigma(gc, mconc, post)
    taus = P.components(mconc, post, None)
    prev = curr = LD(LOWEST)
    decisions = []
    n = min(forced, max_iterations) if forced is not None else max_iterations
    it = 0
    for _ in range(n):
        it += 1
        u = P.lp + P.marginal(sigma, taus)
        lpost = u - _lse(u)
        post = np.exp(lpost)
        gc = P.gc0 + np.sum(sigma, axis=0)
        mconc = np.array([P.mc0[s] + np.concatenate([np.sum(taus[s][t][:P.sizes[t]], axis=1) for t in range(P.T)])
                          for s in range(P.S)], dtype=LD)
        curr = P.evidence(gc, mconc, lpost, post, sigma, taus)
        decisions.append((float(curr), float(prev)))
        stop = bool(curr <= prev or curr - prev < epsilon)
        if forced is not None and it < forced:
            stop = False
        elif forced is not None and it == forced < max_iterations:
            stop = True      # the device stopped here; at max_iterations its own decision says whether sigma and tau moved on
        if stop:
            break
        prev = curr
        sigma = P.update_sigma(gc, mconc, post, taus)
        taus = P.components(mconc, post, taus)
    return dict(lpost=lpost, post=post, group_concentrations=gc, mixture_concentrations=mconc, sigma=sigma, evidence=curr,
                iterations=it, decisions=decisions)


def combine(res):
    """compute_evidence_weighted_latents and the max-evidence seed (:42-46, :644-691)."""
    ev = [r["evidence"] for r in res]
    best = {}
    for i, r in enumerate(res):
        g = int(np.argmax(r["post"]))
        if g not in best or ev[i] > ev[best[g]]:
            best[g] = i
    modes = [best[g] for g in sorted(best)]
    me = np.array([ev[i] for i in modes], dtype=LD)
    w = np.exp(me - _lse(me))
    weighted = np.zeros_like(res[0]["post"])
    wsigma = np.zeros_like(res[0]["sigma"])
    for wi, i in zip(w, modes):
        weighted = weighted + wi * res[i]["post"]
        wsigma = wsigma + wi * res[i]["sigma"]
    mass = np.sum(weighted)
    if mass > 1:
        weighted = weighted / mass
    for s in range(wsigma.shape[0]):
        mass = np.sum(wsigma[s])
        if mass > 1:
            wsigma[s] = wsigma[s] / mass
    ms = int(np.argmax(np.array(ev, dtype=LD)))
    return dict(posteriors=res[ms]["post"], log_posteriors=res[ms]["lpost"], group_concentrations=res[ms]["group_concentrations"],
                mixture_concentrations=res[ms]["mixture_concentrations"], group_responsibilities=res[ms]["sigma"],
                weighted=weighted, weighted_group_responsibilities=wsigma, max_log_evidence=ev[ms], max_seed=ms, modes=modes)


def run(lnl, sample_off, group_sizes, combinations, genotype_log_priors, group_concentrations, mixture_concentrations, seeds,
        group_priors=None, group_prior_mask=None, epsilon=0.05, max_iterations=1000, forced=None, direct=False, quirk=True, free=None):
    """The whole call (concentrations already expanded: (T,) and (S, sum K)). forced: None, or one iteration count per seed (e.g.
    the device's) to run each seed for exactly that long. free: this call's result without `forced`, whose seeds are reused where
    they ran for their forced count (vb_exact._reuse)."""
    P = _Problem(lnl, sample_off, group_sizes, combinations, genotype_log_priors, group_concentrations, mixture_concentrations,
                 group_priors, group_prior_mask, direct, quirk)
    seeds = np.asarray(seeds, dtype=np.float64)
    res = [_reuse(free, forced, i) or run_seed(P, seeds[i], epsilon, max_iterations, None if forced is None else int(forced[i]))
           for i in range(len(seeds))]
    out = combine(res)
    out["seeds"] = res
    return out


# -- forward-error bound of one iteration -----------------------------------------------------------------------------------------
# The first-order error of a double evaluation of a one-seed call with max_iterations = 1: p = exp(seed); the initial sigma and
# tau; one genotype update (its evidence decision always continues: prev is lowest()); the concentrations; the evidence. Rules as
# in vb_exact (u = 2^-53; exp, log, lgamma within 2u relative; the project's digamma within 32u of |psi| + its recurrence terms
# + 1; a sum of n terms adds n u times the sum of their magnitudes). Step by step, d. the absolute error bound of a quantity:
#   W[j][h] = sum of p over its c_jh combinations:          dW = sum dp + c u W
#   m[j][n] = sum_h W lnl over slot j's nk_j haplotypes:     dm = sum_h dW |lnl| + (nk + 1) u sum_h W |lnl|
#   ln E[pi] of exact concentrations:                        dal = dpsi(a_k) + dpsi(a_0) + u |al|   (0 when K_t = 1)
#   x = 0 + (al + m):                                        dx = dal + dm + 2u |x|
#   tau over the maxK components, relative:                  e = 2 max_k dx + 2u (max_k |x| + |norm|) + (maxK + 4) u
#   D[s][j][h] = sum_n tau' lnl:                             dD = sum_n tau' |lnl| (e + (N_s + 2) u)
#   A = sum_n tau; mc = mc0 + A:                             dmc = sum_n tau (e + N_s u) + u mc
#   X[t] = sum_n sum_k tau ln tau:                           dX = sum tau (|1 + ln tau| e + (maxK + N_s + 3) u |ln tau|)
#   sigma's initial ln value v_t = ln E[psi] (+ ln prior) + sum_n sum_k atau_k m_k, atau the approximate tau (relative e' as e):
#                                                            dv = dpsi + sum_n sum_k atau (|m| e' + dm) + (N_s + K_t + 3) u (|.| of the terms)
#   sigma = normalise_exp(v), relative:                      es = 2 max dv + 2u (max |v| + |norm|) + (T + 4) u
#   E[j][h] = sum_s sigma D:                                 dE = sum_s (dsigma |D| + sigma dD) + (S + 1) u sum_s sigma |D|
#   v_c = lp + sum_j E[j][gt]:                               dv = sum_j dE + (K + 1) u (|lp| + sum_j |E|)
#   lpost = v - ln sum exp v; p = exp(lpost):                as vb_exact
#   gconc = gc0 + sum_s sigma:                               dg = sum_s dsigma + (S + 1) u gconc
#   the evidence: sum_c p w, w = lp - lpost + sum_j E, with dw = dlpost + sum dE + (K + 2) u (|lp| + |lpost| + sum |E|);
#       per sample the entropy of sigma, sigma_t X_t and sigma_t (logB(mc) - logB(mc0)) with vb_exact's dlogB, the prior term's
#       log-sum-exp of ln sigma (relative error es) + ln prior; logB(gconc) - logB(gc0); and (C + 4 S T + 4) u times the
#       magnitudes of the terms added.
# The returned sigma is one update further on and is not covered here; the tests hold it to the restatement within 1e-9.
# The tests allow BOUND_UNITS times this, for the second-order terms left out.
from vb_exact import BOUND_UNITS, U, _dlogbeta, _dpsi  # noqa: E402


def _dexp_bound(a):
    """ln E[.] of exact concentrations a and its error bound."""
    a = [float(v) for v in a]
    if len(a) <= 1:
        return np.zeros(len(a)), np.zeros(len(a))
    a0 = sum(a)
    al = np.array([float(mpmath.digamma(v) - mpmath.digamma(a0)) for v in a])
    d0 = _dpsi(a0, len(a) * U * a0)
    return al, np.array([_dpsi(v, 0.0) + d0 for v in a]) + U * np.abs(al)


def _normalised_rel(x, dx, axis):
    """Relative error of exp(x - lse(x)) along axis, from the absolute errors dx of x."""
    ax = np.abs(x)
    mx = np.max(x, axis=axis, keepdims=True)
    norm = np.abs(mx + np.log(np.sum(np.exp(x - mx), axis=axis, keepdims=True)))
    return 2 * np.max(dx, axis=axis) + 2 * U * (np.max(ax, axis=axis) + norm.squeeze(axis)) + (x.shape[axis] + 4) * U


def one_iteration_bound(lnl, sample_off, group_sizes, combinations, genotype_log_priors, group_concentrations,
                        mixture_concentrations, seed, group_priors=None, group_prior_mask=None):
    """Absolute error bounds (times BOUND_UNITS) of a one-seed, max_iterations = 1 call's outputs, derived above: dict of
    log_posteriors[C], posteriors[C], weighted[C], group_concentrations[T], mixture_concentrations[S][K], evidence."""
    P = _Problem(lnl, sample_off, group_sizes, combinations, genotype_log_priors, group_concentrations, mixture_concentrations,
                 group_priors, group_prior_mask, False, True)
    L = np.asarray(P.L, float)
    aL = np.abs(L)
    lp, gc0, mc0 = np.asarray(P.lp, float), np.asarray(P.gc0, float), np.asarray(P.mc0, float)
    p0L = np.exp(np.asarray(seed, dtype=np.float64).astype(LD))
    p0 = np.asarray(p0L, float)
    dp0 = 2 * U * p0
    sig = np.asarray(P.init_sigma(P.gc0, P.mc0, p0L), float)
    taus = [np.asarray(t, float) for t in P.components(P.mc0, p0L, None)]
    W, dW, nk = np.zeros((P.K, P.H)), np.zeros((P.K, P.H)), np.zeros(P.K)
    for j in range(P.K):
        c = np.bincount(P.gt[:, j], minlength=P.H)
        W[j] = np.bincount(P.gt[:, j], weights=p0, minlength=P.H)
        dW[j] = np.bincount(P.gt[:, j], weights=dp0, minlength=P.H) + c * U * W[j]
        nk[j] = np.count_nonzero(c)
    alEpsi, dEpsi = _dexp_bound(gc0)
    cmax = int(np.argmax(p0L))
    D, dD, dsig, dmc, dX, X = [], [], np.zeros((P.S, P.T)), np.zeros((P.S, P.K)), np.zeros((P.S, P.T)), np.zeros((P.S, P.T))
    for s in range(P.S):
        cols = slice(P.off[s], P.off[s + 1])
        N = P.off[s + 1] - P.off[s]
        Ls, aLs = L[:, cols], aL[:, cols]
        m, dm = W @ Ls, dW @ aLs + ((nk + 1) * U)[:, None] * (W @ aLs)
        Ds, dDs = np.zeros((P.K, P.H)), np.zeros((P.K, P.H))
        v, dv = np.zeros(P.T), np.zeros(P.T)
        for t in range(P.T):
            js = slice(P.koff[t], P.koff[t + 1])
            al, dal = _dexp_bound(mc0[s][js])
            x = np.full((P.maxK, N), float(NULL))
            dx = np.zeros((P.maxK, N))
            x[:P.sizes[t]] = al[:, None] + m[js]
            dx[:P.sizes[t]] = dal[:, None] + dm[js] + 2 * U * np.abs(x[:P.sizes[t]])
            tau = taus[s][t]
            e = _normalised_rel(x, dx, 0) if N else np.zeros(0)
            with np.errstate(divide="ignore"):
                lt = np.where(tau > 0, np.log(np.where(tau > 0, tau, 1)), 0.0)
            X[s, t] = float(np.sum(tau * lt))
            dX[s, t] = float(np.sum(tau * (np.abs(1 + lt) * e[None, :] + (P.maxK + N + 3) * U * np.abs(lt))))
            for k in range(P.sizes[t]):
                j = P.koff[t] + k
                tp = tau[k] + (tau[P.sizes[t]:].sum(axis=0) if k == 0 else 0)
                Ds[j] = Ls @ tp
                dDs[j] = aLs @ (tp * (e + (N + 2) * U))
                dmc[s, j] = float(np.sum(tau[k] * (e + N * U))) + U * (mc0[s][j] + float(np.sum(tau[k])))
            a = np.array([al[k] + Ls[P.gt[cmax, P.koff[t] + k]] for k in range(P.sizes[t])]).reshape(P.sizes[t], N)
            da = dal[:, None] + U * np.abs(a)
            lpr = float(P.lprior[s][t]) if P.lprior[s] is not None else 0.0
            v[t] = alEpsi[t] + lpr
            dv[t] = dEpsi[t] + U * (abs(alEpsi[t]) + abs(lpr))
            if N:
                at = np.exp(a - np.max(a, axis=0)) / np.sum(np.exp(a - np.max(a, axis=0)), axis=0)
                ep = _normalised_rel(a, da, 0)
                q = np.sum(at * m[js], axis=0)
                v[t] += float(np.sum(q))
                dv[t] += float(np.sum(at * (np.abs(m[js]) * ep[None, :] + dm[js]))) + \
                    (N + P.sizes[t] + 3) * U * float(np.sum(at * np.abs(m[js])))
        es = _normalised_rel(v[None, :].T, dv[None, :].T, 0)[0] if P.T > 1 else 2 * U
        dsig[s] = sig[s] * es
        D.append(Ds)
        dD.append(dDs)
    E = sum(sig[s, P.slot_t_of()][:, None] * D[s] for s in range(P.S))
    magE = sum(sig[s, P.slot_t_of()][:, None] * np.abs(D[s]) for s in range(P.S))
    dE = sum(dsig[s, P.slot_t_of()][:, None] * np.abs(D[s]) + sig[s, P.slot_t_of()][:, None] * dD[s] for s in range(P.S)) + (P.S + 1) * U * magE
    comb = np.zeros(P.C)
    dcomb = np.zeros(P.C)
    magc = np.zeros(P.C)
    for j in range(P.K):
        comb += E[j, P.gt[:, j]]
        dcomb += dE[j, P.gt[:, j]]
        magc += np.abs(E[j, P.gt[:, j]])
    v = lp + comb
    dvc = dcomb + (P.K + 1) * U * (np.abs(lp) + magc)
    norm = float(_lse(v.astype(LD)))
    lpost = v - norm
    dlpost = dvc + np.max(dvc) + (P.C + 3) * U * (abs(norm) + 1) + U * np.abs(lpost)
    post = np.exp(lpost)
    dpost = post * (dlpost + 2 * U)
    gconc = gc0 + sig.sum(axis=0)
    dg = dsig.sum(axis=0) + (P.S + 1) * U * gconc
    mc = mc0 + np.array([np.concatenate([taus[s][t][:P.sizes[t]].sum(axis=1) for t in range(P.T)]) for s in range(P.S)])
    w = lp - lpost + comb
    dw = dlpost + dcomb + (P.K + 2) * U * (np.abs(lp) + np.abs(lpost) + magc)
    dEv = float(np.sum(dpost * np.abs(w) + post * dw))
    mag = float(np.sum(np.abs(post * w)))
    for s in range(P.S):
        with np.errstate(divide="ignore"):
            ls = np.where(sig[s] > 0, np.log(np.where(sig[s] > 0, sig[s], 1)), 0.0)
        dEv += float(np.sum(np.abs(1 + ls) * dsig[s]))
        mag += float(np.sum(np.abs(sig[s] * ls)))
        for t in range(P.T):
            js = slice(P.koff[t], P.koff[t + 1])
            lb = float(_log_beta(mc[s][js].astype(LD)) - _log_beta(P.mc0[s][js]))
            dEv += dsig[s, t] * (abs(X[s, t]) + abs(lb)) + sig[s, t] * (dX[s, t] + _dlogbeta(mc[s][js], dmc[s][js], P.sizes[t]) +
                                                                     _dlogbeta(mc0[s][js], np.zeros(P.sizes[t]), P.sizes[t]))
            mag += sig[s, t] * (abs(X[s, t]) + abs(lb))
        if P.lprior[s] is not None:
            with np.errstate(divide="ignore"):
                z = np.log(sig[s]) + np.asarray(P.lprior[s], float)
            fin = np.isfinite(z)
            dEv += float(np.max(dsig[s][fin] / sig[s][fin])) + (P.T + 3) * U * (float(np.max(np.abs(z[fin]))) + 1)
            mag += float(np.max(np.abs(z[fin])))
    dEv += _dlogbeta(gconc, dg, P.T) + _dlogbeta(gc0, np.zeros(P.T), P.T)
    mag += abs(float(_log_beta(gconc.astype(LD)))) + abs(float(_log_beta(P.gc0)))
    dEv += (P.C + 4 * P.S * P.T + 4) * U * mag
    dpost_n = dpost + (P.C + 1) * U * post
    return dict(log_posteriors=BOUND_UNITS * dlpost, posteriors=BOUND_UNITS * dpost, weighted=BOUND_UNITS * dpost_n,
                group_concentrations=BOUND_UNITS * dg, mixture_concentrations=BOUND_UNITS * dmc, evidence=BOUND_UNITS * dEv)
