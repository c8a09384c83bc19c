"""The variational Bayes restatement (tests/vb_exact.py) and the engine's __host__ __device__ VB arithmetic, run on the CPU
through tests/cpu_emul/vb_emul.cu, held to each other; no GPU needed."""
import ctypes as C

import mpmath
import numpy as np
import pytest

import vb_cases
import vb_exact

vp = C.c_void_p
REL = 1e-9      # chosen: double against long double over up to a few hundred iterations of sums of up to 10^4 terms


@pytest.fixture(scope="module")
def emul():
    from octopus_b200.build import build_vb_emulation
    lib = C.CDLL(build_vb_emulation())
    lib.emul_vb_seed.restype = C.c_double
    lib.emul_vb_seed.argtypes = [vp, C.c_int, C.c_int, vp, C.c_int, vp, C.c_int, C.c_int, vp, vp, vp, C.c_double, C.c_int, vp, vp, vp]
    lib.emul_vb_digamma.restype = C.c_double
    lib.emul_vb_digamma.argtypes = [C.c_double]
    return lib


def _emul_seed(lib, lnl, off, gt, prior, lp, seed, eps, max_it):
    H, R = lnl.shape
    G, K = gt.shape
    S = len(off) - 1
    lnl, gt, prior, lp, seed = (np.ascontiguousarray(x) for x in (lnl, gt, prior, lp, seed))
    soff = np.ascontiguousarray(off, dtype=np.int32)
    lpost, alpha, it = np.empty(G), np.empty((S, K)), C.c_int(0)
    ev = lib.emul_vb_seed(lnl.ctypes.data, H, R, soff.ctypes.data, S, gt.ctypes.data, G, K, prior.ctypes.data, lp.ctypes.data,
                          seed.ctypes.data, eps, max_it, lpost.ctypes.data, alpha.ctypes.data, C.byref(it))
    return dict(lpost=lpost, alphas=alpha, evidence=ev, iterations=it.value)


@pytest.mark.parametrize("x", [1e-300, 1e-8, 0.3, 1.0, 2.5, 5.999, 6.0, 7.5, 40.0, 1e6, 1e300, -0.5, -2.75])
def test_digamma_matches_mpmath(emul, x):
    want = float(mpmath.digamma(mpmath.mpf(x)))
    tol = 2e-15 if x > 0 else 1e-14     # the recurrence's ten or so roundings; the reflection's cancellation near a pole
    assert abs(emul.emul_vb_digamma(x) - want) <= tol * max(abs(want), 1.0), (x, emul.emul_vb_digamma(x), want)


def test_grouped_form_equals_the_genotype_indexed_form():
    lnl, off, gt, prior, lp, seeds = vb_cases.make(5, [7, 0, 4], 9, 3, 3, seed=1, dup=True)
    a = vb_exact.run(lnl, off, gt, prior, lp, seeds, 0.05, 50, direct=True)
    b = vb_exact.run(lnl, off, gt, prior, lp, seeds, 0.05, 50, direct=False)
    for sa, sb in zip(a["seeds"], b["seeds"]):
        assert sa["iterations"] == sb["iterations"]
        assert np.allclose(np.asarray(sa["lpost"], float), np.asarray(sb["lpost"], float), rtol=1e-15, atol=1e-15)
        assert abs(float(sa["evidence"]) - float(sb["evidence"])) <= 1e-14 * abs(float(sa["evidence"]))


def test_restatement_follows_the_loop_order():
    """One iteration by hand: posteriors start as exp(seed) unnormalised and the responsibilities from the prior alphas."""
    lnl, off, gt, prior, lp, seeds = vb_cases.make(3, [5], 4, 2, 1, seed=2)
    seeds = seeds + 0.3                      # an unnormalised seed must be used as it is
    r = vb_exact.run(lnl, off, gt, prior, lp, seeds, 0.05, 1)["seeds"][0]
    P = vb_exact._Problem(lnl, off, gt, prior, lp, True)
    taus, _ = P.responsibilities(P.prior, np.exp(np.asarray(seeds[0], dtype=vb_exact.LD)))
    u = P.lp + P.marginal_genotypes(taus[0], 0)
    want = u - vb_exact._lse(u)
    assert np.allclose(np.asarray(r["lpost"], float), np.asarray(want, float), rtol=1e-15, atol=1e-15)
    assert r["iterations"] == 1


@pytest.mark.parametrize("case", [
    dict(H=4, reads=[30], G=6, K=1, n_seeds=2, max_it=1000, eps=0.05),
    dict(H=6, reads=[40, 0], G=12, K=2, n_seeds=3, max_it=1000, eps=0.05),
    dict(H=8, reads=[25, 17, 3], G=20, K=3, n_seeds=4, max_it=1000, eps=0.0, dup=True),
    dict(H=5, reads=[33], G=10, K=4, n_seeds=10, max_it=2, eps=0.05),
    dict(H=5, reads=[12, 9], G=8, K=8, n_seeds=2, max_it=1000, eps=1e9),
])
def test_emulation_matches_the_restatement(emul, case):
    lnl, off, gt, prior, lp, seeds = vb_cases.make(case["H"], case["reads"], case["G"], case["K"], case["n_seeds"], seed=3,
                                                   dup=case.get("dup", False))
    want = vb_exact.run(lnl, off, gt, prior, lp, seeds, case["eps"], case["max_it"])
    flagged = 0
    for i, ws in enumerate(want["seeds"]):
        got = _emul_seed(emul, lnl, off, gt, prior, lp, seeds[i], case["eps"], case["max_it"])
        if got["iterations"] != ws["iterations"]:
            assert vb_exact.near_threshold(ws["decisions"], case["eps"]), (i, got["iterations"], ws["iterations"])
            flagged += 1
            continue
        assert np.allclose(got["lpost"], np.asarray(ws["lpost"], float), rtol=REL, atol=REL)
        assert np.allclose(got["alphas"], np.asarray(ws["alphas"], float), rtol=REL)
        assert abs(got["evidence"] - float(ws["evidence"])) <= REL * max(1.0, abs(float(ws["evidence"])))
    if case["eps"] > 0:      # with epsilon 0 every seed stops where its ELBO stalls at rounding level: always near the threshold
        assert flagged < len(seeds)


BOUND_CASES = [(40, [1], 2000, 2), (16, [257, 40], 300, 3), (10, [256], 20, 100), (8, [300], 50, 8)]


@pytest.mark.parametrize("case", BOUND_CASES, ids=lambda c: "H%d R%s G%d K%d" % c)
def test_emulation_within_the_one_iteration_bound(emul, case):
    """With max_iterations = 1 the emulated cores (sequential sums) stay within vb_exact.one_iteration_bound."""
    H, reads, G, K = case
    lnl, off, gt, prior, lp, seeds = vb_cases.make(H, reads, G, K, 1, seed=11)
    bound = vb_exact.one_iteration_bound(lnl, off, gt, prior, lp, seeds[0])
    want = vb_exact.run(lnl, off, gt, prior, lp, seeds, 0.05, 1)["seeds"][0]
    got = _emul_seed(emul, lnl, off, gt, prior, lp, seeds[0], 0.05, 1)
    for name, g, w, b in (("log posteriors", got["lpost"], want["lpost"], bound["log_posteriors"]),
                          ("alphas", got["alphas"], want["alphas"], bound["alphas"]),
                          ("evidence", [got["evidence"]], [want["evidence"]], [bound["evidence"]])):
        ratio = float(np.max(np.abs(np.asarray(g, float) - np.asarray(w, float)) / np.asarray(b, float)))
        print("%s %s: error / bound %.3g" % (case, name, ratio))
        assert ratio <= 1.0, (name, ratio)
