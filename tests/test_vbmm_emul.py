"""The mixture-of-mixtures restatement (tests/vbmm_exact.py) and the engine's __host__ __device__ arithmetic of
phmm_vb_mm.cuh, run on the CPU through tests/cpu_emul/vbmm_emul.cu, held to each other; no GPU needed."""
import ctypes as C

import numpy as np
import pytest

import vbmm_cases
import vbmm_exact

vp = C.c_void_p
REL = 1e-9      # chosen, as the GPU tests choose it: double against long double over a few tens of iterations


@pytest.fixture(scope="module")
def emul():
    from octopus_b200.build import build_vbmm_emulation
    lib = C.CDLL(build_vbmm_emulation())
    lib.emul_vbmm_seed.restype = C.c_double
    lib.emul_vbmm_seed.argtypes = [vp, C.c_int, C.c_int, vp, C.c_int, vp, C.c_int, vp, C.c_int] + [vp] * 6 + \
                                  [C.c_double, C.c_int] + [vp] * 5
    return lib


def _emul_seed(lib, x, i, eps, max_it):
    lnl, gt = np.ascontiguousarray(x["lnl"]), np.ascontiguousarray(x["gt"], dtype=np.int32)
    H, R = lnl.shape
    Cn, K = gt.shape
    soff = np.ascontiguousarray(x["off"], dtype=np.int32)
    S, T = len(soff) - 1, len(x["sizes"])
    sizes = np.ascontiguousarray(x["sizes"], dtype=np.int32)
    lp, gc, mc = (np.ascontiguousarray(v, dtype=np.float64) for v in (x["lp"], x["gc"], x["mc"]))
    seed = np.ascontiguousarray(x["seeds"][i], dtype=np.float64)
    gp = None if x["gp"] is None else np.ascontiguousarray(x["gp"], dtype=np.float64)
    has = np.ascontiguousarray(np.ones(S) if x["mask"] is None else x["mask"], dtype=np.int32)
    lpost, gco, mco, sig, it = np.empty(Cn), np.empty(T), np.empty((S, K)), np.empty((S, T)), C.c_int(0)
    ev = lib.emul_vbmm_seed(lnl.ctypes.data, H, R, soff.ctypes.data, S, sizes.ctypes.data, T, gt.ctypes.data, Cn, lp.ctypes.data,
                            None if gp is None else gp.ctypes.data, has.ctypes.data, gc.ctypes.data, mc.ctypes.data, seed.ctypes.data,
                            eps, max_it, lpost.ctypes.data, gco.ctypes.data, mco.ctypes.data, sig.ctypes.data, C.byref(it))
    return dict(lpost=lpost, group_concentrations=gco, mixture_concentrations=mco, sigma=sig, evidence=ev, iterations=it.value)


CASES = [
    dict(H=6, reads=[7, 0, 5, 1, 9], sizes=[2, 2], C=40, n_seeds=3),
    dict(H=6, reads=[7, 0, 5, 1, 9], sizes=[1, 2, 3], C=40, n_seeds=3, priors="some", conc="full"),
    dict(H=5, reads=[3, 12, 0, 4], sizes=[2, 2, 2, 2, 2], C=30, n_seeds=3, priors="some"),
    dict(H=8, reads=[20, 1, 0, 33, 6], sizes=[1, 3], C=60, n_seeds=3, max_it=1),
    dict(H=8, reads=[12, 9, 4], sizes=[2, 2, 2], C=50, n_seeds=3, max_it=2, dup=True),
    dict(H=7, reads=[10, 10], sizes=[1, 2, 2], C=40, n_seeds=3, lowest=3),
    dict(H=5, reads=[12, 9], sizes=[3, 1], C=20, n_seeds=2, eps=1e9),
]


@pytest.mark.parametrize("case", CASES, ids=lambda c: "K%s reads%s" % (c["sizes"], c["reads"]))
def test_emulation_matches_the_restatement(emul, case):
    x = vbmm_cases.make(case["H"], case["reads"], case["sizes"], case["C"], case["n_seeds"], seed=3, dup=case.get("dup", False),
                        lowest=case.get("lowest", 0), priors=case.get("priors"), concentrations=case.get("conc", "scalar"))
    eps, max_it = case.get("eps", 0.05), case.get("max_it", 1000)
    want = vbmm_exact.run(x["lnl"], x["off"], x["sizes"], x["gt"], x["lp"], x["gc"], x["mc"], x["seeds"], x["gp"], x["mask"], eps, max_it)
    flagged = 0
    for i, ws in enumerate(want["seeds"]):
        got = _emul_seed(emul, x, i, eps, max_it)
        if got["iterations"] != ws["iterations"]:
            assert vbmm_exact.near_threshold(ws["decisions"], eps), (i, got["iterations"], ws["iterations"])
            flagged += 1
            continue
        for key, g, w in (("lpost", got["lpost"], ws["lpost"]), ("sigma", got["sigma"], ws["sigma"]),
                          ("group concentrations", got["group_concentrations"], ws["group_concentrations"]),
                          ("mixture concentrations", got["mixture_concentrations"], ws["mixture_concentrations"])):
            w = np.asarray(w, float)
            assert np.allclose(g, w, rtol=REL, atol=REL), (key, i, float(np.max(np.abs(g - w))))
        assert abs(got["evidence"] - float(ws["evidence"])) <= REL * max(1.0, abs(float(ws["evidence"])))
    assert flagged < len(x["seeds"])


BOUND_CASES = [dict(H=8, reads=[20, 1, 0, 33, 6], sizes=[1, 3], C=60), dict(H=6, reads=[7, 0, 5, 1, 9], sizes=[1, 2, 3], C=40, priors="some"),
               dict(H=10, reads=[4] * 30, sizes=[2, 2, 2], C=300), dict(H=5, reads=[12, 9], sizes=[2, 2, 2, 2, 2], C=30, conc="full")]


@pytest.mark.parametrize("case", BOUND_CASES, ids=lambda c: "K%s S%d C%d" % (c["sizes"], len(c["reads"]), c["C"]))
def test_emulation_within_the_one_iteration_bound(emul, case):
    """With max_iterations = 1 the emulated arithmetic (sequential sums) stays within vbmm_exact.one_iteration_bound."""
    x = vbmm_cases.make(case["H"], case["reads"], case["sizes"], case["C"], 1, seed=11, priors=case.get("priors"),
                        concentrations=case.get("conc", "scalar"))
    bound = vbmm_exact.one_iteration_bound(x["lnl"], x["off"], x["sizes"], x["gt"], x["lp"], x["gc"], x["mc"], x["seeds"][0], x["gp"], x["mask"])
    want = vbmm_exact.run(x["lnl"], x["off"], x["sizes"], x["gt"], x["lp"], x["gc"], x["mc"], x["seeds"], x["gp"], x["mask"], 0.05, 1)["seeds"][0]
    got = _emul_seed(emul, x, 0, 0.05, 1)
    for name, g, w, b in (("log posteriors", got["lpost"], want["lpost"], bound["log_posteriors"]),
                          ("group concentrations", got["group_concentrations"], want["group_concentrations"], bound["group_concentrations"]),
                          ("mixture concentrations", got["mixture_concentrations"], want["mixture_concentrations"], bound["mixture_concentrations"]),
                          ("evidence", [got["evidence"]], [want["evidence"]], [bound["evidence"]])):
        ratio = float(np.max(np.abs(np.asarray(g, float) - np.asarray(w, float)) / np.maximum(np.asarray(b, float), 1e-320)))
        print("%s %s: error / bound %.3g" % (case["sizes"], name, ratio))
        assert ratio <= 1.0, (name, ratio)
