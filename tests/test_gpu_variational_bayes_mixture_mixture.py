"""phmm_variational_bayes_mixture_mixture (PairHMMEngine.variational_bayes_mixture_mixture): SingleCellModel's mixture-of-mixtures
variational Bayes inference on the device, every seed in one call, held to the long-double restatement tests/vbmm_exact.py run
for the device's own per-seed iteration counts.

A seed whose iteration count differs from the restatement's is accepted only when one of the restatement's stopping decisions lies
within rounding of epsilon or of 0 (vb_exact.near_threshold); such seeds are counted as flagged and their values are not compared.
Tolerances are chosen, not derived: posteriors within ABS absolutely, everything else within REL relatively."""
import numpy as np
import pytest

import vbmm_cases
import vbmm_exact

pytestmark = pytest.mark.gpu

DEV = "cuda:0"
ABS = 1e-9
REL = 1e-9
SPIN_CYCLES = 400_000_000
FIELDS = ["genotype_posteriors", "genotype_log_posteriors", "group_concentrations", "mixture_concentrations", "group_responsibilities",
          "max_log_evidence", "weighted_genotype_posteriors", "weighted_group_responsibilities", "max_seed", "seed_log_evidences",
          "seed_iterations"]


def _np(x):
    return x.cpu().numpy() if hasattr(x, "cpu") else np.asarray(x)


def _bits(x):
    if isinstance(x, (int, float)):
        x = np.int32(x) if isinstance(x, int) else np.float64(x)
    return np.ascontiguousarray(_np(x)).view(np.uint8)


def _cells(S, mean, rng):
    """S cells of about `mean` reads, a few with none and a few with one."""
    r = rng.poisson(mean, size=S)
    r[::17] = 0
    r[5::19] = 1
    return [int(v) for v in r]


_rng = np.random.default_rng(7)
CASES = {
    "S1 T2 K[2,2] C1 one seed": dict(H=3, reads=[40], sizes=[2, 2], C=1, n_seeds=1),
    "S200 T3 K[2,2,2] C1000 12 seeds cells": dict(H=20, reads=_cells(200, 20, _rng), sizes=[2, 2, 2], C=1000, n_seeds=12),
    "S40 T3 K[1,2,3] C1000 propose_seeds priors": dict(H=20, reads=_cells(40, 20, _rng), sizes=[1, 2, 3], C=1000, n_seeds=12,
                                                        propose=True, priors="some", conc="full"),
    "S300 T2 K[2,2] C300 cells two iterations": dict(H=12, reads=_cells(300, 8, _rng), sizes=[2, 2], C=300, n_seeds=12, max_it=2),
    "S8 T5 K[2,2,2,2,2] C200 dup eps 0": dict(H=10, reads=_cells(8, 15, _rng), sizes=[2, 2, 2, 2, 2], C=200, n_seeds=4, eps=0.0, dup=True),
    "S6 T4 K[30,30,30,10] C50 sum K 100": dict(H=16, reads=[30, 0, 12, 1, 25, 9], sizes=[30, 30, 30, 10], C=50, n_seeds=3),
    "S4 T2 K[1,3] C20000 one iteration": dict(H=40, reads=[20, 0, 1, 30], sizes=[1, 3], C=20000, n_seeds=2, max_it=1),
    "S10 T3 K[2,2,2] C100 eps 1e9": dict(H=8, reads=_cells(10, 10, _rng), sizes=[2, 2, 2], C=100, n_seeds=12, eps=1e9),
    "S12 T3 K[1,2,2] C60 lowest entries": dict(H=10, reads=_cells(12, 10, _rng), sizes=[1, 2, 2], C=60, n_seeds=6, lowest=4),
}


def _inputs(c, seed=11):
    x = vbmm_cases.make(c["H"], c["reads"], c["sizes"], c["C"], c["n_seeds"], seed=seed, dup=c.get("dup", False),
                        lowest=c.get("lowest", 0), priors=c.get("priors"), concentrations=c.get("conc", "scalar"))
    if c.get("propose"):
        x["seeds"] = vbmm_cases.propose_seeds(c["C"], c["n_seeds"])
    return x


def _call(engine, x, eps, max_it, conv=lambda a: a):
    return engine.variational_bayes_mixture_mixture(conv(x["lnl"]), x["sizes"], conv(x["gt"]), conv(x["lp"]), conv(x["gc"]), conv(x["mc"]),
                                                    conv(x["seeds"]), x["off"], None if x["gp"] is None else conv(x["gp"]), x["mask"],
                                                    eps, max_it)


def _exact(x, eps, max_it, forced=None, free=None):
    return vbmm_exact.run(x["lnl"], x["off"], x["sizes"], x["gt"], x["lp"], x["gc"], x["mc"], x["seeds"], x["gp"], x["mask"],
                          eps, max_it, forced=forced, free=free)


def _rel(got, want):
    got, want = np.asarray(_np(got), float), np.asarray(want, float)
    fin = np.isfinite(want)
    assert np.array_equal(np.isfinite(got), fin)
    return float(np.max(np.abs(got[fin] - want[fin]) / (REL * np.maximum(1.0, np.abs(want[fin]))), initial=0.0))


def _compare(got, x, eps, max_it, name):
    iters = _np(got.seed_iterations)
    free = _exact(x, eps, max_it)
    want = _exact(x, eps, max_it, forced=iters, free=free)
    flagged = 0
    ratios = {"evidences": 0.0}
    for i, ws in enumerate(want["seeds"]):
        if free["seeds"][i]["iterations"] != iters[i]:
            assert vbmm_exact.near_threshold(free["seeds"][i]["decisions"], eps), (name, i, iters[i], free["seeds"][i]["iterations"])
            flagged += 1
            continue
        ratios["evidences"] = max(ratios["evidences"], _rel([_np(got.seed_log_evidences)[i]], [float(ws["evidence"])]))
    assert int(_np(got.max_seed)) == want["max_seed"] or flagged, (name, int(_np(got.max_seed)), want["max_seed"])
    ratios["posteriors"] = float(np.max(np.abs(_np(got.genotype_posteriors) - np.asarray(want["posteriors"], float)))) / ABS
    ratios["weighted"] = float(np.max(np.abs(_np(got.weighted_genotype_posteriors) - np.asarray(want["weighted"], float)))) / ABS
    ratios["log posteriors"] = _rel(got.genotype_log_posteriors, want["log_posteriors"])
    ratios["group concentrations"] = _rel(got.group_concentrations, want["group_concentrations"])
    ratios["mixture concentrations"] = _rel(got.mixture_concentrations, want["mixture_concentrations"])
    ratios["sigma"] = _rel(got.group_responsibilities, want["group_responsibilities"])
    ratios["weighted sigma"] = _rel(got.weighted_group_responsibilities, want["weighted_group_responsibilities"])
    print("%s: flagged %d of %d seeds; largest error / tolerance: %s" % (name, flagged, len(iters),
                                                                         ", ".join("%s %.3g" % kv for kv in ratios.items())))
    assert all(r <= 1.0 for r in ratios.values()), (name, ratios)


@pytest.mark.parametrize("name", list(CASES))
def test_matches_the_restatement(engine, name):
    c = CASES[name]
    x = _inputs(c)
    got = _call(engine, x, c.get("eps", 0.05), c.get("max_it", 1000))
    _compare(got, x, c.get("eps", 0.05), c.get("max_it", 1000), name)


def test_a_padded_component_takes_a_whole_read(engine):
    """Group 0 has one component and group 1 two, so group 0 has a padded one. Read 1's only real likelihood in group 0 is
    lowest(): its ln rho lies below -10000 and the padded component takes its whole responsibility, which then enters the genotype
    update through hap(c, 0, 0)."""
    lnl = np.array([[-1.0, vbmm_cases.LOWEST, -2.0], [-2.0, -3.0, -0.5], [-4.0, -1.0, -1.5]])
    gt = np.array([[0, 0, 1], [0, 1, 2], [0, 2, 2]], np.int32)
    x = dict(lnl=lnl, off=np.array([0, 3]), sizes=[1, 2], gt=gt, lp=np.log(np.full(3, 1 / 3)), gc=np.ones(2), mc=np.ones((1, 3)),
             seeds=np.log(np.full((2, 3), 1 / 3)), gp=None, mask=None)
    x["seeds"][1] = np.log([0.8, 0.1, 0.1])
    P = vbmm_exact._Problem(lnl, x["off"], x["sizes"], gt, x["lp"], x["gc"], x["mc"], None, None, False, True)
    taus = P.components(P.mc0, np.exp(np.asarray(x["seeds"][0]).astype(vbmm_exact.LD)), None)
    assert float(taus[0][0][1][1]) == 1.0
    _compare(_call(engine, x, 0.05, 1000), x, 0.05, 1000, "padded component")


def _agrees_with_reference(got, x, eps, max_it, name):
    """One call's result against the reference's (vbmm_ref.RefVBMM): iteration counts equal (seeds the restatement flags aside),
    weighted posteriors, weighted sigma and max evidence within the float tolerances measured on the CPU (tests/test_vbmm_ref.py).
    Returns False, having compared only the iteration counts, when the restatement flags a seed."""
    from test_vbmm_ref import EVIDENCE_REL, SIGMA_ABS, WEIGHTED_ABS
    from vbmm_ref import RefVBMM
    r = RefVBMM().run(x["lnl"], x["off"], x["sizes"], x["gt"], x["lp"], x["gc"], x["mc"], x["seeds"], x["gp"], x["mask"], eps, max_it)
    free = _exact(x, eps, max_it)
    flagged = [vbmm_exact.near_threshold(s["decisions"], eps, rel=1e-6) for s in free["seeds"]]
    its = _np(got.seed_iterations)
    for i in range(len(its)):
        assert its[i] == r["seed_iterations"][i] or flagged[i], (name, i, its[i], r["seed_iterations"][i])
    if any(flagged):
        return False
    w = float(np.max(np.abs(_np(got.weighted_genotype_posteriors) - r["weighted"]))) / WEIGHTED_ABS
    sg = float(np.max(np.abs(_np(got.weighted_group_responsibilities) - r["weighted_group_responsibilities"]))) / SIGMA_ABS
    e = abs(float(_np(got.max_log_evidence)) - r["max_log_evidence"]) / (EVIDENCE_REL * abs(r["max_log_evidence"]))
    print("%s: device vs reference, error / tolerance: weighted %.3g, weighted sigma %.3g, max evidence %.3g" % (name, w, sg, e))
    assert w <= 1 and sg <= 1 and e <= 1, (name, w, sg, e)
    return True


def test_device_agrees_with_the_reference(engine):
    """The device against the UNMODIFIED reference (oracle/_ref/libref_vbmm.so) on the cases without lowest() entries small
    enough for it (_agrees_with_reference)."""
    from vbmm_ref import RefVBMM
    if not RefVBMM.available():
        pytest.skip("reference mixture-of-mixtures VB not built (oracle/_ref/libref_vbmm.so)")
    checked = 0
    for name, c in CASES.items():
        if c.get("lowest") or c["C"] * sum(c["reads"]) * sum(c["sizes"]) > 3_000_000:
            continue
        x = _inputs(c)
        eps, max_it = c.get("eps", 0.05), c.get("max_it", 1000)
        checked += _agrees_with_reference(_call(engine, x, eps, max_it), x, eps, max_it, name)
    assert checked >= 3


@pytest.mark.parametrize("name", ["S200 T3 K[2,2,2] C1000 12 seeds cells", "S40 T3 K[1,2,3] C1000 propose_seeds priors"])
def test_host_and_device_space_give_the_same_bits_every_run(engine, name):
    import torch
    c = CASES[name]
    x = _inputs(c)
    host = _call(engine, x, c.get("eps", 0.05), c.get("max_it", 1000))
    dev = [_call(engine, x, c.get("eps", 0.05), c.get("max_it", 1000), lambda a: torch.as_tensor(a, device=DEV)) for _ in range(2)]
    for f in FIELDS:
        for d in dev:
            assert np.array_equal(_bits(getattr(host, f)), _bits(getattr(d, f))), f


def test_populated_multi_sample_region(engine):
    """The matrix populate leaves on the device, its columns split into cells, through HaplotypeLikelihoodArray."""
    import torch
    from octopus_b200 import HaplotypeLikelihoodArray, HaplotypeLikelihoodModel, synth
    haps, reads, band = synth.make_batch("C2", n_reads=600)
    cfg = HaplotypeLikelihoodModel.Config(max_indel_error=band)
    arr = HaplotypeLikelihoodArray(engine=engine)
    arr.likelihoods = engine.populate(cfg, haps.to_device(DEV), reads.to_device(DEV))
    widths = [0, 1] + [25] * ((reads.n - 1) // 25)
    widths.append(reads.n - sum(widths))
    names = ["cell%d" % i for i in range(len(widths))]
    arr._set_samples(names, widths)
    assert isinstance(arr.likelihoods, torch.Tensor)
    H = haps.n
    genotypes = [(a, b) for a in range(H) for b in range(a, H)]
    gt = vbmm_cases.combinations_of(genotypes, 2)[:1000]
    lp = np.log(np.full(len(gt), 1.0 / len(gt)))
    seeds = vbmm_cases.propose_seeds(len(gt), 12)
    got = arr.variational_bayes_mixture_mixture(names, [2, 2], gt, lp, 1.0, 1.5, seeds)
    assert got.genotype_posteriors.device.type == "cuda"
    S = len(names)
    x = dict(lnl=arr.likelihoods.cpu().numpy(), off=np.concatenate([[0], np.cumsum(widths)]), sizes=[2, 2], gt=gt, lp=lp,
             gc=np.ones(2), mc=np.full((S, 4), 1.5), seeds=seeds, gp=None, mask=None)
    _compare(got, x, 0.05, 1000, "populated C2 cells")


def _bad_args():
    rng = np.random.default_rng(1)
    return dict(lnl=-rng.uniform(0, 10, (5, 10)), sizes=[2, 1], gt=rng.integers(0, 5, (3, 3)).astype(np.int32), lp=np.log(np.full(3, 1 / 3)),
                gc=np.ones(2), mc=np.ones((2, 3)), seeds=np.log(np.full((2, 3), 1 / 3)), off=[0, 4, 10], max_it=10)


BAD = {
    "T 0": lambda a: a.update(sizes=[], gt=np.zeros((3, 0), np.int32), gc=np.ones(0), mc=np.ones((2, 0))),
    "T 33": lambda a: a.update(sizes=[1] * 33, gt=np.zeros((3, 33), np.int32), gc=np.ones(33), mc=np.ones((2, 33))),
    "K_t 0": lambda a: a.update(sizes=[3, 0]),
    "K_t 101": lambda a: a.update(sizes=[101], gt=np.zeros((3, 101), np.int32), gc=np.ones(1), mc=np.ones((2, 101))),
    "sum K 101": lambda a: a.update(sizes=[51, 50], gt=np.zeros((3, 101), np.int32), mc=np.ones((2, 101))),
    "max_iterations 0": lambda a: a.update(max_it=0),
    "no seeds": lambda a: a.update(seeds=np.zeros((0, 3))),
    "no combinations": lambda a: a.update(gt=np.zeros((0, 3), np.int32), lp=np.zeros(0), seeds=np.zeros((2, 0))),
    "sample_off not from 0": lambda a: a.update(off=[1, 4, 10]),
    "sample_off not to R": lambda a: a.update(off=[0, 4, 9]),
    "sample_off decreasing": lambda a: a.update(off=[0, 6, 4, 10], mc=np.ones((3, 3))),
    "no samples": lambda a: a.update(off=[0], mc=np.ones((0, 3)), lnl=np.zeros((5, 0))),
    "H 50001": lambda a: a.update(lnl=np.zeros((50001, 1)), off=[0, 1], mc=np.ones((1, 3))),
    "index H": lambda a: a["gt"].__setitem__((1, 1), 5),
    "index -1": lambda a: a["gt"].__setitem__((2, 2), -1),
}


@pytest.mark.parametrize("space", ["host", "device"])
@pytest.mark.parametrize("what", list(BAD))
def test_refused(engine, what, space):
    import torch
    from octopus_b200 import PhmmError
    a = _bad_args()
    BAD[what](a)
    conv = (lambda v: torch.as_tensor(v, device=DEV)) if space == "device" else (lambda v: v)
    with pytest.raises((PhmmError, ValueError)) as ei:
        engine.variational_bayes_mixture_mixture(conv(a["lnl"]), a["sizes"], conv(a["gt"]), conv(a["lp"]), conv(a["gc"]), conv(a["mc"]),
                                                 conv(a["seeds"]), a["off"], max_iterations=a["max_it"])
    if isinstance(ei.value, PhmmError):
        assert ei.value.code == -1
    ok = _bad_args()      # the engine still works after a refusal
    r = engine.variational_bayes_mixture_mixture(ok["lnl"], ok["sizes"], ok["gt"], ok["lp"], ok["gc"], ok["mc"], ok["seeds"], ok["off"],
                                                 max_iterations=ok["max_it"])
    assert np.isfinite(r.max_log_evidence)


@pytest.mark.parametrize("side", [False, True])
def test_device_call_orders_after_the_callers_busy_stream(engine, side):
    """Seeds written on torch's current stream behind a spin, passed as float32 so that the call converts them there: the engine
    must read them only after the conversion."""
    import torch
    c = CASES["S40 T3 K[1,2,3] C1000 propose_seeds priors"]
    x = _inputs(c)
    x["seeds"] = np.log(np.random.default_rng(3).dirichlet(np.ones(c["C"]), size=6) + 1e-30).astype(np.float32).astype(np.float64)
    want = _call(engine, x, 0.05, 1000)
    stream = torch.cuda.Stream(DEV) if side else torch.cuda.current_stream(DEV)
    with torch.cuda.stream(stream):
        d = {k: (torch.as_tensor(v, device=DEV) if isinstance(v, np.ndarray) and k not in ("off", "mask") else v) for k, v in x.items()}
        src = torch.as_tensor(x["seeds"].astype(np.float32), device=DEV)
        s32 = torch.zeros_like(src)
        torch.cuda._sleep(SPIN_CYCLES)
        s32.copy_(src)
        assert not torch.cuda.current_stream().query(), "the spin ended before the call, which then tests no ordering"
        d["seeds"] = s32
        got = _call(engine, d, 0.05, 1000)
        for f in FIELDS:
            assert np.array_equal(_bits(getattr(got, f)), _bits(getattr(want, f))), f
    torch.cuda.synchronize(DEV)


def test_scalar_concentrations_expand_on_the_device(engine):
    """A 0-d group concentration and per-sample mixture concentrations as device tensors give the bits of their expansion."""
    import torch
    c = CASES["S40 T3 K[1,2,3] C1000 propose_seeds priors"]
    x = _inputs(c)
    per_sample = np.random.default_rng(2).uniform(0.5, 3.0, size=len(x["off"]) - 1)
    want = _call(engine, dict(x, gc=np.full(3, 1.5), mc=np.repeat(per_sample[:, None], 6, axis=1)), 0.05, 1000)
    conv = lambda a: torch.as_tensor(a, device=DEV)
    got = _call(engine, dict(x, gc=np.float64(1.5), mc=per_sample), 0.05, 1000, conv)
    for f in FIELDS:
        assert np.array_equal(_bits(getattr(got, f)), _bits(getattr(want, f))), f


def test_cpp_adapter_matches_the_python_api(engine):
    """octopus_b200::VariationalBayesMixtureMixtureModel (the C++ adapter) over a populated four-cell array gives the bits the
    Python API gives on the same matrix; its scalar overloads expand as the general one; a refusal surfaces as Error."""
    import os
    import subprocess
    import tempfile
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    exe = os.path.join(tempfile.mkdtemp(prefix="test_vbmm_"), "test_vbmm")
    subprocess.run(["g++", "-std=c++14", "-O1", "-I", os.path.join(root, "include"), "-I", os.path.join(root, "octopus_b200", "cpp"),
                    os.path.join(root, "tests", "cpp", "test_vbmm.cpp"), "-o", exe, "-L", os.path.join(root, "octopus_b200"), "-lphmm_b200",
                    "-Wl,-rpath," + os.path.join(root, "octopus_b200")], check=True)
    out = subprocess.run([exe], capture_output=True, text=True, timeout=120)
    assert out.returncode == 0, out.stdout + out.stderr
    rows = {l.split()[0]: l.split()[1:] for l in out.stdout.strip().splitlines()}
    H, R = int(rows["MATRIX"][0]), int(rows["MATRIX"][1])
    lnl = np.array([float(v) for v in rows["MATRIX"][2:]]).reshape(H, R)
    widths = [int(v) for v in rows["WIDTHS"]]
    genotypes = [[0], [1], [2], [0, 0], [0, 1], [0, 2], [1, 2]]
    gt = np.array([genotypes[a] + genotypes[b] for a in range(3) for b in range(3, 7)], np.int32)
    lp = np.full(12, -2.4849066497880004)
    seeds = [np.full(12, -2.4849066497880004)]
    for i in range(3):
        seeds.append(np.full(12, -11.608235644774552))
        seeds[-1][i] = -0.00010000500033334732
    gp = np.zeros((4, 2))
    gp[1] = [0.7, 0.3]
    want = engine.variational_bayes_mixture_mixture(lnl, [1, 2], gt, lp, 1.0, 0.8, np.array(seeds), np.concatenate([[0], np.cumsum(widths)]),
                                                    gp, np.array([0, 1, 0, 0]))
    got = lambda k: np.array([float(v) for v in rows[k]])
    for key, f in (("POST", "genotype_posteriors"), ("LPOST", "genotype_log_posteriors"), ("GCONC", "group_concentrations"),
                   ("MCONC", "mixture_concentrations"), ("SIGMA", "group_responsibilities"), ("WEIGHTED", "weighted_genotype_posteriors"),
                   ("WSIGMA", "weighted_group_responsibilities")):
        assert np.array_equal(_bits(got(key)), _bits(np.ravel(getattr(want, f)))), key
    assert np.array_equal(_bits(got("EVIDENCE")), _bits(np.array([want.max_log_evidence])))
    assert rows["EXPANSION"] == ["yes"]
    assert rows["REFUSED"] == ["yes"]


ONE_ITERATION = {
    "S5 T2 K[1,3] C20000": dict(H=40, reads=[20, 1, 0, 33, 6], sizes=[1, 3], C=20000),
    "S200 T3 K[2,2,2] C1000 cells": dict(H=20, reads=_cells(200, 20, np.random.default_rng(3)), sizes=[2, 2, 2], C=1000),
    "S5 T3 K[1,2,3] C40 priors": dict(H=6, reads=[7, 0, 5, 1, 9], sizes=[1, 2, 3], C=40, priors="some"),
}


@pytest.mark.parametrize("name", list(ONE_ITERATION))
def test_one_iteration_within_the_derived_bound(engine, name):
    """max_iterations = 1, one seed: every output vbmm_exact.one_iteration_bound covers lies within it of the long-double value."""
    c = ONE_ITERATION[name]
    x = vbmm_cases.make(c["H"], c["reads"], c["sizes"], c["C"], 1, seed=11, priors=c.get("priors"))
    got = _call(engine, x, 0.05, 1)
    assert int(_np(got.seed_iterations)[0]) == 1
    bound = vbmm_exact.one_iteration_bound(x["lnl"], x["off"], x["sizes"], x["gt"], x["lp"], x["gc"], x["mc"], x["seeds"][0], x["gp"], x["mask"])
    want = _exact(x, 0.05, 1)
    ratios = {}
    for key, g, w in (("log_posteriors", got.genotype_log_posteriors, want["log_posteriors"]),
                      ("posteriors", got.genotype_posteriors, want["posteriors"]),
                      ("weighted", got.weighted_genotype_posteriors, want["weighted"]),
                      ("group_concentrations", got.group_concentrations, want["group_concentrations"]),
                      ("mixture_concentrations", got.mixture_concentrations, want["mixture_concentrations"]),
                      ("evidence", [_np(got.max_log_evidence)], [want["max_log_evidence"]])):
        b = np.atleast_1d(np.asarray(bound[key], float))
        ratios[key] = float(np.max(np.abs(np.asarray(_np(g), float) - np.asarray(w, float)) / np.maximum(b, 1e-320)))
    print("%s: largest error / bound: %s" % (name, ", ".join("%s %.3g" % kv for kv in ratios.items())))
    assert all(r <= 1.0 for r in ratios.values()), (name, ratios)
