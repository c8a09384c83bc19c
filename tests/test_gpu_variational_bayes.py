"""phmm_variational_bayes (PairHMMEngine.variational_bayes): SubcloneModel::evaluate's variational Bayes inference on the device,
every seed in one call, held to the long-double restatement tests/vb_exact.py run for the device's own per-seed iteration counts.

A seed whose iteration count differs from the restatement's is accepted only when one of the restatement's stopping decisions lies
within rounding of epsilon or of 0 (vb_exact.near_threshold); such seeds are counted as flagged and their values are not compared.
Tolerances are chosen, not derived: posteriors within ABS absolutely, log posteriors, alphas and evidences within REL relatively
(double against long double over up to a few hundred iterations of sums of up to 10^4 terms)."""
import numpy as np
import pytest

import vb_cases
import vb_exact

pytestmark = pytest.mark.gpu

DEV = "cuda:0"
ABS = 1e-9
REL = 1e-9
SPIN_CYCLES = 400_000_000


def _bits(x):
    if isinstance(x, (int, float)):      # host-space scalars come back as Python numbers
        x = np.int32(x) if isinstance(x, int) else np.float64(x)
    x = x.cpu().numpy() if hasattr(x, "cpu") else np.asarray(x)
    return np.ascontiguousarray(x).view(np.uint8)


def _np(x):
    return x.cpu().numpy() if hasattr(x, "cpu") else np.asarray(x)


CASES = {
    "K1 S1 R255 G1 one seed": dict(H=3, reads=[255], G=1, K=1, n_seeds=1, max_it=1000, eps=0.05),
    "K2 S2 R256+0 G2 exhaustive": dict(H=4, reads=[256, 0], G=2, K=2, n_seeds=2, max_it=1000, eps=0.05),
    "K3 S3 R257+1+0 G1000 12 seeds dup": dict(H=16, reads=[257, 1, 0], G=1000, K=3, n_seeds=12, max_it=1000, eps=0.05, dup=True),
    "K4 S1 R4000 G1000 12 seeds": dict(H=32, reads=[4000], G=1000, K=4, n_seeds=12, max_it=1000, eps=0.05),
    "K8 S2 R255+257 G1000 two iterations": dict(H=24, reads=[255, 257], G=1000, K=8, n_seeds=12, max_it=2, eps=0.05),
    "K100 S1 R256 G20 eps 1e9": dict(H=10, reads=[256], G=20, K=100, n_seeds=1, max_it=1000, eps=1e9),
    "K3 S2 R1000+1000 G20000 12 seeds": dict(H=64, reads=[1000, 1000], G=20000, K=3, n_seeds=12, max_it=1000, eps=0.05),
    "K2 S1 R1 G70000 one iteration": dict(H=40, reads=[1], G=70000, K=2, n_seeds=1, max_it=1, eps=0.05),
    "K4 S1 R257 G60 exhaustive": dict(H=8, reads=[257], G=60, K=4, n_seeds=60, max_it=1000, eps=0.05),
    "K3 S1 R257 G100 eps 0": dict(H=8, reads=[257], G=100, K=3, n_seeds=12, max_it=1000, eps=0.0),
    "K2 S1 R100 G15 lowest entries": dict(H=6, reads=[100], G=15, K=2, n_seeds=12, max_it=1000, eps=0.05, lowest=3),
}


def _inputs(c, seed=11):
    return vb_cases.make(c["H"], c["reads"], c["G"], c["K"], c["n_seeds"], seed=seed, dup=c.get("dup", False), lowest=c.get("lowest", 0))


def _compare(got, lnl, off, gt, prior, lp, seeds, eps, max_it, name):
    iters = _np(got.seed_iterations)
    free = vb_exact.run(lnl, off, gt, prior, lp, seeds, eps, max_it)
    want = vb_exact.run(lnl, off, gt, prior, lp, seeds, eps, max_it, forced=iters, free=free)
    flagged, ratios = 0, {"posteriors": 0.0, "log posteriors": 0.0, "alphas": 0.0, "evidences": 0.0}
    for i, ws in enumerate(want["seeds"]):
        if free["seeds"][i]["iterations"] != iters[i]:
            assert vb_exact.near_threshold(free["seeds"][i]["decisions"], eps), (name, i, iters[i], free["seeds"][i]["iterations"])
            flagged += 1
        e_want = float(ws["evidence"])
        ratios["evidences"] = max(ratios["evidences"], abs(_np(got.seed_log_evidences)[i] - e_want) / (REL * max(1.0, abs(e_want))))
    ms = int(_np(got.max_seed))
    assert ms == want["max_seed"] or flagged, (name, ms, want["max_seed"])
    p_want = np.asarray(want["posteriors"], float)
    ratios["posteriors"] = float(np.max(np.abs(_np(got.genotype_posteriors) - p_want)) / ABS)
    lw = np.asarray(want["log_posteriors"], float)
    fin = np.isfinite(lw)
    assert np.array_equal(np.isfinite(_np(got.genotype_log_posteriors)), fin)
    ratios["log posteriors"] = float(np.max(np.abs(_np(got.genotype_log_posteriors)[fin] - lw[fin]) / (REL * np.maximum(1.0, np.abs(lw[fin])))))
    aw = np.asarray(want["alphas"], float)
    ratios["alphas"] = float(np.max(np.abs(_np(got.alphas) - aw) / (REL * np.abs(aw))))
    ww = np.asarray(want["weighted"], float)
    ratios["weighted"] = float(np.max(np.abs(_np(got.evidence_weighted_genotype_posteriors) - ww)) / ABS)
    assert int(np.argmax(_np(got.genotype_posteriors))) == int(np.argmax(p_want)) or flagged
    print("%s: flagged %d of %d seeds; largest error / tolerance: %s" % (name, flagged, len(seeds),
                                                                         ", ".join("%s %.3g" % kv for kv in ratios.items())))
    assert all(r <= 1.0 for r in ratios.values()), (name, ratios)


@pytest.mark.parametrize("name", list(CASES))
def test_matches_the_restatement(engine, name):
    c = CASES[name]
    lnl, off, gt, prior, lp, seeds = _inputs(c)
    got = engine.variational_bayes(lnl, gt, prior, lp, seeds, off, c["eps"], c["max_it"])
    _compare(got, lnl, off, gt, prior, lp, seeds, c["eps"], c["max_it"], name)


ONE_ITERATION = {
    "K2 S1 R1 G70000": dict(H=40, reads=[1], G=70000, K=2),
    "K3 S2 R257+40 G300": dict(H=16, reads=[257, 40], G=300, K=3),
    "K100 S1 R256 G20": dict(H=10, reads=[256], G=20, K=100),
    "K8 S3 R300+0+255 G1000": dict(H=24, reads=[300, 0, 255], G=1000, K=8),
}


@pytest.mark.parametrize("name", list(ONE_ITERATION))
def test_one_iteration_within_the_derived_bound(engine, name):
    """max_iterations = 1, one seed: every output within vb_exact.one_iteration_bound of the long-double value."""
    c = ONE_ITERATION[name]
    lnl, off, gt, prior, lp, seeds = vb_cases.make(c["H"], c["reads"], c["G"], c["K"], 1, seed=11)
    got = engine.variational_bayes(lnl, gt, prior, lp, seeds, off, 0.05, 1)
    assert int(got.seed_iterations[0]) == 1
    bound = vb_exact.one_iteration_bound(lnl, off, gt, prior, lp, seeds[0])
    want = vb_exact.run(lnl, off, gt, prior, lp, seeds, 0.05, 1)
    ratios = {}
    for key, g, w in (("log_posteriors", got.genotype_log_posteriors, want["log_posteriors"]),
                      ("posteriors", got.genotype_posteriors, want["posteriors"]),
                      ("weighted", got.evidence_weighted_genotype_posteriors, want["weighted"]),
                      ("alphas", got.alphas, want["alphas"]),
                      ("evidence", [got.max_log_evidence], [want["max_log_evidence"]])):
        b = np.atleast_1d(np.asarray(bound[key], float))
        ratios[key] = float(np.max(np.abs(np.asarray(_np(g), float) - np.asarray(w, float)) / np.maximum(b, 1e-320)))
    print("%s: largest error / bound: %s" % (name, ", ".join("%s %.3g" % kv for kv in ratios.items())))
    assert all(r <= 1.0 for r in ratios.values()), (name, ratios)


def _agrees_with_reference(ref, got, lnl, off, gt, prior, lp, seeds, eps, max_it, name):
    """One call's result against the reference's (vb_ref.RefVB): iteration counts, max-evidence seed and MAP genotype equal (seeds
    the restatement flags aside), weighted posteriors and max evidence within the float tolerances measured on the CPU
    (tests/test_vb_ref.py). Returns False, having compared only the iteration counts, when the restatement flags a seed."""
    from test_vb_ref import EVIDENCE_REL, WEIGHTED_ABS
    r = ref.run(lnl, off, gt, prior, lp, seeds, eps, max_it)
    free = vb_exact.run(lnl, off, gt, prior, lp, seeds, eps, max_it)
    flagged = [vb_exact.near_threshold(s["decisions"], eps) for s in free["seeds"]]
    its = _np(got.seed_iterations)
    for i in range(len(seeds)):
        assert its[i] == r["seed_iterations"][i] or flagged[i], (name, i, its[i], r["seed_iterations"][i])
    if any(flagged):
        return False
    ev = sorted((float(x["evidence"]) for x in free["seeds"]), reverse=True)
    tie = len(ev) > 1 and ev[0] - ev[1] <= EVIDENCE_REL * abs(ev[0])     # closer than the float reference resolves
    if not tie:
        assert int(_np(got.max_seed)) == r["max_seed"], name
        assert int(np.argmax(_np(got.genotype_posteriors))) == int(np.argmax(r["posteriors"])), name
    w = float(np.max(np.abs(_np(got.evidence_weighted_genotype_posteriors) - r["weighted"]))) / WEIGHTED_ABS
    e = abs(float(_np(got.max_log_evidence)) - r["max_log_evidence"]) / (EVIDENCE_REL * abs(r["max_log_evidence"]))
    print("%s: device vs reference, error / tolerance: weighted %.3g, max evidence %.3g" % (name, w, e))
    assert w <= 1 and e <= 1, (name, w, e)
    return True


def test_device_agrees_with_the_reference(engine):
    """The device against the UNMODIFIED reference (oracle/_ref/libref_vb.so) on the cases small enough for it
    (_agrees_with_reference)."""
    from vb_ref import REF_K, RefVB
    if not RefVB.available():
        pytest.skip("reference VB not built (oracle/_ref/libref_vb.so)")
    ref = RefVB()
    checked = 0
    for name, c in CASES.items():
        if c["K"] not in REF_K or c["G"] * sum(c["reads"]) > 300_000 or c.get("lowest"):
            continue
        lnl, off, gt, prior, lp, seeds = _inputs(c)
        got = engine.variational_bayes(lnl, gt, prior, lp, seeds, off, c["eps"], c["max_it"])
        checked += _agrees_with_reference(ref, got, lnl, off, gt, prior, lp, seeds, c["eps"], c["max_it"], name)
    assert checked >= 4


@pytest.mark.parametrize("name", ["K3 S3 R257+1+0 G1000 12 seeds dup", "K3 S2 R1000+1000 G20000 12 seeds", "K4 S1 R257 G60 exhaustive"])
def test_host_and_device_space_give_the_same_bits_every_run(engine, name):
    import torch
    c = CASES[name]
    lnl, off, gt, prior, lp, seeds = _inputs(c)
    host = engine.variational_bayes(lnl, gt, prior, lp, seeds, off, c["eps"], c["max_it"])
    dev = [engine.variational_bayes(*(torch.as_tensor(x, device=DEV) for x in (lnl, gt, prior, lp, seeds)), off, c["eps"], c["max_it"])
           for _ in range(2)]
    for f in vb_exact_fields():
        for d in dev:
            assert np.array_equal(_bits(getattr(host, f)), _bits(getattr(d, f))), f


def vb_exact_fields():
    return ["genotype_posteriors", "genotype_log_posteriors", "alphas", "max_log_evidence", "evidence_weighted_genotype_posteriors",
            "max_seed", "seed_log_evidences", "seed_iterations"]


def test_populated_two_sample_region(engine):
    """The matrix populate leaves on the device, its columns split into two samples, as the cancer caller passes it."""
    import torch
    from octopus_b200 import HaplotypeLikelihoodArray, HaplotypeLikelihoodModel, synth
    haps, reads, band = synth.make_batch("C2", n_reads=600)
    cfg = HaplotypeLikelihoodModel.Config(max_indel_error=band)
    arr = HaplotypeLikelihoodArray(engine=engine)
    arr.likelihoods = engine.populate(cfg, haps.to_device(DEV), reads.to_device(DEV))
    half = reads.n // 2
    arr._set_samples(["normal", "tumour"], [half, reads.n - half])
    assert isinstance(arr.likelihoods, torch.Tensor)
    rng = np.random.default_rng(5)
    H = haps.n
    germ = [(a, b) for a in range(H) for b in range(a, H)]
    gt = np.array([(a, b, c) for a, b in germ for c in range(H)], dtype=np.int32)[:2000]
    prior = np.array([[1.0, 1.0, 0.5], [1.0, 1.0, 0.5]])
    lp = np.log(np.full(len(gt), 1.0 / len(gt)))
    seeds = np.log(rng.dirichlet(np.ones(len(gt)) * 0.5, size=12) + 1e-300)
    got = arr.variational_bayes(["normal", "tumour"], gt, prior, lp, seeds)
    assert got.genotype_posteriors.device.type == "cuda"
    _compare(got, arr.likelihoods.cpu().numpy(), [0, half, reads.n], gt, prior, lp, seeds, 0.05, 1000, "populated C2 two samples")


BAD = {
    "K 0": lambda a: a.update(gt=np.zeros((3, 0), np.int32), prior=np.zeros((1, 0))),
    "K 101": lambda a: a.update(gt=np.zeros((3, 101), np.int32), prior=np.ones((1, 101))),
    "max_iterations 0": lambda a: a.update(max_it=0),
    "no seeds": lambda a: a.update(seeds=np.zeros((0, 3))),
    "sample_off not from 0": lambda a: a.update(off=[1, 10]),
    "sample_off not to R": lambda a: a.update(off=[0, 9]),
    "sample_off decreasing": lambda a: a.update(off=[0, 6, 4, 10], prior=np.ones((3, 2))),
    "H 50001": lambda a: a.update(lnl=np.zeros((50001, 1)), off=[0, 1]),
    "index H": lambda a: a["gt"].__setitem__((1, 1), 5),
    "index -1": lambda a: a["gt"].__setitem__((2, 0), -1),
}


@pytest.mark.parametrize("space", ["host", "device"])
@pytest.mark.parametrize("what", list(BAD))
def test_refused(engine, what, space):
    import torch
    from octopus_b200 import PhmmError
    rng = np.random.default_rng(1)
    a = dict(lnl=-rng.uniform(0, 10, (5, 10)), gt=rng.integers(0, 5, (3, 2)).astype(np.int32), prior=np.ones((1, 2)),
             lp=np.log(np.full(3, 1 / 3)), seeds=np.log(np.full((2, 3), 1 / 3)), off=[0, 10], max_it=10)
    BAD[what](a)
    args = [a[k] for k in ("lnl", "gt", "prior", "lp", "seeds")]
    if space == "device":
        args = [torch.as_tensor(x, device=DEV) for x in args]
    with pytest.raises((PhmmError, ValueError)) as ei:
        engine.variational_bayes(*args, a["off"], 0.05, a["max_it"])
    if isinstance(ei.value, PhmmError):
        assert ei.value.code == -1
    # the engine still works after a refusal
    ok = engine.variational_bayes(-rng.uniform(0, 10, (5, 10)), rng.integers(0, 5, (3, 2)).astype(np.int32), np.ones((1, 2)),
                                  np.log(np.full(3, 1 / 3)), np.log(np.full((2, 3), 1 / 3)), [0, 10], 0.05, 10)
    assert np.isfinite(ok.max_log_evidence)


@pytest.mark.parametrize("side", [False, True])
def test_device_call_orders_after_the_callers_busy_stream(engine, side):
    """Seeds written on torch's current stream behind a spin, passed as float32 so that the call converts them there: the engine
    must read them only after the conversion."""
    import torch
    c = CASES["K3 S3 R257+1+0 G1000 12 seeds dup"]
    lnl, off, gt, prior, lp, seeds = _inputs(c)
    seeds = seeds.astype(np.float32).astype(np.float64)
    _, _, _, _, _, warm = _inputs(c, seed=99)
    want = engine.variational_bayes(lnl, gt, prior, lp, seeds, off, c["eps"], c["max_it"])
    stream = torch.cuda.Stream(DEV) if side else torch.cuda.current_stream(DEV)
    with torch.cuda.stream(stream):
        m, g, p, l = (torch.as_tensor(x, device=DEV) for x in (lnl, gt, prior, lp))
        src = torch.as_tensor(seeds.astype(np.float32), device=DEV)
        engine.variational_bayes(m, g, p, l, torch.as_tensor(warm.astype(np.float32), device=DEV), off, c["eps"], c["max_it"])
        s32 = torch.zeros_like(src)
        torch.cuda._sleep(SPIN_CYCLES)
        s32.copy_(src)
        assert not torch.cuda.current_stream().query(), "the spin ended before the call, which then tests no ordering"
        got = engine.variational_bayes(m, g, p, l, s32, off, c["eps"], c["max_it"])
        for f in vb_exact_fields():
            assert np.array_equal(_bits(getattr(got, f)), _bits(getattr(want, f))), f
    torch.cuda.synchronize(DEV)


def test_cpp_adapter_matches_the_python_api(engine):
    """octopus_b200::run_variational_bayes (the C++ adapter) over a populated two-sample array gives the bits the Python API gives
    on the same matrix, and surfaces a refusal as Error."""
    import os
    import subprocess
    import tempfile
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    exe = os.path.join(tempfile.mkdtemp(prefix="test_vb_"), "test_vb")
    subprocess.run(["g++", "-std=c++14", "-O1", "-I", os.path.join(root, "include"), "-I", os.path.join(root, "octopus_b200", "cpp"),
                    os.path.join(root, "tests", "cpp", "test_vb.cpp"), "-o", exe, "-L", os.path.join(root, "octopus_b200"), "-lphmm_b200",
                    "-Wl,-rpath," + os.path.join(root, "octopus_b200")], check=True)
    out = subprocess.run([exe], capture_output=True, text=True, timeout=120)
    assert out.returncode == 0, out.stdout + out.stderr
    rows = {l.split()[0]: l.split()[1:] for l in out.stdout.strip().splitlines()}
    H, R = int(rows["MATRIX"][0]), int(rows["MATRIX"][1])
    lnl = np.array([float(v) for v in rows["MATRIX"][2:]]).reshape(H, R)
    w0 = int(rows["WIDTHS"][0])
    gt = np.array([[0, 0], [0, 1], [0, 2], [1, 2], [1, 1]], np.int32)
    prior = np.array([[1.0, 0.5], [1.0, 0.8]])
    lp = np.full(5, -1.6094379124341003)
    seeds = np.full((5, 5), -13.815510557964274)
    np.fill_diagonal(seeds, -4e-6)
    want = engine.variational_bayes(lnl, gt, prior, lp, seeds, [0, w0, R])
    got = lambda k: np.array([float(v) for v in rows[k]])
    assert np.array_equal(_bits(got("POST")), _bits(want.genotype_posteriors))
    assert np.array_equal(_bits(got("LPOST")), _bits(want.genotype_log_posteriors))
    assert np.array_equal(_bits(got("WEIGHTED")), _bits(want.evidence_weighted_genotype_posteriors))
    assert np.array_equal(_bits(np.stack([got("ALPHA_normal"), got("ALPHA_tumour")])), _bits(want.alphas))
    assert np.array_equal(_bits(got("EVIDENCE")), _bits(np.array([want.max_log_evidence])))
    assert rows["REFUSED"] == ["yes"]
