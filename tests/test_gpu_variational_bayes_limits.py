"""phmm_variational_bayes and phmm_variational_bayes_mixture_mixture where their launch shapes and limits bind: a block that runs
several seeds in turn over one workspace, a grid cut down by the 2 GiB workspace budget, k_vb_index's shared memory above the
48 KB default (up to H = 50 000) shared by two engines, and calls with no reads at all.

Each case first restates the host's grid formula and asserts that its shape reaches the path it is named after, so the test
keeps its point on a GPU with another SM count. Seeds run independently, so cutting a call into calls of at most `grid` seeds
(one seed per block) must give every seed the same bits; left-over per-block state from a block's previous seed would not.
Whole results are held to the long-double restatements under the neighbouring modules' rules (_compare)."""
import threading

import numpy as np
import pytest

import vb_cases
import vb_exact
import vbmm_cases
import vbmm_exact
from test_gpu_variational_bayes import REL, _agrees_with_reference as _vb_agrees_with_reference, _bits, _compare as _vb_compare, _np
from test_gpu_variational_bayes import vb_exact_fields
from test_gpu_variational_bayes_mixture_mixture import FIELDS as VBMM_FIELDS
from test_gpu_variational_bayes_mixture_mixture import _agrees_with_reference as _vbmm_agrees_with_reference, _call, _cells
from test_gpu_variational_bayes_mixture_mixture import _compare as _vbmm_compare

pytestmark = pytest.mark.gpu

BUDGET_DOUBLES = ((2 << 30) // 8)     # kVbWorkspaceBudget (phmm_engine.cu:751), in doubles
DEFAULT_SMEM = 48 * 1024              # a kernel's shared memory (static and dynamic) above this needs the attribute raised
MAX_H = 50000                         # kVbMaxHaplotypes (phmm_engine.cu:752)
CHUNK = 32                            # phmm::vbmm::kChunk (phmm_vb_mm.cuh:175)


def _vb_workspace(H, R, S, G, K):
    """phmm::vb::Workspace::doubles (phmm_vb.cuh:270-274)."""
    KH = K * H
    return KH + S * KH + K * R + R + G + 3 * S * K + S


def _vbmm_workspace(H, off, sizes, C):
    """phmm::vbmm::Workspace::doubles (phmm_vb_mm.cuh:206-209) at the host's P = Pmax = K min(H, C) and NC read chunks
    (phmm_engine.cu: chunks of at most kChunk reads of one sample)."""
    K, T, S, R = int(sum(sizes)), len(sizes), len(off) - 1, int(off[-1])
    P = K * min(H, C)
    NC = sum(-(-int(off[s + 1] - off[s]) // CHUNK) for s in range(S))
    return 2 * K * H + C + K * R + 3 * T * R + NC * (P + K + T) + S * P + 3 * S * K + 2 * S * T


def _sms():
    import torch
    return torch.cuda.get_device_properties(0).multi_processor_count


def _grid(n_seeds, ws):
    """The seed kernels' grid (phmm_engine.cu): min(n_seeds, 2 per SM, max(1, budget / one workspace)), its budget term and the
    SM count."""
    sms = _sms()
    by_budget = max(1, BUDGET_DOUBLES // ws)
    return min(n_seeds, 2 * sms, by_budget), by_budget, sms


def _trips(n_seeds, grid):
    """The most seeds one block runs (block b runs seeds b, b + grid, ...)."""
    return -(-n_seeds // grid)


def _seed_bits_equal(whole, part, rows, name):
    for f in ("seed_log_evidences", "seed_iterations"):
        w, p = _np(getattr(whole, f))[rows], _np(getattr(part, f))
        assert np.array_equal(_bits(w), _bits(p)), (name, f, rows[:1], rows[-1:], w[w != p][:3], p[w != p][:3])


def _check_seed_loop(call, n_seeds, grid, name, one_seed_rows=None):
    """(a): every seed's evidence and iteration count of the whole call equal, bit for bit, those of the call cut into calls of at
    most `grid` seeds (each seed alone in its block), and those of a one-seed call for every seed of the last trip (or of
    one_seed_rows). call(rows) runs the call on seeds[rows]. Returns the whole call's result."""
    whole = call(np.arange(n_seeds))
    for lo in range(0, n_seeds, grid):
        rows = np.arange(lo, min(lo + grid, n_seeds))
        _seed_bits_equal(whole, call(rows), rows, name)
    if one_seed_rows is None:
        one_seed_rows = range((_trips(n_seeds, grid) - 1) * grid, n_seeds)
    for i in one_seed_rows:
        _seed_bits_equal(whole, call(np.array([i])), np.array([i]), name)
    return whole


def _duplicate_the_best(seeds, best, grid):
    """Moves the max-evidence seed `best` to row 5 and copies it to row grid + 6: a later block in a later trip."""
    seeds = seeds.copy()
    j, d = 5, grid + 6
    seeds[[j, best]] = seeds[[best, j]]
    seeds[d] = seeds[j]
    return seeds, j, d


# -- more seeds than blocks --------------------------------------------------------------------------------------------------------

VB_LOOP = {
    "K2 S2 exhaustive G 2SM+37": dict(H=40, reads=[180, 120], K=2, extra=37),
    "K3 S2 exhaustive G1300": dict(H=48, reads=[200, 150], K=3, G=1300),
}


@pytest.mark.parametrize("name", list(VB_LOOP))
def test_vb_blocks_run_many_seeds(engine, name):
    """Exhaustive seeds (one point mass per genotype, so seeds i and i + grid sit on different genotypes), more than the grid: each
    block runs several seeds over its workspace, the mode kernels run more than one block and, at G = 1300, k_vb_modes_compact's
    loops stride past 1024 seeds. The max-evidence seed also sits at row 5 and again at row grid + 6, in another block and trip:
    both get the same bits, and max_seed is the first (std::max_element)."""
    c = VB_LOOP[name]
    R, S = sum(c["reads"]), len(c["reads"])
    G = c.get("G", 2 * _sms() + c.get("extra", 0))
    lnl, off, gt, prior, lp, seeds = vb_cases.make(c["H"], c["reads"], G, c["K"], G, seed=21)
    grid, by_budget, sms = _grid(G, _vb_workspace(c["H"], R, S, G, c["K"]))
    trips = _trips(G, grid)
    print("%s: %d seeds, grid %d (2 x %d SMs, by_budget %d), up to %d seeds per block, %d mode-kernel blocks"
          % (name, G, grid, sms, by_budget, trips, -(-G // 256)))
    assert G > grid and trips >= 2 and G > 256
    if c.get("G"):
        assert G > 1024 and trips >= 4

    first = engine.variational_bayes(lnl, gt, prior, lp, seeds, off)
    seeds, j, d = _duplicate_the_best(seeds, int(first.max_seed), grid)
    assert d > grid and d % grid != j % grid
    call = lambda rows: engine.variational_bayes(lnl, gt, prior, lp, seeds[rows], off)
    got = _check_seed_loop(call, G, grid, name)
    ev = _np(got.seed_log_evidences)
    assert _bits(ev[j]).tobytes() == _bits(ev[d]).tobytes()
    assert int(got.max_seed) == j, (int(got.max_seed), j, d)
    _vb_compare(got, lnl, off, gt, prior, lp, seeds, 0.05, 1000, name)


VBMM_LOOP = {
    "S8 T3 K[2,2,2] C200 300 seeds": dict(H=12, S=8, sizes=[2, 2, 2], C=200, n_seeds=300),
    "S6 T3 K[1,2,2] C120 1100 seeds": dict(H=10, S=6, sizes=[1, 2, 2], C=120, n_seeds=1100),
}


@pytest.mark.parametrize("name", list(VBMM_LOOP))
def test_vbmm_blocks_run_many_seeds(engine, name):
    """Random seeds over cells, more than the grid, near-uniform in a block's odd trips and peaked in its even ones: each block runs
    a peaked seed after a flat one over the same workspace, where left-over sigma, tau or group concentrations would show. The
    max-evidence seed also sits at row 5 and again at row grid + 6."""
    c = VBMM_LOOP[name]
    x = vbmm_cases.make(c["H"], _cells(c["S"], 10, np.random.default_rng(13)), c["sizes"], c["C"], c["n_seeds"], seed=23)
    n, C = c["n_seeds"], c["C"]
    grid, by_budget, sms = _grid(n, _vbmm_workspace(c["H"], x["off"], c["sizes"], C))
    trips = _trips(n, grid)
    print("%s: %d seeds, grid %d (2 x %d SMs, by_budget %d), up to %d seeds per block, %d mode-kernel blocks"
          % (name, n, grid, sms, by_budget, trips, -(-n // 256)))
    assert n > grid and trips >= 2 and n > 256
    if n > 1024:
        assert trips >= 4

    rng = np.random.default_rng(29)
    flat = np.log(rng.dirichlet(np.full(C, 200.0), size=n))
    peaked = np.full((n, C), np.log(1e-4 / (C - 1)))
    peaked[np.arange(n), rng.integers(0, C, n)] = np.log1p(-1e-4)
    x["seeds"] = np.where(((np.arange(n) // grid) % 2 == 0)[:, None], peaked, flat)
    first = _call(engine, x, 0.05, 1000)
    x["seeds"], j, d = _duplicate_the_best(x["seeds"], int(first.max_seed), grid)
    call = lambda rows: _call(engine, dict(x, seeds=x["seeds"][rows]), 0.05, 1000)
    got = _check_seed_loop(call, n, grid, name)
    ev = _np(got.seed_log_evidences)
    assert _bits(ev[j]).tobytes() == _bits(ev[d]).tobytes()
    assert int(got.max_seed) == j, (int(got.max_seed), j, d)
    _vbmm_compare(got, x, 0.05, 1000, name)


# -- the workspace budget binds ----------------------------------------------------------------------------------------------------

def _restated_seeds(run_seed, near, got, seeds, rows, eps, max_it, name):
    """Per-seed evidences (and iteration counts) of `rows` against the restatement's run_seed; returns the restated seeds."""
    out, worst = {}, 0.0
    its = _np(got.seed_iterations)
    for i in rows:
        r = run_seed(seeds[i], eps, max_it)
        if r["iterations"] != its[i]:
            assert near(r["decisions"], eps), (name, i, its[i], r["iterations"])
            r = run_seed(seeds[i], eps, max_it, int(its[i]))
        want = float(r["evidence"])
        worst = max(worst, abs(_np(got.seed_log_evidences)[i] - want) / (REL * max(1.0, abs(want))))
        out[i] = r
    return out, worst


def test_vb_workspace_budget_binds(engine):
    """K = 100 slots over R reads: one seed's workspace is so large that the 2 GiB budget, not the SM count, sets the grid, and each
    block runs at least three seeds. Every seed equals its one-seed call; three seeds of block 0 (one per trip) and the
    max-evidence seed's evidence and alphas equal the restatement's at max_iterations = 2."""
    H, K, G, R = 10, 100, 50, 26000
    ws = _vb_workspace(H, R, 1, G, K)
    n = 3 * (BUDGET_DOUBLES // ws) + 7
    grid, by_budget, sms = _grid(n, ws)
    lnl, off, gt, prior, lp, seeds = vb_cases.make(H, [R], G, K, n, seed=31)
    print("VB budget: workspace %d doubles (%.1f MB), by_budget %d, grid %d (2 x %d SMs), %d seeds, up to %d per block"
          % (ws, ws * 8 / 1e6, by_budget, grid, sms, n, _trips(n, grid)))
    assert grid == by_budget < min(n, 2 * sms) and n >= 3 * grid
    call = lambda rows: engine.variational_bayes(lnl, gt, prior, lp, seeds[rows], off, 0.05, 2)
    got = _check_seed_loop(call, n, grid, "VB budget", one_seed_rows=range(n))
    P = vb_exact._Problem(lnl, off, gt, prior, lp, False)
    run_seed = lambda sd, eps, max_it, forced=None: vb_exact.run_seed(P, sd, eps, max_it, forced)
    ms = int(got.max_seed)
    rows = sorted({0, grid, 2 * grid, ms})
    res, worst = _restated_seeds(run_seed, vb_exact.near_threshold, got, seeds, rows, 0.05, 2, "VB budget")
    aw = np.asarray(res[ms]["alphas"], float)
    alphas = float(np.max(np.abs(_np(got.alphas) - aw) / (REL * np.abs(aw))))
    print("VB budget: seeds %s; largest error / tolerance: evidences %.3g, max-evidence seed's alphas %.3g" % (rows, worst, alphas))
    assert worst <= 1 and alphas <= 1


def test_vbmm_workspace_budget_binds(engine):
    """Two groups of 50 components over four samples of R / 4 reads: the budget sets the grid and each block runs at least three
    seeds. Every seed equals its one-seed call; three seeds of block 0 and the max-evidence seed's evidence and mixture
    concentrations equal the restatement's at max_iterations = 2."""
    H, sizes, C, S, R = 8, [50, 50], 50, 4, 20000
    reads = [R // S] * S
    x = vbmm_cases.make(H, reads, sizes, C, 1, seed=37)
    ws = _vbmm_workspace(H, x["off"], sizes, C)
    n = 3 * (BUDGET_DOUBLES // ws) + 7
    grid, by_budget, sms = _grid(n, ws)
    x["seeds"] = np.log(np.random.default_rng(41).dirichlet(np.full(C, 0.5), size=n) + 1e-300)
    print("VBMM budget: workspace %d doubles (%.1f MB), by_budget %d, grid %d (2 x %d SMs), %d seeds, up to %d per block"
          % (ws, ws * 8 / 1e6, by_budget, grid, sms, n, _trips(n, grid)))
    assert grid == by_budget < min(n, 2 * sms) and n >= 3 * grid
    call = lambda rows: _call(engine, dict(x, seeds=x["seeds"][rows]), 0.05, 2)
    got = _check_seed_loop(call, n, grid, "VBMM budget", one_seed_rows=range(n))
    P = vbmm_exact._Problem(x["lnl"], x["off"], sizes, x["gt"], x["lp"], x["gc"], x["mc"], x["gp"], x["mask"], False, True)
    run_seed = lambda sd, eps, max_it, forced=None: vbmm_exact.run_seed(P, sd, eps, max_it, forced)
    ms = int(got.max_seed)
    rows = sorted({0, grid, 2 * grid, ms})
    res, worst = _restated_seeds(run_seed, vbmm_exact.near_threshold, got, x["seeds"], rows, 0.05, 2, "VBMM budget")
    mw = np.asarray(res[ms]["mixture_concentrations"], float)
    mconc = float(np.max(np.abs(_np(got.mixture_concentrations) - mw) / (REL * np.abs(mw))))
    print("VBMM budget: seeds %s; largest error / tolerance: evidences %.3g, max-evidence seed's mixture concentrations %.3g"
          % (rows, worst, mconc))
    assert worst <= 1 and mconc <= 1


# -- many haplotypes ---------------------------------------------------------------------------------------------------------------

def _spread(gt, H, rng, few):
    """Haplotypes from the whole range, 0 and H - 1 included; with `few`, slot 1 takes only a handful of them (nk << H)."""
    gt[0, 0], gt[-1, -1], gt[1, 0] = 0, H - 1, H - 1
    if few:
        gt[:, 1] = rng.choice([0, 1, H // 2, H - 2, H - 1], size=len(gt))
    return gt


MANY_H = {
    "H12288": dict(H=12288),
    "H12289": dict(H=12289),
    "H50000": dict(H=50000),
    "H50000 handful in slot 1": dict(H=50000, few=True),
}


@pytest.mark.parametrize("name", list(MANY_H))
def test_vb_many_haplotypes(engine, name):
    """k_vb_index keeps one int per haplotype in dynamic shared memory: at H = 12 288 that is exactly the 48 KB default limit, which
    the kernel's own static shared int then exceeds (a launch that only raised the limit above 48 KB of dynamic memory failed here
    with 'invalid argument' while no earlier call had raised it); 12 289 is the first H whose dynamic memory alone exceeds it;
    50 000 is the largest the call takes. This runs before any other call of the module needs more than 48 KB."""
    c = MANY_H[name]
    H = c["H"]
    lnl, off, gt, prior, lp, seeds = vb_cases.make(H, [150, 130], 300, 3, 12, seed=43)
    gt = _spread(gt, H, np.random.default_rng(47), c.get("few"))
    smem = 4 * H
    print("%s: k_vb_index dynamic shared memory %d B (default limit %d B)" % (name, smem, DEFAULT_SMEM))
    assert (smem >= DEFAULT_SMEM) == (H >= 12288) and (smem > DEFAULT_SMEM) == (H >= 12289)
    got = engine.variational_bayes(lnl, gt, prior, lp, seeds, off)
    _vb_compare(got, lnl, off, gt, prior, lp, seeds, 0.05, 1000, name)
    from vb_ref import RefVB
    if RefVB.available():         # the existing size rule: G * R <= 300 000
        assert len(gt) * lnl.shape[1] <= 300_000
        _vb_agrees_with_reference(RefVB(), got, lnl, off, gt, prior, lp, seeds, 0.05, 1000, name)


def _vbmm_many_h(H, few=False, seed=53):
    x = vbmm_cases.make(H, [50, 40, 0, 60, 1, 50], [1, 2], 300, 12, seed=seed)
    x["gt"] = _spread(x["gt"], H, np.random.default_rng(seed + 1), few)
    return x


@pytest.mark.parametrize("name", list(MANY_H))
def test_vbmm_many_haplotypes(engine, name):
    """As test_vb_many_haplotypes, for the mixture-of-mixtures call (which shares k_vb_index)."""
    c = MANY_H[name]
    x = _vbmm_many_h(c["H"], c.get("few"))
    print("%s: k_vb_index dynamic shared memory %d B (default limit %d B)" % (name, 4 * c["H"], DEFAULT_SMEM))
    got = _call(engine, x, 0.05, 1000)
    _vbmm_compare(got, x, 0.05, 1000, name)
    from vbmm_ref import RefVBMM
    if RefVBMM.available():       # the existing size rule: C * R * sum K <= 3 000 000
        assert len(x["gt"]) * x["lnl"].shape[1] * sum(x["sizes"]) <= 3_000_000
        _vbmm_agrees_with_reference(got, x, 0.05, 1000, name)


# -- two engines, one shared-memory limit ------------------------------------------------------------------------------------------

def _limit_calls():
    """A VB and a mixture-of-mixtures call at each of two haplotype counts, both above the 48 KB default."""
    calls = {}
    for H in (MAX_H, 13000):
        lnl, off, gt, prior, lp, seeds = vb_cases.make(H, [150, 130], 300, 3, 12, seed=59)
        gt = _spread(gt, H, np.random.default_rng(61), False)
        calls[("vb", H)] = lambda e, a=(lnl, gt, prior, lp, seeds, off): e.variational_bayes(*a)
        x = _vbmm_many_h(H, seed=67)
        calls[("vbmm", H)] = lambda e, x=x: _call(e, x, 0.05, 1000)
    return calls


def _same_bits(a, b, kind):
    for f in (vb_exact_fields() if kind == "vb" else VBMM_FIELDS):
        assert np.array_equal(_bits(getattr(a, f)), _bits(getattr(b, f))), (kind, f)


def test_two_engines_share_k_vb_index_shared_memory_limit(engine):
    """k_vb_index's dynamic shared-memory limit belongs to the process, not to an engine: engine B's call at H = 13 000 must not
    lower the limit engine A's H = 50 000 call relies on. Sequentially, then from two threads with an engine each alternating the
    two sizes and both calls. The threads cannot force the window between one engine setting the limit and the other launching,
    so this guards the rule (the limit is only ever raised, through the engine's per-process high-water mark) against regressing
    rather than proving it; the sequential part passes whenever each call sets the limit it needs just before its launch."""
    from octopus_b200 import PairHMMEngine
    calls = _limit_calls()
    solo = {key: fn(engine) for key, fn in calls.items()}
    other = PairHMMEngine(0)
    try:
        for kind in ("vb", "vbmm"):
            first = calls[(kind, MAX_H)](engine)
            _same_bits(first, solo[(kind, MAX_H)], kind)
            _same_bits(calls[(kind, 13000)](other), solo[(kind, 13000)], kind)
            _same_bits(calls[(kind, MAX_H)](engine), first, kind)

        errors = []

        def worker(eng, t):
            try:
                for c in range(6):       # (vb, vbmm) at one size, then at the other
                    key = (("vb", "vbmm")[c % 2], (MAX_H, 13000)[(c // 2 + t) % 2])
                    _same_bits(calls[key](eng), solo[key], key[0])
            except Exception as ex:      # noqa: BLE001  (reported from the main thread)
                errors.append(repr(ex))

        threads = [threading.Thread(target=worker, args=(eng, t)) for t, eng in enumerate((engine, other))]
        for th in threads:
            th.start()
        for th in threads:
            th.join()
        assert not errors, errors
    finally:
        other.close()


# -- no reads ----------------------------------------------------------------------------------------------------------------------

def _finite_or_like(got, want):
    got, want = np.asarray(_np(got), float), np.asarray(want, float)
    assert np.array_equal(np.isfinite(got), np.isfinite(want)) and np.array_equal(np.isnan(got), np.isnan(want))


@pytest.mark.parametrize("n_seeds", [1, 12, 300])
def test_vb_no_reads(engine, n_seeds):
    """R = 0: every sample is empty and the matrix has no columns. The responsibilities are empty sums, so alphas stay at the priors
    and the second iteration's ELBO repeats the first; with 300 seeds each block also runs a second seed."""
    S, H, K, G = 3, 6, 2, 40
    lnl, off, gt, prior, lp, seeds = vb_cases.make(H, [0] * S, G, K, n_seeds, seed=71)
    assert lnl.shape == (H, 0) and list(off) == [0] * (S + 1)
    got = engine.variational_bayes(lnl, gt, prior, lp, seeds, off)
    want = vb_exact.run(lnl, off, gt, prior, lp, seeds)
    for f, w in (("genotype_posteriors", want["posteriors"]), ("genotype_log_posteriors", want["log_posteriors"]),
                 ("alphas", want["alphas"]), ("evidence_weighted_genotype_posteriors", want["weighted"]),
                 ("seed_log_evidences", [s["evidence"] for s in want["seeds"]])):
        _finite_or_like(getattr(got, f), w)
    _vb_compare(got, lnl, off, gt, prior, lp, seeds, 0.05, 1000, "VB no reads, %d seeds" % n_seeds)
    from vb_ref import RefVB
    if RefVB.available():
        # Not _agrees_with_reference: with nothing to move, the reference's per-seed count (the fewest iterations that end in the
        # final latents) is 1 where the loop runs 2, and the evidence cancels to about 1e-16, below a relative tolerance.
        from test_vb_ref import EVIDENCE_REL, WEIGHTED_ABS
        r = RefVB().run(lnl, off, gt, prior, lp, seeds)
        w = float(np.max(np.abs(_np(got.evidence_weighted_genotype_posteriors) - r["weighted"]))) / WEIGHTED_ABS
        p = float(np.max(np.abs(_np(got.genotype_posteriors) - r["posteriors"]))) / WEIGHTED_ABS
        e = abs(float(got.max_log_evidence) - r["max_log_evidence"]) / EVIDENCE_REL
        print("VB no reads, %d seeds: device vs reference, error / tolerance: weighted %.3g, posteriors %.3g, max evidence %.3g"
              % (n_seeds, w, p, e))
        assert w <= 1 and p <= 1 and e <= 1 and np.array_equal(_np(got.alphas), prior)


@pytest.mark.parametrize("n_seeds", [1, 12, 300])
def test_vbmm_no_reads(engine, n_seeds):
    """R = 0 over several cells: no read chunks; sigma starts from the concentrations alone."""
    x = vbmm_cases.make(6, [0] * 5, [1, 2, 2], 40, n_seeds, seed=73)
    assert x["lnl"].shape == (6, 0)
    got = _call(engine, x, 0.05, 1000)
    want = vbmm_exact.run(x["lnl"], x["off"], x["sizes"], x["gt"], x["lp"], x["gc"], x["mc"], x["seeds"], x["gp"], x["mask"])
    for f, w in (("genotype_posteriors", want["posteriors"]), ("genotype_log_posteriors", want["log_posteriors"]),
                 ("group_concentrations", want["group_concentrations"]), ("mixture_concentrations", want["mixture_concentrations"]),
                 ("group_responsibilities", want["group_responsibilities"]), ("weighted_genotype_posteriors", want["weighted"]),
                 ("weighted_group_responsibilities", want["weighted_group_responsibilities"]),
                 ("seed_log_evidences", [s["evidence"] for s in want["seeds"]])):
        _finite_or_like(getattr(got, f), w)
    _vbmm_compare(got, x, 0.05, 1000, "VBMM no reads, %d seeds" % n_seeds)
    from vbmm_ref import RefVBMM
    if RefVBMM.available():
        _vbmm_agrees_with_reference(got, x, 0.05, 1000, "VBMM no reads, %d seeds" % n_seeds)
