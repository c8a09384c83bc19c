"""The long-double restatement (tests/vb_exact.py) against the UNMODIFIED reference run_variational_bayes (oracle/_ref/libref_vb.so),
on the CPU. The reference keeps alphas, digamma differences and its likelihood copy in float (fmath fast_exp / fast_log), so values
agree only to float tolerance. Tolerances, measured on an x86-64 CPU over the cases below with two input seeds each (the largest
difference seen, times 10): weighted posteriors 1.03e-5 absolute -> WEIGHTED_ABS 1e-4; max log evidence 4e-7 relative ->
EVIDENCE_REL 4e-6. The max-evidence seed and its MAP genotype must be equal unless the two largest exact evidences lie within
EVIDENCE_REL of each other, a tie the float reference cannot resolve. Iteration counts must be equal unless the restatement flags the seed (vb_exact.near_threshold): with K = 1
every responsibility is 1, so the reference's latents are the same after one trip as after two, and its inferred count is 1."""
import numpy as np
import pytest

import vb_cases
import vb_exact
from vb_ref import RefVB

pytestmark = pytest.mark.skipif(not RefVB.available(), reason="reference VB not built (oracle/_ref/libref_vb.so)")

WEIGHTED_ABS = 1e-4
EVIDENCE_REL = 4e-6

CASES = [(4, [30], 6, 1, 2), (6, [40, 0], 12, 2, 3), (8, [25, 17, 3], 20, 3, 4), (5, [33], 10, 4, 10), (5, [12, 9], 8, 8, 2),
         (6, [60], 10, 100, 1), (16, [257, 1, 0], 200, 3, 12)]


def assert_agrees_with_reference(ref, exact, eps, name):
    """Iteration counts (flagged seeds aside), max-evidence seed and MAP genotype equal; weighted posteriors and the max evidence
    within the measured float tolerances. Returns the number of flagged seeds."""
    flagged = 0
    for i, s in enumerate(exact["seeds"]):
        if int(ref["seed_iterations"][i]) != s["iterations"]:
            assert vb_exact.near_threshold(s["decisions"], eps), (name, i, ref["seed_iterations"][i], s["iterations"])
            flagged += 1
    if not flagged:
        ev = sorted((float(x["evidence"]) for x in exact["seeds"]), reverse=True)
        if len(ev) < 2 or ev[0] - ev[1] > EVIDENCE_REL * abs(ev[0]):    # a closer tie is below what the float reference resolves
            assert ref["max_seed"] == exact["max_seed"], name
            assert int(np.argmax(ref["posteriors"])) == int(np.argmax(np.asarray(exact["posteriors"], float))), name
        w = np.abs(ref["weighted"] - np.asarray(exact["weighted"], float)).max() / WEIGHTED_ABS
        e = abs(ref["max_log_evidence"] - float(exact["max_log_evidence"])) / (EVIDENCE_REL * abs(float(exact["max_log_evidence"])))
        print("%s: reference vs exact, error / tolerance: weighted %.3g, max evidence %.3g" % (name, w, e))
        assert w <= 1 and e <= 1, (name, w, e)
    return flagged


@pytest.mark.parametrize("seed", [3, 4])
@pytest.mark.parametrize("case", CASES, ids=lambda c: "H%d R%s G%d K%d seeds%d" % c)
def test_restatement_agrees_with_the_reference(case, seed):
    H, reads, G, K, n = case
    lnl, off, gt, prior, lp, seeds = vb_cases.make(H, reads, G, K, n, seed=seed)
    ref = RefVB().run(lnl, off, gt, prior, lp, seeds, 0.05, 1000)
    exact = vb_exact.run(lnl, off, gt, prior, lp, seeds, 0.05, 1000)
    flagged = assert_agrees_with_reference(ref, exact, 0.05, str(case))
    assert flagged == 0 or K == 1
