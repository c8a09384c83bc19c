"""The mixture-of-mixtures restatement (tests/vbmm_exact.py) against the UNMODIFIED reference VariationalBayesMixtureMixtureModel
(oracle/_ref/libref_vbmm.so); no GPU needed.

Tolerances, measured on an x86-64 CPU (the reference keeps its expanded likelihoods and its component update's sums in float):
the largest errors seen over these cases were 2e-9 relative on seed evidences, 4e-8 absolute on weighted posteriors and 1e-6
relative on mixture concentrations, and the limits below allow about 50 times that. Group responsibilities are a normalise_exp of
sums over a cell's reads, so their float error grows with the cell count: 8e-9 here, 1.5e-5 on the 200-cell copy-number workload
of tools/bench_variational_bayes_mixture_mixture.py; SIGMA_ABS allows about 7 times the latter."""
import numpy as np
import pytest

import vbmm_cases
import vbmm_exact
from vbmm_ref import RefVBMM

EVIDENCE_REL = 1e-7
WEIGHTED_ABS = 2e-6
SIGMA_ABS = 1e-4
CONCENTRATION_REL = 5e-5

pytestmark = pytest.mark.skipif(not RefVBMM.available(), reason="reference mixture-of-mixtures VB not built (oracle/_ref/libref_vbmm.so)")

CASES = {
    "T2 K[2,2] scalar": dict(H=6, reads=[7, 0, 5, 1, 9], sizes=[2, 2], C=40, n_seeds=4),
    "T3 K[1,2,3] priors full": dict(H=6, reads=[7, 0, 5, 1, 9], sizes=[1, 2, 3], C=40, n_seeds=4, priors="some", conc="full"),
    "T4 K[2,2,2,2] priors": dict(H=5, reads=[3, 12, 0, 4], sizes=[2, 2, 2, 2], C=30, n_seeds=3, priors="some"),
    "T5 K[2,2,2,2,2] priors scalar": dict(H=6, reads=[7, 0, 5, 1, 9], sizes=[2, 2, 2, 2, 2], C=40, n_seeds=4, priors="some"),
    "T3 K[1,1,1] full dup": dict(H=4, reads=[6, 6, 2], sizes=[1, 1, 1], C=20, n_seeds=3, conc="full", dup=True),
}


def _args(c, seed=3):
    x = vbmm_cases.make(c["H"], c["reads"], c["sizes"], c["C"], c["n_seeds"], seed=seed, dup=c.get("dup", False),
                        priors=c.get("priors"), concentrations=c.get("conc", "scalar"))
    return (x["lnl"], x["off"], x["sizes"], x["gt"], x["lp"], x["gc"], x["mc"], x["seeds"], x["gp"], x["mask"])


@pytest.mark.parametrize("name", list(CASES))
def test_restatement_matches_the_reference(name):
    args = _args(CASES[name])
    r = RefVBMM().run(*args, epsilon=0.05, max_iterations=1000)
    want = vbmm_exact.run(*args, epsilon=0.05, max_iterations=1000)
    flagged = [vbmm_exact.near_threshold(s["decisions"], 0.05, rel=1e-6) for s in want["seeds"]]
    for i, s in enumerate(want["seeds"]):
        assert s["iterations"] == r["seed_iterations"][i] or flagged[i], (i, s["iterations"], r["seed_iterations"][i])
        if not flagged[i]:
            assert abs(float(s["evidence"]) - r["seed_log_evidences"][i]) <= EVIDENCE_REL * abs(r["seed_log_evidences"][i])
    assert not any(flagged), "a case near a stopping threshold compares nothing; pick another seed"
    assert want["max_seed"] == r["max_seed"]
    assert np.max(np.abs(np.asarray(want["weighted"], float) - r["weighted"])) <= WEIGHTED_ABS
    assert np.max(np.abs(np.asarray(want["weighted_group_responsibilities"], float) - r["weighted_group_responsibilities"])) <= SIGMA_ABS
    assert np.max(np.abs(np.asarray(want["group_responsibilities"], float) - r["group_responsibilities"])) <= SIGMA_ABS
    mc = np.asarray(want["mixture_concentrations"], float)
    assert np.max(np.abs(mc - r["mixture_concentrations"]) / mc) <= CONCENTRATION_REL
    gc = np.asarray(want["group_concentrations"], float)
    assert np.max(np.abs(gc - r["group_concentrations"]) / gc) <= CONCENTRATION_REL
    assert abs(float(want["max_log_evidence"]) - r["max_log_evidence"]) <= EVIDENCE_REL * abs(r["max_log_evidence"])


def test_the_reference_does_not_reset_tau_for_later_groups():
    """Without the t > 0 quirk (tau reset for every group, as the model would have it) the restatement leaves the reference's
    evidences by far more than the float tolerance; with it, it agrees."""
    args = _args(CASES["T3 K[1,2,3] priors full"])
    r = RefVBMM().run(*args, epsilon=0.05, max_iterations=1000)
    with_quirk = vbmm_exact.run(*args, epsilon=0.05, max_iterations=1000)
    without = vbmm_exact.run(*args, epsilon=0.05, max_iterations=1000, quirk=False)
    dev = lambda res: max(abs(float(s["evidence"]) - e) / abs(e) for s, e in zip(res["seeds"], r["seed_log_evidences"]))
    assert dev(with_quirk) <= EVIDENCE_REL
    assert dev(without) > 100 * EVIDENCE_REL, dev(without)


def test_grouped_form_equals_the_combination_indexed_form():
    args = _args(CASES["T3 K[1,2,3] priors full"])
    a = vbmm_exact.run(*args, epsilon=0.05, max_iterations=50, direct=True)
    b = vbmm_exact.run(*args, epsilon=0.05, max_iterations=50)
    for sa, sb in zip(a["seeds"], b["seeds"]):
        assert sa["iterations"] == sb["iterations"]
        assert np.allclose(np.asarray(sa["lpost"], float), np.asarray(sb["lpost"], float), rtol=1e-14, atol=1e-14)
        assert abs(float(sa["evidence"]) - float(sb["evidence"])) <= 1e-14 * abs(float(sa["evidence"]))


def test_a_padded_component_can_take_a_whole_read():
    """A read whose real components' ln rho all lie below -10000 (lowest() likelihoods) goes wholly to the padded components."""
    lnl = np.array([[-1.0, vbmm_cases.LOWEST], [-2.0, -3.0]])
    P = vbmm_exact._Problem(lnl, [0, 2], [1, 2], np.array([[0, 0, 1]], np.int32), [0.0], [1.0, 1.0], [[1.0, 1.0, 1.0]], None, None,
                            False, True)
    taus = P.components(P.mc0, np.ones(1, dtype=vbmm_exact.LD), None)
    assert float(taus[0][0][0][1]) == 0.0 and float(taus[0][0][1][1]) == 1.0      # group 0 (K_t = 1): read 1 is the padded slot's
    assert abs(float(taus[0][0][0][0]) - 1.0) < 1e-15
