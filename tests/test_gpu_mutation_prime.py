"""phmm_mutation_prime (DeNovoModel::prime + evaluate on the device) against the UNMODIFIED reference DeNovoModel compiled from the
checkout (oracle/_ref/libref_mutation.so): every HMM / SELF value bit for bit, and the pairs sent to the approximate path exactly those
whose Haplotype::difference stand-in was called. Also constructed edge cases, a multi-tile call against phmm_align_pairs + the C
re-scoring, and the argument checks."""
import os
import subprocess
import tempfile

import numpy as np
import pytest

from mutation_oracle import SOMATIC_PRIORS, TRIO_PRIORS, RefMutation, align_pairs_recipe, haplotype_set, mutate, repeat_sequence
from octopus_b200 import MutationModel, PhmmError, _lib

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
pytestmark = pytest.mark.gpu
needs_ref = pytest.mark.skipif(not RefMutation.available(), reason="reference mutation model not built (oracle/_ref/libref_mutation.so)")
APPROX = (_lib.MUT_APPROX_LENGTH, _lib.MUT_APPROX_OFFSET, _lib.MUT_APPROX_OVERFLOW)


@pytest.fixture(scope="module")
def ref():
    return RefMutation()


def _model(ref, priors):
    o, e = ref.table(priors[1])
    return MutationModel(priors[0], o, e), o, e


def _check(engine, ref, priors, seqs):
    model, _, _ = _model(ref, priors)
    out, status = engine.mutation_prime(model, seqs)
    want, approx = ref.prime(priors[0], priors[1], seqs)
    H = len(seqs)
    assert (np.diag(status) == _lib.MUT_SELF).all() and (np.diag(out) == 0.0).all()
    got_approx = np.isin(status, APPROX)
    assert np.array_equal(got_approx, approx), np.argwhere(got_approx != approx)[:10]
    hmm = status == _lib.MUT_HMM
    assert np.array_equal(out[hmm].view(np.uint64), want[hmm].view(np.uint64)), np.argwhere(hmm & (out != want))[:10]
    # an indel past the given haplotype: the reference reads past its model (no defined value); never an approximate pair there
    assert not (approx & (status == _lib.MUT_OUT_OF_MODEL)).any()
    assert ((status >= 0) & (status <= _lib.MUT_OUT_OF_MODEL)).all() and hmm.sum() + np.isin(status, APPROX).sum() + H + (status == 5).sum() == H * H
    return out, status


@needs_ref
@pytest.mark.parametrize("priors", [TRIO_PRIORS, SOMATIC_PRIORS], ids=["trio", "somatic"])
@pytest.mark.parametrize("n", [2, 12, 50, 51, 200])
def test_prime_matches_reference(engine, ref, priors, n):
    rng = np.random.default_rng(1000 + n)
    seqs = haplotype_set(rng, n, max_len=260 if n < 200 else 160, n_events=(0, 8))
    _, status = _check(engine, ref, priors, seqs)
    assert (status == _lib.MUT_HMM).sum() >= n * (n - 1) // 5


@needs_ref
def test_constructed_cases(engine, ref):
    rng = np.random.default_rng(5)
    base = repeat_sequence(rng, 200, n_runs=False) + "ACGTTGCA" * 5
    seqs = [base,
            base + "T" * 31,                                  # length distance 31: through the HMM
            base + "G" * 32,                                  # 32: approximate
            base[:len(base) - 20],                            # a prefix of the given haplotype: the naive alignment
            base,                                             # identical sequences
            base[:60] + base[91:],                            # a 31 bp deletion
            base[:60] + "ACGTACGTTTGACCAGTACCATTGCAACGTG" + base[60:],   # a 31 bp insertion
            base[:40] + "N" * 12 + base[52:],                 # an N run
            "NNNNNN" + base[6:]]
    _, status = _check(engine, ref, TRIO_PRIORS, seqs)
    assert _lib.MUT_APPROX_LENGTH not in (status[1, 0], status[0, 1], status[3, 0])
    assert status[2, 0] == _lib.MUT_APPROX_LENGTH and status[0, 2] == _lib.MUT_APPROX_LENGTH
    assert status[4, 0] == _lib.MUT_HMM


@needs_ref
def test_long_haplotypes(engine, ref):
    rng = np.random.default_rng(9)
    base = "".join(rng.choice(list("ACGT"), 1100)) + "CA" * 40 + "".join(rng.choice(list("ACGT"), 150))
    seqs = [base] + [mutate(rng, base, int(rng.integers(1, 10))) for _ in range(7)]
    _check(engine, ref, SOMATIC_PRIORS, seqs)


def test_multi_tile_call_matches_align_pairs_recipe(engine):
    """1 047 552 ordered pairs (two tiles) against phmm_align_pairs + host re-scoring of the same pairs, bit for bit."""
    rng = np.random.default_rng(21)
    o = np.full((11, 51), 1e-6, np.float32)
    o[1:6, 3:] = np.linspace(2e-6, 0.9, 48, dtype=np.float32)
    e = np.full((11, 51, 50), 0.3, np.float32)
    e[1:6, 3:, :] = 0.85
    model = MutationModel(1e-4, o, e)
    seqs = []
    for _ in range(32):                                       # 32 regions of 32 haplotypes, 40-70 bp, each with a short STR
        base = "".join(rng.choice(list("ACGT"), 40)) + "".join(rng.choice(list("ACGT"), int(rng.integers(1, 4)))) * int(rng.integers(2, 7))
        seqs += [base] + [mutate(rng, base, int(rng.integers(0, 3)))[:70] for _ in range(31)]
    assert len(seqs) == 1024
    small_out, _ = engine.mutation_prime(model, seqs[:16])
    one_tile = engine.launch_count()
    out, status = engine.mutation_prime(model, seqs)
    assert engine.launch_count() >= 2 * one_tile
    want, want_status = align_pairs_recipe(engine, model, o, e, seqs)
    assert np.array_equal(status, want_status)
    assert np.array_equal(out.view(np.uint64), want.view(np.uint64))
    assert np.array_equal(out[:16, :16].view(np.uint64), small_out.view(np.uint64))
    through_dp = np.isin(status, (_lib.MUT_HMM, _lib.MUT_APPROX_OFFSET, _lib.MUT_APPROX_OVERFLOW, _lib.MUT_OUT_OF_MODEL))
    assert through_dp.sum() > 524288 and (status == _lib.MUT_HMM).sum() > 20000      # more aligned pairs than one tile holds


def test_argument_checks(engine):
    o = np.full((11, 51), 1e-9, np.float32)
    e = np.full((11, 51, 50), 0.5, np.float32)
    model = MutationModel(1e-8, o, e)
    lib = _lib.load()
    off = np.array([0, 4, 8], np.int64)
    seq = np.frombuffer(b"ACGTACGA", np.uint8)
    out = np.zeros(4, np.float64)
    st = np.zeros(4, np.int32)
    h = engine._h
    args = [h, model._h, 2, off.ctypes.data, seq.ctypes.data, out.ctypes.data, st.ctypes.data]
    assert lib.phmm_mutation_prime(*args) == _lib.PHMM_OK
    for k in (1, 3, 4, 5, 6):
        bad = list(args)
        bad[k] = None
        assert lib.phmm_mutation_prime(*bad) == _lib.PHMM_ERR_INVALID
    assert lib.phmm_mutation_prime(None, *args[1:]) == _lib.PHMM_ERR_INVALID
    for n in (0, -1):
        bad = list(args)
        bad[2] = n
        assert lib.phmm_mutation_prime(*bad) == _lib.PHMM_ERR_INVALID
    with pytest.raises(PhmmError):
        engine.mutation_prime(model, ["ACGT", ""])                          # an empty haplotype
    with pytest.raises(PhmmError):
        engine.mutation_prime(model, ["A" * 65536, "A" * 65536])            # longer than the limit
    with pytest.raises(PhmmError):
        engine.mutation_prime(model, ["ACGT"] * 4097)                       # more haplotypes than the limit
    assert "4096" in lib.phmm_last_error(h).decode()


@needs_ref
def test_cpp_denovo_model(ref):
    """octopus_b200::SomaticMutationModel (= DeNovoModel) from a plain C++ program: prime, evaluate with the approx function for exactly
    the pairs the reference sends to its approximate path, the kept values on a second pass, unprime."""
    from octopus_b200 import build
    build.build()
    exe = os.path.join(tempfile.mkdtemp(prefix="test_denovo_"), "test_denovo")
    subprocess.run(["g++", "-std=c++14", "-O1", "-I", os.path.join(ROOT, "include"), "-I", os.path.join(ROOT, "octopus_b200", "cpp"),
                    os.path.join(ROOT, "tests", "cpp", "test_denovo.cpp"), "-o", exe, "-L", os.path.join(ROOT, "octopus_b200"), "-lphmm_b200",
                    "-Wl,-rpath," + os.path.join(ROOT, "octopus_b200")], check=True)
    snv, indel = SOMATIC_PRIORS
    o, e = ref.table(indel)
    rng = np.random.default_rng(77)
    seqs = haplotype_set(rng, 14, max_len=200, n_events=(0, 8)) + ["ACGT" * 30]          # the last one: length distance >= 32
    spec = os.path.join(os.path.dirname(exe), "set.txt")
    with open(spec, "w") as f:
        f.write("%r %d %d %d %d\n" % (snv, o.shape[0] - 1, o.shape[1] - 1, e.shape[2], len(seqs)))
        f.write(" ".join("%.9g" % x for x in o.reshape(-1)) + "\n")
        f.write(" ".join("%.9g" % x for x in e.reshape(-1)) + "\n")
        f.write("\n".join(seqs) + "\n")
    run = subprocess.run([exe, spec], capture_output=True, text=True, timeout=300)
    assert run.returncode == 0, run.stdout + run.stderr
    lines = [l.split() for l in run.stdout.splitlines()]
    want, approx = ref.prime(snv, indel, seqs)
    H = len(seqs)
    got = np.zeros((H, H))
    status = np.zeros((H, H), np.int32)
    for l in lines:
        if l[0] == "V":
            got[int(l[1]), int(l[2])] = float.fromhex(l[3])
            status[int(l[1]), int(l[2])] = int(l[4])
    asked = np.zeros((H, H), bool)
    for l in lines:
        if l[0] == "A":
            asked[int(l[1]), int(l[2])] = True
    assert np.array_equal(asked & ~(status == _lib.MUT_OUT_OF_MODEL), approx) and approx.any()
    t, g = np.nonzero(asked)
    assert np.array_equal(got[t, g], -1000.0 - (t * H + g))
    hmm = (status == _lib.MUT_HMM) | (status == _lib.MUT_SELF)
    assert np.array_equal(got[hmm].view(np.uint64), want[hmm].view(np.uint64))
    assert [l for l in lines if l[0] == "PRIMED"] == [["PRIMED", "1"], ["PRIMED", "0"]]
