"""DeNovoModel's context indel model (phmm_mutation_context, host C++) against the UNMODIFIED reference IndelMutationModel::evaluate
(oracle/_ref/libref_mutation.so), value for value; and the C restatement of recalculate_log_probability (tests/cpp/mutation_oracle.c)
against the reference DeNovoModel on the pairs it aligns with the HMM. No GPU needed."""
import os
import subprocess
import tempfile

import numpy as np
import pytest

from mutation_oracle import SOMATIC_PRIORS, TRIO_PRIORS, RefMutation, haplotype_set, log_table, penalty, recalculate, repeat_sequence
from octopus_b200 import MutationModel, PhmmError
from oracle import oracle as O
from oracle.oracle import RefHMM

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))

needs_ref = pytest.mark.skipif(not RefMutation.available(), reason="reference mutation model not built (oracle/_ref/libref_mutation.so)")
# a high indel prior makes several cells reach the 0.9 open cap: equal open probabilities from different cells, where order decides
INDEL_PRIORS = [TRIO_PRIORS[1], SOMATIC_PRIORS[1], 1e-2, 0.2]


def _check_context(ref, model, indel_prior, sequences):
    o, e = ref.table(indel_prior)
    flat_o, flat_e = o.reshape(-1), e.reshape(o.size, -1)
    cell, op, ep = model.context(sequences)
    at = 0
    for s in sequences:
        go, ge = ref.context(indel_prior, s)
        c = cell[at:at + len(s)]
        assert np.array_equal(flat_o[c].view(np.uint32), go.view(np.uint32)), s
        assert np.array_equal(flat_e[c].view(np.uint32), ge.view(np.uint32)), s
        assert np.array_equal(op[at:at + len(s)], [penalty(float(x)) for x in go]), s
        assert np.array_equal(ep[at:at + len(s)], [penalty(float(x)) for x in ge[:, 1]]), s
        at += len(s)


@needs_ref
@pytest.mark.parametrize("indel_prior", INDEL_PRIORS)
def test_context_random(indel_prior):
    ref = RefMutation()
    o, e = ref.table(indel_prior)
    model = MutationModel(TRIO_PRIORS[0], o, e)
    rng = np.random.default_rng(int(indel_prior * 1e12) % 1000 + 7)
    _check_context(ref, model, indel_prior, [repeat_sequence(rng) for _ in range(1500)])


@needs_ref
def test_context_constructed():
    ref = RefMutation()
    prior = 1e-2
    o, e = ref.table(prior)
    model = MutationModel(TRIO_PRIORS[0], o, e)
    seqs = ["A" * 120, "AC" * 60 + "G", "T" + "ACG" * 70, "ACGTA" * 55, "GATTACA" + "CA" * 52,       # > 50 periods, touching either end
            "CA" * 8 + "T" + "CAG" * 6 + "T" + "AAAAAAAA",                                          # capped cells of equal open probability
            "NNNN" + "AC" * 10 + "NN" + "A" * 9 + "N" + "CT" * 4 + "NNNNNNN",                       # N runs around and between repeats
            "ACACACNNNNNAC", "AAAANNNNAAAA", "N", "NN", "A", "ACGT" * 3 + "NNN", "NACNNACNN" * 4,
            "ACGTN" * 12, "C" * 3 + "N" * 20 + "G" * 3]
    _check_context(ref, model, prior, seqs)


@needs_ref
@pytest.mark.skipif(not RefHMM.available(), reason="reference HMM layer not built (oracle/_ref/libref_hmm.so)")
@pytest.mark.parametrize("priors", [TRIO_PRIORS, SOMATIC_PRIORS])
def test_rescoring_matches_reference(priors):
    """On every pair the reference scores with the HMM: its own alignment (the compiled hmm::align), re-scored by the C restatement over
    the library's context model, equals DeNovoModel::evaluate bit for bit."""
    ref, hmm = RefMutation(), RefHMM()
    snv, indel = priors
    o, e = ref.table(indel)
    model = MutationModel(snv, o, e)
    logp = log_table(o, e)
    rng = np.random.default_rng(11)
    checked = 0
    for _ in range(6):
        seqs = haplotype_set(rng, 10, max_len=160)
        want, approx = ref.prime(snv, indel, seqs)
        cell, op, ep = model.context(seqs)
        starts = np.concatenate([[0], np.cumsum([len(s) for s in seqs])])
        for t in range(len(seqs)):
            for g in range(len(seqs)):
                if t == g or approx[t, g]:
                    continue
                given, target = seqs[g], seqs[t]
                size = max(len(given), len(target)) + 64                      # pad_given (denovo_model.cpp:135-143)
                truth = "N" * 32 + given + "N" * (size - 32 - len(given))
                go = np.full(size, 60, np.int8); ge = np.full(size, 60, np.int8)
                go[32:32 + len(given)] = op[starts[g]:starts[g + 1]]
                ge[32:32 + len(given)] = ep[starts[g]:starts[g + 1]]
                rc, off, _, cigar = hmm.align_mutation_model(truth, target, penalty(snv), go, ge)
                assert rc == 0 and off == 32
                st, v = recalculate(cigar, cell[starts[g]:starts[g + 1]], logp, snv)
                assert st == 0
                assert np.float64(v).view(np.uint64) == np.float64(want[t, g]).view(np.uint64), (t, g, cigar, v, want[t, g])
                checked += 1
    assert checked > 200


def test_model_argument_checks():
    o = np.full((11, 51), 1e-9, np.float32)
    e = np.full((11, 51, 50), 0.5, np.float32)
    MutationModel(1e-8, o, e)
    for snv in (0.0, -1e-3, 1.5, float("nan")):
        with pytest.raises(PhmmError):
            MutationModel(snv, o, e)
    with pytest.raises(PhmmError):                       # periods up to 5 must exist
        MutationModel(1e-8, o[:5], e[:5])
    with pytest.raises(PhmmError):                       # extend[1] must exist
        MutationModel(1e-8, o, e[:, :, :1])
    for bad in (0.0, 1.5, float("nan")):
        o2 = o.copy(); o2[3, 7] = bad
        with pytest.raises(PhmmError):
            MutationModel(1e-8, o2, e)
        e2 = e.copy(); e2[2, 4, 9] = bad
        with pytest.raises(PhmmError):
            MutationModel(1e-8, o, e2)


@needs_ref
@pytest.mark.skipif(not O.have_reference(), reason="needs the reference checkout's indel_mutation_model_config.hpp")
@pytest.mark.parametrize("indel_prior", INDEL_PRIORS)
def test_cpp_adapter_table_from_reference_header(indel_prior):
    """MutationRepeatTable::from_reference, compiled against the reference's own config header, equals the compiled constructor's table."""
    exe = os.path.join(tempfile.mkdtemp(prefix="test_mutation_table_"), "test_mutation_table")
    subprocess.run(["g++", "-std=c++14", "-O1", "-I", os.path.join(O.REFERENCE, "src"), "-I", os.path.join(ROOT, "include"),
                    "-I", os.path.join(ROOT, "octopus_b200", "cpp"), os.path.join(ROOT, "tests", "cpp", "test_mutation_table.cpp"), "-o", exe,
                    "-L", os.path.join(ROOT, "octopus_b200"), "-lphmm_b200", "-Wl,-rpath," + os.path.join(ROOT, "octopus_b200")], check=True)
    lines = subprocess.run([exe, repr(indel_prior)], capture_output=True, text=True, check=True).stdout.splitlines()
    o, e = RefMutation().table(indel_prior)
    assert [int(x) for x in lines[0].split()] == [o.shape[0] - 1, o.shape[1] - 1, e.shape[2]]
    got_o = np.array([float.fromhex(x) for x in lines[1].split()], dtype=np.float32)
    got_e = np.array([float.fromhex(x) for x in lines[2].split()], dtype=np.float32)
    assert np.array_equal(got_o.view(np.uint32), o.reshape(-1).view(np.uint32))
    assert np.array_equal(got_e.view(np.uint32), e.reshape(-1).view(np.uint32))
