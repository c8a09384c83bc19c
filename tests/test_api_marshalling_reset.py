"""The ctypes mirror's populate calls with an error model, against the recording stand-in for libphmm_b200.so of
test_api_marshalling.py: which _reset entry point each method calls, with the sequences block and the model handle in place of the
haplotype block. Needs neither a GPU nor the built library."""
import numpy as np
import pytest

from octopus_b200 import _lib
from octopus_b200.api import ErrorModel, HaplotypeLikelihoodArray, HaplotypeLikelihoodModel, PairHMMEngine, PopulateBatcher
from octopus_b200.batch import HaplotypeSequences, pack_reads
from test_api_marshalling import CFG, CS, FLANK, RS, Stub, host  # noqa: F401

SEQS = {"n": 2, "off": "seqs.off", "seq": "seqs.seq", "is_substitution": "seqs.is_substitution", "begin": "seqs.begin"}


@pytest.fixture
def stub(monkeypatch):
    s = Stub()
    monkeypatch.setattr(_lib, "load", lambda: s)
    return s


@pytest.fixture
def blocks(stub):
    seqs = HaplotypeSequences.pack([b"ACGTACGTACGTACGT", b"ACGTACGTACGTACGTAC"], begin=[5, 6],
                                   is_substitution=[np.zeros(16, np.uint8), np.ones(18, np.uint8)])
    reads = pack_reads([b"ACGT", b"CGTAC", b"GTACGT"], [np.full(n, 30, np.uint8) for n in (4, 5, 6)])
    stub.register("seqs.", seqs.arrays())
    stub.register("reads.", reads.arrays())
    return seqs, reads


def test_sequences_block_packs_flags_and_begins():
    s = HaplotypeSequences.pack(["ACG", b"TTTT"], begin=[1, 2], is_substitution=[[0, 1, 0], [1, 1, 0, 0]])
    assert s.n == 2 and list(s.off) == [0, 3, 7] and bytes(s.seq) == b"ACGTTTT"
    assert list(s.is_substitution) == [0, 1, 0, 1, 1, 0, 0] and list(s.begin) == [1, 2]
    bare = HaplotypeSequences.pack(["AC"])
    assert bare.is_substitution is None and bare.begin is None


def test_engine_populate_calls_the_reset_twins(stub, blocks):
    seqs, reads = blocks
    model = ErrorModel("PCR.NovaSeq")
    e = PairHMMEngine(0)
    stub.calls.clear()
    out = e.populate(CFG, seqs, reads, flank_state=(3, 4), error_model=model)
    assert out.shape == (2, 3) and out.dtype == np.float64
    assert stub.only("phmm_populate_reset")[:7] == ["handle", CS, "handle", SEQS, RS, None, FLANK]
    assert stub.only("phmm_populate_reset")[-1] == _lib.SPACE_HOST
    e.populate_regions(CFG, seqs, reads, [0, 1, 2], [0, 2, 3], error_model=model)
    args = stub.only("phmm_populate_regions_reset")
    assert args[:5] == ["handle", CS, "handle", SEQS, RS] and args[5]["hap_first"] == [0, 1, 2]
    t = e.populate_templates(CFG, seqs, reads, [0, 1, 3], error_model=model)
    assert t.shape == (2, 2) and stub.only("phmm_populate_templates_reset")[:5] == ["handle", CS, "handle", SEQS, RS]
    assert not [n for n, _ in stub.calls if n in ("phmm_populate", "phmm_populate_regions", "phmm_populate_templates")]
    with pytest.raises(TypeError):
        e.populate(CFG, model.reset([b"ACGT"]), reads, error_model=model)


def test_batcher_and_array_call_the_reset_twins(stub, blocks):
    seqs, reads = blocks
    model = ErrorModel()
    b = PopulateBatcher()
    b.populate(CFG, seqs, reads, error_model=model)
    assert stub.only("phmm_batcher_populate_reset")[:5] == ["handle", CS, "handle", SEQS, RS]
    b.populate_templates(CFG, seqs, reads, [0, 3], error_model=model, want_status=True)
    assert stub.only("phmm_batcher_populate_templates_reset")[:5] == ["handle", CS, "handle", SEQS, RS]
    arr = HaplotypeLikelihoodArray(HaplotypeLikelihoodModel(CFG), PairHMMEngine(), error_model=model)
    arr.populate({"s1": reads, "s2": reads}, seqs)
    assert len([n for n, _ in stub.calls if n == "phmm_populate_reset"]) == 1
    merged = arr.merge_samples()
    assert merged.error_model is model
