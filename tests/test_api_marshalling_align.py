"""The ctypes mirror's assign and realign requests through the shared engine, against the recording stand-in for libphmm_b200.so of
test_api_marshalling.py: PopulateBatcher.assign_reads / realign_reads call the batcher's entry points with the arguments the
engine's methods pass (without the memory space), return what the engine's methods return, and raise with the batcher's message.
Needs neither a GPU nor the built library."""
import ctypes as C

import numpy as np
import pytest

from octopus_b200 import _lib
from octopus_b200.api import PopulateBatcher, ShortHaplotypeError
from octopus_b200.batch import pack_haplotypes, pack_reads
from test_api_marshalling import CFG, CS, ERRORS, FLANK, HS, RS, STRIDE, Stub, host, raises, write_cigars  # noqa: F401


@pytest.fixture
def stub(monkeypatch):
    s = Stub()
    monkeypatch.setattr(_lib, "load", lambda: s)
    return s


@pytest.fixture
def blocks(stub):
    seqs = [b"ACGTACGTACGTACGT", b"ACGTACGTACGTACGTAC"]
    z = lambda dt: [np.zeros(len(s), dt) for s in seqs]      # noqa: E731
    haps = pack_haplotypes(seqs, z(np.uint8), z(np.int8), z(np.uint8), z(np.int8), z(np.int8), z(np.int8))
    reads = pack_reads([b"ACGT", b"CGTAC", b"GTACGT"], [np.full(n, 30, np.uint8) for n in (4, 5, 6)])
    stub.register("haps.", haps.arrays())
    stub.register("reads.", reads.arrays())
    return haps, reads


@pytest.fixture
def batcher(stub):
    b = PopulateBatcher()
    stub.calls.clear()
    return b


def test_batcher_assign_reads(stub, batcher, blocks):
    haps, reads = blocks
    hf, rf = [0, 2], [0, 3]
    pri = np.log([0.25, 0.75])
    stub.register("", {"pri": pri})

    def effect(h, c, hs, rs, regs, p, top, lnl, status):
        host(top, C.c_uint64, 3)[:] = [1, 2, 3]
        if lnl:
            host(lnl, C.c_double, 6)[:] = -4
        if status:
            host(status, C.c_int32, 6)[:] = 1
    stub.effects["phmm_batcher_assign_reads"] = effect
    top = batcher.assign_reads(CFG, haps, reads, hf, rf)
    args = stub.only("phmm_batcher_assign_reads")
    assert args[:6] == ["handle", CS, HS, RS, {"n": 1, "hap_first": [0, 2], "read_first": [0, 3], "flank": None}, None]
    assert args[7:] == [None, None]
    assert top.dtype == np.uint64 and top.tolist() == [1, 2, 3]
    stub.calls.clear()
    top, lnl, status = batcher.assign_reads(CFG, haps, reads, hf, rf, pri, want_likelihoods=True, want_status=True)
    assert stub.only("phmm_batcher_assign_reads")[5] == "pri"
    assert lnl.tolist() == [-4] * 6 and status.dtype == np.int32 and status.tolist() == [1] * 6
    with pytest.raises(ValueError):
        batcher.assign_reads(CFG, haps, reads, hf, rf, [0.0])
    raises(stub, "phmm_batcher_assign_reads", lambda: batcher.assign_reads(CFG, haps, reads, hf, rf), "batcher says no")
    # with statuses a short haplotype is no failure, as on the engine
    stub.rc["phmm_batcher_assign_reads"] = _lib.PHMM_ERR_SHORT_HAPLOTYPE
    batcher.assign_reads(CFG, haps, reads, hf, rf, want_status=True)
    with pytest.raises(ShortHaplotypeError):
        batcher.assign_reads(CFG, haps, reads, hf, rf)


def test_batcher_realign_reads(stub, batcher, blocks):
    haps, reads = blocks
    pairs = np.array([[0, 0], [2, 1]], np.int32)
    stub.register("", {"pairs": pairs})
    stub.effects["phmm_batcher_realign_reads"] = write_cigars(STRIDE, cg=9, st=11)
    mp, lk, cigars, st = batcher.realign_reads(CFG, haps, reads, pairs, flank_state=(3, 4))
    args = stub.only("phmm_batcher_realign_reads")
    assert args[:7] == ["handle", CS, HS, RS, "pairs", 2, FLANK] and args[10] == STRIDE and len(args) == 12
    assert cigars == ["1M", "2M"] and mp.tolist() == [100, 101] and st.tolist() == [0, 1] and lk.dtype == np.float64
    stub.calls.clear()
    batcher.realign_reads(CFG, haps, reads, pairs, cigar_stride=30)
    args = stub.only("phmm_batcher_realign_reads")
    assert args[6] is None and args[10] == 30
    raises(stub, "phmm_batcher_realign_reads", lambda: batcher.realign_reads(CFG, haps, reads, pairs), "batcher says no")


def test_batcher_reruns(stub, batcher):
    stub.effects["phmm_batcher_reruns"] = lambda h: 3
    assert batcher.reruns() == 3
