"""The ctypes mirror's template assignment, against the recording stand-in for libphmm_b200.so of test_api_marshalling.py:
PairHMMEngine.assign_templates and PopulateBatcher.assign_templates call phmm_assign_templates / phmm_batcher_assign_templates with
the groups' read bounds derived from their first templates, the template offsets in host memory and outputs sized per template
(top, likelihoods) and per read (statuses); they return what the call wrote and raise with the handle's message. Needs neither a GPU
nor the built library."""
import ctypes as C

import numpy as np
import pytest

from octopus_b200 import _lib
from octopus_b200.api import PairHMMEngine, PopulateBatcher, ShortHaplotypeError
from test_api_marshalling import CFG, CS, HS, RS, Stub, host, raises

TOFF = [0, 2, 3]          # templates {0, 1} and {2}
TF = [0, 1, 2]            # group 0: template 0 (reads 0-1), group 1: template 1 (read 2)
HF = [0, 1, 2]


@pytest.fixture
def stub(monkeypatch):
    s = Stub()
    monkeypatch.setattr(_lib, "load", lambda: s)
    return s


@pytest.fixture
def blocks(stub):
    from octopus_b200.batch import pack_haplotypes, pack_reads
    seqs = [b"ACGTACGTACGTACGT", b"ACGTACGTACGTACGTAC"]
    z = lambda dt: [np.zeros(len(s), dt) for s in seqs]      # noqa: E731
    haps = pack_haplotypes(seqs, z(np.uint8), z(np.int8), z(np.uint8), z(np.int8), z(np.int8), z(np.int8))
    reads = pack_reads([b"ACGT", b"CGTAC", b"GTACGT"], [np.full(n, 30, np.uint8) for n in (4, 5, 6)])
    stub.register("haps.", haps.arrays())
    stub.register("reads.", reads.arrays())
    return haps, reads


def effect(seen):
    """Records the template offsets the call was given; writes top per template, likelihoods per (haplotype, template) of the
    groups and statuses per (haplotype, read)."""
    def call(h, c, hs, rs, regs, toff, n, p, top, lnl, status, *space):
        seen.append(list(host(toff, C.c_int64, n + 1)))
        host(top, C.c_uint64, n)[:] = [3, 1]
        if lnl:
            host(lnl, C.c_double, 2)[:] = [-4, -5]
        if status:
            host(status, C.c_int32, 3)[:] = [1, 2, 3]
    return call


def check(stub, name, method, args_tail):
    seen = []
    stub.effects[name] = effect(seen)
    top = method(CFG, *stub.blocks, TOFF, HF, TF)
    args = stub.only(name)
    assert args[:5] == ["handle", CS, HS, RS, {"n": 2, "hap_first": HF, "read_first": [0, 2, 3], "flank": None}]
    assert args[6] == 2 and args[7] is None and args[9:] == [None, None] + args_tail
    assert seen == [TOFF] and top.dtype == np.uint64 and top.tolist() == [3, 1]
    stub.calls.clear()
    pri = np.log([0.25, 0.75])
    stub.register("", {"pri": pri})
    top, lnl, status = method(CFG, *stub.blocks, np.array(TOFF, np.int64), HF, TF, pri, want_likelihoods=True, want_status=True)
    assert stub.only(name)[7] == "pri"
    assert lnl.tolist() == [-4, -5] and status.dtype == np.int32 and status.tolist() == [1, 2, 3]
    with pytest.raises(ValueError):
        method(CFG, *stub.blocks, TOFF, HF, TF, [0.0])
    with pytest.raises(ValueError):
        method(CFG, *stub.blocks, TOFF, HF, [0, 1, 7])
    stub.effects.pop(name)


def test_engine_assign_templates(stub, blocks):
    e = PairHMMEngine(0)
    stub.calls.clear()
    stub.blocks = blocks
    check(stub, "phmm_assign_templates", e.assign_templates, [_lib.SPACE_HOST])
    raises(stub, "phmm_assign_templates", lambda: e.assign_templates(CFG, *blocks, TOFF, HF, TF), "engine says no")
    stub.rc["phmm_assign_templates"] = _lib.PHMM_ERR_SHORT_HAPLOTYPE
    e.assign_templates(CFG, *blocks, TOFF, HF, TF, want_status=True)
    with pytest.raises(ShortHaplotypeError):
        e.assign_templates(CFG, *blocks, TOFF, HF, TF)


def test_batcher_assign_templates(stub, blocks):
    b = PopulateBatcher()
    stub.calls.clear()
    stub.blocks = blocks
    check(stub, "phmm_batcher_assign_templates", b.assign_templates, [])
    raises(stub, "phmm_batcher_assign_templates", lambda: b.assign_templates(CFG, *blocks, TOFF, HF, TF), "batcher says no")
    stub.rc["phmm_batcher_assign_templates"] = _lib.PHMM_ERR_SHORT_HAPLOTYPE
    b.assign_templates(CFG, *blocks, TOFF, HF, TF, want_status=True)
    with pytest.raises(ShortHaplotypeError):
        b.assign_templates(CFG, *blocks, TOFF, HF, TF)
