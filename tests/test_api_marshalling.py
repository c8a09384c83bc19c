"""The ctypes mirror's marshalling on the host path, against a recording stand-in for libphmm_b200.so: which entry point each
public method calls, with which struct contents, sizes, strides and memory space; the shapes and dtypes it returns; which
exception each failure code becomes; and the second call of the grow-and-retry loops. Needs neither a GPU nor the built library."""
import ctypes as C

import numpy as np
import pytest

from octopus_b200 import _lib
from octopus_b200.api import (ErrorModel, HaplotypeLikelihoodModel, MutationModel, PairHMMEngine, PhmmError, PopulateBatcher,
                              ShortHaplotypeError, TooLargeBandSizeError)
from octopus_b200.batch import pack_haplotypes, pack_reads

HANDLE = 0x5150
MESSAGES = {"phmm_last_error": b"engine says no", "phmm_batcher_last_error": b"batcher says no",
            "phmm_error_model_last_error": b"model says no"}
CREATE = ("phmm_create", "phmm_batcher_create", "phmm_error_model_create", "phmm_error_model_create_custom",
          "phmm_mutation_model_create")
ERRORS = [(_lib.PHMM_ERR_SHORT_HAPLOTYPE, ShortHaplotypeError), (_lib.PHMM_ERR_BAND, TooLargeBandSizeError),
          (_lib.PHMM_ERR_INVALID, PhmmError)]


def host(ptr, ctype, n):
    """numpy view of n host values at a pointer the stub was given."""
    return np.ctypeslib.as_array((ctype * n).from_address(ptr)) if n else np.zeros(0, np.dtype(ctype))


def fields(s):
    return {f: getattr(s, f) for f, _ in s._fields_}


class Stub:
    """Answers every phmm_* call: records (name, arguments decoded to values), runs effects[name](raw arguments) if set, and returns
    rc[name] (PHMM_OK by default) or what the effect returns. The create functions hand out HANDLE."""

    def __init__(self):
        self.calls, self.rc, self.effects, self.names = [], {}, {}, {}

    def register(self, prefix, arrays):
        for f, a in arrays.items():
            self.names[a.ctypes.data] = (prefix + f, a)       # the array itself is kept alive, so its address stays its own

    def decode(self, x):
        if isinstance(x, int):
            return self.names[x][0] if x in self.names else x
        if isinstance(x, C.c_void_p):
            return "handle" if x.value == HANDLE else x.value
        x = getattr(x, "_obj", x)                             # C.byref(...)
        if isinstance(x, _lib.Regions):
            flank = None if not x.flank else [tuple(fields(f).values()) for f in (_lib.FlankState * x.n).from_address(x.flank)]
            return {"n": x.n, "hap_first": list(host(x.hap_first, C.c_int32, x.n + 1)),
                    "read_first": list(host(x.read_first, C.c_int32, x.n + 1)), "flank": flank}
        if isinstance(x, C.Structure):
            return {f: self.decode(v) for f, v in fields(x).items()}
        if isinstance(x, C.Array):
            return "buffer[%d]" % len(x)
        if isinstance(x, C._SimpleCData):
            return x.value
        return x

    def __getattr__(self, name):
        if not name.startswith("phmm_"):
            raise AttributeError(name)
        if name in MESSAGES:
            return lambda *a: MESSAGES[name]

        def call(*args):
            if name in CREATE:
                self.calls.append((name, [self.decode(a) for a in args[1:]]))
            else:
                self.calls.append((name, [self.decode(a) for a in args]))
            got = self.effects[name](*args) if name in self.effects else None
            rc = self.rc.get(name, _lib.PHMM_OK)
            if name in CREATE and rc == _lib.PHMM_OK:
                args[0]._obj.value = HANDLE
            return got if got is not None else rc
        return call

    def only(self, name):
        got = [a for n, a in self.calls if n == name]
        assert len(got) == 1, (name, self.calls)
        return got[0]


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


HS = {"n": 2, "off": "haps.off", "seq": "haps.seq", "snv_mask_fwd": "haps.snv_mask_fwd", "snv_prior_fwd": "haps.snv_prior_fwd",
      "snv_mask_rev": "haps.snv_mask_rev", "snv_prior_rev": "haps.snv_prior_rev", "gap_open": "haps.gap_open",
      "gap_extend": "haps.gap_extend", "begin": None}
RS = {"n": 3, "off": "reads.off", "bases": "reads.bases", "quals": "reads.quals", "mapq": "reads.mapq", "reverse": "reads.reverse",
      "begin": "reads.begin"}
STRIDE = 4 * 6 + 64          # the default CIGAR stride: 4 x the longest read + 64
CFG = HaplotypeLikelihoodModel.Config(max_indel_error=16, mapping_quality_cap_trigger=100, use_flank_state=False)
CS = fields(CFG.c_struct())
FLANK = {"has_flank": 1, "lhs_flank": 3, "rhs_flank": 4}


@pytest.fixture
def engine(stub):
    e = PairHMMEngine(2)
    assert stub.calls == [("phmm_create", [2])]
    stub.calls.clear()
    return e


def raises(stub, name, call, message, codes=ERRORS):
    """Each failure code of `name` raises its exception class with the handle's own message."""
    for rc, cls in codes:
        stub.rc[name] = rc
        with pytest.raises(cls) as e:
            call()
        assert e.value.code == rc and str(e.value) == "phmm error %d: %s" % (rc, message)
    stub.rc.pop(name)


def write_cigars(stride, cg=10, st=12, mp=None):
    """Effect for the aligning calls: CIGAR j is '<j+1>M', status j is j, mapping position j is 100 + j."""
    def effect(*a):
        n = a[5] if mp is None else a[mp]
        for j in range(n):
            text = b"%dM" % (j + 1)
            C.memmove(a[cg] + j * a[cg + 1], text, len(text))
        host(a[st], C.c_int32, n)[:] = np.arange(n)
        host(a[cg - 2], C.c_int64, n)[:] = 100 + np.arange(n)
    return effect


# -- handles -----------------------------------------------------------------------------------------------------------
def test_engine_handle_lifetime_and_creation_failure(stub):
    with PairHMMEngine() as e:
        assert stub.calls == [("phmm_create", [-1])]
    assert stub.calls[-1] == ("phmm_destroy", ["handle"])
    e.close()
    assert len(stub.calls) == 2
    stub.rc["phmm_create"] = _lib.PHMM_ERR_BAND
    with pytest.raises(PhmmError) as ex:
        PairHMMEngine(0)
    assert type(ex.value) is PhmmError and str(ex.value) == "phmm error -3: engine says no"


def test_engine_stream_calls(stub, engine):
    engine.wait_event(7)
    engine.reserve_sms(4)
    assert stub.calls == [("phmm_wait_event", ["handle", 7]), ("phmm_reserve_sms", ["handle", 4])]
    raises(stub, "phmm_reserve_sms", lambda: engine.reserve_sms(1), "engine says no")


def test_batcher_handle_options_stats_and_creation_failure(stub):
    PopulateBatcher().close()
    PopulateBatcher(clients=4).close()
    with PopulateBatcher(max_wait_us=100) as b:
        pass
    created = [a for n, a in stub.calls if n == "phmm_batcher_create"]
    assert created == [[-1, None], [-1, {"clients": 4, "max_wait_us": 500}], [-1, {"clients": 0, "max_wait_us": 100}]]
    assert [n for n, _ in stub.calls].count("phmm_batcher_destroy") == 3

    def fill(h, s):
        for i, (f, _) in enumerate(_lib.BatcherStats._fields_):
            setattr(s._obj, f, i + 1)
    stub.effects["phmm_batcher_stats_get"] = fill
    assert b.stats() == {"requests": 1, "gpu_calls": 2, "merged_calls": 3, "max_regions_per_call": 4, "dp_cells": 5}
    stub.rc["phmm_batcher_create"] = _lib.PHMM_ERR_SHORT_HAPLOTYPE
    with pytest.raises(PhmmError) as ex:
        PopulateBatcher()
    assert type(ex.value) is PhmmError and str(ex.value) == "phmm error -4: batcher says no"


def test_model_handles_are_destroyed(stub):
    m = ErrorModel("PCR.NovaSeq")
    del m
    t = MutationModel(1e-8, np.zeros((2, 3), np.float32), np.zeros((2, 3, 4), np.float32))
    del t
    names = [n for n, _ in stub.calls]
    assert names == ["phmm_error_model_create", "phmm_error_model_destroy", "phmm_mutation_model_create", "phmm_mutation_model_destroy"]


# -- PairHMMEngine ------------------------------------------------------------------------------------------------------
def test_mutation_prime(stub, engine):
    open_, extend = np.full((2, 3), 0.5, np.float32), np.full((2, 3, 4), 0.25, np.float32)
    stub.register("table.", {"open": open_, "extend": extend})
    model = MutationModel(1e-8, open_, extend)
    assert stub.calls[-1] == ("phmm_mutation_model_create", [1e-8, "table.open", "table.extend", 1, 2, 4])
    seen = {}

    def effect(h, m, n, off, seq, out, status):
        o = host(off, C.c_int64, n + 1)
        seen.update(off=list(o), seq=C.string_at(seq, int(o[-1])))
        host(out, C.c_double, n * n)[:] = np.arange(n * n)
        host(status, C.c_int32, n * n)[:] = 5
    stub.effects["phmm_mutation_prime"] = effect
    out, status = engine.mutation_prime(model, ["ACG", b"TT", np.frombuffer(b"GGGG", np.uint8)])
    assert stub.only("phmm_mutation_prime")[:3] == ["handle", "handle", 3]
    assert seen == {"off": [0, 3, 5, 9], "seq": b"ACGTTGGGG"}
    assert out.dtype == np.float64 and out.shape == (3, 3) and (out.reshape(-1) == np.arange(9)).all()
    assert status.dtype == np.int32 and status.shape == (3, 3) and (status == 5).all()
    raises(stub, "phmm_mutation_prime", lambda: engine.mutation_prime(model, ["A"]), "engine says no")


def test_align_scores(stub, engine, blocks):
    haps, reads = blocks
    tasks = [0, 1, 0, 0, 2, 0, 1, 1]                                   # reshaped to (-1, 4) rows on the host path
    seen = {}

    def effect(h, band, bits, nuc, hs, rs, t, n, out, space):
        seen["tasks"] = host(t, C.c_int32, 4 * n).reshape(-1, 4).tolist()
        host(out, C.c_int32, n)[:] = [-7, -9]
    stub.effects["phmm_align_scores"] = effect
    out = engine.align_scores(16, haps, reads, tasks, nuc_prior=3, precision_bits=32)
    args = stub.only("phmm_align_scores")
    assert args[:6] == ["handle", 16, 32, 3, HS, RS] and args[7] == 2 and args[9] == _lib.SPACE_HOST
    assert seen["tasks"] == [[0, 1, 0, 0], [2, 0, 1, 1]]
    assert out.dtype == np.int32 and out.tolist() == [-7, -9]
    raises(stub, "phmm_align_scores", lambda: engine.align_scores(8, haps, reads, tasks), "engine says no")


def test_align_traceback(stub, engine):
    def effect(*a):
        a[13]._obj.value, a[14]._obj.value = -12, 5
        a[15].value, a[16].value = b"AC-GT", b"ACTGT"
    stub.effects["phmm_align_traceback"] = effect
    q, go = np.full(4, 30, np.int8), np.full(9, 40, np.int8)
    assert engine.align(8, "ACGTACGTA", b"ACGT", q, go, 3) == (-12, 5, "AC-GT", "ACTGT")
    args = stub.only("phmm_align_traceback")
    n = 2 * (4 + 8) + 1
    assert args[:4] == ["handle", 8, b"ACGTACGTA", b"ACGT"] and args[5:9] == [9, 4, None, None]
    assert args[10:13] == [None, 3, 2] and args[15:] == ["buffer[%d]" % (n + 8)] * 2
    stub.calls.clear()
    engine.align(8, "ACGTACGTA", b"ACGT", q, go, np.full(9, 2, np.int8), nuc_prior=4, snv_mask="ACGTACGTA", snv_prior=np.full(9, 9))
    args = stub.only("phmm_align_traceback")
    assert args[7] == b"ACGTACGTA" and isinstance(args[8], int) and isinstance(args[10], int) and args[11:13] == [0, 4]
    raises(stub, "phmm_align_traceback", lambda: engine.align(8, "ACGTACGTA", b"ACGT", q, go, 3), "engine says no")


def test_align_reads(stub, engine, blocks):
    haps, reads = blocks
    pairs = np.array([[0, 0], [1, 0], [2, 1]], np.int32)
    poff, ppos = np.array([0, 1, 1, 3], np.int64), np.array([5, 6, 7], np.int32)
    stub.register("", {"pairs": pairs, "pos.off": poff, "pos.pos": ppos})
    stub.effects["phmm_align_reads"] = write_cigars(STRIDE)
    mp, lk, cigars, st = engine.align_reads(CFG, haps, reads, pairs, positions=(poff, ppos), flank_state=(3, 4))
    args = stub.only("phmm_align_reads")
    assert args[:8] == ["handle", CS, HS, RS, "pairs", 3, {"off": "pos.off", "pos": "pos.pos"}, FLANK]
    assert args[11] == STRIDE and args[13] == _lib.SPACE_HOST
    assert cigars == ["1M", "2M", "3M"] and mp.dtype == np.int64 and mp.tolist() == [100, 101, 102]
    assert lk.dtype == np.float64 and lk.shape == (3,) and st.dtype == np.int32 and st.tolist() == [0, 1, 2]
    stub.calls.clear()
    _, _, cigars, _ = engine.align_reads(CFG, haps, reads, [[0, 1], [1, 1]], cigar_stride=40)
    args = stub.only("phmm_align_reads")
    assert args[5:8] == [2, None, None] and args[11] == 40 and cigars == ["1M", "2M"]
    raises(stub, "phmm_align_reads", lambda: engine.align_reads(CFG, haps, reads, pairs), "engine says no")


def test_align_pairs(stub, engine, blocks):
    haps, reads = blocks
    pairs, offs = np.array([[0, 0], [2, 1]], np.int32), np.array([4, 9], np.int32)
    stub.register("", {"pairs": pairs, "offs": offs})
    stub.effects["phmm_align_pairs"] = write_cigars(STRIDE, mp=6)
    mp, lk, cigars, st = engine.align_pairs(CFG, haps, reads, pairs, offs, flank_state=(3, 4))
    args = stub.only("phmm_align_pairs")
    assert args[:8] == ["handle", CS, HS, RS, "pairs", "offs", 2, FLANK]
    assert args[11] == STRIDE and args[13] == _lib.SPACE_HOST
    assert cigars == ["1M", "2M"] and mp.dtype == np.int64 and mp.tolist() == [100, 101]
    assert lk.dtype == np.float64 and lk.shape == (2,) and st.dtype == np.int32 and st.tolist() == [0, 1]
    stub.calls.clear()
    engine.align_pairs(CFG, haps, reads, pairs, offs, cigar_stride=24)
    args = stub.only("phmm_align_pairs")
    assert args[7] is None and args[11] == 24
    raises(stub, "phmm_align_pairs", lambda: engine.align_pairs(CFG, haps, reads, pairs, offs), "engine says no")


@pytest.mark.parametrize("extra", [0, 5])
def test_map_pairs_grows_and_retries(stub, engine, blocks, extra):
    haps, reads = blocks
    pairs = [[0, 0], [1, 0], [2, 1]]
    n, cap = 3, 4 * 3 + 16
    total = cap + extra

    def effect(h, hs, rs, pp, n_, off, pos, cap_, space):
        o = host(off, C.c_int64, n_ + 1)
        o[:] = np.linspace(0, total, n_ + 1).astype(np.int64)
        host(pos, C.c_int32, min(cap_, total))[:] = 11
    stub.effects["phmm_map_pairs"] = effect
    off, pos = engine.map_pairs(haps, reads, pairs)
    calls = [a for name, a in stub.calls if name == "phmm_map_pairs"]
    assert [a[7] for a in calls] == ([cap] if extra == 0 else [cap, total])
    assert all(a[:3] == ["handle", HS, RS] and a[4] == n and a[8] == _lib.SPACE_HOST for a in calls)
    assert off.dtype == np.int64 and off.shape == (n + 1,) and int(off[-1]) == total
    assert pos.dtype == np.int32 and pos.shape == (total,) and (pos == 11).all()
    raises(stub, "phmm_map_pairs", lambda: engine.map_pairs(haps, reads, pairs), "engine says no")


def test_realign_reads_outputs_start_zeroed(stub, engine, blocks):
    haps, reads = blocks
    pairs = np.array([[0, 0], [2, 1]], np.int32)
    stub.register("", {"pairs": pairs})
    zeroed = []

    def effect(*a):
        n, stride = a[5], a[10]
        zeroed.append(all(not host(p, t, k).any() for p, t, k in ((a[7], C.c_int64, n), (a[8], C.c_double, n),
                                                                 (a[9], C.c_uint8, n * stride), (a[11], C.c_int32, n))))
        write_cigars(stride, cg=9, st=11)(*a)
    stub.effects["phmm_realign_reads"] = effect
    mp, lk, cigars, st = engine.realign_reads(CFG, haps, reads, pairs, flank_state=(3, 4))
    args = stub.only("phmm_realign_reads")
    assert args[:7] == ["handle", CS, HS, RS, "pairs", 2, FLANK] and args[10] == STRIDE and args[12] == _lib.SPACE_HOST
    assert zeroed == [True] and cigars == ["1M", "2M"] and mp.tolist() == [100, 101] and st.tolist() == [0, 1]
    assert mp.dtype == np.int64 and lk.dtype == np.float64 and lk.shape == (2,) and st.dtype == np.int32
    stub.calls.clear()
    engine.realign_reads(CFG, haps, reads, pairs, cigar_stride=30)
    args = stub.only("phmm_realign_reads")
    assert args[6] is None and args[10] == 30
    raises(stub, "phmm_realign_reads", lambda: engine.realign_reads(CFG, haps, reads, pairs), "engine says no")


def test_genotype_likelihoods(stub, engine):
    lnl, gts = np.zeros((3, 5)), np.array([[0, 1], [2, 2], [1, 0], [0, 0]], np.int32)
    stub.register("", {"lnl": lnl, "gts": gts})
    stub.effects["phmm_genotype_likelihoods"] = lambda h, m, H, R, g, G, P, out, space: host(out, C.c_double, G).__setitem__(slice(None), -1.5)
    out = engine.genotype_likelihoods(lnl, gts)
    assert stub.only("phmm_genotype_likelihoods")[:7] == ["handle", "lnl", 3, 5, "gts", 4, 2]
    assert stub.only("phmm_genotype_likelihoods")[8] == _lib.SPACE_HOST
    assert out.dtype == np.float64 and out.tolist() == [-1.5] * 4
    raises(stub, "phmm_genotype_likelihoods", lambda: engine.genotype_likelihoods(lnl, gts), "engine says no")


def test_populate_templates(stub, engine, blocks):
    haps, reads = blocks
    toff = np.array([0, 2, 3], np.int64)
    stub.register("", {"toff": toff})
    stub.effects["phmm_populate_templates"] = lambda *a: host(a[8], C.c_double, 4).__setitem__(slice(None), -2.0)
    out = engine.populate_templates(CFG, haps, reads, toff, flank_state=(3, 4))
    args = stub.only("phmm_populate_templates")
    assert args[:8] == ["handle", CS, HS, RS, "toff", 2, None, FLANK] and args[9:] == [None, _lib.SPACE_HOST]
    assert out.dtype == np.float64 and out.shape == (2, 2) and (out == -2.0).all()
    stub.calls.clear()
    engine.populate_templates(CFG, haps, reads, toff)
    assert stub.only("phmm_populate_templates")[7] is None
    raises(stub, "phmm_populate_templates", lambda: engine.populate_templates(CFG, haps, reads, toff), "engine says no")


@pytest.mark.parametrize("raw_config", [False, True])
def test_populate_regions(stub, engine, blocks, raw_config):
    haps, reads = blocks
    cfg = CFG.c_struct() if raw_config else CFG
    hf, rf = [0, 1, 2], [0, 1, 3]                                      # regions of 1 x 1 and 1 x 2 pairs

    def effect(h, c, hs, rs, regs, out, status, space):
        host(out, C.c_double, 3)[:] = [-1, -2, -3]
        if status:
            host(status, C.c_int32, 3)[:] = 7
    stub.effects["phmm_populate_regions"] = effect
    out, off = engine.populate_regions(cfg, haps, reads, hf, rf, flank_states=[(1, 2), None])
    args = stub.only("phmm_populate_regions")
    assert args[:5] == ["handle", CS, HS, RS, {"n": 2, "hap_first": [0, 1, 2], "read_first": [0, 1, 3], "flank": [(1, 1, 2), (0, 0, 0)]}]
    assert args[6] is None and args[7] == _lib.SPACE_HOST
    assert out.dtype == np.float64 and out.tolist() == [-1, -2, -3] and off.dtype == np.int64 and off.tolist() == [0, 1, 3]
    stub.calls.clear()
    got = engine.populate_regions(cfg, haps, reads, hf, rf, want_status=True)
    assert stub.only("phmm_populate_regions")[4]["flank"] is None
    assert len(got) == 3 and got[2].dtype == np.int32 and got[2].tolist() == [7, 7, 7]
    mine = np.zeros(3)
    assert engine.populate_regions(cfg, haps, reads, hf, rf, out=mine)[0] is mine and mine.tolist() == [-1, -2, -3]
    call = lambda: engine.populate_regions(cfg, haps, reads, hf, rf)                       # noqa: E731
    raises(stub, "phmm_populate_regions", call, "engine says no")
    stub.rc["phmm_populate_regions"] = _lib.PHMM_ERR_SHORT_HAPLOTYPE
    assert len(engine.populate_regions(cfg, haps, reads, hf, rf, want_status=True)) == 3
    call = lambda: engine.populate_regions(cfg, haps, reads, hf, rf, want_status=True)     # noqa: E731
    raises(stub, "phmm_populate_regions", call, "engine says no", ERRORS[1:])


@pytest.mark.parametrize("raw_config", [False, True])
def test_assign_reads(stub, engine, blocks, raw_config):
    haps, reads = blocks
    cfg = CFG.c_struct() if raw_config else CFG
    hf, rf = [0, 2], [0, 3]
    pri = np.log([0.25, 0.75])
    stub.register("", {"pri": pri})

    def effect(h, c, hs, rs, regs, p, top, lnl, status, space):
        host(top, C.c_uint64, 3)[:] = [1, 2, 3]
        if lnl:
            host(lnl, C.c_double, 6)[:] = -4
        if status:
            host(status, C.c_int32, 6)[:] = 1
    stub.effects["phmm_assign_reads"] = effect
    top = engine.assign_reads(cfg, haps, reads, hf, rf)
    args = stub.only("phmm_assign_reads")
    assert args[:6] == ["handle", CS, HS, RS, {"n": 1, "hap_first": [0, 2], "read_first": [0, 3], "flank": None}, None]
    assert args[7:] == [None, None, _lib.SPACE_HOST]
    assert isinstance(top, np.ndarray) and top.dtype == np.uint64 and top.tolist() == [1, 2, 3]
    stub.calls.clear()
    top, lnl, status = engine.assign_reads(cfg, haps, reads, hf, rf, pri, want_likelihoods=True, want_status=True)
    assert stub.only("phmm_assign_reads")[5] == "pri"
    assert lnl.dtype == np.float64 and lnl.tolist() == [-4] * 6 and status.dtype == np.int32 and status.tolist() == [1] * 6
    top, lnl = engine.assign_reads(cfg, haps, reads, hf, rf, want_likelihoods=True)
    top, status = engine.assign_reads(cfg, haps, reads, hf, rf, want_status=True)
    assert status.shape == (6,)
    stub.calls.clear()
    with pytest.raises(ValueError):
        engine.assign_reads(cfg, haps, reads, hf, rf, [0.0])
    assert stub.calls == []
    raises(stub, "phmm_assign_reads", lambda: engine.assign_reads(cfg, haps, reads, hf, rf), "engine says no")
    stub.rc["phmm_assign_reads"] = _lib.PHMM_ERR_SHORT_HAPLOTYPE
    assert len(engine.assign_reads(cfg, haps, reads, hf, rf, want_status=True)) == 2
    call = lambda: engine.assign_reads(cfg, haps, reads, hf, rf, want_status=True)     # noqa: E731
    raises(stub, "phmm_assign_reads", call, "engine says no", ERRORS[1:])


@pytest.mark.parametrize("raw_config", [False, True])
def test_populate(stub, engine, blocks, raw_config):
    haps, reads = blocks
    cfg = CFG.c_struct() if raw_config else CFG
    poff, ppos = np.array([0, 1, 1, 1, 1, 1, 2], np.int64), np.array([5, 6], np.int32)
    stub.register("", {"pos.off": poff, "pos.pos": ppos})

    def effect(h, c, hs, rs, p, f, out, status, space):
        host(out, C.c_double, 6)[:] = -3
        if status:
            host(status, C.c_int32, 6)[:] = 2
    stub.effects["phmm_populate"] = effect
    out = engine.populate(cfg, haps, reads, positions=(poff, ppos), flank_state=(3, 4))
    args = stub.only("phmm_populate")
    assert args[:6] == ["handle", CS, HS, RS, {"off": "pos.off", "pos": "pos.pos"}, FLANK] and args[7:] == [None, _lib.SPACE_HOST]
    assert isinstance(out, np.ndarray) and out.dtype == np.float64 and out.shape == (2, 3) and (out == -3).all()
    stub.calls.clear()
    out, status = engine.populate(cfg, haps, reads, want_status=True)
    assert stub.only("phmm_populate")[4:6] == [None, None]
    assert status.dtype == np.int32 and status.shape == (2, 3) and (status == 2).all()
    mine = np.zeros((2, 3))
    assert engine.populate(cfg, haps, reads, out=mine) is mine and (mine == -3).all()
    raises(stub, "phmm_populate", lambda: engine.populate(cfg, haps, reads), "engine says no")
    stub.rc["phmm_populate"] = _lib.PHMM_ERR_SHORT_HAPLOTYPE
    out, status = engine.populate(cfg, haps, reads, want_status=True)
    assert out.shape == status.shape == (2, 3)
    raises(stub, "phmm_populate", lambda: engine.populate(cfg, haps, reads, want_status=True), "engine says no", ERRORS[1:])


# -- PopulateBatcher ----------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("raw_config", [False, True])
def test_batcher_populate(stub, blocks, raw_config):
    haps, reads = blocks
    cfg = CFG.c_struct() if raw_config else CFG
    b = PopulateBatcher()
    stub.calls.clear()
    poff, ppos = np.array([0, 1, 1, 1, 1, 1, 2], np.int64), np.array([5, 6], np.int32)
    stub.register("", {"pos.off": poff, "pos.pos": ppos})
    stub.effects["phmm_batcher_populate"] = lambda *a: host(a[6], C.c_double, 6).__setitem__(slice(None), -5)
    out = b.populate(cfg, haps, reads, positions=(poff, ppos), flank_state=(3, 4))
    args = stub.only("phmm_batcher_populate")
    assert args[:6] == ["handle", CS, HS, RS, {"off": "pos.off", "pos": "pos.pos"}, FLANK] and args[7] is None
    assert out.dtype == np.float64 and out.shape == (2, 3) and (out == -5).all()
    out, status = b.populate(cfg, haps, reads, want_status=True)
    assert status.dtype == np.int32 and status.shape == (2, 3)
    raises(stub, "phmm_batcher_populate", lambda: b.populate(cfg, haps, reads), "batcher says no")
    stub.rc["phmm_batcher_populate"] = _lib.PHMM_ERR_SHORT_HAPLOTYPE
    assert len(b.populate(cfg, haps, reads, want_status=True)) == 2
    raises(stub, "phmm_batcher_populate", lambda: b.populate(cfg, haps, reads, want_status=True), "batcher says no", ERRORS[1:])


@pytest.mark.parametrize("raw_config", [False, True])
def test_batcher_populate_templates(stub, blocks, raw_config):
    haps, reads = blocks
    cfg = CFG.c_struct() if raw_config else CFG
    b = PopulateBatcher()
    stub.calls.clear()
    toff = np.array([0, 2, 3], np.int64)
    stub.register("", {"toff": toff})
    out = b.populate_templates(cfg, haps, reads, toff, flank_state=(3, 4))
    args = stub.only("phmm_batcher_populate_templates")
    assert args[:7] == ["handle", CS, HS, RS, "toff", 2, FLANK] and args[8] is None
    assert out.dtype == np.float64 and out.shape == (2, 2)
    out, status = b.populate_templates(cfg, haps, reads, toff, want_status=True)
    assert out.shape == (2, 2) and status.dtype == np.int32 and status.shape == (2, 3)
    raises(stub, "phmm_batcher_populate_templates", lambda: b.populate_templates(cfg, haps, reads, toff), "batcher says no")
    stub.rc["phmm_batcher_populate_templates"] = _lib.PHMM_ERR_SHORT_HAPLOTYPE
    assert len(b.populate_templates(cfg, haps, reads, toff, want_status=True)) == 2


# -- ErrorModel and MutationModel ---------------------------------------------------------------------------------------
def test_error_model_creation(stub):
    ErrorModel()
    ErrorModel("PCR.NovaSeq")
    ErrorModel(custom_model_text="text")
    created = [(n, a) for n, a in stub.calls if n.startswith("phmm_error_model_create")]
    assert created == [("phmm_error_model_create", [None]), ("phmm_error_model_create", [b"PCR.NovaSeq"]),
                       ("phmm_error_model_create_custom", [b"text"])]
    stub.rc["phmm_error_model_create"] = _lib.PHMM_ERR_INVALID
    with pytest.raises(PhmmError, match="model says no"):
        ErrorModel("nope")


@pytest.mark.parametrize("sequences", [["ACGT", b"GG", np.frombuffer(b"TTA", np.uint8), np.array([0x4341], np.int16)], []])
def test_error_model_reset(stub, sequences):
    m = ErrorModel()
    stub.calls.clear()
    seen = {}

    def effect(h, n, off, seq, sub, *outs):
        o = host(off, C.c_int64, n + 1)
        seen.update(n=n, off=list(o), seq=C.string_at(seq, int(o[-1])), sub=sub, threads=outs[-1])
        for p in outs[:-1]:
            host(p, C.c_int8, int(o[-1]))[:] = 1
    stub.effects["phmm_reset_haplotypes"] = effect
    block = m.reset(sequences, n_threads=3)
    parts = [x.encode() if isinstance(x, str) else bytes(x) for x in sequences]
    want = b"".join(parts)
    assert seen == {"n": len(parts), "off": list(np.cumsum([0] + [len(x) for x in parts])), "seq": want, "sub": None, "threads": 3}
    assert block.n == len(sequences) and block.seq.tobytes() == want and (block.gap_open == 1).all()
    assert block.gap_open.dtype == np.int8 and block.snv_mask_fwd.dtype == np.uint8 and len(block.gap_extend) == len(want)
    if sequences:
        m.reset(["AC", "G"], is_substitution=[[1, 0], [True]])
        stub.rc["phmm_reset_haplotypes"] = _lib.PHMM_ERR_INVALID
        with pytest.raises(PhmmError, match="model says no"):
            m.reset(["A"])


@pytest.mark.parametrize("extra", [0, 3])
def test_tandem_repeats_grows_and_retries(stub, extra):
    m = ErrorModel()
    stub.calls.clear()
    cap = 4 * 6 + 16
    total = cap + extra

    def effect(s, n, lo, hi, out, cap_):
        if total <= cap_:
            host(out, C.c_uint32, 3 * total)[:] = 9
        return total
    stub.effects["phmm_tandem_repeats"] = effect
    out = m.tandem_repeats("ACACAC", 2, 4)
    calls = [a for n, a in stub.calls if n == "phmm_tandem_repeats"]
    assert [a[5] for a in calls] == ([cap] if extra == 0 else [cap, total])
    assert all(a[1:4] == [6, 2, 4] for a in calls)
    assert out.dtype == np.uint32 and out.shape == (total, 3) and (out == 9).all()
    stub.effects["phmm_tandem_repeats"] = lambda *a: _lib.PHMM_ERR_INVALID
    with pytest.raises(PhmmError, match="model says no"):
        m.tandem_repeats("ACGT")


def test_mutation_model_context(stub):
    with pytest.raises(ValueError):
        MutationModel(1e-8, np.zeros((2, 3)), np.zeros((3, 3, 4)))
    assert stub.calls == []
    t = MutationModel(1e-8, np.zeros((2, 3)), np.zeros((2, 3, 4)))
    assert (t.max_period, t.max_periodicity, t.max_indel_length, t.snv_prior) == (1, 2, 4, 1e-8)
    stub.calls.clear()
    seen = {}

    def effect(h, n, off, seq, cell, op, ep, threads):
        o = host(off, C.c_int64, n + 1)
        seen.update(off=list(o), seq=C.string_at(seq, int(o[-1])))
        host(cell, C.c_int32, int(o[-1]))[:] = 3
    stub.effects["phmm_mutation_context"] = effect
    cell, op, ep = t.context(["ACG", b"T"], n_threads=2)
    args = stub.only("phmm_mutation_context")
    assert args[:2] == ["handle", 2] and args[7] == 2 and seen == {"off": [0, 3, 4], "seq": b"ACGT"}
    assert cell.dtype == np.int32 and cell.tolist() == [3] * 4 and op.dtype == ep.dtype == np.int8 and op.shape == ep.shape == (4,)
    stub.rc["phmm_mutation_context"] = _lib.PHMM_ERR_INVALID
    with pytest.raises(PhmmError, match="model says no"):
        t.context(["A"])
    stub.rc["phmm_mutation_model_create"] = _lib.PHMM_ERR_INVALID
    with pytest.raises(PhmmError, match="model says no"):
        MutationModel(1e-8, np.zeros((2, 3)), np.zeros((2, 3, 4)))
