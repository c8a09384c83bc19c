"""Many haplotype sets per call (phmm_mutation_prime_sets, PairHMMEngine.mutation_prime_sets) and concurrent primes on one shared
engine (phmm_batcher_mutation_prime, PopulateBatcher.mutation_prime, the C++ DeNovoModel over a SharedEngine): every set's statuses
equal the one-set call's, and its values bit for bit where the status is HMM or SELF; against the reference DeNovoModel where it is
built. The marshalling tests at the end need neither a GPU nor the library."""
import ctypes as C
import os
import subprocess
import tempfile
import threading

import numpy as np
import pytest

from helpers import random_region
from mutation_oracle import SOMATIC_PRIORS, TRIO_PRIORS, RefMutation, mutate
from octopus_b200 import HaplotypeLikelihoodModel, MutationModel, PhmmError, PopulateBatcher, _lib
from octopus_b200.api import PairHMMEngine

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
APPROX = (_lib.MUT_APPROX_LENGTH, _lib.MUT_APPROX_OFFSET, _lib.MUT_APPROX_OVERFLOW)
needs_ref = pytest.mark.skipif(not RefMutation.available(), reason="reference mutation model not built (oracle/_ref/libref_mutation.so)")


def _table(priors):
    """The reference's repeat table for the indel prior where it is built, else a stand-in rising with the repeat count."""
    if RefMutation.available():
        return RefMutation().table(priors[1])
    o = np.full((11, 51), priors[1], np.float32)
    o[1:6, 3:] = np.geomspace(priors[1], 1e-3, 48, dtype=np.float32)
    e = np.full((11, 51, 50), 0.5, np.float32)
    e[1:6, 3:, :] = 0.85
    return o, e


def _model(priors):
    return MutationModel(priors[0], *_table(priors))


def region(rng, n, length):
    """n haplotypes of about `length` bp: a base with a short tandem repeat, and copies 0-8 SNVs / 1-20 bp indels away from it."""
    unit = "".join(rng.choice(list("ACGT"), int(rng.integers(1, 5))))
    base = "".join(rng.choice(list("ACGT"), max(1, length - 40))) + unit * int(rng.integers(4, 10))
    return [base] + [mutate(rng, base, int(rng.integers(0, 9))) for _ in range(n - 1)]


def all_approx_set(rng):
    """Haplotypes whose lengths differ pairwise by >= 32: every off-diagonal pair is APPROX_LENGTH, so the set lists nothing."""
    return ["".join(rng.choice(list("ACGT"), 100 + 40 * k)) for k in range(5)]


def assert_same(got, want, where):
    (out, status), (wout, wstatus) = got, want
    assert out.shape == wout.shape and status.shape == wstatus.shape, where
    assert np.array_equal(status, wstatus), (where, np.argwhere(status != wstatus)[:10])
    exact = (wstatus == _lib.MUT_HMM) | (wstatus == _lib.MUT_SELF)
    assert np.array_equal(out[exact].view(np.uint64), wout[exact].view(np.uint64)), (where, np.argwhere(exact & (out != wout))[:10])


def assert_sets_equal_per_set_calls(engine, model, sets):
    got = engine.mutation_prime_sets(model, sets)
    assert len(got) == len(sets)
    for s, seqs in enumerate(sets):
        if not seqs:
            assert got[s][0].shape == (0, 0) and got[s][1].shape == (0, 0)
            continue
        assert_same(got[s], engine.mutation_prime(model, seqs), s)
    return got


@pytest.mark.gpu
@pytest.mark.parametrize("priors", [TRIO_PRIORS, SOMATIC_PRIORS], ids=["trio", "somatic"])
@pytest.mark.parametrize("length", [300, 1000])
def test_sets_call_equals_one_call_per_set(engine, priors, length):
    rng = np.random.default_rng(length + int(priors[0] * 1e9))
    model = _model(priors)
    sets = [region(rng, n, length) for n in (1, 2, 12, 50)] + [[]] + [region(rng, n, length) for n in (51, 200)] + [all_approx_set(rng)]
    got = assert_sets_equal_per_set_calls(engine, model, sets)
    assert (got[-1][1] == _lib.MUT_APPROX_LENGTH).sum() == 5 * 4 and (np.diag(got[-1][1]) == _lib.MUT_SELF).all()
    assert (got[3][1] == _lib.MUT_HMM).sum() >= 50 * 49 // 5


@pytest.mark.gpu
@needs_ref
@pytest.mark.parametrize("priors", [TRIO_PRIORS, SOMATIC_PRIORS], ids=["trio", "somatic"])
def test_sets_call_matches_reference(engine, priors):
    rng = np.random.default_rng(77)
    model = _model(priors)
    sets = [region(rng, n, 280) for n in (3, 20, 40)] + [[]] + [region(rng, 9, 900)]
    got = engine.mutation_prime_sets(model, sets)
    ref = RefMutation()
    for s, seqs in enumerate(sets):
        if not seqs:
            continue
        out, status = got[s]
        want, approx = ref.prime(priors[0], priors[1], seqs)
        assert np.array_equal(np.isin(status, APPROX), approx), (s, np.argwhere(np.isin(status, APPROX) != approx)[:10])
        hmm = (status == _lib.MUT_HMM) | (status == _lib.MUT_SELF)
        assert np.array_equal(out[hmm].view(np.uint64), want[hmm].view(np.uint64)), (s, np.argwhere(hmm & (out != want))[:10])


@pytest.mark.gpu
def test_tile_boundary_inside_a_set(engine):
    """Seven sets of 300 haplotypes of about 100 bp: 630 000 ordered pairs, the first tile (2^19 pairs) ends inside set 5."""
    rng = np.random.default_rng(31)
    model = _model(TRIO_PRIORS)
    sets = [region(rng, 300, 100) for _ in range(7)]
    assert 5 * 300 * 300 < 1 << 19 < 6 * 300 * 300
    got = assert_sets_equal_per_set_calls(engine, model, sets)
    # set 5 aligns pairs on both sides of the tile boundary
    hmm = np.flatnonzero(got[5][1].reshape(-1) == _lib.MUT_HMM) + 5 * 300 * 300
    assert (hmm < 1 << 19).sum() > 1000 and (hmm >= 1 << 19).sum() > 1000


@pytest.mark.gpu
def test_one_long_set_among_short_ones(engine):
    """A 5 kb set among 300 bp sets: every truth padded to its own set's longest haplotype, the CIGAR stride the call's."""
    rng = np.random.default_rng(41)
    model = _model(SOMATIC_PRIORS)
    sets = [region(rng, 20, 300), region(rng, 6, 5000), region(rng, 30, 300), region(rng, 1, 300)]
    got = assert_sets_equal_per_set_calls(engine, model, sets)
    assert (got[1][1] == _lib.MUT_HMM).sum() > 0 and (got[2][1] == _lib.MUT_HMM).sum() > 0


@pytest.mark.gpu
def test_argument_checks(engine):
    lib = _lib.load()
    model = _model(TRIO_PRIORS)
    off = np.array([0, 4, 8, 0], np.int64)                    # two haplotypes; the trailing 0 is not an offset of theirs
    seq = np.frombuffer(b"ACGTACGA", np.uint8)
    out = np.zeros(8, np.float64)
    st = np.zeros(8, np.int32)

    def call(set_first, n_sets=None, **swap):
        sf = np.ascontiguousarray(set_first, np.int32)
        args = dict(e=engine._h, m=model._h, sf=sf.ctypes.data, off=off.ctypes.data, seq=seq.ctypes.data, out=out.ctypes.data, st=st.ctypes.data)
        args.update(swap)
        rc = lib.phmm_mutation_prime_sets(args["e"], args["m"], len(sf) - 1 if n_sets is None else n_sets, args["sf"], args["off"], args["seq"],
                                          args["out"], args["st"])
        return rc, lib.phmm_last_error(engine._h).decode() if rc and args["e"] else ""

    assert call([0, 1, 2]) == (_lib.PHMM_OK, "")
    assert call([0, 2, 2, 2]) == (_lib.PHMM_OK, "")              # empty sets
    assert call([0, 2], n_sets=0) == (_lib.PHMM_OK, "")
    for bad, message in (([1, 2], "set_first[0] must be 0"), ([0, 2, 1], "set_first must be non-decreasing"),
                         ([0, 3], "haplotype length outside [1, 65535]")):         # a last entry past the haplotypes the offsets describe
        assert call(bad) == (_lib.PHMM_ERR_INVALID, message), bad
    for k in ("m", "sf", "off", "seq", "out", "st"):
        assert call([0, 1, 2], **{k: None}) == (_lib.PHMM_ERR_INVALID, "null argument"), k
    assert call([0, 1, 2], e=None)[0] == _lib.PHMM_ERR_INVALID
    with pytest.raises(PhmmError, match=r"haplotype count outside \[1, 4096\]"):
        engine.mutation_prime_sets(model, [["ACGT"], ["ACGT"] * 4097])
    # five full sets: 5 x 4096^2 ordered pairs > 2^26 (refused before anything is written or allocated)
    big_off = np.arange(5 * 4096 + 1, dtype=np.int64)
    big_seq = np.full(5 * 4096, ord("A"), np.uint8)
    rc, msg = call(np.arange(6, dtype=np.int32) * 4096, off=big_off.ctypes.data, seq=big_seq.ctypes.data)
    assert rc == _lib.PHMM_ERR_INVALID and "PHMM_MUT_MAX_PAIRS" in msg
    assert (4 * 4096 * 4096 <= _lib.MUT_MAX_PAIRS < 5 * 4096 * 4096) and _lib.MUT_MAX_PAIRS >= 4096 ** 2


@pytest.mark.gpu
def test_batcher_threads_merge_and_equal_solo_calls(engine):
    """8 threads on one PopulateBatcher, each with its own model objects: mutation requests of equal models merge, a model with
    other priors never shares their call, populate requests interleave, and a request that fails its checks fails alone."""
    n_threads = 8
    trio_table, somatic_table = _table(TRIO_PRIORS), _table(SOMATIC_PRIORS)
    work = {}
    for k in range(n_threads):
        rng = np.random.default_rng(500 + k)
        items = []
        for i in range(4):
            if k in (2, 5) and i % 2 == 1:
                haps, reads = random_region(rng, 16, n_haps=int(rng.integers(2, 10)), n_reads=int(rng.integers(10, 60)), hap_len=300,
                                            read_len_choices=[76, 100, 150])
                items.append(("populate", (haps, reads)))
            elif k == 3 and i == 2:
                items.append(("bad", ["ACGTACGT", ""]))                             # an empty haplotype
            else:
                items.append(("prime", region(rng, int(rng.integers(2, 40)), int(rng.choice([250, 400])))))
        work[k] = items
    cfg = HaplotypeLikelihoodModel.Config(max_indel_error=16)
    got, errors = {}, []
    batcher = PopulateBatcher(0, clients=n_threads, max_wait_us=200000)
    start = threading.Barrier(n_threads)

    def worker(k):
        try:
            priors, table = (SOMATIC_PRIORS, somatic_table) if k == n_threads - 1 else (TRIO_PRIORS, trio_table)
            start.wait()
            for i, (kind, item) in enumerate(work[k]):
                if kind == "populate":
                    got[(k, i)] = batcher.populate(cfg, *item, want_status=True)
                elif kind == "bad":
                    with pytest.raises(PhmmError, match=r"haplotype length outside \[1, 65535\]"):
                        batcher.mutation_prime(MutationModel(priors[0], *table), item)
                    got[(k, i)] = "refused"
                else:
                    got[(k, i)] = batcher.mutation_prime(MutationModel(priors[0], *table), item)     # a new model per region
        except Exception as ex:          # noqa: BLE001
            errors.append((k, repr(ex)))

    threads = [threading.Thread(target=worker, args=(k,)) for k in range(n_threads)]
    for t in threads:
        t.start()
    for t in threads:
        t.join(timeout=300)
    assert not any(t.is_alive() for t in threads), "a request never returned"
    assert not errors, errors
    stats = batcher.stats()
    batcher.close()

    models = {False: _model(TRIO_PRIORS), True: _model(SOMATIC_PRIORS)}
    for (k, i), res in got.items():
        kind, item = work[k][i]
        if kind == "populate":
            assert_same_populate(res, engine.populate(cfg, *item, want_status=True), (k, i))
        elif kind == "prime":
            assert_same(res, engine.mutation_prime(models[k == n_threads - 1], item), (k, i))
    assert len(got) == 4 * n_threads
    assert stats["requests"] == 4 * n_threads - 1, stats                     # the refused request never reached the GPU
    assert stats["merged_calls"] >= 1 and stats["max_regions_per_call"] > 1, stats


def assert_same_populate(got, want, where):
    (out, st), (wout, wst) = got, want
    assert np.array_equal(st, wst), where
    ok = (wst & 0xFFFF) == 0
    assert np.array_equal(out.view(np.int64)[ok], wout.view(np.int64)[ok]), where


@pytest.mark.gpu
def test_models_with_other_priors_never_merge(engine):
    """Two threads with equal models and one with other priors, all at once: the equal pair share one call, the third runs on its
    own, and each result equals its solo call."""
    rng = np.random.default_rng(3)
    sets = [region(rng, 12, 300) for _ in range(3)]
    priors = [TRIO_PRIORS, TRIO_PRIORS, SOMATIC_PRIORS]
    tables = {p: _table(p) for p in (TRIO_PRIORS, SOMATIC_PRIORS)}
    got = {}
    with PopulateBatcher(0, clients=3, max_wait_us=500000) as batcher:
        start = threading.Barrier(3)

        def worker(k):
            model = MutationModel(priors[k][0], *tables[priors[k]])
            start.wait()
            got[k] = batcher.mutation_prime(model, sets[k])
        threads = [threading.Thread(target=worker, args=(k,)) for k in range(3)]
        for t in threads:
            t.start()
        for t in threads:
            t.join(timeout=120)
        stats = batcher.stats()
    assert stats["gpu_calls"] == 2 and stats["merged_calls"] == 1 and stats["max_regions_per_call"] == 2, stats
    for k in range(3):
        assert_same(got[k], engine.mutation_prime(_model(priors[k]), sets[k]), k)


# ---------------------------------------------------------------------------------------------------------------------
# The C++ adapter: DeNovoModel over a SharedEngine from many std::threads
# ---------------------------------------------------------------------------------------------------------------------
def _build_cpp():
    from octopus_b200 import build
    build.build()
    exe = os.path.join(tempfile.mkdtemp(prefix="test_denovo_shared_"), "test_denovo_shared")
    subprocess.run(["g++", "-std=c++14", "-O1", "-pthread", "-I", os.path.join(ROOT, "include"), "-I", os.path.join(ROOT, "octopus_b200", "cpp"),
                    os.path.join(ROOT, "tests", "cpp", "test_denovo_shared.cpp"), "-o", exe, "-L", os.path.join(ROOT, "octopus_b200"),
                    "-lphmm_b200", "-Wl,-rpath," + os.path.join(ROOT, "octopus_b200")], check=True)
    return exe


def test_cpp_shared_denovo_driver_compiles():
    exe = _build_cpp()
    assert subprocess.run([exe, "--compile-only"]).returncode == 0


@pytest.mark.gpu
def test_cpp_threads_prime_on_one_shared_engine():
    run = subprocess.run([_build_cpp()], capture_output=True, text=True, timeout=600)
    assert run.returncode == 0 and "SHARED ok" in run.stdout, run.stdout + run.stderr
    requests, gpu_calls, merged, most = (int(x) for x in run.stdout.split()[2:6])
    assert requests == 6 * 4 and gpu_calls < requests and merged >= 1 and most > 1, run.stdout


# ---------------------------------------------------------------------------------------------------------------------
# Marshalling of the Python mirror against a recording stand-in for the library (no GPU, no library)
# ---------------------------------------------------------------------------------------------------------------------
HANDLE = 0x5150


class Stub:
    """Records every phmm_* call with its raw arguments, runs effects[name](*args) if set, returns rc[name] (PHMM_OK by default).
    The create functions hand out HANDLE."""

    def __init__(self):
        self.calls, self.rc, self.effects = [], {}, {}

    def __getattr__(self, name):
        if not name.startswith("phmm_"):
            raise AttributeError(name)
        if name.endswith("last_error"):
            return lambda *a: b"stub says no"

        def call(*args):
            self.calls.append((name, args))
            if name in self.effects:
                self.effects[name](*args)
            rc = self.rc.get(name, _lib.PHMM_OK)
            if name.endswith("_create") and rc == _lib.PHMM_OK:
                args[0]._obj.value = HANDLE
            return rc
        return call

    def only(self, name):
        got = [a for n, a in self.calls if n == name]
        assert len(got) == 1, (name, [n for n, _ in self.calls])
        return got[0]


@pytest.fixture
def stub(monkeypatch):
    s = Stub()
    monkeypatch.setattr(_lib, "load", lambda: s)
    return s


def _host(ptr, ctype, n):
    return np.ctypeslib.as_array((ctype * n).from_address(ptr)) if n else np.zeros(0, np.dtype(ctype))


def test_mutation_prime_sets_marshalling(stub):
    engine = PairHMMEngine(1)
    model = MutationModel(1e-8, np.full((2, 3), 0.5, np.float32), np.full((2, 3, 4), 0.25, np.float32))
    seen = {}

    def effect(h, m, n_sets, set_first, off, seq, out, status):
        sf = _host(set_first, C.c_int32, n_sets + 1)
        o = _host(off, C.c_int64, int(sf[-1]) + 1)
        seen.update(handles=(h.value if isinstance(h, C.c_void_p) else h, m.value if isinstance(m, C.c_void_p) else m), n_sets=n_sets,
                    set_first=list(sf), off=list(o), seq=C.string_at(seq, int(o[-1])))
        total = int(sum(b * b for b in np.diff(sf)))
        _host(out, C.c_double, total)[:] = np.arange(total)
        _host(status, C.c_int32, total)[:] = np.arange(total) % 6
    stub.effects["phmm_mutation_prime_sets"] = effect
    got = engine.mutation_prime_sets(model, [["ACG", b"TT"], [], [np.frombuffer(b"GGGG", np.uint8)], ["A", "CC", "GGG"]])
    assert seen == {"handles": (HANDLE, HANDLE), "n_sets": 4, "set_first": [0, 2, 2, 3, 6], "off": [0, 3, 5, 9, 10, 12, 15],
                    "seq": b"ACGTTGGGGACCGGG"}
    assert [o.shape for o, _ in got] == [(2, 2), (0, 0), (1, 1), (3, 3)] and [s.shape for _, s in got] == [(2, 2), (0, 0), (1, 1), (3, 3)]
    assert all(o.dtype == np.float64 and s.dtype == np.int32 for o, s in got)
    assert got[0][0].reshape(-1).tolist() == [0, 1, 2, 3] and got[2][0].tolist() == [[4]] and got[3][0].reshape(-1).tolist() == list(range(5, 14))
    assert got[3][1].reshape(-1).tolist() == [x % 6 for x in range(5, 14)]
    assert engine.mutation_prime_sets(model, []) == [] and stub.calls[-1][1][2] == 0
    stub.rc["phmm_mutation_prime_sets"] = _lib.PHMM_ERR_INVALID
    with pytest.raises(PhmmError, match="stub says no") as ex:
        engine.mutation_prime_sets(model, [["A"]])
    assert ex.value.code == _lib.PHMM_ERR_INVALID


def test_batcher_mutation_prime_marshals_as_mutation_prime(stub):
    engine = PairHMMEngine(1)
    batcher = PopulateBatcher()
    model = MutationModel(1e-8, np.full((2, 3), 0.5, np.float32), np.full((2, 3, 4), 0.25, np.float32))
    seqs = ["ACG", b"TT", np.frombuffer(b"GGGG", np.uint8)]
    seen = []

    def effect(h, m, n, off, seq, out, status):
        o = _host(off, C.c_int64, n + 1)
        seen.append((n, list(o), C.string_at(seq, int(o[-1]))))
        _host(out, C.c_double, n * n)[:] = np.arange(n * n)
        _host(status, C.c_int32, n * n)[:] = 1
    stub.effects["phmm_mutation_prime"] = stub.effects["phmm_batcher_mutation_prime"] = effect
    want = engine.mutation_prime(model, seqs)
    got = batcher.mutation_prime(model, seqs)
    assert seen[0] == seen[1] == (3, [0, 3, 5, 9], b"ACGTTGGGG")
    assert stub.only("phmm_batcher_mutation_prime")[0].value == HANDLE
    for a, b in zip(got, want):
        assert a.dtype == b.dtype and a.shape == b.shape == (3, 3) and np.array_equal(a, b)
    stub.rc["phmm_batcher_mutation_prime"] = _lib.PHMM_ERR_INVALID
    with pytest.raises(PhmmError, match="stub says no"):
        batcher.mutation_prime(model, seqs)
