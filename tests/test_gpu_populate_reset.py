"""Populate from haplotype sequences (phmm_populate*_reset, phmm_batcher_populate*_reset): the engine runs the error model's reset()
on the device inside the populate call. Every result is held bit for bit (return code, statuses, values at OK pairs) to the two-step
path: host phmm_reset_haplotypes, then the plain populate call."""
import ctypes as C
import threading

import numpy as np
import pytest

from helpers import random_positions, random_region
from test_error_model import LABELS, repeat_rich_sequence
from test_gpu_reset import CUSTOM_TEXTS

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def engine():
    import torch
    if not torch.cuda.is_available():
        pytest.skip("no GPU")
    from octopus_b200 import PairHMMEngine
    return PairHMMEngine(0)


@pytest.fixture(scope="module")
def models():
    from octopus_b200 import ErrorModel
    out = {label: ErrorModel(label) for label in LABELS}
    out.update({"custom%d" % i: ErrorModel(custom_model_text=t) for i, t in enumerate(CUSTOM_TEXTS)})
    return out


def _cfg(band=16, **kw):
    from octopus_b200 import HaplotypeLikelihoodModel
    return HaplotypeLikelihoodModel.Config(max_indel_error=band, **kw)


def _region(rng, band=16, n_haps=8, n_reads=60, hap_len=220, read_lens=(40, 80, 100), repeats=True, subs=False):
    """(HaplotypeSequences, ReadBlock): random_region's reads over haplotypes with tandem repeats where `repeats`."""
    from octopus_b200 import HaplotypeSequences
    haps, reads = random_region(rng, band, n_haps, n_reads, hap_len, read_lens)
    seqs = [haps.seq[haps.off[h]:haps.off[h + 1]].copy() for h in range(haps.n)]
    if repeats:
        for s in seqs:
            r = np.frombuffer(repeat_rich_sequence(rng, 60), dtype=np.uint8)[:len(s) // 3]
            a = int(rng.integers(0, len(s) - len(r) + 1))
            s[a:a + len(r)] = r
    flags = [(rng.random(len(s)) < 0.05).astype(np.uint8) for s in seqs] if subs else None
    return HaplotypeSequences.pack(seqs, begin=haps.begin, is_substitution=flags), reads


def _two_step(model, seqs):
    """The HaplotypeBlock host reset() gives for a sequences block."""
    return model.reset_block(seqs.off, seqs.seq, seqs.begin, seqs.is_substitution)


def _same(a, b, what):
    """(rc, out, status) results equal bit for bit: codes, statuses, and values at OK pairs."""
    (rc_a, out_a, st_a), (rc_b, out_b, st_b) = a, b
    assert rc_a == rc_b, (what, rc_a, rc_b)
    if rc_a not in (0, -4):
        return
    st_a, st_b = np.asarray(st_a), np.asarray(st_b)
    assert np.array_equal(st_a, st_b), what
    ok = st_a == 0
    assert np.array_equal(np.asarray(out_a)[ok].view(np.int64), np.asarray(out_b)[ok].view(np.int64)), what


def _run(call):
    from octopus_b200 import PhmmError
    try:
        out, st = call()
        return 0, out, st
    except PhmmError as e:
        return e.code, None, None


def _host(x):
    return x.cpu().numpy() if hasattr(x, "cpu") else x


def _populate_both(engine, cfg, model, seqs, reads, positions=None, flank=None):
    got = _run(lambda: engine.populate(cfg, seqs, reads, positions, flank, want_status=True, error_model=model))
    want = _run(lambda: engine.populate(cfg, _two_step(model, seqs), reads, positions, flank, want_status=True))
    return got, want


def test_every_model_equals_host_reset_then_populate(engine, models):
    rng = np.random.default_rng(101)
    for name, model in models.items():
        seqs, reads = _region(rng, subs=name.startswith("PCR-free.H"))
        got, want = _populate_both(engine, _cfg(), model, seqs, reads, flank=(5, 7))
        assert got[0] == 0
        _same(got, want, name)


@pytest.mark.parametrize("band", [8, 16, 32, 64])
def test_bands_mapper_flank_and_mapping_quality(engine, models, band):
    rng = np.random.default_rng(200 + band)
    model = models["custom0"] if band == 32 else models["PCR.NovaSeq"]
    for map_positions in (True, False):
        for flank in (None, (4, 9)):
            for use_mq in (True, False):
                seqs, reads = _region(rng, band=band, hap_len=160 + 2 * band)
                cfg = _cfg(band, map_positions=map_positions, use_mapping_quality=use_mq, use_flank_state=flank is not None)
                got, want = _populate_both(engine, cfg, model, seqs, reads, flank=flank)
                _same(got, want, (band, map_positions, flank, use_mq))


def test_explicit_positions_and_substitution_flags(engine, models):
    rng = np.random.default_rng(303)
    model = models["PCR-free.HiSeq-2500"]
    seqs, reads = _region(rng, subs=True)
    plain = _two_step(model, seqs)
    positions = random_positions(rng, plain, reads)
    got, want = _populate_both(engine, _cfg(), model, seqs, reads, positions, (3, 3))
    _same(got, want, "positions")
    # the flags matter: without them the arrays, and so some values, differ
    unflagged = model.reset_block(seqs.off, seqs.seq, seqs.begin)
    assert not np.array_equal(unflagged.snv_prior_fwd, plain.snv_prior_fwd)


def test_short_haplotypes_keep_their_statuses(engine, models):
    rng = np.random.default_rng(404)
    seqs, reads = _region(rng, hap_len=120, read_lens=(100, 118))
    without = [_run(lambda: (engine.populate(_cfg(32), h, reads, error_model=m), None)) for h, m in
               ((seqs, models["custom1"]), (_two_step(models["custom1"], seqs), None))]
    assert without[0][0] == without[1][0] == -4
    got = _run(lambda: engine.populate(_cfg(32), seqs, reads, want_status=True, error_model=models["custom1"]))
    assert got[0] == 0 and ((got[2] & 0xFFFF) == 2).any()       # with statuses requested the short pairs are reported, not raised
    _same(got, _run(lambda: engine.populate(_cfg(32), _two_step(models["custom1"], seqs), reads, want_status=True)), "short")


def test_200_regions_in_one_call_equal_per_region_calls(engine, models):
    from octopus_b200.batch import concat_reads, concat_sequences
    rng = np.random.default_rng(505)
    model = models["PCR.HiSeq-4000"]
    regions = [_region(rng, n_haps=int(rng.integers(1, 9)), n_reads=int(rng.integers(1, 40)), hap_len=int(rng.integers(150, 320)),
                       subs=bool(rng.random() < 0.3)) for _ in range(200)]
    seqs = concat_sequences([s for s, _ in regions])
    reads = concat_reads([r for _, r in regions])
    hap_first = np.concatenate([[0], np.cumsum([s.n for s, _ in regions])])
    read_first = np.concatenate([[0], np.cumsum([r.n for _, r in regions])])
    flanks = [(int(rng.integers(0, 20)), int(rng.integers(0, 20))) if rng.random() < 0.5 else None for _ in regions]
    cfg = _cfg(16)
    flat, off, st = engine.populate_regions(cfg, seqs, reads, hap_first, read_first, flanks, want_status=True, error_model=model)
    flat2, _, st2 = engine.populate_regions(cfg, _two_step(model, seqs), reads, hap_first, read_first, flanks, want_status=True)
    _same((0, flat, st), (0, flat2, st2), "regions vs two-step")
    for g, (s, r) in enumerate(regions):
        one = _run(lambda: engine.populate(cfg, s, r, None, flanks[g], want_status=True, error_model=model))
        _same((0, flat[off[g]:off[g + 1]].reshape(s.n, r.n), st[off[g]:off[g + 1]].reshape(s.n, r.n)), one, g)


def test_templates(engine, models):
    rng = np.random.default_rng(606)
    model = models["10X.X10"] if "10X.X10" in models else models["PCR-free.X10"]
    seqs, reads = _region(rng, n_reads=64)
    toff = np.concatenate([[0], np.sort(rng.choice(np.arange(1, 64), 20, replace=False)), [64]])
    got = engine.populate_templates(_cfg(), seqs, reads, toff, (2, 2), error_model=model)
    want = engine.populate_templates(_cfg(), _two_step(model, seqs), reads, toff, (2, 2))
    assert np.array_equal(got.view(np.int64), want.view(np.int64))


def test_pipelined_host_call(engine, models):
    """32 haplotypes x 131 072 reads: the size at which the plain populate pipelines over two sub-engines."""
    from octopus_b200.batch import pack_reads
    rng = np.random.default_rng(707)
    model = models["PCR-free.NovaSeq"]
    seqs, small = _region(rng, n_haps=32, n_reads=64, hap_len=300, read_lens=(50,))
    R = 131072
    pick = rng.integers(0, small.n, R)
    reads = pack_reads([small.bases[small.off[i]:small.off[i + 1]] for i in pick], [small.quals[small.off[i]:small.off[i + 1]] for i in pick],
                       small.mapq[pick], small.reverse[pick], small.begin[pick])
    got, want = _populate_both(engine, _cfg(), model, seqs, reads, flank=(10, 10))
    assert got[0] == 0
    _same(got, want, "pipelined")


def test_device_space_equals_host_space(engine, models):
    rng = np.random.default_rng(808)
    for name in ("custom0", "PCR-free.HiSeq-2500"):
        seqs, reads = _region(rng, subs=True)
        host = _run(lambda: engine.populate(_cfg(), seqs, reads, None, (6, 2), want_status=True, error_model=models[name]))
        dev = _run(lambda: engine.populate(_cfg(), seqs.to_device(), reads.to_device(), None, (6, 2), want_status=True, error_model=models[name]))
        _same(host, (dev[0], _host(dev[1]), _host(dev[2])), name)
        dev_two_step = engine.populate(_cfg(), _two_step(models[name], seqs).to_device(), reads.to_device(), None, (6, 2))
        assert np.array_equal(_host(dev[1])[host[2] == 0].view(np.int64), _host(dev_two_step)[host[2] == 0].view(np.int64))


def _raw(engine, model_h, seqs_struct, reads, space=0, cfg=None):
    from octopus_b200 import _lib
    cfg = (cfg or _cfg()).c_struct()
    out = np.zeros(64 * max(reads.n, 1))
    rc = engine._lib.phmm_populate_reset(engine._h, C.byref(cfg), model_h, seqs_struct, C.byref(reads.c_struct()), None, None,
                                         out.ctypes.data, None, space)
    return rc, engine._lib.phmm_last_error(engine._h).decode() if rc else ""


def test_argument_errors(engine, models):
    from octopus_b200 import HaplotypeSequences, _lib
    rng = np.random.default_rng(909)
    model = models["PCR.NovaSeq"]
    seqs, reads = _region(rng, n_haps=2, n_reads=4)
    ok = C.byref(seqs.c_struct())
    assert _raw(engine, model._h, ok, reads) == (0, "")
    assert _raw(engine, None, ok, reads) == (_lib.PHMM_ERR_INVALID, "null argument")
    assert _raw(engine, model._h, None, reads) == (_lib.PHMM_ERR_INVALID, "null argument")
    s = seqs.c_struct(); s.seq = None
    assert _raw(engine, model._h, C.byref(s), reads) == (_lib.PHMM_ERR_INVALID, "null argument")
    assert _raw(engine, model._h, ok, reads, space=3) == (_lib.PHMM_ERR_INVALID, "bad memory space")
    bad = HaplotypeSequences(np.array([0, 10, 5], np.int64), seqs.seq)
    assert _raw(engine, model._h, C.byref(bad.c_struct()), reads) == (_lib.PHMM_ERR_INVALID, "bad haplotype offsets")
    long = HaplotypeSequences.pack([b"ACGT" * 16384 + b"A"])
    assert _raw(engine, model._h, C.byref(long.c_struct()), reads) == (_lib.PHMM_ERR_INVALID, "haplotype longer than 65535 bases")
    # n == 0 and a bad config: what the plain twin reports
    empty = HaplotypeSequences(np.zeros(1, np.int64), np.zeros(0, np.uint8))
    want = engine._lib.phmm_populate(engine._h, C.byref(_cfg().c_struct()), C.byref(model.reset([]).c_struct()), C.byref(reads.c_struct()),
                                     None, None, np.zeros(4).ctypes.data, None, 0)
    assert _raw(engine, model._h, C.byref(empty.c_struct()), reads) == (want, engine._lib.phmm_last_error(engine._h).decode())
    assert _raw(engine, model._h, ok, reads, cfg=_cfg(300)) == (_lib.PHMM_ERR_BAND, "max_indel_error > 256")
    with pytest.raises(TypeError):
        engine.populate(_cfg(), _two_step(model, seqs), reads, error_model=model)


def test_last_dp_kernel_time_and_cells_are_populate_s(engine, models):
    rng = np.random.default_rng(1001)
    seqs, reads = _region(rng, n_haps=16, n_reads=200)
    model = models["PCR.NovaSeq"]
    engine.populate(_cfg(disable_naive_shortcut=True), _two_step(model, seqs), reads)
    cells = engine.last_dp_cells()
    engine.populate(_cfg(disable_naive_shortcut=True), seqs, reads, error_model=model)
    assert engine.last_dp_cells() == cells and engine.last_dp_kernel_ms() > 0


def test_against_c_oracle_with_reference_model_arrays(engine, coracle):
    from oracle.oracle import RefErrorModel
    if not RefErrorModel.available():
        pytest.skip("reference error models not built")
    from octopus_b200 import ErrorModel
    from octopus_b200.batch import pack_haplotypes
    ref = RefErrorModel()
    rng = np.random.default_rng(1101)
    seqs, reads = _region(rng, n_haps=6, n_reads=80)
    label = "PCR.HiSeq-2500"
    arrs = [ref.reset(bytes(seqs.seq[seqs.off[h]:seqs.off[h + 1]]), label=label) for h in range(seqs.n)]
    fields = ("snv_mask_fwd", "snv_prior_fwd", "snv_mask_rev", "snv_prior_rev", "gap_open", "gap_extend")
    haps = pack_haplotypes([seqs.seq[seqs.off[h]:seqs.off[h + 1]] for h in range(seqs.n)], *[[a[f] for a in arrs] for f in fields],
                           begin=seqs.begin)
    band, flanks = 16, (8, 8)
    rc, want, wst = coracle.populate(band, haps, reads, None, flanks, use_mapping_quality=False, map_positions=True)
    got, st = engine.populate(_cfg(band, use_mapping_quality=False), seqs, reads, None, flanks, want_status=True, error_model=ErrorModel(label))
    ok = wst == 0
    assert np.array_equal(st[~ok], wst[~ok]) and np.array_equal(got[ok], want[ok])


# ---------------------------------------------------------------------------------------------------------------------
# the shared engine
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("threads", [8, 32])
def test_batcher_mixes_plain_and_reset_requests_under_two_models(engine, models, threads):
    from octopus_b200 import PopulateBatcher
    rng = np.random.default_rng(1200 + threads)
    two = [models["PCR.NovaSeq"], models["custom0"]]
    reqs = []
    for i in range(threads * 3):
        short = i == 5
        seqs, reads = _region(rng, n_haps=int(rng.integers(2, 9)), n_reads=int(rng.integers(5, 50)), hap_len=90 if short else 220,
                              read_lens=(100,) if short else (40, 80, 100), subs=bool(i % 3 == 0))
        kind = "plain" if i % 4 == 0 else "reset"
        reqs.append((kind, two[i % 2], seqs, reads, (3, 4) if i % 2 else None))
    cfg = _cfg(16)

    def solo(kind, model, seqs, reads, flank):
        if kind == "plain":
            return _run(lambda: engine.populate(cfg, _two_step(model, seqs), reads, None, flank, want_status=True))
        return _run(lambda: engine.populate(cfg, seqs, reads, None, flank, want_status=True, error_model=model))
    want = [solo(*q) for q in reqs]
    short = [i for i, w in enumerate(want) if ((w[2] & 0xFFFF) == 2).any()]
    assert short == [5]
    got = [None] * len(reqs)
    with PopulateBatcher(0, clients=threads, max_wait_us=2000) as b:
        def work(t):
            for i in range(t, len(reqs), threads):
                kind, model, seqs, reads, flank = reqs[i]
                haps = _two_step(model, seqs) if kind == "plain" else seqs
                got[i] = _run(lambda: b.populate(cfg, haps, reads, None, flank, want_status=True,
                                                 error_model=None if kind == "plain" else model))
        ts = [threading.Thread(target=work, args=(t,)) for t in range(threads)]
        for t in ts:
            t.start()
        for t in ts:
            t.join()
        stats = b.stats()
    for i, (g, w) in enumerate(zip(got, want)):
        _same(g, w, i)
    assert stats["merged_calls"] > 0


def test_batcher_reset_templates_and_run_alone(engine, models):
    from octopus_b200 import PopulateBatcher
    rng = np.random.default_rng(1300)
    model = models["PCR-free.HiSeq-2500"]
    seqs, reads = _region(rng, n_reads=30)
    toff = np.array([0, 2, 5, 9, 30])
    want = engine.populate_templates(_cfg(), seqs, reads, toff, (1, 2), error_model=model)
    positions = random_positions(rng, _two_step(model, seqs), reads)
    want_pos = engine.populate(_cfg(), seqs, reads, positions, None, error_model=model)
    with PopulateBatcher(0) as b:
        assert np.array_equal(b.populate_templates(_cfg(), seqs, reads, toff, (1, 2), error_model=model).view(np.int64), want.view(np.int64))
        assert np.array_equal(b.populate(_cfg(), seqs, reads, positions, error_model=model).view(np.int64), want_pos.view(np.int64))


# ---------------------------------------------------------------------------------------------------------------------
# the host recompute of haplotypes that overflow their device slot, and the C++ adapter
# ---------------------------------------------------------------------------------------------------------------------
OVERFLOW_SCRIPT = r"""
import numpy as np, sys
sys.path.insert(0, sys.argv[1]); sys.path.insert(0, sys.argv[1] + "/tests")
from test_gpu_populate_reset import _cfg, _region, _two_step, _run, _same, _host
from octopus_b200 import ErrorModel, PairHMMEngine
e = PairHMMEngine(0)
rng = np.random.default_rng(1400)
for name, model in (("PCR.NovaSeq", ErrorModel("PCR.NovaSeq")), ("custom", ErrorModel(custom_model_text="A:30,25,20\nAC:26,20,14\nNN:24,18\n"))):
    seqs, reads = _region(rng, n_haps=12, subs=True)
    want = _run(lambda: e.populate(_cfg(), _two_step(model, seqs), reads, None, (3, 3), want_status=True))
    _same(_run(lambda: e.populate(_cfg(), seqs, reads, None, (3, 3), want_status=True, error_model=model)), want, name + " host")
    dev = _run(lambda: e.populate(_cfg(), seqs.to_device(), reads.to_device(), None, (3, 3), want_status=True, error_model=model))
    _same((dev[0], _host(dev[1]), _host(dev[2])), want, name + " device")
print("OVERFLOW ok")
"""


def test_haplotypes_that_overflow_their_device_slot_are_recomputed_on_the_host():
    """PHMM_RESET_CAP forces a device run capacity of 4: nearly every haplotype overflows, and its arrays come from the host recompute,
    written into the engine's buffers (host space from off[0] = 0, and device space)."""
    import os
    import subprocess
    import sys
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    env = dict(os.environ, PHMM_RESET_CAP="4", PHMM_TRACE="1")
    run = subprocess.run([sys.executable, "-c", OVERFLOW_SCRIPT, root], capture_output=True, text=True, timeout=600, env=env)
    assert run.returncode == 0 and "OVERFLOW ok" in run.stdout, run.stdout + run.stderr
    counts = [int(line.split("reset: ")[1].split()[0]) for line in run.stderr.splitlines() if "reset: " in line]
    assert len(counts) == 4 and all(c > 0 for c in counts), run.stderr


def test_cpp_threads_populate_from_sequences_on_one_shared_engine(engine):
    import os
    import subprocess
    import tempfile
    from octopus_b200 import build
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    build.build()
    exe = os.path.join(tempfile.mkdtemp(prefix="test_populate_reset_"), "test_populate_reset")
    subprocess.run(["g++", "-std=c++14", "-O1", "-pthread", "-I", os.path.join(root, "include"), "-I", os.path.join(root, "octopus_b200", "cpp"),
                    os.path.join(root, "tests", "cpp", "test_populate_reset.cpp"), "-o", exe, "-L", os.path.join(root, "octopus_b200"),
                    "-lphmm_b200", "-Wl,-rpath," + os.path.join(root, "octopus_b200")], check=True)
    run = subprocess.run([exe], capture_output=True, text=True, timeout=600)
    assert run.returncode == 0 and "RESET ok" in run.stdout, run.stdout + run.stderr
    requests, gpu_calls, merged = (int(x) for x in run.stdout.split()[2:5])
    assert gpu_calls < requests and merged >= 1, run.stdout
