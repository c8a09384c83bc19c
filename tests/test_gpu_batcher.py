"""The shared engine (phmm_batcher_*, PopulateBatcher, the C++ adapter's SharedEngine): populate requests from many threads merged
into one multi-region kernel chain, each request with exactly the result it gets alone on an engine of its own."""
import ctypes as C
import os
import subprocess
import tempfile
import threading

import numpy as np
import pytest

from exact import assert_same_penalties
from helpers import random_positions, random_region

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SRC = os.path.join(ROOT, "tests", "cpp", "test_batcher.cpp")
BAD_PENALTY = "snv prior / gap penalty outside [0,127]"


def _build_cpp():
    """Compile the driver into a fresh temporary directory (the source tree may be read-only) and return its path."""
    from octopus_b200 import build
    build.build()
    exe = os.path.join(tempfile.mkdtemp(prefix="test_batcher_"), "test_batcher")
    subprocess.run(["g++", "-std=c++14", "-O1", "-pthread", "-I", os.path.join(ROOT, "include"), "-I", os.path.join(ROOT, "octopus_b200", "cpp"),
                    SRC, "-o", exe, "-L", os.path.join(ROOT, "octopus_b200"), "-lphmm_b200",
                    "-Wl,-rpath," + os.path.join(ROOT, "octopus_b200")], check=True)
    return exe


def test_cpp_shared_engine_driver_compiles():
    assert os.path.exists(_build_cpp())


def test_batcher_create_without_gpu_is_a_cuda_error():
    import torch
    if torch.cuda.is_available():
        pytest.skip("GPU present")
    from octopus_b200 import PhmmError, PopulateBatcher
    with pytest.raises(PhmmError) as ei:
        PopulateBatcher(0, clients=4)
    assert ei.value.code == -2          # PHMM_ERR_CUDA


# ---------------------------------------------------------------------------------------------------------------------
# helpers: one request through the raw C calls, alone on an engine or through a batcher
# ---------------------------------------------------------------------------------------------------------------------
def _structs(cfg, haps, reads, positions, flank):
    from octopus_b200 import _lib
    keep = [cfg.c_struct(), haps.c_struct(), reads.c_struct()]
    ps = None
    if positions is not None:
        off, pos = np.ascontiguousarray(positions[0], np.int64), np.ascontiguousarray(positions[1], np.int32)
        keep += [off, pos]
        ps = _lib.Positions(off.ctypes.data, pos.ctypes.data)
    fs = None if flank is None else _lib.FlankState(1, int(flank[0]), int(flank[1]))
    ref = lambda s: C.byref(s) if s is not None else None       # noqa: E731
    return keep, ref(keep[0]), ref(keep[1]), ref(keep[2]), ref(ps), ref(fs), ps, fs


def _alone(engine, req):
    """(rc, message, out, status) of phmm_populate / phmm_populate_templates for the request on its own engine."""
    cfg, haps, reads, positions, flank, toff = req
    keep, c, h, r, p, f, ps, fs = _structs(cfg, haps, reads, positions, flank)
    st = np.full((haps.n, reads.n), -7, np.int32)
    lib = engine._lib
    if toff is not None:
        t = np.ascontiguousarray(toff, np.int64)
        out = np.zeros((haps.n, len(t) - 1))
        rc = lib.phmm_populate_templates(engine._h, c, h, r, t.ctypes.data, len(t) - 1, None, f, out.ctypes.data, st.ctypes.data, 0)
    else:
        out = np.zeros((haps.n, reads.n))
        rc = lib.phmm_populate(engine._h, c, h, r, p, f, out.ctypes.data, st.ctypes.data, 0)
    return rc, (lib.phmm_last_error(engine._h).decode() if rc else ""), out, st


def _batched(batcher, req):
    """(rc, message, out, status) of phmm_batcher_populate / _templates, on the calling thread."""
    cfg, haps, reads, positions, flank, toff = req
    keep, c, h, r, p, f, ps, fs = _structs(cfg, haps, reads, positions, flank)
    st = np.full((haps.n, reads.n), -7, np.int32)
    lib = batcher._lib
    if toff is not None:
        t = np.ascontiguousarray(toff, np.int64)
        out = np.zeros((haps.n, len(t) - 1))
        rc = lib.phmm_batcher_populate_templates(batcher._h, c, h, r, t.ctypes.data, len(t) - 1, f, out.ctypes.data, st.ctypes.data)
    else:
        out = np.zeros((haps.n, reads.n))
        rc = lib.phmm_batcher_populate(batcher._h, c, h, r, p, f, out.ctypes.data, st.ctypes.data)
    return rc, (lib.phmm_batcher_last_error().decode() if rc else ""), out, st


def _truncate_haplotype(haps, h, length):
    from octopus_b200.batch import pack_haplotypes
    parts = [haps.hap(i) for i in range(haps.n)]
    parts[h] = {k: v[:length] for k, v in parts[h].items()}
    fields = ("seq", "snv_mask_fwd", "snv_prior_fwd", "snv_mask_rev", "snv_prior_rev", "gap_open", "gap_extend")
    return pack_haplotypes(*[[p[f] for p in parts] for f in fields], begin=haps.begin)


def _make_request(k, i):
    """Thread k's request i. Every thread's request i has the same config, so concurrent requests can share a batch."""
    from octopus_b200 import HaplotypeLikelihoodModel
    rng = np.random.default_rng(7000 + 100 * k + i)
    band = (8, 16, 32)[i % 3]
    mapit = i % 2 == 0
    hap_len = 2 * band + int(rng.choice([200, 260]))
    haps, reads = random_region(rng, band, n_haps=int(rng.integers(2, 20)), n_reads=int(rng.integers(10, 90)), hap_len=hap_len,
                                read_len_choices=[40, 76, 100, 150], read_n_rate=0.05, edge_reads=(k % 2 == 0))
    cfg = HaplotypeLikelihoodModel.Config(max_indel_error=band, map_positions=mapit)
    flank = (int(rng.integers(0, 80)), int(rng.integers(0, 80))) if (k + i) % 2 else None
    positions, toff, kind = None, None, "reads"
    if k in (2, 7) and i == 5:
        haps = _truncate_haplotype(haps, 0, 90)          # shorter than the 100 / 150 bp reads
        kind = "short"
    if k == 4 and i == 6:
        haps.gap_open.view(np.uint8)[5] = 200            # a gap penalty of 200: outside [0,127]
        kind = "bad_penalty"
    if k == 6 and i == 4:
        positions = random_positions(rng, haps, reads)
        kind = "positions"
    if kind == "reads" and i % 4 == 3:
        sizes = rng.integers(1, 3, reads.n)
        toff = np.concatenate([[0], np.cumsum(sizes)])
        toff = toff[toff < reads.n].tolist() + [reads.n]
        kind = "templates"
    if kind == "reads" and i % 4 == 1:
        kind = "samples"                                 # a two-sample ReadMap through HaplotypeLikelihoodArray
    return kind, (cfg, haps, reads, positions, flank, None if toff is None else np.asarray(toff, np.int64))


@pytest.mark.gpu
def test_concurrent_requests_equal_one_engine_each(engine):
    from octopus_b200 import HaplotypeLikelihoodArray, HaplotypeLikelihoodModel, PopulateBatcher
    from octopus_b200.batch import ReadBlock
    n_threads, n_requests = 12, 8
    reqs = {(k, i): _make_request(k, i) for k in range(n_threads) for i in range(n_requests)}
    got, errors = {}, []
    batcher = PopulateBatcher(0, clients=n_threads, max_wait_us=20000)
    start = threading.Barrier(n_threads)

    def worker(k):
        try:
            start.wait()
            for i in range(n_requests):
                kind, req = reqs[(k, i)]
                if kind == "samples":
                    cfg, haps, reads = req[:3]
                    half = reads.n // 2
                    split = [ReadBlock(reads.off[a:b + 1] - reads.off[a], reads.bases[reads.off[a]:reads.off[b]], reads.quals[reads.off[a]:reads.off[b]],
                                       reads.mapq[a:b], reads.reverse[a:b], reads.begin[a:b]) for a, b in ((0, half), (half, reads.n))]
                    arr = HaplotypeLikelihoodArray(HaplotypeLikelihoodModel(cfg), engine=batcher)
                    arr.populate({"S1": split[0], "S2": split[1]}, haps, flank_state=req[4])
                    got[(k, i)] = (0, "", np.asarray(arr.likelihoods), None)
                else:
                    got[(k, i)] = _batched(batcher, req)
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

    seen = set()
    for key, (kind, req) in reqs.items():
        rc, msg, out, st = got[key]
        wrc, wmsg, want, wst = _alone(engine, req)
        seen.add(kind)
        assert rc == wrc, (key, kind, rc, wrc, msg, wmsg)
        if kind == "short":
            assert rc == -4, (key, rc)
        elif kind == "bad_penalty":
            assert rc == -1 and msg == BAD_PENALTY == wmsg, (key, msg, wmsg)
            continue
        else:
            assert rc == 0, (key, kind, rc, msg)
        if st is not None:
            assert np.array_equal(st, wst), (key, kind, np.argwhere(st != wst)[:10])
        ok = (wst & 0xFFFF) == 0
        if req[5] is not None:                           # a template's value is compared where all its reads are OK
            toff = req[5]
            ok = np.stack([ok[:, toff[t]:toff[t + 1]].all(axis=1) for t in range(len(toff) - 1)], axis=1)
        assert np.array_equal(out.view(np.int64)[ok], want.view(np.int64)[ok]), (key, kind, np.argwhere(ok & (out != want))[:10])
    assert seen == {"reads", "samples", "templates", "short", "bad_penalty", "positions"}, seen
    # the bad-penalty request never reaches the GPU; everything else does, merged
    assert stats["requests"] == n_threads * n_requests - 1, stats
    assert stats["gpu_calls"] * 4 <= stats["requests"], stats
    assert stats["max_regions_per_call"] >= 8 and stats["merged_calls"] >= 1 and stats["dp_cells"] > 0, stats


@pytest.mark.gpu
def test_short_haplotype_raises_in_its_own_thread_only():
    from octopus_b200 import HaplotypeLikelihoodModel, PopulateBatcher, ShortHaplotypeError
    rng = np.random.default_rng(5)
    cfg = HaplotypeLikelihoodModel.Config(max_indel_error=16)
    regions = [random_region(rng, 16, n_haps=6, n_reads=40, hap_len=300, read_len_choices=[100, 150]) for _ in range(4)]
    regions[1] = (_truncate_haplotype(regions[1][0], 2, 80), regions[1][1])
    outcome = {}
    with PopulateBatcher(0, clients=4, max_wait_us=20000) as batcher:
        def worker(g):
            try:
                batcher.populate(cfg, *regions[g])
                outcome[g] = "ok"
            except ShortHaplotypeError:
                outcome[g] = "short"
        threads = [threading.Thread(target=worker, args=(g,)) for g in range(4)]
        for t in threads:
            t.start()
        for t in threads:
            t.join(timeout=120)
        assert batcher.stats()["max_regions_per_call"] >= 2
    assert outcome == {0: "ok", 1: "short", 2: "ok", 3: "ok"}, outcome


@pytest.mark.gpu
def test_merged_batch_matches_oracle(coracle):
    """One merged batch without mapping quality: every request's values bit-equal the oracle's integer penalties."""
    from octopus_b200 import HaplotypeLikelihoodModel, PopulateBatcher
    rng = np.random.default_rng(91)
    band, n = 16, 6
    cfg = HaplotypeLikelihoodModel.Config(max_indel_error=band, use_mapping_quality=False)
    regions = []
    for g in range(n):
        haps, reads = random_region(rng, band, n_haps=int(rng.integers(2, 12)), n_reads=int(rng.integers(10, 60)), hap_len=2 * band + 230,
                                    read_len_choices=[76, 100, 150], read_n_rate=0.05, edge_reads=(g % 2 == 0))
        regions.append((haps, reads, (int(rng.integers(0, 80)), int(rng.integers(0, 80))) if g % 2 else None))
    got = {}
    with PopulateBatcher(0, clients=n, max_wait_us=200000) as batcher:
        def worker(g):
            haps, reads, flank = regions[g]
            got[g] = batcher.populate(cfg, haps, reads, flank_state=flank, want_status=True)
        threads = [threading.Thread(target=worker, args=(g,)) for g in range(n)]
        for t in threads:
            t.start()
        for t in threads:
            t.join(timeout=120)
        stats = batcher.stats()
    assert stats["gpu_calls"] == 1 and stats["max_regions_per_call"] == n, stats
    for g, (haps, reads, flank) in enumerate(regions):
        rc, want, wst = coracle.populate(band, haps, reads, None, flank, use_mapping_quality=False, map_positions=True)
        out, st = got[g]
        assert_same_penalties(out, want, st, wst, g)


@pytest.mark.gpu
def test_lone_thread_is_never_stuck_waiting_for_clients():
    """clients = 8 but only one thread submits: every request goes out after max_wait_us, alone."""
    from octopus_b200 import HaplotypeLikelihoodModel, PopulateBatcher
    rng = np.random.default_rng(13)
    cfg = HaplotypeLikelihoodModel.Config(max_indel_error=8)
    regions = [random_region(rng, 8, n_haps=4, n_reads=20, hap_len=220, read_len_choices=[76]) for _ in range(20)]
    batcher = PopulateBatcher(0, clients=8, max_wait_us=2000)
    done = []

    def worker():
        for haps, reads in regions:
            batcher.populate(cfg, haps, reads)
            done.append(1)
    t = threading.Thread(target=worker)
    t.start()
    t.join(timeout=120)
    assert not t.is_alive() and len(done) == 20
    assert batcher.stats()["gpu_calls"] == 20
    batcher.close()


@pytest.mark.gpu
def test_cpp_threads_share_one_engine():
    exe = _build_cpp()
    out = subprocess.run([exe], capture_output=True, text=True, timeout=300)
    assert out.returncode == 0 and "BATCHER ok" in out.stdout, out.stdout + out.stderr
