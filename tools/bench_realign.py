#!/usr/bin/env python
"""Throughput of phmm_realign_reads (ReadRealigner::realign: uncapped k-mer mapping + HaplotypeLikelihoodModel::align per pair) on a
ReadAssignments-shaped workload: many groups, each of 2 haplotypes of 400-800 bases and 20-300 reads of 150 bases, one pair per read
(the read against its assigned haplotype). Bands 8 (the realigner's default model) and 16; a plain and a repeat-rich variant (a third
of every haplotype is a short tandem repeat, so reads tie on many diagonals).

Per (variant, band) one JSON line:
  realign_ms / realign_pairs_per_s
                          wall time of one phmm_realign_reads C call on host arrays, copies included (median of --reps calls; a
                          call returns after its final synchronisation)
  kernels_ms / mapper_share
                          all kernel time of one realign call, and the mapper's part of it (read hashes, haplotype tables,
                          k_kmer_map_pairs, offset scan), from torch.profiler in a separate run
  host_map_s / host_align_ms / host_path_pairs_per_s
                          the same pairs mapped on the host (the C oracle's uncapped mapper, one ctypes call per pair, so Python's
                          loop overhead is included) followed by one phmm_align_reads C call on those positions
The device name, power limit and SM clock limit are printed beside the figures. Needs a GPU; writes nothing but stdout (and --out)."""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

ACGT = np.frombuffer(b"ACGT", dtype=np.uint8)
MAPPER_KERNELS = ("k_kmer_map_pairs", "k_csr_scan", "k_read_kmers", "k_build_kmer_table")


def workload(rng, n_groups, repeat_rich, read_len=150):
    from octopus_b200.batch import HaplotypeBlock, ReadBlock
    seqs, reads, quals, begins, pairs = [], [], [], [], []
    r = 0
    for g in range(n_groups):
        L = int(rng.integers(400, 801))
        a = ACGT[rng.integers(0, 4, L)].copy()
        if repeat_rich:
            unit = ACGT[rng.integers(0, 4, int(rng.integers(1, 5)))]
            p, n = int(rng.integers(0, L // 2)), L // 3
            a[p:p + n] = np.tile(unit, n // len(unit) + 1)[:n]
        b = a.copy()
        b[rng.integers(0, L, 2)] = ACGT[rng.integers(0, 4, 2)]
        seqs += [a, b]
        for _ in range(int(rng.integers(20, 301))):
            h = int(rng.integers(0, 2))
            s = (a, b)[h]
            p = int(rng.integers(0, L - read_len + 1))
            x = s[p:p + read_len].copy()
            x[rng.integers(0, read_len, int(rng.integers(0, 3)))] = ACGT[rng.integers(0, 4)]
            reads.append(x); quals.append(rng.integers(10, 41, read_len).astype(np.uint8)); begins.append(p)
            pairs.append((r, 2 * g + h))
            r += 1
    hoff = np.concatenate([[0], np.cumsum([len(s) for s in seqs])]).astype(np.int64)
    seq = np.concatenate(seqs)
    T = len(seq)
    haps = HaplotypeBlock(hoff, seq, np.roll(seq, 1), rng.integers(20, 126, T).astype(np.int8), np.roll(seq, -1),
                          rng.integers(20, 126, T).astype(np.int8), rng.integers(8, 46, T).astype(np.int8), rng.integers(1, 11, T).astype(np.int8),
                          begin=np.zeros(len(seqs), np.int64))
    roff = np.concatenate([[0], np.cumsum([len(x) for x in reads])]).astype(np.int64)
    rb = ReadBlock(roff, np.concatenate(reads), np.concatenate(quals), rng.choice([20, 60], r).astype(np.uint8),
                   (rng.random(r) < 0.5).astype(np.uint8), np.asarray(begins, np.int64))
    return haps, rb, np.asarray(pairs, np.int32)


def device_info():
    import torch
    info = {"device": torch.cuda.get_device_name(0)}
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=power.limit,clocks.max.sm,clocks.sm", "--format=csv,noheader"],
                           capture_output=True, text=True, timeout=30).stdout.strip().splitlines()[0]
        info["power_limit"], info["sm_clock_max"], info["sm_clock_now"] = [x.strip() for x in q.split(",")]
    except Exception as ex:        # the figures are still printed, marked as lacking their conditions
        info["nvidia_smi"] = "unavailable: %s" % ex
    return info


def abi_call(engine, cfg, haps, reads, pairs, positions=None):
    """A zero-argument call of phmm_realign_reads (positions None) or phmm_align_reads (positions = CSR) on preallocated host
    buffers: times the C ABI call itself, without the Python wrapper's allocation and CIGAR decoding."""
    import ctypes as C
    from octopus_b200 import _lib
    n = len(pairs)
    stride = 4 * int(np.diff(reads.off).max()) + 64
    pr = np.ascontiguousarray(pairs, dtype=np.int32)
    mp, lk, st, cg = np.zeros(n, np.int64), np.zeros(n, np.float64), np.zeros(n, np.int32), np.zeros(n * stride, np.uint8)
    keep = (pr, mp, lk, st, cg, haps.c_struct(), reads.c_struct(), cfg.c_struct())
    hs, rs, cs = keep[5:]
    lib, h = engine._lib, engine._h
    if positions is None:
        def call():
            return lib.phmm_realign_reads(h, C.byref(cs), C.byref(hs), C.byref(rs), pr.ctypes.data, n, None, mp.ctypes.data, lk.ctypes.data,
                                          cg.ctypes.data, stride, st.ctypes.data, _lib.SPACE_HOST)
    else:
        off, pos = (np.ascontiguousarray(positions[0], np.int64), np.ascontiguousarray(positions[1], np.int32))
        ps = _lib.Positions(off.ctypes.data, pos.ctypes.data)
        keep += (off, pos, ps)

        def call():
            return lib.phmm_align_reads(h, C.byref(cs), C.byref(hs), C.byref(rs), pr.ctypes.data, n, C.byref(ps), None, mp.ctypes.data,
                                        lk.ctypes.data, cg.ctypes.data, stride, st.ctypes.data, _lib.SPACE_HOST)
    call.keep = keep
    return call


def median_ms(call, reps):
    assert call() == 0                 # warm-up: allocations, module load
    times = []
    for _ in range(reps):
        t0 = time.perf_counter()
        assert call() == 0             # returns after the call's final synchronisation
        times.append(time.perf_counter() - t0)
    return 1e3 * float(np.median(times))


def mapper_share(engine, cfg, haps, reads, pairs):
    import torch
    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        engine.realign_reads(cfg, haps, reads, pairs)
        torch.cuda.synchronize()
    total = mapper = 0.0
    for ev in prof.events():
        if ev.device_type.name != "CUDA" or "memcpy" in ev.name.lower() or "memset" in ev.name.lower():
            continue
        t = ev.device_time_total if hasattr(ev, "device_time_total") else ev.cuda_time_total
        total += t
        if any(k in ev.name for k in MAPPER_KERNELS):
            mapper += t
    return mapper / total if total else float("nan"), total / 1e3


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--groups", type=int, default=400)
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    import torch
    assert torch.cuda.is_available(), "bench_realign needs a GPU"
    from octopus_b200 import HaplotypeLikelihoodModel, PairHMMEngine
    from oracle.oracle import COracle
    co = COracle()
    eng = PairHMMEngine(0)
    info = device_info()
    print(json.dumps(info))
    rows = []
    for repeat_rich in (False, True):
        haps, reads, pairs = workload(np.random.default_rng(11 + repeat_rich), a.groups, repeat_rich)
        for band in (8, 16):
            cfg = HaplotypeLikelihoodModel.Config(max_indel_error=band)
            got = eng.realign_reads(cfg, haps, reads, pairs)
            realign_ms = median_ms(abi_call(eng, cfg, haps, reads, pairs), a.reps)
            share, kernels_ms = mapper_share(eng, cfg, haps, reads, pairs)
            # host path: the C oracle's uncapped mapper per pair, then phmm_align_reads on its positions
            t0 = time.perf_counter()
            lists = []
            for r, h in pairs:
                hb, he = int(haps.off[h]), int(haps.off[h + 1])
                rb, re_ = int(reads.off[r]), int(reads.off[r + 1])
                lists.append(co.kmer_map(reads.bases[rb:re_].tobytes().decode("latin1"), haps.seq[hb:he].tobytes().decode("latin1"), he - hb))
            t_map = time.perf_counter() - t0
            off = np.concatenate([[0], np.cumsum([len(x) for x in lists])]).astype(np.int64)
            pos = np.concatenate([np.asarray(x, np.int32) for x in lists] + [np.zeros(1, np.int32)])
            align_ms = median_ms(abi_call(eng, cfg, haps, reads, pairs, (off, pos)), a.reps)
            want = eng.align_reads(cfg, haps, reads, pairs, (off, pos))
            same = bool(np.array_equal(got[0], want[0]) and np.array_equal(got[1].view(np.int64), want[1].view(np.int64)) and got[2] == want[2]
                        and np.array_equal(got[3], want[3]))
            row = dict(what="phmm_realign_reads", variant="repeat_rich" if repeat_rich else "plain", band=band, groups=a.groups,
                       pairs=len(pairs), positions_per_pair=float(off[-1]) / len(pairs), max_positions=int(np.diff(off).max()),
                       realign_ms=realign_ms, realign_pairs_per_s=len(pairs) / (realign_ms / 1e3), kernels_ms=kernels_ms, mapper_share=share,
                       host_map_s=t_map, host_align_ms=align_ms, host_path_pairs_per_s=len(pairs) / (t_map + align_ms / 1e3),
                       same_as_host_path=same, **info)
            rows.append(row)
            print(json.dumps(row), flush=True)
    if a.out:
        with open(a.out, "w") as f:
            json.dump(rows, f, indent=1)


if __name__ == "__main__":
    main()
