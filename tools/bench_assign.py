#!/usr/bin/env python
"""One phmm_assign_reads call (compute_haplotype_support's scoring and choice for many genotypes) against the recipe it replaces: one
phmm_map_pairs call over every pair, the positions copied to the host, one phmm_populate per genotype with its positions, and the
find_map_haplotypes choice in numpy. Filter-shaped groups: 2-3 haplotypes of 400-800 bases, 20-300 reads of 150 bases, every fourth
group repeat-rich (a third of the haplotype is a short tandem repeat). Bands 8 and 16, mapping quality on, random log priors.

Per band one JSON line:
  assign_ms / assign_pairs_per_s   wall time of one assign_reads call (top and the likelihoods back on the host; median of --reps)
  recipe_ms / recipe_pairs_per_s   wall time of the recipe above (median of --reps)
  same_top / same_lnl              whether both ways gave identical top sets and bit-identical likelihoods
The device name, power limit and SM clock limit are printed beside the figures. Needs a GPU; writes nothing but stdout (and --out)."""
import argparse
import json
import os
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))

from bench_realign import device_info  # noqa: E402

ACGT = np.frombuffer(b"ACGT", dtype=np.uint8)
EPS = 2.0 ** -52
LOWEST = -1.7976931348623157e308


def workload(rng, n_groups, read_len=150):
    from octopus_b200.batch import HaplotypeBlock, ReadBlock
    seqs, reads, quals, begins, hf, rf = [], [], [], [], [0], [0]
    for g in range(n_groups):
        L = int(rng.integers(400, 801))
        a = ACGT[rng.integers(0, 4, L)].copy()
        if g % 4 == 0:
            unit = ACGT[rng.integers(0, 4, int(rng.integers(1, 5)))]
            p, n = int(rng.integers(0, L // 2)), L // 3
            a[p:p + n] = np.tile(unit, n // len(unit) + 1)[:n]
        group = [a]
        for _ in range(int(rng.integers(1, 3))):
            b = a.copy()
            b[rng.integers(0, L, 2)] = ACGT[rng.integers(0, 4, 2)]
            group.append(b)
        seqs += group
        nr = int(rng.integers(20, 301))
        for _ in range(nr):
            s = group[int(rng.integers(0, len(group)))]
            p = int(rng.integers(0, L - read_len + 1))
            x = s[p:p + read_len].copy()
            x[rng.integers(0, read_len, int(rng.integers(0, 3)))] = ACGT[rng.integers(0, 4)]
            reads.append(x); quals.append(rng.integers(10, 41, read_len).astype(np.uint8)); begins.append(p)
        hf.append(hf[-1] + len(group)); rf.append(rf[-1] + nr)
    hoff = np.concatenate([[0], np.cumsum([len(s) for s in seqs])]).astype(np.int64)
    seq = np.concatenate(seqs)
    T = len(seq)
    haps = HaplotypeBlock(hoff, seq, np.roll(seq, 1), rng.integers(20, 126, T).astype(np.int8), np.roll(seq, -1),
                          rng.integers(20, 126, T).astype(np.int8), rng.integers(8, 46, T).astype(np.int8), rng.integers(1, 11, T).astype(np.int8),
                          begin=np.zeros(len(seqs), np.int64))
    R = len(reads)
    roff = np.concatenate([[0], np.cumsum([len(x) for x in reads])]).astype(np.int64)
    rb = ReadBlock(roff, np.concatenate(reads), np.concatenate(quals), rng.choice([20, 60], R).astype(np.uint8),
                   (rng.random(R) < 0.5).astype(np.uint8), np.asarray(begins, np.int64))
    return haps, rb, np.asarray(hf, np.int32), np.asarray(rf, np.int32)


def find_map_numpy(lnl, pri):
    """find_map_haplotypes for every read of one group ((H, R) matrix, log priors [H]) as uint64 masks."""
    H, R = lnl.shape
    mx = np.full(R, LOWEST)
    top = np.zeros(R, np.uint64)
    for k in range(H):
        cur = lnl[k] + pri[k]
        with np.errstate(invalid="ignore", over="ignore"):
            eq = (cur == mx) | (np.abs(cur - mx) < EPS * np.abs(cur + mx))
            gt = ~eq & (cur > mx)
        bit = np.uint64(1 << k)
        top = np.where(eq, top | bit, np.where(gt, bit, top))
        mx = np.where(gt, cur, mx)
    return np.where(top == 0, np.uint64((1 << H) - 1), top)


def sub_block(haps, reads, hf, rf, g):
    from octopus_b200.batch import HaplotypeBlock, ReadBlock
    h0, h1, r0, r1 = int(hf[g]), int(hf[g + 1]), int(rf[g]), int(rf[g + 1])
    a, b = int(haps.off[h0]), int(haps.off[h1])
    hs = HaplotypeBlock(haps.off[h0:h1 + 1] - a, *[getattr(haps, f)[a:b] for f in HaplotypeBlock._fields[1:8]], haps.begin[h0:h1])
    c, d = int(reads.off[r0]), int(reads.off[r1])
    rs = ReadBlock(reads.off[r0:r1 + 1] - c, reads.bases[c:d], reads.quals[c:d], reads.mapq[r0:r1], reads.reverse[r0:r1], reads.begin[r0:r1])
    return hs, rs


def recipe(eng, cfg, haps, reads, hf, rf, pri, subs, pairs):
    """map_pairs, positions to the host, one populate per group with its positions, the choice in numpy."""
    off, pos = eng.map_pairs(haps, reads, pairs)
    tops, lnls = [], []
    j = 0
    for g, (hs, rs) in enumerate(subs):
        n = hs.n * rs.n
        o = off[j:j + n + 1]
        p = pos[o[0]:o[-1]] if o[-1] > o[0] else np.zeros(1, np.int32)
        lnl = eng.populate(cfg, hs, rs, positions=(o - o[0], p))
        j += n
        tops.append(find_map_numpy(lnl, pri[int(hf[g]):int(hf[g + 1])]))
        lnls.append(lnl.reshape(-1))
    return np.concatenate(tops), np.concatenate(lnls)


def median_ms(f, reps):
    f()
    times = []
    for _ in range(reps):
        t0 = time.perf_counter()
        f()
        times.append(time.perf_counter() - t0)
    return 1e3 * float(np.median(times))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--groups", type=int, default=300)
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    import torch
    assert torch.cuda.is_available(), "bench_assign needs a GPU"
    from octopus_b200 import HaplotypeLikelihoodModel, PairHMMEngine
    eng = PairHMMEngine(0)
    info = device_info()
    print(json.dumps(info))
    rng = np.random.default_rng(23)
    haps, reads, hf, rf = workload(rng, a.groups)
    pri = np.log(rng.dirichlet(np.ones(haps.n)))
    subs = [sub_block(haps, reads, hf, rf, g) for g in range(len(hf) - 1)]
    pairs = np.concatenate([np.stack(np.meshgrid(np.arange(rf[g], rf[g + 1]), np.arange(hf[g], hf[g + 1])), -1).reshape(-1, 2)
                            for g in range(len(hf) - 1)]).astype(np.int32)     # (read, hap) in slot order
    rows = []
    for band in (8, 16):
        cfg = HaplotypeLikelihoodModel.Config(max_indel_error=band)
        top, lnl = eng.assign_reads(cfg, haps, reads, hf, rf, pri, want_likelihoods=True)
        rtop, rlnl = recipe(eng, cfg, haps, reads, hf, rf, pri, subs, pairs)
        assign_ms = median_ms(lambda: eng.assign_reads(cfg, haps, reads, hf, rf, pri, want_likelihoods=True), a.reps)
        recipe_ms = median_ms(lambda: recipe(eng, cfg, haps, reads, hf, rf, pri, subs, pairs), a.reps)
        n = len(pairs)
        row = dict(what="phmm_assign_reads", band=band, groups=a.groups, reads=int(reads.n), pairs=n, assign_ms=assign_ms,
                   assign_pairs_per_s=n / (assign_ms / 1e3), recipe_ms=recipe_ms, recipe_pairs_per_s=n / (recipe_ms / 1e3),
                   speedup=recipe_ms / assign_ms, same_top=bool(np.array_equal(top, rtop)),
                   same_lnl=bool(np.array_equal(lnl.view(np.int64), rlnl.view(np.int64))), **info)
        rows.append(row)
        print(json.dumps(row), flush=True)
    if a.out:
        with open(a.out, "w") as f:
            json.dump(rows, f, indent=1)


if __name__ == "__main__":
    main()
