#!/usr/bin/env python
"""One phmm_assign_templates call (compute_haplotype_support over paired templates for many genotypes, BAMRealigner's call under
--read-linkage paired) against phmm_assign_reads on the same reads, and against the host-side workaround an integrator would otherwise
write: assign_reads with the likelihoods, each template's reads summed on the host, find_map_haplotypes in numpy.

Workload: --groups genotypes (default 300) of 2-3 haplotypes of 700-1 000 bases; --templates templates in all (default 25 000), each two
150-base mates from one haplotype (the second on the reverse strand, 150-450 bases further on), with 0-2 mismatches. Host arrays, bands
8 and 16, mapping quality on, random log priors.

Per band one JSON line:
  templates_ms      wall time of one assign_templates call (top and the template likelihoods back on the host; median of --reps)
  reads_ms          wall time of one assign_reads call on the same reads (top and the read likelihoods back)
  workaround_ms     assign_reads with the likelihoods, then the template sums and the choice in numpy
  *_min_ms / *_max_ms   the fastest and slowest of the --reps runs of each: the spread the medians come with
  same_top / same_lnl   whether the template call and the workaround give identical top sets and bit-identical template values
The device name, power limit and SM clock limit are read in the same run and printed beside the figures. Needs a GPU; writes nothing
but stdout (and --out)."""
import argparse
import json
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))

from bench_assign import find_map_numpy, median_ms  # noqa: E402
from bench_realign import device_info  # noqa: E402

ACGT = np.frombuffer(b"ACGT", dtype=np.uint8)


def workload(rng, n_groups, n_templates, read_len=150):
    """(haps, reads, template_off, hap_first, template_first): the templates spread evenly over the groups."""
    from octopus_b200.batch import HaplotypeBlock, ReadBlock
    seqs, reads, quals, begins, rev, hf, tf = [], [], [], [], [], [0], [0]
    per_group = np.diff(np.linspace(0, n_templates, n_groups + 1).astype(int))
    for g in range(n_groups):
        L = int(rng.integers(700, 1001))
        a = ACGT[rng.integers(0, 4, L)].copy()
        group = [a]
        for _ in range(int(rng.integers(1, 3))):
            b = a.copy()
            b[rng.integers(0, L, 2)] = ACGT[rng.integers(0, 4, 2)]
            group.append(b)
        seqs += group
        for _ in range(int(per_group[g])):
            s = group[int(rng.integers(0, len(group)))]
            p = int(rng.integers(0, L - 2 * read_len - 300 + 1))
            for mate, q in enumerate((p, p + read_len + int(rng.integers(0, 301)))):
                x = s[q:q + read_len].copy()
                x[rng.integers(0, read_len, int(rng.integers(0, 3)))] = ACGT[rng.integers(0, 4)]
                reads.append(x); quals.append(rng.integers(10, 41, read_len).astype(np.uint8)); begins.append(q); rev.append(mate)
        hf.append(hf[-1] + len(group)); tf.append(tf[-1] + int(per_group[g]))
    hoff = np.concatenate([[0], np.cumsum([len(s) for s in seqs])]).astype(np.int64)
    seq = np.concatenate(seqs)
    T = len(seq)
    haps = HaplotypeBlock(hoff, seq, np.roll(seq, 1), rng.integers(20, 126, T).astype(np.int8), np.roll(seq, -1),
                          rng.integers(20, 126, T).astype(np.int8), rng.integers(8, 46, T).astype(np.int8), rng.integers(1, 11, T).astype(np.int8),
                          begin=np.zeros(len(seqs), np.int64))
    R = len(reads)
    roff = np.concatenate([[0], np.cumsum([len(x) for x in reads])]).astype(np.int64)
    rb = ReadBlock(roff, np.concatenate(reads), np.concatenate(quals), rng.choice([20, 60], R).astype(np.uint8),
                   np.asarray(rev, np.uint8), np.asarray(begins, np.int64))
    toff = np.arange(0, R + 1, 2, dtype=np.int64)
    return haps, rb, toff, np.asarray(hf, np.int32), np.asarray(tf, np.int32)


def workaround(eng, cfg, haps, reads, toff, hf, rf, tf, pri):
    """assign_reads with the likelihoods, the template sums (read order from 0.0: two mates, so one add after 0.0 + the first), the
    choice per group in numpy."""
    _, lnl = eng.assign_reads(cfg, haps, reads, hf, rf, pri, want_likelihoods=True)
    tops, values, slot = [], [], 0
    for g in range(len(hf) - 1):
        nh, nr = int(hf[g + 1] - hf[g]), int(rf[g + 1] - rf[g])
        m = lnl[slot:slot + nh * nr].reshape(nh, nr)
        s = (0.0 + m[:, 0::2]) + m[:, 1::2]
        tops.append(find_map_numpy(s, pri[int(hf[g]):int(hf[g + 1])]))
        values.append(s.reshape(-1))
        slot += nh * nr
    return np.concatenate(tops), np.concatenate(values)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--groups", type=int, default=300)
    ap.add_argument("--templates", type=int, default=25000)
    ap.add_argument("--reps", type=int, default=7)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    import torch
    assert torch.cuda.is_available(), "bench_assign_templates needs a GPU"
    from octopus_b200 import HaplotypeLikelihoodModel, PairHMMEngine
    eng = PairHMMEngine(0)
    info = device_info()
    print(json.dumps(info))
    rng = np.random.default_rng(29)
    haps, reads, toff, hf, tf = workload(rng, a.groups, a.templates)
    rf = toff[tf].astype(np.int32)
    pri = np.log(rng.dirichlet(np.ones(haps.n)))
    pairs = int((np.diff(hf).astype(np.int64) * np.diff(rf)).sum())
    rows = []
    for band in (8, 16):
        cfg = HaplotypeLikelihoodModel.Config(max_indel_error=band)
        top, lnl = eng.assign_templates(cfg, haps, reads, toff, hf, tf, pri, want_likelihoods=True)
        wtop, wlnl = workaround(eng, cfg, haps, reads, toff, hf, rf, tf, pri)
        times = {}
        # the three ways alternate rep by rep, so that a drift of the shared machine falls on all of them
        for _ in range(a.reps):
            for name, f in (("templates_ms", lambda: eng.assign_templates(cfg, haps, reads, toff, hf, tf, pri, want_likelihoods=True)),
                            ("reads_ms", lambda: eng.assign_reads(cfg, haps, reads, hf, rf, pri, want_likelihoods=True)),
                            ("workaround_ms", lambda: workaround(eng, cfg, haps, reads, toff, hf, rf, tf, pri))):
                times.setdefault(name, []).append(median_ms(f, 1))
        row = dict(what="phmm_assign_templates", band=band, groups=a.groups, templates=int(len(toff) - 1), reads=int(reads.n), pairs=pairs,
                   **{k: float(np.median(v)) for k, v in times.items()},
                   **{k[:-3] + "_min_ms": float(np.min(v)) for k, v in times.items()},
                   **{k[:-3] + "_max_ms": float(np.max(v)) for k, v in times.items()},
                   same_top=bool(np.array_equal(top, wtop)), same_lnl=bool(np.array_equal(lnl.view(np.int64), wlnl.view(np.int64))), **info)
        rows.append(row)
        print(json.dumps(row), flush=True)
    if a.out:
        with open(a.out, "w") as f:
            json.dump(rows, f, indent=1)


if __name__ == "__main__":
    main()
