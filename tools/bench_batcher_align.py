"""What merging read assignment and realignment gains, on Octopus's call pattern: T host threads, each sending K seeded regions one
after the other to

  (a) a PairHMMEngine of its own (one stream and one set of scratch pools per thread), or
  (b) one PopulateBatcher shared by all threads;

for two workloads in the shape of make_default-model calls (band 8, no mapping quality, no flank state, device k-mer mapper on):

  assign:  compute_haplotype_support for one 2-haplotype genotype (two ~600-bp haplotypes) and its 200 reads of 150 bp;
  realign: ReadRealigner::realign of 200 reads of 150 bp against one ~600-bp haplotype.

The two modes alternate over --runs runs after a warm-up; the script prints, per workload and thread count, the median and the range
of regions/s and of host CPU per region (the submitting threads' own CPU time, time.thread_time), requests per GPU call, and the card's
name and power limit read in the same process; and it checks that (a) and (b) give identical outputs in every run.

  python tools/bench_batcher_align.py [--threads 1,8,32] [--regions 16] [--runs 3] [--json PATH]
"""
import argparse
import json
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))

from bench_batcher import card  # noqa: E402
from bench_populate_reset import run  # noqa: E402

ACGT = np.frombuffer(b"ACGT", np.uint8)


def region(rng, n_haps, n_reads=200, hap_len=600, read_len=150):
    """n_haps haplotypes (variants of one sequence, random penalties) and n_reads reads drawn from them."""
    from octopus_b200.batch import pack_haplotypes, pack_reads
    base = ACGT[rng.integers(0, 4, hap_len)]
    seqs = []
    for _ in range(n_haps):
        s = base.copy()
        s[rng.integers(0, hap_len, 3)] = ACGT[rng.integers(0, 4, 3)]
        seqs.append(s)
    pen = lambda lo, hi, s: rng.integers(lo, hi, len(s)).astype(np.int8)     # noqa: E731
    haps = pack_haplotypes(seqs, [np.roll(s, 1) for s in seqs], [pen(1, 126, s) for s in seqs], [np.roll(s, -1) for s in seqs],
                           [pen(1, 126, s) for s in seqs], [pen(3, 46, s) for s in seqs], [pen(1, 11, s) for s in seqs],
                           begin=np.zeros(n_haps, np.int64))
    bases, begins = [], []
    for _ in range(n_reads):
        s = seqs[int(rng.integers(0, n_haps))]
        p = int(rng.integers(0, hap_len - read_len + 1))
        b = s[p:p + read_len].copy()
        b[rng.integers(0, read_len, 2)] = ACGT[rng.integers(0, 4, 2)]
        bases.append(b)
        begins.append(p)
    reads = pack_reads(bases, [rng.integers(8, 41, read_len).astype(np.uint8) for _ in bases], mapq=np.full(n_reads, 60, np.uint8),
                       reverse=(rng.random(n_reads) < 0.5).astype(np.uint8), begin=np.asarray(begins, np.int64))
    return haps, reads


def workloads(n, seed):
    from octopus_b200 import HaplotypeLikelihoodModel
    cfg = HaplotypeLikelihoodModel.Config(max_indel_error=8, use_mapping_quality=False, use_flank_state=False, map_positions=True)
    rng = np.random.default_rng(seed)
    assign = [region(rng, 2) for _ in range(n)]
    realign = [region(rng, 1) for _ in range(n)]
    pairs = np.stack([np.arange(200, dtype=np.int32), np.zeros(200, np.int32)], axis=1)
    return {
        "assign": (assign, lambda c, r: c.assign_reads(cfg, r[0], r[1], [0, 2], [0, r[1].n], want_likelihoods=True, want_status=True)),
        "realign": (realign, lambda c, r: c.realign_reads(cfg, r[0], r[1], pairs)),
    }


def identical(x, y):
    if isinstance(x, (tuple, list)):
        return len(x) == len(y) and all(identical(a, b) for a, b in zip(x, y))
    if isinstance(x, np.ndarray):
        return x.dtype == y.dtype and x.shape == y.shape and x.tobytes() == y.tobytes()
    return x == y


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--threads", default="1,8,32")
    ap.add_argument("--regions", type=int, default=16, help="regions per thread and run")
    ap.add_argument("--runs", type=int, default=3)
    ap.add_argument("--max-wait-us", type=int, default=500)
    ap.add_argument("--json", default=None)
    a = ap.parse_args()
    from octopus_b200 import PairHMMEngine, PopulateBatcher
    Ts = [int(x) for x in a.threads.split(",")]
    K = a.regions
    info = card()
    print("card: %s, power limit %s W, max SM clock %s MHz" % (info["name"], info["power_limit_w"], info["max_sm_mhz"]))
    work = workloads(max(Ts) * K, 0xA551)
    report = {"card": info, "regions_per_thread": K, "runs": a.runs, "rows": []}
    ok = True
    for wname, (regions, one) in work.items():
        for T in Ts:
            engines = {}
            rows = {"a": [], "b": []}
            first = None
            for rep in range(a.runs):
                for mode in "ab":
                    if mode == "a":
                        dt, res, cpu = run(T, K, regions, lambda t: engines.setdefault(t, PairHMMEngine(0)), one)
                        per_call = 1.0
                    else:
                        b = PopulateBatcher(0, clients=T, max_wait_us=a.max_wait_us)
                        dt, res, cpu = run(T, K, regions, lambda t: b, one)
                        st = b.stats()
                        b.close()
                        per_call = st["requests"] / max(1, st["gpu_calls"])
                    first = first or res
                    ok = ok and identical(first, res)
                    rows[mode].append((T * K / dt, 1e3 * cpu / (T * K), per_call))
            for e in engines.values():
                e.close()
            for mode, what in (("a", "an engine per thread"), ("b", "one shared engine")):
                r = np.array(rows[mode])
                row = {"workload": wname, "threads": T, "mode": mode, "what": what,
                       "regions_per_s": [float(x) for x in r[:, 0]], "host_cpu_ms_per_region": [float(x) for x in r[:, 1]],
                       "requests_per_gpu_call": float(np.median(r[:, 2]))}
                report["rows"].append(row)
                print("%-7s T=%-3d (%s) %-21s %8.1f regions/s [%7.1f .. %7.1f]  %6.3f host CPU ms/region [%6.3f .. %6.3f]  %5.1f requests/GPU call" %
                      (wname, T, mode, what, np.median(r[:, 0]), r[:, 0].min(), r[:, 0].max(), np.median(r[:, 1]), r[:, 1].min(), r[:, 1].max(),
                       row["requests_per_gpu_call"]))
    print("identical outputs in every run: %s" % ok)
    report["identical"] = ok
    if a.json:
        os.makedirs(os.path.dirname(os.path.abspath(a.json)), exist_ok=True)
        with open(a.json, "w") as f:
            json.dump(report, f, indent=1)
    return 0 if ok else 1


if __name__ == "__main__":
    sys.exit(main())
