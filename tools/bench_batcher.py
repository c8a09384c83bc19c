"""Throughput of the shared engine (PopulateBatcher / phmm_batcher) against one engine per thread, on Octopus's call pattern:
T host threads, each submitting K seeded regions one after the other.

  (a) one PairHMMEngine per thread, one populate per region (the per-thread integration);
  (b) one PopulateBatcher with clients = T.

Workloads: "c1" (1000 reads x 8 haplotypes, 150 bp reads, band 8) and "octopus" (300 reads x 32 haplotypes, band 16, a flank
state, device k-mer mapper on). Checks that (a) and (b) give identical statuses and identical values at every OK pair, and prints
regions/s, GCUPS (DP cells from the engines' / batcher's counters over wall time), mean regions per GPU call, and a max_wait_us
sweep, with the card's name and power limit read in the same run. The harness is Python threads over ctypes (the GIL is released
inside every call, not between calls), so per-call Python overhead is part of every number.

  python tools/bench_batcher.py [--threads 1,8,32] [--regions 24] [--sweep 0,100,250,500,1000,2000] [--json PATH]
"""
import argparse
import json
import os
import subprocess
import sys
import threading
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def card():
    import torch
    name = torch.cuda.get_device_name(0)
    try:
        q = subprocess.run(["nvidia-smi", "-i", "0", "--query-gpu=power.limit,clocks.max.sm", "--format=csv,noheader,nounits"],
                           capture_output=True, text=True, timeout=20).stdout.strip().split(",")
        return {"name": name, "power_limit_w": float(q[0]), "max_sm_mhz": float(q[1])}
    except Exception:                       # noqa: BLE001
        return {"name": name, "power_limit_w": None, "max_sm_mhz": None}


def workload(kind, n, seed0):
    from octopus_b200 import HaplotypeLikelihoodModel, synth
    regions = []
    for i in range(n):
        if kind == "c1":
            haps, reads, band = synth.make_batch("C1", seed=seed0 + i)
            regions.append((haps, reads, None))
        else:
            haps, reads, band = synth.make_batch("C2", n_reads=300, n_haps=32, seed=seed0 + i)
            regions.append((haps, reads, (40, 40)))
    cfg = HaplotypeLikelihoodModel.Config(max_indel_error=8 if kind == "c1" else 16, map_positions=(kind != "c1"))
    return cfg, regions


def run_threads(T, K, cfg, regions, make_client, cells_of):
    """Each of T threads submits its K regions; returns (seconds, results, dp cells). A warm-up region per thread runs first."""
    clients = [make_client(t) for t in range(T)]
    results = [[None] * K for _ in range(T)]
    cells = [0] * T
    barrier = threading.Barrier(T + 1)
    errors = []

    def worker(t):
        try:
            c = clients[t]
            haps, reads, flank = regions[t * K]
            c.populate(cfg, haps, reads, flank_state=flank, want_status=True)      # warm-up
            barrier.wait()
            barrier.wait()
            for i in range(K):
                haps, reads, flank = regions[t * K + i]
                results[t][i] = c.populate(cfg, haps, reads, flank_state=flank, want_status=True)
                cells[t] += cells_of(c)
        except Exception as ex:             # noqa: BLE001
            errors.append(repr(ex))
            barrier.abort()

    threads = [threading.Thread(target=worker, args=(t,)) for t in range(T)]
    for th in threads:
        th.start()
    barrier.wait()
    t0 = time.perf_counter()
    barrier.wait()
    for th in threads:
        th.join()
    dt = time.perf_counter() - t0
    if errors:
        raise RuntimeError(errors[0])
    return dt, results, sum(cells)


def per_thread_engines(T, K, cfg, regions):
    from octopus_b200 import PairHMMEngine
    engines = {}
    dt, res, cells = run_threads(T, K, cfg, regions, lambda t: engines.setdefault(t, PairHMMEngine(0)), lambda e: e.last_dp_cells())
    for e in engines.values():
        e.close()
    return dt, res, cells


def batched(T, K, cfg, regions, max_wait_us):
    from octopus_b200 import PopulateBatcher
    b = PopulateBatcher(0, clients=T, max_wait_us=max_wait_us)
    dt, res, _ = run_threads(T, K, cfg, regions, lambda t: b, lambda c: 0)
    s = b.stats()          # includes the T warm-up requests
    b.close()
    return dt, res, s


def same(ra, rb):
    for (oa, sa), (ob, sb) in zip(ra, rb):
        if not np.array_equal(sa, sb):
            return False
        ok = (sa & 0xFFFF) == 0
        if not np.array_equal(oa.view(np.int64)[ok], ob.view(np.int64)[ok]):
            return False
    return True


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--threads", default="1,8,32")
    ap.add_argument("--regions", type=int, default=24, help="regions per thread")
    ap.add_argument("--sweep", default="0,100,250,500,1000,2000", help="max_wait_us values swept at the largest thread count")
    ap.add_argument("--default-wait", type=int, default=500)
    ap.add_argument("--json", default=None)
    a = ap.parse_args()
    Ts = [int(x) for x in a.threads.split(",")]
    K = a.regions
    info = card()
    print("card: %s, power limit %s W, max SM clock %s MHz" % (info["name"], info["power_limit_w"], info["max_sm_mhz"]))
    report = {"card": info, "regions_per_thread": K, "runs": [], "sweep": []}
    for kind in ("c1", "octopus"):
        cfg, regions = workload(kind, max(Ts) * K, 0xBA7C0 + (0 if kind == "c1" else 50_000))
        for T in Ts:
            dta, ra, cells_a = per_thread_engines(T, K, cfg, regions)
            dtb, rb, st = batched(T, K, cfg, regions, a.default_wait)
            ident = all(same(ra[t], rb[t]) for t in range(T))
            n = T * K
            # the batcher's counters include the T warm-up requests: scale its cells to the measured requests
            cells_b = st["dp_cells"] * n / max(1, st["requests"])
            row = {"workload": kind, "threads": T, "regions": n, "identical": ident,
                   "a_regions_per_s": n / dta, "a_gcups": cells_a / dta / 1e9,
                   "b_regions_per_s": n / dtb, "b_gcups": cells_b / dtb / 1e9,
                   "b_regions_per_call": st["requests"] / max(1, st["gpu_calls"]), "b_max_regions_per_call": st["max_regions_per_call"],
                   "max_wait_us": a.default_wait}
            report["runs"].append(row)
            print("%-8s T=%-3d (a) per-thread engines %8.1f regions/s %7.1f GCUPS | (b) batcher %8.1f regions/s %7.1f GCUPS, %.1f regions/call "
                  "(max %d) | identical=%s" % (kind, T, row["a_regions_per_s"], row["a_gcups"], row["b_regions_per_s"], row["b_gcups"],
                                               row["b_regions_per_call"], row["b_max_regions_per_call"], ident))
            if not ident:
                print("MISMATCH between (a) and (b)")
        T = max(Ts)
        for w in [int(x) for x in a.sweep.split(",") if x]:
            dtb, rb, st = batched(T, K, cfg, regions, w)
            row = {"workload": kind, "threads": T, "max_wait_us": w, "b_regions_per_s": T * K / dtb,
                   "b_gcups": st["dp_cells"] * T * K / max(1, st["requests"]) / dtb / 1e9,
                   "b_regions_per_call": st["requests"] / max(1, st["gpu_calls"])}
            report["sweep"].append(row)
            print("%-8s T=%-3d sweep max_wait_us=%-5d %8.1f regions/s %7.1f GCUPS, %.1f regions/call" %
                  (kind, T, w, row["b_regions_per_s"], row["b_gcups"], row["b_regions_per_call"]))
    ok = all(r["identical"] for r in report["runs"])
    print("identical outputs (a) == (b): %s" % ok)
    if a.json:
        os.makedirs(os.path.dirname(os.path.abspath(a.json)), exist_ok=True)
        with open(a.json, "w") as f:
            json.dump(report, f, indent=1)
    return 0 if ok else 1


if __name__ == "__main__":
    sys.exit(main())
