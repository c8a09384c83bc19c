"""Where HaplotypeLikelihoodModel::reset runs, on Octopus's call pattern: T host threads, each populating K seeded regions one after
the other (32 haplotypes, 300 reads, band 16, a flank state, device k-mer mapper on), every region starting from haplotype sequences.

  (a) reset on the calling thread (ErrorModel.reset_block, one host thread) + PopulateBatcher.populate;
  (b) PopulateBatcher.populate(error_model=): the reset runs on the GPU inside the merged call;
  (c) ErrorModel.reset_block(engine=) + PairHMMEngine.populate, one engine per thread;
  (d) PairHMMEngine.populate(error_model=), one engine per thread.

Prints regions/s, host CPU seconds per region (the submitting threads' own CPU time, time.thread_time), regions per GPU call, and the
card's name and power limit read in the same run; checks that all four give identical statuses and identical values at every OK pair.

  python tools/bench_populate_reset.py [--threads 1,8,32] [--regions 16] [--json PATH]
"""
import argparse
import json
import os
import sys
import threading
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))

from bench_batcher import card, same  # noqa: E402


def workload(n, seed0):
    """n regions of (HaplotypeSequences, ReadBlock, flank): synth's C2 reads over 32 haplotypes."""
    from octopus_b200 import HaplotypeLikelihoodModel, HaplotypeSequences, synth
    regions = []
    for i in range(n):
        haps, reads, _ = synth.make_batch("C2", n_reads=300, n_haps=32, seed=seed0 + i)
        regions.append((HaplotypeSequences(haps.off, haps.seq, haps.begin), reads, (40, 40)))
    return HaplotypeLikelihoodModel.Config(max_indel_error=16, map_positions=True), regions


def run(T, K, regions, make_client, one):
    """Each of T threads runs one(client, region) over its K regions after a warm-up; returns (seconds, results, thread CPU seconds)."""
    clients = [make_client(t) for t in range(T)]
    results = [[None] * K for _ in range(T)]
    cpu = [0.0] * T
    barrier = threading.Barrier(T + 1)
    errors = []

    def worker(t):
        try:
            one(clients[t], regions[t * K])
            barrier.wait()
            barrier.wait()
            c0 = time.thread_time()
            for i in range(K):
                results[t][i] = one(clients[t], regions[t * K + i])
            cpu[t] = time.thread_time() - c0
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
    return dt, results, sum(cpu)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--threads", default="1,8,32")
    ap.add_argument("--regions", type=int, default=16, help="regions per thread")
    ap.add_argument("--max-wait-us", type=int, default=500)
    ap.add_argument("--json", default=None)
    a = ap.parse_args()
    from octopus_b200 import ErrorModel, PairHMMEngine, PopulateBatcher
    Ts = [int(x) for x in a.threads.split(",")]
    K = a.regions
    info = card()
    print("card: %s, power limit %s W, max SM clock %s MHz" % (info["name"], info["power_limit_w"], info["max_sm_mhz"]))
    cfg, regions = workload(max(Ts) * K, 0x5E5E7)
    lengths = np.concatenate([np.diff(s.off) for s, _, _ in regions[:8]])
    print("regions: 32 haplotypes (mean %.0f bp) x 300 reads, band 16, flank state, mapper on" % lengths.mean())
    model = ErrorModel()

    def host_reset(s):
        return model.reset_block(s.off, s.seq, s.begin, n_threads=1)

    modes = {
        "a": ("host reset + batcher", True, lambda b, r: b.populate(cfg, host_reset(r[0]), r[1], flank_state=r[2], want_status=True)),
        "b": ("batcher(error_model=)", True, lambda b, r: b.populate(cfg, r[0], r[1], flank_state=r[2], want_status=True, error_model=model)),
        "c": ("device reset + engine", False, lambda e, r: e.populate(cfg, model.reset_block(r[0].off, r[0].seq, r[0].begin, engine=e), r[1],
                                                                     flank_state=r[2], want_status=True)),
        "d": ("engine(error_model=)", False, lambda e, r: e.populate(cfg, r[0], r[1], flank_state=r[2], want_status=True, error_model=model)),
    }
    report = {"card": info, "regions_per_thread": K, "runs": []}
    ok = True
    for T in Ts:
        outs = {}
        for key, (name, shared, one) in modes.items():
            if shared:
                b = PopulateBatcher(0, clients=T, max_wait_us=a.max_wait_us)
                dt, res, cpu = run(T, K, regions, lambda t: b, one)
                st = b.stats()
                b.close()
                per_call = st["requests"] / max(1, st["gpu_calls"])
            else:
                engines = {}
                dt, res, cpu = run(T, K, regions, lambda t: engines.setdefault(t, PairHMMEngine(0)), one)
                for e in engines.values():
                    e.close()
                per_call = 1.0
            outs[key] = res
            n = T * K
            row = {"threads": T, "mode": key, "what": name, "regions_per_s": n / dt, "host_cpu_ms_per_region": 1e3 * cpu / n,
                   "regions_per_gpu_call": per_call}
            report["runs"].append(row)
            print("T=%-3d (%s) %-24s %8.1f regions/s  %7.3f host CPU ms/region  %5.1f regions/GPU call" %
                  (T, key, name, row["regions_per_s"], row["host_cpu_ms_per_region"], per_call))
        ident = all(same(outs["a"][t], outs[k][t]) for k in "bcd" for t in range(T))
        ok = ok and ident
        print("T=%-3d identical outputs (a) == (b) == (c) == (d): %s" % (T, ident))
    report["identical"] = ok
    if a.json:
        os.makedirs(os.path.dirname(os.path.abspath(a.json)), exist_ok=True)
        with open(a.json, "w") as f:
            json.dump(report, f, indent=1)
    return 0 if ok else 1


if __name__ == "__main__":
    sys.exit(main())
