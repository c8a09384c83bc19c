"""Times phmm_variational_bayes_mixture_mixture on two workloads shaped like the single-cell caller, on one GPU:
  cells:        200 cells of about 20 reads, 20 haplotypes, T = 3 clones of ploidy 2, 1 000 combinations, 12 seeds
  copy-number:  the same cells and haplotypes, groups of ploidy 1, 2 and 3
Each call is timed with CUDA events around synchronised calls after warm-up; the card's name and power limit are read in the same
run. Where oracle/_ref/libref_vbmm.so was built, the UNMODIFIED reference VariationalBayesMixtureMixtureModel::evaluate is timed on
the same host's CPU (one thread, wall clock, median of --ref-calls) and its weighted posteriors, weighted group responsibilities
and max evidence are compared with the device's within the float tolerances of tests/test_vbmm_ref.py. Prints one JSON line per
workload: time per call, total iterations, time per iteration and seed, and the reference's time and agreement."""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

WORKLOADS = {"cells": dict(H=20, S=200, mean_reads=20, sizes=[2, 2, 2], C=1000, n_seeds=12),
             "copy-number": dict(H=20, S=200, mean_reads=20, sizes=[1, 2, 3], C=1000, n_seeds=12)}


def main():
    import torch
    import vbmm_cases
    from octopus_b200 import PairHMMEngine
    from test_vbmm_ref import EVIDENCE_REL, SIGMA_ABS, WEIGHTED_ABS
    from vbmm_ref import RefVBMM
    ap = argparse.ArgumentParser()
    ap.add_argument("--calls", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--ref-calls", type=int, default=1)
    args = ap.parse_args()
    gpu = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True).stdout.strip()
    eng = PairHMMEngine(0)
    for name, w in WORKLOADS.items():
        reads = [int(v) for v in np.random.default_rng(5).poisson(w["mean_reads"], size=w["S"])]
        x = vbmm_cases.make(w["H"], reads, w["sizes"], w["C"], 1, seed=7)
        seeds = vbmm_cases.propose_seeds(w["C"], w["n_seeds"])
        call_args = lambda conv: (conv(x["lnl"]), x["sizes"], conv(x["gt"]), conv(x["lp"]), conv(x["gc"]), conv(x["mc"]), conv(seeds), x["off"])
        host = eng.variational_bayes_mixture_mixture(*call_args(lambda a: a))
        d = call_args(lambda a: torch.as_tensor(a, device="cuda:0"))
        for _ in range(args.warmup):
            eng.variational_bayes_mixture_mixture(*d)
        times = []
        for _ in range(args.calls):
            torch.cuda.synchronize()
            a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            a.record()
            r = eng.variational_bayes_mixture_mixture(*d)
            b.record()
            torch.cuda.synchronize()
            times.append(a.elapsed_time(b))
        same = all(np.array_equal(np.asarray(getattr(host, f)), getattr(r, f).cpu().numpy())
                   for f in ("genotype_posteriors", "weighted_genotype_posteriors", "weighted_group_responsibilities", "seed_iterations"))
        its = int(r.seed_iterations.sum().item())
        ms = float(np.median(times))
        ref = "not measured (oracle/_ref/libref_vbmm.so not built)"
        if RefVBMM.available():
            rv, rt = RefVBMM(), []
            for _ in range(args.ref_calls):
                t0 = time.perf_counter()
                want = rv.run(x["lnl"], x["off"], x["sizes"], x["gt"], x["lp"], x["gc"], x["mc"], seeds, per_seed=False)
                rt.append(1000 * (time.perf_counter() - t0))
            agree = bool(np.max(np.abs(r.weighted_genotype_posteriors.cpu().numpy() - want["weighted"])) <= WEIGHTED_ABS and
                         np.max(np.abs(r.weighted_group_responsibilities.cpu().numpy() - want["weighted_group_responsibilities"])) <= SIGMA_ABS and
                         abs(float(r.max_log_evidence) - want["max_log_evidence"]) <= EVIDENCE_REL * abs(want["max_log_evidence"]))
            ref = dict(ms_per_call=round(float(np.median(rt)), 1), threads=1, agrees=agree)
        print(json.dumps(dict(workload=name, gpu=gpu, reads=sum(reads), ms_per_call=round(ms, 3), ms_min=round(min(times), 3),
                              iterations=its, us_per_iteration_and_seed=round(1000 * ms / max(its, 1), 2), host_equals_device=bool(same),
                              reference_cpu=ref)), flush=True)


if __name__ == "__main__":
    main()
