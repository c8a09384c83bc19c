"""Times phmm_variational_bayes on two workloads shaped like the callers that use it, on one GPU:
  cancer-shaped:    2 samples x 1 000 reads, 64 haplotypes, K = 3, 20 000 genotypes, 12 seeds
  polyclone-shaped: 1 sample x 1 000 reads, 64 haplotypes, K = 4, 10 000 genotypes, 12 seeds
Each call is timed with CUDA events around synchronised calls after warm-up; the card's name and power limit are read in the same
run. Where oracle/_ref/libref_vb.so was built, the UNMODIFIED reference run_variational_bayes is timed on the same host's CPU (one
thread, wall clock, median of --ref-calls) and its weighted posteriors and max evidence are compared with the device's within the
float tolerances of tests/test_vb_ref.py. Prints one JSON line per workload: time per call, total iterations, time per iteration
and seed, and the reference's time and agreement."""
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

WORKLOADS = {"cancer": dict(H=64, reads=[1000, 1000], G=20000, K=3, n_seeds=12),
             "polyclone": dict(H=64, reads=[1000], G=10000, K=4, n_seeds=12)}


def main():
    import torch
    import vb_cases
    from octopus_b200 import PairHMMEngine
    from test_vb_ref import EVIDENCE_REL, WEIGHTED_ABS
    from vb_ref import RefVB
    ap = argparse.ArgumentParser()
    ap.add_argument("--calls", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--ref-calls", type=int, default=3)
    args = ap.parse_args()
    gpu = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True).stdout.strip()
    eng = PairHMMEngine(0)
    for name, w in WORKLOADS.items():
        lnl, off, gt, prior, lp, seeds = vb_cases.make(w["H"], w["reads"], w["G"], w["K"], w["n_seeds"], seed=7)
        d = [torch.as_tensor(x, device="cuda:0") for x in (lnl, gt, prior, lp, seeds)]
        host = eng.variational_bayes(lnl, gt, prior, lp, seeds, off)
        for _ in range(args.warmup):
            eng.variational_bayes(*d, off)
        times = []
        for _ in range(args.calls):
            torch.cuda.synchronize()
            a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            a.record()
            r = eng.variational_bayes(*d, off)
            b.record()
            torch.cuda.synchronize()
            times.append(a.elapsed_time(b))
        same = all(np.array_equal(np.asarray(getattr(host, f)), getattr(r, f).cpu().numpy())
                   for f in ("genotype_posteriors", "evidence_weighted_genotype_posteriors", "seed_iterations"))
        its = int(r.seed_iterations.sum().item())
        ms = float(np.median(times))
        ref = "not measured (oracle/_ref/libref_vb.so not built)"
        if RefVB.available():
            rv, rt = RefVB(), []
            for _ in range(args.ref_calls):
                t0 = time.perf_counter()
                want = rv.run(lnl, off, gt, prior, lp, seeds, per_seed=False)
                rt.append(1000 * (time.perf_counter() - t0))
            agree = bool(np.max(np.abs(r.evidence_weighted_genotype_posteriors.cpu().numpy() - want["weighted"])) <= WEIGHTED_ABS and
                         abs(float(r.max_log_evidence) - want["max_log_evidence"]) <= EVIDENCE_REL * abs(want["max_log_evidence"]))
            ref = dict(ms_per_call=round(float(np.median(rt)), 1), threads=1, agrees=agree)
        print(json.dumps(dict(workload=name, gpu=gpu, ms_per_call=round(ms, 3), ms_min=round(min(times), 3), iterations=its,
                              us_per_iteration_and_seed=round(1000 * ms / max(its, 1), 2), host_equals_device=bool(same),
                              reference_cpu=ref)))


if __name__ == "__main__":
    main()
