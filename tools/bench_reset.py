"""HaplotypeLikelihoodModel::reset: the host threads (phmm_reset_haplotypes) against the GPU (phmm_engine_reset_haplotypes) on
repeat-rich haplotypes. Per shape: host time on every hardware thread and on one thread (µs per haplotype), the device call's wall
time including its copies (host-space arrays in and out), and its kernel time from CUDA events after a warm-up. Every timed
device output is compared byte for byte with the host's. Fails without a GPU.

    python tools/bench_reset.py [--shapes 128x300,1024x300,1024x2000,100000x300] [--out FILE]"""
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
FIELDS = ("snv_mask_fwd", "snv_prior_fwd", "snv_mask_rev", "snv_prior_rev", "gap_open", "gap_extend")


def haplotypes(rng, n, length):
    """n haplotypes of `length` bases: random bases with tandem repeats (period 1..6, 2..20 copies) injected every ~40 bases."""
    out = []
    for _ in range(n):
        parts, total = [], 0
        while total < length:
            if rng.random() < 0.35:
                p, k = int(rng.integers(1, 7)), int(rng.integers(2, 21))
                part = np.tile(ACGT[rng.integers(0, 4, p)], k)
            else:
                part = ACGT[rng.integers(0, 4, int(rng.integers(5, 40)))]
            parts.append(part)
            total += len(part)
        out.append(np.concatenate(parts)[:length])
    return out


def best_of(fn, reps):
    times = []
    for _ in range(reps):
        t = time.perf_counter()
        fn()
        times.append(time.perf_counter() - t)
    return min(times), float(np.median(times))


def gpu_info():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True, text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 and q.stdout.strip() else "unknown"


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--shapes", default="128x300,1024x300,1024x2000,100000x300")
    ap.add_argument("--out", default=None)
    ap.add_argument("--seed", type=int, default=2026)
    args = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        sys.exit("bench_reset.py needs a GPU")
    from octopus_b200 import ErrorModel, PairHMMEngine, build
    from octopus_b200.batch import pack_sequences
    build.build()
    engine = PairHMMEngine(0)
    model = ErrorModel()
    rng = np.random.default_rng(args.seed)
    threads = os.cpu_count()
    result = {"gpu": gpu_info(), "host_threads": threads, "shapes": []}
    print("GPU (name, power limit, max SM clock):", result["gpu"], "| host threads:", threads, flush=True)
    for shape in args.shapes.split(","):
        n, length = (int(x) for x in shape.split("x"))
        off, seq = pack_sequences(haplotypes(rng, n, length))
        # warm-up: the device path once (module load, buffers), the host path once
        dev = model.reset_block(off, seq, engine=engine)
        host = model.reset_block(off, seq)
        for f in FIELDS:
            assert np.array_equal(getattr(host, f).view(np.uint8), getattr(dev, f).view(np.uint8)), (shape, f)
        reps = 5 if n * length <= 2_000_000 else 3
        host_all = best_of(lambda: model.reset_block(off, seq, n_threads=0), reps)
        # one thread: on at most 10 000 haplotypes (the per-haplotype cost does not depend on the count)
        n1 = min(n, 10000)
        off1, seq1 = off[:n1 + 1], seq[:int(off[n1])]
        host_one = best_of(lambda: model.reset_block(off1, seq1, n_threads=1), 2 if n1 * length > 1_000_000 else reps)
        kernel_ms = []

        def device():
            out = model.reset_block(off, seq, engine=engine)
            kernel_ms.append(engine._lib.phmm_last_dp_kernel_ms(engine._h))
            return out
        dev_wall = best_of(device, reps)
        dev = device()
        for f in FIELDS:
            assert np.array_equal(getattr(host, f).view(np.uint8), getattr(dev, f).view(np.uint8)), (shape, f)
        row = {"shape": shape, "haplotypes": n, "length": length,
               "host_all_threads_ms": 1e3 * host_all[1], "host_all_threads_us_per_hap": 1e6 * host_all[1] / n,
               "host_one_thread_us_per_hap": 1e6 * host_one[1] / n1, "host_one_thread_haplotypes": n1,
               "device_wall_ms": 1e3 * dev_wall[1], "device_wall_best_ms": 1e3 * dev_wall[0],
               "device_kernel_ms": float(np.median(kernel_ms)), "device_us_per_hap": 1e6 * dev_wall[1] / n,
               "device_beats_all_host_threads": dev_wall[1] < host_all[1], "outputs_equal": True}
        result["shapes"].append(row)
        print(json.dumps(row), flush=True)
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as f:
            json.dump(result, f, indent=1)


if __name__ == "__main__":
    main()
