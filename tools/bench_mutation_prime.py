"""DeNovoModel::prime on trio-shaped haplotype sets: one phmm_mutation_prime call per set, against the reference's own prime on one host
thread (the compiled oracle, oracle/_ref/libref_mutation.so, where present) and against the recipe it replaces (phmm_align_pairs over
host-built padded truths, every CIGAR copied back and re-scored on the host). Checks that the three agree and prints one JSON line per
shape, with the card's name and power limit read in the same run.

Sets: 50 haplotypes (the reference's largest eagerly primed set, 2 450 ordered pairs) of one region, from synth.make_haplotypes's base
sequence with injected STRs, each haplotype carrying SNVs and 1-20 bp indels (tests/mutation_oracle.py's mutate).
    python tools/bench_mutation_prime.py [--sets 20] [--out results.json]

With --sets-per-call K and / or --threads T, the same seeded sets instead run three ways, alternated round by round in one process
after a warm-up of every mode and shape: one phmm_mutation_prime per set ("per_set"), K sets per phmm_mutation_prime_sets call
("sets_per_call"), and T Python threads priming their share of the sets on one PopulateBatcher, each with a model object of its own
("threads"). One JSON row per mode and shape: sets per second, median call time, median DP kernel time, the batcher's merged-call
statistics, and whether every status and every HMM / SELF value equals the per-set call's.
    python tools/bench_mutation_prime.py --sets 20,100 --sets-per-call 20 --threads 8 [--rounds 3]
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
sys.path.insert(0, os.path.join(ROOT, "tests"))

from bench_realign import device_info  # noqa: E402
from mutation_oracle import TRIO_PRIORS, RefMutation, align_pairs_recipe, mutate  # noqa: E402


def trio_set(rng, n, length):
    """n haplotypes of about `length` bp: a base sequence with two injected STRs, each haplotype 0-6 SNVs / indels away from it."""
    from octopus_b200 import synth
    base = bytes(synth.make_haplotypes(rng, 1, length).seq).decode().replace("N", "A")
    for _ in range(2):
        unit = "".join(rng.choice(list("ACGT"), int(rng.integers(1, 6))))
        at = int(rng.integers(0, len(base)))
        k = int(rng.integers(4, 16))
        base = base[:at] + unit * k + base[at + len(unit) * k:]
    return [base] + [mutate(rng, base, int(rng.integers(0, 7))) for _ in range(n - 1)]


def synthetic_table():
    """A stand-in repeat table where the reference's is not available: rising open probabilities with the repeat count."""
    o = np.full((11, 51), 1e-9, np.float32)
    o[1:, 2:] = np.geomspace(1e-9, 1e-5, 49, dtype=np.float32)
    e = np.full((11, 51, 50), 0.5, np.float32)
    e[1:, 2:, :] = 0.8
    return o, e


def same(got, want):
    """Statuses identical and HMM / SELF values bit-equal."""
    (out, st), (wout, wst) = got, want
    exact = (wst == 0) | (wst == 1)
    return bool(np.array_equal(st, wst) and np.array_equal(out[exact].view(np.uint64), wout[exact].view(np.uint64)))


def run_per_set(eng, model, sets, K, T):
    ms, dp, res = [], [], []
    for seqs in sets:
        t0 = time.perf_counter()
        res.append(eng.mutation_prime(model, seqs))
        ms.append(1e3 * (time.perf_counter() - t0))
        dp.append(eng.last_dp_kernel_ms())
    return res, ms, dp


def run_sets_per_call(eng, model, sets, K, T):
    ms, dp, res = [], [], []
    for i in range(0, len(sets), K):
        t0 = time.perf_counter()
        res += eng.mutation_prime_sets(model, sets[i:i + K])
        ms.append(1e3 * (time.perf_counter() - t0))
        dp.append(eng.last_dp_kernel_ms())
    return res, ms, dp


def run_threads(batcher, make_model, sets, K, T):
    """T threads, thread k priming sets k, k + T, ... one after the other, each with a model of its own (as a caller builds one per
    region). Call time = one request's latency."""
    res, ms, errors = [None] * len(sets), [], []
    start = threading.Barrier(T)

    def worker(k):
        try:
            start.wait()
            for i in range(k, len(sets), T):
                model = make_model()
                t0 = time.perf_counter()
                res[i] = batcher.mutation_prime(model, sets[i])
                ms.append(1e3 * (time.perf_counter() - t0))
        except Exception as ex:          # noqa: BLE001
            errors.append(repr(ex))
    threads = [threading.Thread(target=worker, args=(k,)) for k in range(T)]
    for t in threads:
        t.start()
    for t in threads:
        t.join()
    assert not errors, errors
    return res, ms, []


def compare_modes(a, info, snv, o, e):
    """Per shape: the three modes on the same seeded sets, alternated round by round after a warm-up of each."""
    from octopus_b200 import MutationModel, PairHMMEngine, PopulateBatcher
    eng = PairHMMEngine(0)
    model = MutationModel(snv, o, e)
    make_model = lambda: MutationModel(snv, o, e)       # noqa: E731
    rows = []
    for length in [int(x) for x in a.lengths.split(",")]:
        for n_sets in [int(x) for x in str(a.sets).split(",")]:
            rng = np.random.default_rng(1000 * length + n_sets)
            sets = [trio_set(rng, a.haplotypes, length) for _ in range(n_sets)]
            K, T = a.sets_per_call or n_sets, a.threads or 1
            batcher = PopulateBatcher(0, clients=T, max_wait_us=a.max_wait_us)
            modes = [("per_set", lambda: run_per_set(eng, model, sets, K, T)),
                     ("sets_per_call", lambda: run_sets_per_call(eng, model, sets, K, T)),
                     ("threads", lambda: run_threads(batcher, make_model, sets, K, T))]
            for _, run in modes:                          # warm-up: module load, scratch and staging growth
                run()
            acc = {name: dict(wall=[], ms=[], dp=[], same=True, stats=[]) for name, _ in modes}
            baseline = None
            for r in range(a.rounds):
                order = modes if r % 2 == 0 else modes[::-1]
                for name, run in order:
                    before = batcher.stats()
                    t0 = time.perf_counter()
                    res, ms, dp = run()
                    acc[name]["wall"].append(time.perf_counter() - t0)
                    after = batcher.stats()
                    acc[name]["ms"] += ms
                    acc[name]["dp"] += dp
                    if name == "threads":
                        acc[name]["stats"].append({k: after[k] - before[k] for k in ("requests", "gpu_calls", "merged_calls")})
                        acc[name]["max_regions_per_call"] = after["max_regions_per_call"]
                    if name == "per_set" and baseline is None:
                        baseline = res
                    acc[name]["res"] = res
                for name, _ in modes:
                    if "res" in acc[name]:
                        acc[name]["same"] &= all(same(g, w) for g, w in zip(acc[name].pop("res"), baseline))
            batcher.close()
            for name, _ in modes:
                m = acc[name]
                wall = float(np.median(m["wall"]))
                row = dict(what="mutation_prime_modes", mode=name, haplotypes=a.haplotypes, length=length, sets=n_sets,
                           sets_per_call=K if name == "sets_per_call" else 1, threads=T if name == "threads" else 1, rounds=a.rounds,
                           sets_per_s=n_sets / wall, wall_ms=1e3 * wall, median_call_ms=float(np.median(m["ms"])),
                           dp_kernel_ms=float(np.median(m["dp"])) if m["dp"] else "not measured (the batcher's engine)",
                           same_as_per_set=m["same"], **info)
                if name == "threads":
                    row.update(batcher_calls_per_round=m["stats"], max_regions_per_call=m["max_regions_per_call"], max_wait_us=a.max_wait_us)
                rows.append(row)
                print(json.dumps(row), flush=True)
    return rows


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--sets", default="20", help="sets per shape; a comma list with --sets-per-call / --threads")
    ap.add_argument("--haplotypes", type=int, default=50)
    ap.add_argument("--lengths", default="300,1000")
    ap.add_argument("--sets-per-call", type=int, default=0)
    ap.add_argument("--threads", type=int, default=0)
    ap.add_argument("--max-wait-us", type=int, default=2000)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    import torch
    assert torch.cuda.is_available(), "bench_mutation_prime needs a GPU"
    from octopus_b200 import MutationModel, PairHMMEngine, _lib
    info = device_info()
    print(json.dumps(info), flush=True)
    snv, indel = TRIO_PRIORS
    ref = RefMutation() if RefMutation.available() else None
    o, e = ref.table(indel) if ref else synthetic_table()
    if a.sets_per_call or a.threads:
        rows = compare_modes(a, info, snv, o, e)
        if a.out:
            with open(a.out, "w") as f:
                json.dump(rows, f, indent=1)
        return
    a.sets = int(a.sets)
    eng = PairHMMEngine(0)
    model = MutationModel(snv, o, e)
    rows = []
    for length in [int(x) for x in a.lengths.split(",")]:
        rng = np.random.default_rng(length)
        sets = [trio_set(rng, a.haplotypes, length) for _ in range(a.sets)]
        eng.mutation_prime(model, sets[0])                    # warm-up: module load, scratch allocation
        align_pairs_recipe(eng, model, o, e, sets[0])
        prime_ms, dp_ms, recipe_ms, ref_ms = [], [], [], []
        same_recipe, same_ref, hmm_pairs = True, True, 0
        for seqs in sets:
            t0 = time.perf_counter()
            out, status = eng.mutation_prime(model, seqs)
            prime_ms.append(1e3 * (time.perf_counter() - t0))
            dp_ms.append(eng.last_dp_kernel_ms())
            t0 = time.perf_counter()
            rout, rstatus = align_pairs_recipe(eng, model, o, e, seqs)
            recipe_ms.append(1e3 * (time.perf_counter() - t0))
            same_recipe &= bool(np.array_equal(status, rstatus) and np.array_equal(out.view(np.uint64), rout.view(np.uint64)))
            hmm = (status == _lib.MUT_HMM) | (status == _lib.MUT_SELF)
            hmm_pairs += int((status == _lib.MUT_HMM).sum())
            if ref:
                t0 = time.perf_counter()
                want, approx = ref.prime(snv, indel, seqs)
                ref_ms.append(1e3 * (time.perf_counter() - t0))
                approx_got = np.isin(status, (_lib.MUT_APPROX_LENGTH, _lib.MUT_APPROX_OFFSET, _lib.MUT_APPROX_OVERFLOW))
                same_ref &= bool(np.array_equal(out[hmm].view(np.uint64), want[hmm].view(np.uint64)) and np.array_equal(approx_got, approx))
        row = dict(what="phmm_mutation_prime", haplotypes=a.haplotypes, length=length, sets=a.sets, pairs_per_set=a.haplotypes * (a.haplotypes - 1),
                   hmm_pairs_per_set=hmm_pairs / a.sets, prime_ms=float(np.median(prime_ms)), dp_kernel_ms=float(np.median(dp_ms)),
                   recipe_ms=float(np.median(recipe_ms)), reference_cpu_ms=float(np.median(ref_ms)) if ref else "not measured",
                   speedup_vs_recipe=float(np.median(recipe_ms) / np.median(prime_ms)),
                   speedup_vs_reference_cpu=float(np.median(ref_ms) / np.median(prime_ms)) if ref else "not measured",
                   same_as_recipe=same_recipe, same_as_reference=same_ref if ref else "not checked",
                   repeat_table="reference" if ref else "synthetic", **info)
        rows.append(row)
        print(json.dumps(row), flush=True)
    if a.out:
        with open(a.out, "w") as f:
            json.dump(rows, f, indent=1)


if __name__ == "__main__":
    main()
