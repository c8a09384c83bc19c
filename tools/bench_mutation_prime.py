"""DeNovoModel::prime on trio-shaped haplotype sets: one phmm_mutation_prime call per set, against the reference's own prime on one host
thread (the compiled oracle, oracle/_ref/libref_mutation.so, where present) and against the recipe it replaces (phmm_align_pairs over
host-built padded truths, every CIGAR copied back and re-scored on the host). Checks that the three agree and prints one JSON line per
shape, with the card's name and power limit read in the same run.

Sets: 50 haplotypes (the reference's largest eagerly primed set, 2 450 ordered pairs) of one region, from synth.make_haplotypes's base
sequence with injected STRs, each haplotype carrying SNVs and 1-20 bp indels (tests/mutation_oracle.py's mutate).
    python tools/bench_mutation_prime.py [--sets 20] [--out results.json]
"""
import argparse
import json
import os
import sys
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


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--sets", type=int, default=20)
    ap.add_argument("--haplotypes", type=int, default=50)
    ap.add_argument("--lengths", default="300,1000")
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    import torch
    assert torch.cuda.is_available(), "bench_mutation_prime needs a GPU"
    from octopus_b200 import MutationModel, PairHMMEngine, _lib
    eng = PairHMMEngine(0)
    info = device_info()
    print(json.dumps(info), flush=True)
    snv, indel = TRIO_PRIORS
    ref = RefMutation() if RefMutation.available() else None
    o, e = ref.table(indel) if ref else synthetic_table()
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
