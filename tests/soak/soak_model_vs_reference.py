"""Long-running CPU soak (test infrastructure, not collected by pytest): oracle_model_evaluate against the reference's own HaplotypeLikelihoodModel (compiled from
the reference checkout, oracle/_ref/libref_hmm.so) on adversarial inputs: low-complexity and N-rich haplotypes, zero penalties,
qualities 0..93, reads with N, out-of-range positions, short haplotypes.

usage: python tests/soak/soak_model_vs_reference.py [seed] [cases]
"""
import os, sys, numpy as np
ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT); sys.path.insert(0, os.path.join(ROOT, 'tests'))
from oracle.oracle import COracle, RefHMM
co, rh = COracle(), RefHMM()
seed = int(sys.argv[1]); N = int(sys.argv[2])
rng = np.random.default_rng(seed)
acgt = np.frombuffer(b"ACGT", dtype=np.uint8)
bad = 0
for it in range(N):
    band_req = int(rng.choice([3, 8, 12, 16, 30])); band = next(b for b in (8, 16, 32) if band_req <= b)
    L = int(rng.integers(6, 100))
    Lh = int(rng.integers(max(8, L + 2 * band - 6), L + 2 * band + 120))
    style = rng.integers(0, 3)
    if style == 0: hap = acgt[rng.integers(0, 4, Lh)].copy()
    elif style == 1:
        unit = acgt[rng.integers(0, 4, int(rng.integers(1, 5)))]; hap = np.tile(unit, Lh // len(unit) + 1)[:Lh].copy()
        for _ in range(int(rng.integers(0, 5))): hap[rng.integers(0, Lh)] = acgt[rng.integers(0, 4)]
    else:
        hap = acgt[rng.integers(0, 4, Lh)].copy(); hap[rng.random(Lh) < 0.05] = ord("N")
    ext = rng.random() < 0.3
    gen = lambda hi: (rng.choice([0, 1, hi], Lh) if ext else rng.integers(0, hi + 1, Lh)).astype(np.int8)
    mask_f = np.frombuffer(b"ACGTN", dtype=np.uint8)[rng.integers(0, 5, Lh)].copy(); mask_r = np.roll(hap, -1)
    prior_f, prior_r, go, ge = gen(125), gen(125), gen(45), gen(10)
    p0 = int(rng.integers(0, max(1, Lh - L + 1)))
    read = hap[p0:p0 + L].copy()
    if len(read) < L: read = np.concatenate([read, acgt[rng.integers(0, 4, L - len(read))]])
    read[read == ord("N")] = ord("A")
    for _ in range(int(rng.choice([0, 0, 1, 1, 2, 3, 5]))): read[rng.integers(0, L)] = acgt[rng.integers(0, 4)]
    if rng.random() < 0.2:
        i = int(rng.integers(1, L - 1)); read = np.concatenate([read[:i], read[i + 1:], acgt[rng.integers(0, 4, 1)]])
    if rng.random() < 0.1: read[rng.integers(0, L)] = ord("N")
    q = (rng.integers(0, 94, L) if rng.random() < 0.7 else rng.choice([0, 1, 2, 93], L)).astype(np.uint8)
    positions = None if rng.random() < 0.5 else [int(x) for x in rng.integers(0, Lh + 3, int(rng.integers(0, 5)))]
    orig = int(np.clip(p0 + int(rng.choice([0, 0, 0, -3, 4, -40, 40])), 0, Lh))
    flanks = None if rng.random() < 0.4 else (int(rng.integers(0, Lh // 2 + 1)), int(rng.integers(0, Lh // 2 + 1)))
    mq = int(rng.choice([0, 10, 29, 60, 255])); trig = int(rng.choice([-1, 40, 200])); cap = int(rng.choice([120, 50])); usemq = bool(rng.random() < 0.8)
    rev = bool(rng.random() < 0.5)
    w = rh.model_evaluate(band_req, hap, read, q, go, ge, mask_f, prior_f, mask_r, prior_r, positions, hap_begin=7, read_begin=7 + orig, mapping_quality=mq, reverse=rev, flanks=flanks, use_mapping_quality=usemq, mapq_cap=cap, mapq_cap_trigger=trig)
    pos = positions if positions is not None else co.kmer_map(read.tobytes().decode('latin1'), hap.tobytes().decode('latin1'), 10)
    mask, prior = (mask_r, prior_r) if rev else (mask_f, prior_f)
    g = co.model_evaluate(band, hap, read, q, go, ge, mask, prior, pos, orig, mapping_quality=mq, flanks=flanks, use_mapping_quality=usemq, mapq_cap=cap, mapq_cap_trigger=trig)
    ok = g[0] == w[0] and ((w[0] == 1 and g[2] == w[2]) or (w[0] == 0 and (g[1] == w[1] or abs(g[1]-w[1]) <= 1e-12*abs(w[1]))))
    if not ok:
        bad += 1
        if bad <= 6: print('MISMATCH', seed, it, 'band', band, 'L', L, 'Lh', Lh, g, w, 'flanks', flanks, 'pos', positions, 'orig', orig, flush=True)
print('seed', seed, 'cases', N, 'bad', bad, flush=True)
