"""Seeded inputs for the mixture-of-mixtures variational Bayes tests (CPU and GPU), shaped as SingleCellModel::evaluate_model
passes them: many samples (cells) of few reads, some with none; combinations of one genotype per group (clone)."""
import itertools

import numpy as np

LOWEST = -1.7976931348623157e308


def make(H, reads_per_sample, group_sizes, C, n_seeds, seed=0, dup=False, lowest=0, priors=None, concentrations="scalar"):
    """priors: None, or "some" (group priors on every other sample, one of them 0); concentrations: "scalar" (one value per
    sample) or "full" (one per sample and component). Returns a dict of the call's inputs, concentrations expanded."""
    rng = np.random.default_rng(seed)
    R = int(sum(reads_per_sample))
    T, K = len(group_sizes), int(sum(group_sizes))
    lnl = -rng.gamma(2.0, 6.0, size=(H, R))
    true = rng.integers(0, H, size=R)
    lnl[true, np.arange(R)] = -rng.uniform(0.0, 1.0, size=R)
    if lowest:      # at most one per haplotype row, so that no sum of two of them overflows
        rows = rng.choice(H, size=min(lowest, H), replace=False)
        lnl[rows, rng.integers(0, max(R, 1), size=len(rows))] = LOWEST
    off = np.concatenate([[0], np.cumsum(reads_per_sample)]).astype(np.int64)
    gt = rng.integers(0, H, size=(C, K)).astype(np.int32)
    if dup and K > 1:
        gt[::2, 1] = gt[::2, 0]
    if lowest:      # the lowest() haplotypes only in slot 0: a combination carrying one in several slots sums to -inf in double
        for j in range(1, K):      # (as the reference's double marginalise does), not in the long-double restatement
            while np.isin(gt[:, j], rows).any():
                gt[:, j] = np.where(np.isin(gt[:, j], rows), (gt[:, j] + 1) % H, gt[:, j])
    S = len(reads_per_sample)
    gc = np.full(T, 1.0) if concentrations == "scalar" else rng.uniform(0.5, 2.0, size=T)
    mc = np.repeat(rng.uniform(0.5, 3.0, size=S)[:, None], K, axis=1) if concentrations == "scalar" else rng.uniform(0.5, 3.0, size=(S, K))
    gp = mask = None
    if priors == "some":
        gp = rng.dirichlet(np.ones(T), size=S)
        gp[0, 0] = 0.0
        mask = (np.arange(S) % 2 == 0).astype(np.int32)
    lp = np.log(rng.dirichlet(np.ones(C)) + 1e-300)
    seeds = np.log(rng.dirichlet(np.ones(C) * 0.5, size=n_seeds) + 1e-300)
    return dict(lnl=lnl, off=off, sizes=list(group_sizes), gt=gt, lp=lp, gc=gc, mc=mc, seeds=seeds, gp=gp, mask=mask)


def propose_seeds(C, max_seeds=12):
    """Seeds as SingleCellModel::propose_seeds builds them (single_cell_model.cpp:855-885): log uniform; range seeds of
    p = 0.9999999 over the first C/100 and C/10 combinations (when C > 100, C > 10); point seeds of p = 0.9999 on the first
    combinations up to max_seeds in all."""
    def range_seed(n, p=0.9999999):
        r = np.full(C, np.log((1 - p) / (C - n)))
        r[:n] = np.log(p / n)
        return r
    seeds = [np.full(C, -np.log(float(C)))]
    if max_seeds > 1 and C > 100:
        seeds.append(range_seed(C // 100))
    if max_seeds > 2 and C > 10:
        seeds.append(range_seed(C // 10))
    for idx in range(min(max_seeds - len(seeds), C)):
        r = np.full(C, np.log((1 - 0.9999) / (C - 1)) if C > 1 else 0.0)
        if C > 1:
            r[idx] = np.log(0.9999)
        seeds.append(r)
    return np.array(seeds)


def combinations_of(genotypes, T):
    """Every ordered choice of one genotype per group, as rows of the combination matrix."""
    return np.array([np.concatenate(c) for c in itertools.product(genotypes, repeat=T)], dtype=np.int32)
