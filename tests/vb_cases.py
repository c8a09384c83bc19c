"""Seeded inputs for the variational Bayes tests (CPU and GPU): a likelihood matrix whose reads favour a few haplotypes,
genotypes, prior alphas, genotype log priors and seeds shaped as SubcloneModel::evaluate passes them."""
import numpy as np


def make(H, reads_per_sample, G, K, n_seeds, seed=0, dup=False, lowest=0):
    rng = np.random.default_rng(seed)
    R = int(sum(reads_per_sample))
    lnl = -rng.gamma(2.0, 6.0, size=(H, R))
    true = rng.integers(0, H, size=R)
    lnl[true, np.arange(R)] = -rng.uniform(0.0, 1.0, size=R)
    if lowest:
        idx = rng.choice(H * R, size=min(lowest, H * R), replace=False)
        lnl.ravel()[idx] = -1.7976931348623157e308
    off = np.concatenate([[0], np.cumsum(reads_per_sample)]).astype(np.int64)
    gt = rng.integers(0, H, size=(G, K)).astype(np.int32)
    if dup and K > 1:
        gt[::2, 1] = gt[::2, 0]
    S = len(reads_per_sample)
    prior = rng.uniform(0.5, 3.0, size=(S, K))
    lp = np.log(rng.dirichlet(np.ones(G)) + 1e-300)
    if n_seeds == G:       # generate_exhaustive_seeds: one near-point mass per genotype
        seeds = np.full((G, G), np.log(1e-6 / max(G - 1, 1)))
        np.fill_diagonal(seeds, np.log1p(-1e-6) if G > 1 else 0.0)
    else:
        seeds = np.log(rng.dirichlet(np.ones(G) * 0.5, size=n_seeds) + 1e-300)
    return lnl, off, gt, prior, lp, seeds
