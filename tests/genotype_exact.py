"""High-precision reference for the genotype-likelihood reduction (phmm_genotype_likelihoods, k_genotype_likelihoods, and the
reference-form oracle_genotype_likelihoods), plain numpy + decimal as tests/exact.py.

For a genotype g = (h_1 .. h_p) over an [H][R] matrix x of ln-likelihoods the value is
    L(g) = sum_r t_r,   t_r = ln sum_k e^{x[h_k][r]} - ln p,
with every copy of a haplotype counted (ConstantMixtureGenotypeLikelihoodModel::evaluate). exact_genotypes computes it at 40+
digits; genotype_bound is the forward-error bound of a double evaluation of it; kernel_model restates the kernel's operation
order in numpy so that the bound can be tried on the CPU; assert_within_bound is the checker the GPU tests use.

The bound. Let u = eps / 2 (eps = 2^-52) be the unit roundoff, and let exp / log be faithful to 1 ulp (CUDA's double exp and
log are, glibc's are closer). Per read of a heterozygous genotype the double evaluation does one max (exact), p subtractions
x_k - mx and p exps, a p-term sum, one log, and two adds (+ mx, - ln p, with ln p itself one log):
  * e_k = exp(fl(x_k - mx)) carries a relative error of at most |x_k - mx| u + 2u; since y e^-y <= 1/e the sum S = sum_k e_k
    (S >= 1: the max term is 1) carries at most ((p - 1)/e + 2) u from them, and p - 1 more u from its p - 1 additions of
    positive terms: |dS / S| <= 2p u;
  * ln S moves by |dS / S| and the log adds 2u ln S <= 2u ln p; mx + ln S rounds by u (|mx| + ln p); ln p is off by 2u ln p; the
    last subtraction rounds by u |t_r|.
So |fl(t_r) - t_r| <= u (|mx| + 5 ln p + 2p + |t_r|) <= eps (|mx_r| + ln p + 2p + 4) + eps |t_r| / 2 (c = 1 below). The
reference's special forms (log_sum_exp(ln 2 + a, b), log1p, ...) add one rounding of ln m + x, which is at most u (|mx| + ln p)
more, and still fit: u (2|mx| + 7 ln p + 2p + 2) <= eps (|mx| + ln p + 2p + 4). A homozygous genotype's t_r is x exactly.
Summing the computed t_r along chains of at most n_seq additions adds at most n_seq u sum_r |t_r| (first order). With the
per-read |t_r| term folded in,
    |fl(L) - L| <= eps [ (n_seq + 8) sum_r |t_r| + sum_r c (|mx_r| + ln p + 2p + 4) ],   c = 1,
and the tests allow BOUND_UNITS times that, for the second-order terms left out above. n_seq = kernel_chain(R) for the
kernel's 256 strided partial sums followed by its shared-memory tree, and R for the reference's read-by-read std::accumulate.

Entries equal to lowest() (-DBL_MAX) are values like any other: e^{x - mx} underflows to 0 unless x is the max, which counts
as it is. -inf contributes e^-inf = 0; a read on which every value of the genotype is -inf has t_r = -inf. A result whose
exact value is not finite, or whose exact value lies beyond the largest double, is reported by class ("-inf", "+inf", "nan")
and must be met by a result of the same class."""
import math
from decimal import Decimal, localcontext

import numpy as np

EPS = 2.0 ** -52
LOWEST = -1.7976931348623157e308
C = 0.230258509299404568401799145468436420760110148862877297603     # ln10 / 10, the populate value scale
BOUND_UNITS = 2.0           # safety factor over the first-order bound derived above
_PREC = 48
_NEGLIGIBLE = -2000         # e^-2000 < 10^-868: a term this far below the max (which contributes 1) is nothing at _PREC digits
_exp_cache, _ln_cache = {}, {}


def kernel_chain(R):
    """The longest chain of additions any read's term goes through in k_genotype_likelihoods: ceil(R / 256) strided adds per
    thread, then 8 levels of the 256-wide shared-memory tree."""
    return -(-int(R) // 256) + 8


def _cls(v):
    return "finite" if math.isfinite(v) else ("nan" if math.isnan(v) else ("-inf" if v < 0 else "+inf"))


def _row_term(row, p, ln_p):
    """t for one read's finite values sorted descending (p values in all, the others -inf): (Decimal t, |t| as float)."""
    mx = row[0]
    if len(row) == p and row[-1] == mx:  # every value equal: ln(p e^x) - ln p = x
        return Decimal(mx), abs(mx)
    dmx = Decimal(mx)
    with localcontext() as ctx:
        ctx.prec = _PREC
        s = Decimal(0)
        for x in row:
            key = (x, mx)
            e = _exp_cache.get(key)
            if e is None:
                d = Decimal(x) - dmx
                e = _exp_cache[key] = Decimal(0) if d < _NEGLIGIBLE else d.exp()
            s += e
        ln_s = _ln_cache.get(s)
        if ln_s is None:
            ln_s = _ln_cache[s] = s.ln()
        t = dmx + ln_s - ln_p
    return t, abs(float(t))


class Exact:
    """The exact value of every genotype's L(g) and the pieces of its bound.
    value[g]: Decimal (None where cls[g] is not "finite"); cls[g]: "finite", "-inf", "+inf" or "nan";
    abs_t[g] = sum_r |t_r|; mx_terms[g] = sum_r (|mx_r| + ln p + 2p + 4); R, p: the shape."""

    def __init__(self, lnl, genotypes):
        lnl = np.asarray(lnl, dtype=np.float64)
        gts = np.asarray(genotypes, dtype=np.int64)
        G, p = gts.shape
        R = lnl.shape[1]
        self.R, self.p, self.G = R, p, G
        self.value = [Decimal(0)] * G
        self.cls = ["finite"] * G
        self.abs_t = np.zeros(G)
        self.mx_terms = np.zeros(G)
        if p == 0 or G == 0:
            return
        with localcontext() as ctx:
            ctx.prec = _PREC
            ln_p = Decimal(p).ln()
        extra = math.log(p) + 2 * p + 4
        step = max(1, (1 << 22) // (p * R))
        for g0 in range(0, G, step):
            X = lnl[gts[g0:g0 + step]]                                      # (g, p, R)
            rows = -np.sort(-X.transpose(0, 2, 1).reshape(-1, p), axis=1)   # one row per (genotype, read), descending
            uniq, inv = np.unique(rows, axis=0, return_inverse=True)
            inv = inv.reshape(-1, R)
            terms = []
            for row in uniq:
                if np.isnan(row).any():
                    terms.append(("nan", None, 0.0, 0.0))
                elif row[0] == np.inf:
                    terms.append(("+inf", None, 0.0, 0.0))
                elif row[0] == -np.inf:
                    terms.append(("-inf", None, 0.0, 0.0))
                else:
                    fin = [float(v) for v in row if v != -np.inf]
                    t, a = _row_term(fin, p, ln_p)
                    terms.append(("finite", t, a, abs(fin[0]) + extra))
            for j in range(inv.shape[0]):
                u, cnt = np.unique(inv[j], return_counts=True)
                classes = {terms[i][0] for i in u}
                g = g0 + j
                if "nan" in classes or {"-inf", "+inf"} <= classes:
                    self.cls[g] = "nan"
                elif "-inf" in classes or "+inf" in classes:
                    self.cls[g] = "-inf" if "-inf" in classes else "+inf"
                else:
                    with localcontext() as ctx:
                        ctx.prec = _PREC + 8
                        total = sum((terms[i][1] * int(c) for i, c in zip(u, cnt)), Decimal(0))
                    self.value[g] = total
                    self.abs_t[g] = sum(terms[i][2] * int(c) for i, c in zip(u, cnt))
                    self.mx_terms[g] = sum(terms[i][3] * int(c) for i, c in zip(u, cnt))
                    if math.isinf(float(total)):                                    # beyond the largest double
                        self.cls[g] = "-inf" if total < 0 else "+inf"
                        self.value[g] = None


def exact_genotypes(lnl, genotypes):
    """Exact per-genotype values and classes; see Exact."""
    return Exact(lnl, genotypes)


def genotype_bound(ex, n_seq):
    """eps [ (n_seq + 8) sum_r |t_r| + sum_r (|mx_r| + ln p + 2p + 4) ] per genotype (the module docstring derives it), before
    the BOUND_UNITS safety factor. ex: an Exact."""
    return EPS * ((n_seq + 8) * ex.abs_t + ex.mx_terms)


def assert_within_bound(got, ex, n_seq, what=""):
    """Every got[g] within BOUND_UNITS * genotype_bound of the exact value, or of the exact value's non-finite class. Returns the
    largest |error| / genotype_bound (the check allows BOUND_UNITS)."""
    got = np.asarray(got, dtype=np.float64)
    assert got.shape == (ex.G,), (what, got.shape, ex.G)
    unit = genotype_bound(ex, n_seq)
    worst, bad = 0.0, []
    for g in range(ex.G):
        c = _cls(float(got[g]))
        if ex.cls[g] != "finite" or c != "finite":
            if c != ex.cls[g]:
                bad.append((g, float(got[g]), ex.cls[g]))
            continue
        err = float(abs(Decimal(float(got[g])) - ex.value[g]))
        r = err / unit[g] if unit[g] > 0 else (0.0 if err == 0 else math.inf)
        if not r <= BOUND_UNITS:
            bad.append((g, float(got[g]), float(ex.value[g]), err, float(unit[g])))
        worst = max(worst, r)
    assert not bad, "%s: %d of %d genotypes outside %g x the bound; (g, got, exact, |error|, bound): %s" % (
        what, len(bad), ex.G, BOUND_UNITS, bad[:8])
    return worst


MUTATIONS = ("drop_read", "ln_p_once", "float32", "max_short")


def kernel_model(lnl, genotypes, mutation=None):
    """k_genotype_likelihoods' operation order in float64 numpy: per read (homozygous: the value; else fmax over the p values,
    a sum from 0.0 of exp(x_k - mx) in k order, then (mx + log(sum)) - log(p)), 256 strided partial sums acc[t] over reads
    t, t + 256, ..., then the shared-memory tree partial[i] += partial[i + s] for s = 128 .. 1.
    mutation (the checker's self-test): "drop_read" leaves out each genotype's first read with |t_r| >= 0.1; "ln_p_once"
    subtracts ln p once per genotype instead of once per read; "float32" evaluates exp and log in float32; "max_short" takes
    the max over the first p - 1 values only."""
    assert mutation is None or mutation in MUTATIONS, mutation
    lnl = np.asarray(lnl, dtype=np.float64)
    gts = np.asarray(genotypes, dtype=np.int64)
    G, p = gts.shape
    R = lnl.shape[1]
    out = np.zeros(G)
    if p == 0 or G == 0:
        return out
    ln_p = np.log(np.float64(p))
    exp, log = np.exp, np.log
    if mutation == "float32":
        exp = lambda v: np.exp(v.astype(np.float32)).astype(np.float64)             # noqa: E731
        log = lambda v: np.log(v.astype(np.float32)).astype(np.float64)             # noqa: E731
    step = max(1, (1 << 22) // (p * R))
    with np.errstate(all="ignore"):
        for g0 in range(0, G, step):
            gt = gts[g0:g0 + step]
            X = lnl[gt]                                                  # (g, p, R)
            homo = (gt == gt[:, :1]).all(axis=1)
            mx = X[:, 0]
            for k in range(1, p - 1 if mutation == "max_short" and p > 1 else p):
                mx = np.fmax(mx, X[:, k])
            s = np.zeros_like(mx)
            for k in range(p):
                s = s + exp(X[:, k] - mx)
            t = (mx + log(s)) - (0.0 if mutation == "ln_p_once" else ln_p)
            t = np.where(homo[:, None], X[:, 0], t)
            if mutation == "drop_read":
                big = np.abs(t) >= 0.1
                first = np.argmax(big, axis=1)
                rows = np.nonzero(big.any(axis=1))[0]
                t[rows, first[rows]] = 0.0
            T = np.concatenate([t, np.zeros((len(gt), (-R) % 256))], axis=1).reshape(len(gt), -1, 256)
            acc = np.zeros((len(gt), 256))
            for i in range(T.shape[1]):
                acc = acc + T[:, i]
            s_ = 128
            while s_ > 0:
                acc[:, :s_] = acc[:, :s_] + acc[:, s_:2 * s_]
                s_ >>= 1
            res = acc[:, 0]
            if mutation == "ln_p_once":
                res = np.where(homo, res, res - ln_p)
            out[g0:g0 + len(gt)] = res
    return out


# -- inputs shared by the GPU tests and the CPU validation of the bound --------------------------------------------------------

PLOIDIES = (1, 2, 3, 4, 5, 8, 16, 64)
READ_COUNTS = (1, 31, 255, 256, 257, 4000)


def penalty_matrix(rng, H, R, s_max=400):
    """Values as populate leaves them with mapping quality off: -ln10/10 * s for integer penalties s."""
    return -C * rng.integers(0, s_max + 1, size=(H, R)).astype(np.float64)


def uniform_genotypes(rng, H, p, G, homozygous=True):
    """G genotypes of ploidy p with every index drawn uniformly from [0, H) (sorted, as the reference's genotypes are), and with
    `homozygous` the last row one haplotype p times."""
    gts = np.sort(rng.integers(0, H, size=(G, p)), axis=1).astype(np.int32)
    if homozygous and G:
        gts[-1] = rng.integers(0, H)
    return gts


def duplicate_patterns(rng, H, p):
    """Every sequence of length p over p distinct haplotypes (sorted and unsorted; every run pattern of the reference's special
    forms), p in (3, 4)."""
    hs = rng.choice(H, size=p, replace=False)
    idx = np.array(np.meshgrid(*([np.arange(p)] * p), indexing="ij")).reshape(p, -1).T
    return hs[idx].astype(np.int32)


def value_matrix(rng, kind, H, R):
    """Matrices of the edge values: "lowest" (lowest() entries in the even haplotypes: genotypes of
    even haplotypes only sum several lowest() reads past the largest double), "neg_inf" (-inf entries everywhere but
    haplotype 0), "zeros" (0.0 entries), "spread" (per read one value near 0, the others 700 to 1000 below it: exp underflows
    to subnormals and 0), "equal" (every haplotype the same row: the exact answer is the plain sum)."""
    m = penalty_matrix(rng, H, R)
    if kind == "lowest":
        m[0::2][rng.random(((H + 1) // 2, R)) < 0.2] = LOWEST
    elif kind == "neg_inf":
        m[1:][rng.random((H - 1, R)) < 0.3] = -np.inf
    elif kind == "zeros":
        m[rng.random((H, R)) < 0.3] = 0.0
    elif kind == "spread":
        top = rng.integers(0, H, size=R)
        m = -rng.uniform(0.0, 5.0, size=(1, R)) - rng.uniform(700.0, 1000.0, size=(H, R))
        m[top, np.arange(R)] = -rng.uniform(0.0, 5.0, size=R)
    elif kind == "equal":
        m[:] = m[0]
    else:
        raise ValueError(kind)
    return m


VALUE_KINDS = ("lowest", "neg_inf", "zeros", "spread", "equal")


def synthetic_cases(seed=2024):
    """(name, lnl, genotypes) of every synthetic input the GPU tests run: each ploidy at each read count, the edge values, every
    duplicate pattern of ploidy 3 and 4, one heterozygous copy among 63, H = 1024 with uniform draws, G = 1. Generated from the
    seed so that the CPU validation of the bound sees the same inputs."""
    rng = np.random.default_rng(seed)
    out = []
    for p in PLOIDIES:
        for R in READ_COUNTS:
            out.append(("ploidy %d R %d" % (p, R), penalty_matrix(rng, 64, R), uniform_genotypes(rng, 64, p, 4)))
    for kind in VALUE_KINDS:
        for p in PLOIDIES:
            m = value_matrix(rng, kind, 48, 300)
            gts = uniform_genotypes(rng, 48, p, 6)
            if kind == "neg_inf":
                # haplotype 0 is finite everywhere: every genotype holds it, so no read has all its values -inf
                gts[:, 0] = 0
                gts = np.sort(gts, axis=1)
                gts[-1] = 0
            out.append(("%s ploidy %d" % (kind, p), m, gts))
    for p in (3, 4):
        out.append(("every duplicate pattern, ploidy %d" % p, penalty_matrix(rng, 32, 500), duplicate_patterns(rng, 32, p)))
    one = np.full((3, 64), 5, dtype=np.int32)
    one[0, 0], one[1, 31], one[2, 63] = 9, 9, 9
    out.append(("one heterozygous copy among 63", penalty_matrix(rng, 16, 700), one))
    for p in (2, 3, 8):
        out.append(("H 1024 ploidy %d" % p, penalty_matrix(rng, 1024, 257), uniform_genotypes(rng, 1024, p, 64, homozygous=False)))
    out.append(("G 1", penalty_matrix(rng, 8, 333), np.array([[1, 6]], dtype=np.int32)))
    return out


def many_genotypes_case(seed=7):
    """G = 70 000 > 65 535 genotypes of ploidy 2 over H = 1024, R = 3 (one block per genotype: a grid wider than 2^16 - 1)."""
    rng = np.random.default_rng(seed)
    return penalty_matrix(rng, 1024, 3, s_max=40), uniform_genotypes(rng, 1024, 2, 70_000)
