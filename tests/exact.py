"""Comparators for populate's output (plain numpy + decimal).

With mapping quality off a pair's value is the double ``-ln10/10 * s`` of its integer penalty s (or lowest()), so the engine and
the oracle must agree bit for bit. With mapping quality on the value is ``ln((1 - p) * 10^(-s/10) + p)``, p = 10^(-mapq/10), which
saturates at ln p once s passes mapq by a few tens; a relative tolerance there hides any error in s. The mixed value is instead
held to the forward-error bound of the reference's double formula around the exact value, computed here at 40 digits."""
from decimal import Decimal, localcontext

import numpy as np

C = 0.230258509299404568401799145468436420760110148862877297603     # ln10 / 10 as the engine's double (utils/maths.hpp:41)
EPS = 2.0 ** -52
LOWEST = -1.7976931348623157e308
LOWEST_S = 1 << 62          # penalties(): the stand-in for lowest() (no candidate position produced a score)
BOUND_UNITS = 4.0           # the reference's own formula under glibc stays within 0.58 of these units
_PREC = 40
_D_C = Decimal("0.2302585092994045684017999454684364207601101488628772976033327900967572609677352480235997205089598298")


def penalties(values):
    """The integer penalty behind each mapping-quality-free value (LOWEST_S for lowest()). Clamped values (0.0) give 0. Every
    value must be exactly the double -C * s of the recovered s."""
    v = np.asarray(values, dtype=np.float64)
    low = v == LOWEST
    s = np.rint(-np.where(low, 0.0, v) / C).astype(np.int64)
    s[low] = LOWEST_S
    back = np.where(low, LOWEST, -C * s.astype(np.float64))
    back[(v == 0.0) & ~low] = 0.0
    bad = np.nonzero(back.view(np.int64) != v.view(np.int64))
    assert bad[0].size == 0, "values that are not -ln10/10 * integer: %s" % [
        (tuple(int(i) for i in ix), float(v[ix])) for ix in list(zip(*bad))[:10]]
    return s


def assert_same_penalties(got, want, st, wst, what=""):
    """Statuses equal everywhere (st None: not reported); values bit-equal wherever the oracle's status is 0 (mapping quality off).
    On failure, reports up to 10 (h, r, got s, want s)."""
    got, want, wst = (np.asarray(a) for a in (got, want, wst))
    assert got.shape == want.shape, (what, got.shape, want.shape)
    ok = wst == 0
    if st is not None:
        # the engine also flags lowest() values (PHMM_STATUS_OVERFLOW, 1), a status the oracle does not report
        st, wst1 = np.asarray(st), np.where(ok & (want == LOWEST), 1, wst)
        sbad = np.argwhere(st != wst1)
        assert sbad.size == 0, (what, "status", [(tuple(int(i) for i in ix), int(st[tuple(ix)]), int(wst1[tuple(ix)])) for ix in sbad[:10]])
    g, w = np.ascontiguousarray(got, np.float64), np.ascontiguousarray(want, np.float64)
    bad = np.argwhere(ok & (g.view(np.int64) != w.view(np.int64)))
    if bad.size:
        def s_of(x):
            if x == LOWEST:
                return "lowest"
            k = int(round(-x / C))
            return k if -C * k == x or (x == 0.0 and k == 0) else "not an integer: %r" % x
        rows = [tuple(int(i) for i in ix) + (s_of(float(g[tuple(ix)])), s_of(float(w[tuple(ix)]))) for ix in bad[:10]]
        raise AssertionError("%s: %d of %d values differ; (index, got s, want s): %s" % (what, len(bad), int(ok.sum()), rows))
    penalties(w[ok])


def effective_mapq(mapq, cap=120, trigger=None):
    """haplotype_likelihood_model.cpp:49-51, 285-303: a trigger at or above the cap is dropped; mapq >= trigger becomes the cap."""
    m = np.asarray(mapq, dtype=np.int64).copy()
    if trigger is not None and 0 <= trigger < cap:
        m[m >= trigger] = cap
    return m


_ln_mapped, _p, _q, _mixed = {}, {}, {}, {}


def _tab(tab, key, f):
    v = tab.get(key)
    if v is None:
        with localcontext() as ctx:
            ctx.prec = _PREC
            v = tab[key] = f(key)
    return v


def _mix1(s, m):
    p = _tab(_p, m, lambda k: (-_D_C * k).exp())
    if s == LOWEST_S:
        x = -_D_C * m                                   # ln p: the mixture of lowest() and the miss term
    else:
        if m == 0:
            return 0.0, 0.0
        q = _tab(_q, s, lambda k: (-_D_C * k).exp())
        ln1p = _tab(_ln_mapped, m, lambda k: (1 - _p[k]).ln())
        with localcontext() as ctx:
            ctx.prec = _PREC
            # ln((1-p) q + p) = ln(1-p) + ln(q + p / (1-p)): both terms of the sum are positive, no cancellation
            x = ln1p + (q + p / (1 - p)).ln()
    if x > Decimal("-1e-15"):
        return 0.0, 0.0
    with localcontext() as ctx:
        ctx.prec = _PREC
        return float(x), float(x - Decimal(float(x)))       # the double nearest the exact value, and what rounding left out


def _exact(s, m):
    """[value rounded to a double, exact value - that double] of every (s, mapq) entry."""
    out = np.empty((2,) + s.shape, dtype=np.float64)
    for ix in np.ndindex(s.shape):
        key = (int(s[ix]), int(m[ix]))
        v = _mixed.get(key)
        if v is None:
            v = _mixed[key] = _mix1(*key)
        out[(0,) + ix], out[(1,) + ix] = v
    return out


def mix_reference(s, mapq, cap=120, trigger=None):
    """The exact mixed ln-likelihood of penalty s (LOWEST_S for lowest()) at mapping quality mapq, under the cap / trigger rule,
    rounded once to a double, with the reference's clamp above -1e-15."""
    s = np.asarray(s, dtype=np.int64)
    m = np.broadcast_to(effective_mapq(mapq, cap, trigger), s.shape)
    return _exact(s, m)[0]


def mix_bound(s, mapq_eff):
    """The forward-error bound of the double formula, 4 eps (1 + c|s| + c mapq), in absolute terms."""
    s = np.asarray(s, dtype=np.int64)
    sf = np.where(s == LOWEST_S, 0, np.abs(s)).astype(np.float64)
    return BOUND_UNITS * EPS * (1.0 + C * sf + C * np.asarray(mapq_eff, dtype=np.float64))


def assert_mix_within_bound(got, s, mapq_eff, what=""):
    """|got - exact| <= 4 eps (1 + c|s| + c mapq_eff) for every entry. Returns the largest error in units of eps (1 + c|s| + c mapq)
    (the bound is 4 of them)."""
    got = np.asarray(got, dtype=np.float64)
    s = np.asarray(s, dtype=np.int64)
    m = np.broadcast_to(np.asarray(mapq_eff, dtype=np.int64), s.shape)
    exact, rest = _exact(s, m)
    unit = mix_bound(s, m) / BOUND_UNITS
    err = np.abs((got - exact) - rest) / unit
    bad = np.argwhere(~(err <= BOUND_UNITS))
    assert bad.size == 0, "%s: %d of %d mixed values outside the bound; (index, s, mapq, got, exact, units): %s" % (
        what, len(bad), got.size, len(bad) and [(tuple(int(i) for i in ix), int(s[tuple(ix)]), int(m[tuple(ix)]), float(got[tuple(ix)]),
                                                 float(exact[tuple(ix)]), float(err[tuple(ix)])) for ix in bad[:10]])
    return float(err.max()) if err.size else 0.0


def assert_sums_within_bound(got, s, mapq_eff, template_off, what=""):
    """Templates: got[h, t] against the exact sum of its reads' exact mixed values. The bound adds the reads' bounds and the
    rounding of the running double sum (one eps of each partial sum's magnitude per addition). s / mapq_eff: [H, R] / [R]."""
    got = np.asarray(got, dtype=np.float64)
    s = np.asarray(s, dtype=np.int64)
    m = np.broadcast_to(np.asarray(mapq_eff, dtype=np.int64), s.shape)
    exact = mix_reference(s, m)
    per = mix_bound(s, m)
    worst = 0.0
    for t in range(len(template_off) - 1):
        lo, hi = int(template_off[t]), int(template_off[t + 1])
        for h in range(got.shape[0]):
            terms = [Decimal(float(x)) for x in exact[h, lo:hi]]
            want = sum(terms, Decimal(0))
            run, ulps = Decimal(0), 0.0
            for x in terms:
                run += x
                ulps += float(abs(run)) * EPS
            bound = float(per[h, lo:hi].sum()) + ulps
            err = abs(float(Decimal(float(got[h, t])) - want))
            assert err <= bound, (what, h, t, float(got[h, t]), float(want), err, bound)
            worst = max(worst, err / bound if bound else 0.0)
    return worst
