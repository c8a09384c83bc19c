"""The C restatement of find_map_haplotypes (tests/cpp/find_map_oracle.c, read_assigner.cpp:45-64) pinned on constructed cases: exact
ties, values either side of maths::almost_equal's boundary (ulp = 1), the maximum that an almost-equal value does NOT raise, lowest(),
-inf priors (the every-haplotype fallback) and NaN. A Python statement of the same loop cross-checks random cases."""
import math

import numpy as np

from find_map_oracle import find_map, find_map_group

EPS = 2.0 ** -52
LOWEST = -1.7976931348623157e308
INF = math.inf
NAN = math.nan


def py_find_map(values, priors=None):
    """The reference's loop in Python floats (IEEE doubles, every operation rounded on its own)."""
    result, mx = [], LOWEST
    for k, v in enumerate(values):
        cur = v + (0.0 if priors is None else priors[k])
        if cur == mx or abs(cur - mx) < EPS * abs(cur + mx) * 1:
            result.append(k)
        elif cur > mx:
            result, mx = [k], cur
    if not result:
        result = list(range(len(values)))
    return sum(1 << k for k in result)


def up(x, n):
    """x moved n ulps towards +inf."""
    for _ in range(n):
        x = float(np.nextafter(x, INF))
    return x


def test_exact_ties():
    assert find_map([-5.0, -5.0, -7.0]) == 0b011
    assert find_map([-7.0, -5.0, -5.0]) == 0b110
    assert find_map([-2.5] * 5) == 0b11111
    assert find_map([-1.0, -3.0], [-2.0, 0.0]) == 0b11          # equal after the prior
    assert find_map([0.0, -0.0]) == 0b11


def test_almost_equal_boundary():
    # around -100, |l - r| < eps * |l + r| holds up to 3 ulps (2^-46 each) and fails at 4
    v0 = -100.0
    assert find_map([v0, up(v0, 3)]) == 0b11                      # almost equal and larger: joins the set
    assert find_map([v0, up(v0, 4)]) == 0b10                      # larger and not almost equal: restarts it
    assert find_map([up(v0, 4), v0]) == 0b01                      # smaller and not almost equal: ignored
    assert find_map([up(v0, 3), v0]) == 0b11
    # the boundary measured by the formula itself, on both sides, at several magnitudes
    for base in (-0.001, -1.0, -37.5, -1234.5678, -1e6):
        n = 1
        while abs(up(base, n) - base) < EPS * abs(up(base, n) + base):
            n += 1
        assert n >= 2
        assert find_map([base, up(base, n - 1)]) == 0b11, base
        assert find_map([base, up(base, n)]) == 0b10, base


def test_the_maximum_is_not_raised_by_an_almost_equal_value():
    v0 = -100.0
    v1, v2 = up(v0, 3), up(v0, 6)
    # v1 almost equal to v0 and above it: kept, the maximum stays v0
    assert find_map([v0, v1]) == 0b11
    # v2 is almost equal to v1 but not to v0: it is compared with v0, is larger, and restarts the set
    assert abs(v2 - v1) < EPS * abs(v2 + v1) and not abs(v2 - v0) < EPS * abs(v2 + v0)
    assert find_map([v0, v1, v2]) == 0b100
    # in the other order v2 leads: v1 joins it, v0 is out of its reach
    assert find_map([v2, v1, v0]) == 0b011
    # the same through the priors
    assert find_map([-100.0, -100.0, -100.0], [0.0, v1 - v0, v2 - v0]) == 0b100


def test_lowest_inf_and_nan():
    assert find_map([LOWEST, -5.0]) == 0b10                       # lowest() equals the starting maximum: joins, then -5 restarts
    assert find_map([LOWEST, LOWEST]) == 0b11
    assert find_map([LOWEST - 1.0, -3.0]) == 0b10                 # still lowest() after rounding
    assert find_map([-INF, -INF, -INF]) == 0b111                  # nothing joins: every haplotype
    assert find_map([-3.0, -4.0], [-INF, -INF]) == 0b11           # -inf priors: the fallback
    assert find_map([-3.0, -4.0], [-INF, 0.0]) == 0b10
    assert find_map([-3.0, -4.0, -1.0], [-INF, 0.0, -INF]) == 0b010
    assert find_map([NAN, -5.0]) == 0b10
    assert find_map([-5.0, NAN]) == 0b01
    assert find_map([NAN, NAN]) == 0b11
    assert find_map([NAN, -INF]) == 0b11
    assert find_map([-INF] * 64) == (1 << 64) - 1
    assert find_map([-INF] * 63 + [-1.0]) == 1 << 63


def test_random_cases_match_the_python_statement():
    rng = np.random.default_rng(9101)
    specials = np.array([LOWEST, -INF, NAN, 0.0, -0.0])
    for it in range(3000):
        n = int(rng.integers(1, 65))
        base = -float(rng.integers(1, 400)) * 0.2302585092994046
        v = base + rng.integers(-2, 3, n) * 0.2302585092994046
        v = np.array([up(x, int(rng.integers(0, 5))) if rng.random() < 0.3 else x for x in v])
        if rng.random() < 0.2:
            v[rng.integers(0, n, int(rng.integers(1, 3)))] = specials[rng.integers(0, len(specials))]
        pri = None
        if rng.random() < 0.5:
            pri = np.log(rng.dirichlet(np.ones(n)))
            if rng.random() < 0.3:
                pri[rng.integers(0, n, int(rng.integers(1, n + 1)))] = -INF
        assert find_map(v, pri) == py_find_map(list(v), None if pri is None else list(pri)), (it, v, pri)


def test_group_layout_is_haplotype_major():
    lnl = np.array([[-1.0, -5.0, -3.0], [-2.0, -5.0, -1.0]])
    assert find_map_group(lnl).tolist() == [0b01, 0b11, 0b10]
    assert find_map_group(lnl, [-INF, 0.0]).tolist() == [0b10, 0b10, 0b10]
