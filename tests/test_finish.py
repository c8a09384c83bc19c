"""The FP64 finish (mapq_terms / finish_mixed / finish_likelihood in phmm_device.cuh, the code k_epilogue, k_mapq_terms, direct
mode, k_list_slots and k_align_reads run), host-compiled from the same source, against the exact mixed value (tests/exact.py)
within the forward-error bound of the reference's formula: every mapping quality, the cap / trigger rules, penalties 0..28 000."""
import ctypes as C

import numpy as np
import pytest

from exact import C as C_LN
from exact import EPS, LOWEST, LOWEST_S, assert_mix_within_bound, effective_mapq, penalties

vp = C.c_void_p

# (cap, trigger): none; a trigger below the cap; equal and above (both dropped); a cap of 0
CAPS = [(120, None), (60, 40), (60, 60), (50, 200), (120, 0)]
SCORES = np.unique(np.concatenate([np.arange(0, 201), np.arange(200, 2000, 13), np.arange(2000, 28001, 311), [27648, 27649, 13312, 13313]]))


@pytest.fixture(scope="module")
def emul():
    from octopus_b200.build import build_cpu_emulation
    lib = C.CDLL(build_cpu_emulation())
    lib.emul_mapq_terms.argtypes = [C.c_int, C.c_int, C.c_int, vp, vp]
    for f in (lib.emul_finish_mixed, lib.emul_finish_likelihood):
        f.argtypes = [C.c_int, vp, vp, C.c_int, C.c_int, C.c_int, vp]
    return lib


def _finish(emul, fn, s, mapq, use_mq, cap, trig):
    s = np.ascontiguousarray(np.where(s == LOWEST_S, np.iinfo(np.int32).min, s), dtype=np.int32)
    m = np.ascontiguousarray(np.broadcast_to(mapq, s.shape), dtype=np.int32)
    out = np.empty(s.shape, dtype=np.float64)
    getattr(emul, fn)(len(s), s.ctypes.data, m.ctypes.data, int(use_mq), cap, -1 if trig is None else trig, out.ctypes.data)
    return out


@pytest.mark.parametrize("cap,trig", CAPS)
def test_finish_source_within_bound_of_exact_mix(emul, cap, trig):
    s = np.concatenate([SCORES, [LOWEST_S]]).astype(np.int64)
    worst = 0.0
    for mq in range(256):
        me = int(effective_mapq([mq], cap, trig)[0])
        a = _finish(emul, "emul_finish_mixed", s, mq, True, cap, trig)
        b = _finish(emul, "emul_finish_likelihood", s, mq, True, cap, trig)
        assert np.array_equal(a.view(np.int64), b.view(np.int64)), mq          # the tabulated and the inline finish are one function
        worst = max(worst, assert_mix_within_bound(a, s, me, "cap %d trigger %s mapq %d" % (cap, trig, mq)))
    print("finish source vs exact mix, cap %d trigger %s: largest error %.3f bound units" % (cap, trig, worst))


def test_finish_without_mapping_quality_is_the_scaled_penalty(emul):
    s = np.concatenate([SCORES, [LOWEST_S]]).astype(np.int64)
    got = _finish(emul, "emul_finish_likelihood", s, 60, False, 120, None)
    assert got[-1] == LOWEST and got[0] == 0.0
    assert np.array_equal(penalties(got), s)            # bit for bit -ln10/10 * s


def test_mapq_terms_and_the_cap_rule(emul):
    """The read's share: ln p of the effective mapping quality exactly (the trigger rule as the reference applies it), and
    ln(1 - p) close to exact."""
    from decimal import Decimal, localcontext
    lm, lp = C.c_double(), C.c_double()
    for cap, trig in CAPS:
        for mq in range(256):
            emul.emul_mapq_terms(mq, cap, -1 if trig is None else trig, C.byref(lm), C.byref(lp))
            me = int(effective_mapq([mq], cap, trig)[0])
            assert lp.value == -C_LN * me, (cap, trig, mq)
            if me:
                with localcontext() as ctx:
                    ctx.prec = 40
                    want = float((1 - (Decimal(-me) * Decimal(10).ln() / 10).exp()).ln())
                # exp(ln p) carries a few ulp of p and 1 - p its own rounding: ln(1 - p) inherits both over 1 - p
                p = 10.0 ** (-me / 10)
                assert abs(lm.value - want) <= 4 * EPS * ((1 + C_LN * me) * p + 1) / (1 - p), (cap, trig, mq, lm.value, want)
    assert effective_mapq([10, 39, 40, 255], 60, 40).tolist() == [10, 39, 60, 60]
    assert effective_mapq([10, 60, 255], 60, 60).tolist() == [10, 60, 255]
    assert effective_mapq([10, 255], 50, 200).tolist() == [10, 255]
