"""dp_pair's first and last 2B columns (the prologue, entered at the column's first cell, and the epilogue, left after the
row-L cell) on the CPU emulation of the kernels' own source, against the oracle: read lengths around 2B, alignments whose
optimum lies in those columns, both deletion-update forms, and scores near the 16-bit lanes' bound."""
import ctypes as C

import numpy as np
import pytest

from helpers import ACGT

vp = C.c_void_p


@pytest.fixture(scope="module")
def emul():
    from octopus_b200.build import build_cpu_emulation
    lib = C.CDLL(build_cpu_emulation())
    lib.emul_dp_pair.argtypes = [C.c_int, C.c_int] + [vp] * 14 + [C.c_int, vp, vp]
    lib.emul_force_form.argtypes = [C.c_int]
    return lib


def P(a):
    return a.ctypes.data


def _window(rng, band, L, qmax):
    W = L + 2 * band - 1
    go = rng.integers(3, 46, W).astype(np.int8)
    return dict(truth=ACGT[rng.integers(0, 4, W)].copy(),
                quals=rng.integers(max(2, qmax - 40), qmax + 1, L).astype(np.uint8),
                gap_open=go, gap_extend=np.minimum(rng.integers(1, 11, W), go).astype(np.int8),
                snv_mask=np.frombuffer(b"ACGTN", dtype=np.uint8)[rng.integers(0, 5, W)].copy(),
                snv_prior=rng.integers(1, 126, W).astype(np.int8))


def _case(rng, band, L, kind, qmax=41):
    """kind: 'start' / 'end' (the read copies the window from its first / last possible offset), 'ins_start' / 'del_start' /
    'ins_end' / 'del_end' (the same with an indel of 1-3 bases within 2B bases of that end), 'random' (no alignment)."""
    c = _window(rng, band, L, qmax)
    W = len(c["truth"])
    if kind == "random":
        c["read"] = ACGT[rng.integers(0, 4, L)].copy()
        return c
    n = min(int(rng.integers(1, 4)), L)
    pos = int(rng.integers(0, min(2 * band, L)))
    at_end = kind.endswith("end")
    if kind.startswith("del"):
        src = c["truth"][:L + n] if not at_end else c["truth"][W - L - n:]
        cut = pos if not at_end else L + n - pos - n
        read = np.concatenate([src[:cut], src[cut + n:]])
    elif kind.startswith("ins"):
        src = c["truth"][:L - n] if not at_end else c["truth"][W - L + n:]
        cut = pos if not at_end else max(L - n - pos, 0)
        read = np.concatenate([src[:cut], ACGT[rng.integers(0, 4, n)], src[cut:]])
    else:
        read = c["truth"][:L] if not at_end else c["truth"][W - L:]
    c["read"] = np.ascontiguousarray(read[:L], dtype=np.uint8)
    assert len(c["read"]) == L
    return c


def _run(emul, coracle, band, L, nuc, a, b):
    want = [coracle.align(band, c["truth"].tobytes(), c["read"].tobytes(), c["quals"].astype(np.int8), c["gap_open"],
                          c["gap_extend"], nuc, c["snv_mask"].tobytes(), c["snv_prior"]) for c in (a, b)]
    args = [P(a["read"]), P(a["quals"]), P(b["read"]), P(b["quals"]),
            P(a["truth"]), P(a["snv_mask"]), P(a["snv_prior"]), P(a["gap_open"]), P(a["gap_extend"]),
            P(b["truth"]), P(b["snv_mask"]), P(b["snv_prior"]), P(b["gap_open"]), P(b["gap_extend"])]
    for form in (0, 1):
        emul.emul_force_form(form)
        s0, s1 = C.c_int(0), C.c_int(0)
        try:
            assert emul.emul_dp_pair(band, L, *args, nuc, C.byref(s0), C.byref(s1)) == 0
        finally:
            emul.emul_force_form(-1)
        assert [s0.value, s1.value] == want, (band, L, nuc, form)
    return want


KINDS = ["start", "end", "ins_start", "del_start", "ins_end", "del_end", "random"]


@pytest.mark.parametrize("band", [8, 16])
def test_ramp_columns_match_oracle(emul, coracle, band):
    rng = np.random.default_rng(band)
    K = 2 * band
    for L in list(range(1, K + 9)) + [150]:          # L < 2B-1: the short-read columns, L >= 2B-1: prologue and epilogue
        for i, kind in enumerate(KINDS):
            for rep in range(3):
                nuc = int(rng.integers(0, 5))
                a = _case(rng, band, L, kind)
                b = _case(rng, band, L, KINDS[(i + rep + 1) % len(KINDS)])
                _run(emul, coracle, band, L, nuc, a, b)


@pytest.mark.parametrize("band", [8, 16])
def test_ramp_columns_near_the_16_bit_bound(emul, coracle, band):
    """Quality 127 on reads that match no base of the window, with gaps dearer than a mismatch: the score is the quality sum.
    At L = 217 that is 27 559, just below kMaxScore16 (27 648), the quality sum below which the engine sends a read to the 16-bit lanes,
    and within 1 113 of their +inf (0x7000)."""
    rng = np.random.default_rng(100 + band)
    top = 0
    for L in (2 * band - 1, 2 * band, 2 * band + 5, 150, 217):
        assert 127 * L < 0x7000 - 1024
        for kind in ("start", "end", "del_end"):
            a = _case(rng, band, L, kind, qmax=127)
            a["truth"] = ACGT[rng.integers(0, 2, len(a["truth"]))].copy()      # A / C only
            a["read"] = ACGT[rng.integers(2, 4, L)].copy()                      # G / T only
            a["quals"][:] = 127
            a["snv_mask"][:] = ord("N")
            a["gap_open"][:] = 127
            a["gap_extend"][:] = 127
            b = _case(rng, band, L, kind, qmax=127)
            got = _run(emul, coracle, band, L, int(rng.integers(0, 5)), a, b)
            assert got[0] == 127 * L
            top = max(top, max(got))
    assert top == 127 * 217
