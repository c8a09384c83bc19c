"""The engine's __host__ __device__ DP cores (octopus_b200/csrc/phmm_device.cuh) executed on the CPU with the
sm_90a packed-16 (DPX) instructions emulated, checked against the oracle. This is the same source the kernels compile."""
import ctypes as C
import os

import numpy as np
import pytest

from helpers import random_alignment_case

vp = C.c_void_p


@pytest.fixture(scope="module")
def emul():
    from octopus_b200.build import build_cpu_emulation
    lib = C.CDLL(build_cpu_emulation())
    lib.emul_dp_pair.argtypes = [C.c_int, C.c_int] + [vp] * 14 + [C.c_int, vp, vp]
    lib.emul_generic.argtypes = [C.c_int, C.c_int, C.c_int] + [vp] * 7 + [C.c_int, C.c_int, C.c_int, vp, vp, vp]
    lib.emul_pair_evaluate.argtypes = [C.c_int, vp, C.c_int, vp, vp, vp, vp, vp, vp, C.c_int, C.c_int, C.c_int, C.c_int, vp, C.c_int,
                                       C.c_longlong, C.c_int, C.c_int, C.c_int, C.c_int, C.c_int, C.c_int, vp, vp]
    lib.emul_dp_band.argtypes = [C.c_int, C.c_int, C.c_int] + [vp] * 14 + [C.c_int, vp, vp]
    lib.emul_force_form.argtypes = [C.c_int]
    return lib


def P(a):
    return a.ctypes.data


def test_packed_dp_pair_matches_oracle(emul, coracle):
    rng = np.random.default_rng(11)
    for it in range(1200):
        band = int(rng.choice([8, 16, 32]))
        L = int(rng.integers(1, 200))
        nuc = int(rng.integers(0, 5))
        a = random_alignment_case(rng, band, L, qmax=93 if it % 3 == 0 else 41)
        b = random_alignment_case(rng, band, L)
        s0, s1 = C.c_int(0), C.c_int(0)
        rc = emul.emul_dp_pair(band, L, P(a["read"]), P(a["quals"]), P(b["read"]), P(b["quals"]),
                               P(a["truth"]), P(a["snv_mask"]), P(a["snv_prior"]), P(a["gap_open"]), P(a["gap_extend"]),
                               P(b["truth"]), P(b["snv_mask"]), P(b["snv_prior"]), P(b["gap_open"]), P(b["gap_extend"]),
                               nuc, C.byref(s0), C.byref(s1))
        assert rc == 0
        e = [coracle.align(band, c["truth"].tobytes(), c["read"].tobytes(), c["quals"].astype(np.int8), c["gap_open"], c["gap_extend"],
                           nuc, c["snv_mask"].tobytes(), c["snv_prior"]) for c in (a, b)]
        assert [s0.value, s1.value] == e, (band, L, nuc)


def _oracle_pair(coracle, band, nuc, cases):
    return [coracle.align(band, c["truth"].tobytes(), c["read"].tobytes(), c["quals"].astype(np.int8), c["gap_open"], c["gap_extend"],
                          nuc, c["snv_mask"].tobytes(), c["snv_prior"]) for c in cases]


def test_open_ge_extend_form_of_the_deletion_update(emul, coracle):
    """dp_pair<.., OGE> / dp_band<.., OGE>: with gap_open >= gap_extend in every column the deletion update re-uses min(m, i, d)
    and must give the oracle's score (this is the form the kernels run on every error-model penalty array); the general form on
    the same inputs agrees; and on inputs that break the precondition the kernels' own choice (the general form) is exact while
    the OGE form is allowed to differ — at least once in this sample it does, which is why the flag exists."""
    rng = np.random.default_rng(411)
    differs = 0
    for it in range(900):
        band = int(rng.choice([8, 16, 32, 64]))
        L = int(rng.integers(1, 180))
        nuc = int(rng.integers(0, 5))
        ordered = it % 3 != 0
        a = random_alignment_case(rng, band, L, open_ge_extend=ordered)
        b = random_alignment_case(rng, band, L, open_ge_extend=ordered)
        if it % 7 == 0:      # equality everywhere: the boundary of the precondition
            a["gap_extend"] = a["gap_open"].copy()
        want = _oracle_pair(coracle, band, nuc, (a, b))
        args = [P(a["read"]), P(a["quals"]), P(b["read"]), P(b["quals"]),
                P(a["truth"]), P(a["snv_mask"]), P(a["snv_prior"]), P(a["gap_open"]), P(a["gap_extend"]),
                P(b["truth"]), P(b["snv_mask"]), P(b["snv_prior"]), P(b["gap_open"]), P(b["gap_extend"])]
        for form in ((-1, 1, 0) if ordered else (-1, 0, 1)):
            emul.emul_force_form(form)
            got = []
            s0, s1 = C.c_int(0), C.c_int(0)
            if band <= 32:
                assert emul.emul_dp_pair(band, L, *args, nuc, C.byref(s0), C.byref(s1)) == 0
                got.append([s0.value, s1.value])
            assert emul.emul_dp_band(0, band, L, *args, nuc, C.byref(s0), C.byref(s1)) == 0
            got.append([s0.value, s1.value])
            assert emul.emul_dp_band(1, band, L, *args, nuc, C.byref(s0), C.byref(s1)) == 0
            got.append([s0.value, want[1]])
            if ordered or form != 1:
                assert all(g == want for g in got), (band, L, nuc, form, got, want)
            else:
                differs += any(g != want for g in got)
        emul.emul_force_form(-1)
    assert differs > 0


def test_multi_lane_band_matches_oracle(emul, coracle):
    """dp_band (the band's diagonals split over lanes, stepped in lock-step here): packed and 32-bit lanes, bands 8 .. 256."""
    rng = np.random.default_rng(412)
    for it in range(500):
        band = int(rng.choice([8, 16, 32, 64, 128, 256]))
        L = int(rng.integers(1, 260))
        nuc = int(rng.integers(0, 5))
        a = random_alignment_case(rng, band, L, open_ge_extend=(it % 2 == 0))
        b = random_alignment_case(rng, band, L, open_ge_extend=(it % 2 == 0))
        want = _oracle_pair(coracle, band, nuc, (a, b))
        args = [P(a["read"]), P(a["quals"]), P(b["read"]), P(b["quals"]),
                P(a["truth"]), P(a["snv_mask"]), P(a["snv_prior"]), P(a["gap_open"]), P(a["gap_extend"]),
                P(b["truth"]), P(b["snv_mask"]), P(b["snv_prior"]), P(b["gap_open"]), P(b["gap_extend"])]
        s0, s1 = C.c_int(0), C.c_int(0)
        assert emul.emul_dp_band(0, band, L, *args, nuc, C.byref(s0), C.byref(s1)) == 0
        assert [s0.value, s1.value] == want, (band, L, nuc)
        n = random_alignment_case(rng, band, L, read_n=True)
        wn = _oracle_pair(coracle, band, nuc, (n,))[0]
        nargs = [P(n["read"]), P(n["quals"]), P(n["read"]), P(n["quals"])] + [P(n[k]) for k in ("truth", "snv_mask", "snv_prior", "gap_open", "gap_extend")] * 2
        assert emul.emul_dp_band(1, band, L, *nargs, nuc, C.byref(s0), C.byref(s1)) == 0
        assert s0.value == wn, (band, L, nuc)


def test_packed_dp_pair_reference_kats(emul, kats):
    """The reference's KATs use the no-SNV overload with a scalar gap_extend: a mask byte that matches no base and a
    constant gap_extend array are the same recurrence."""
    for c in kats:
        if c["band"] > 32:
            continue
        L, W = len(c["read"]), len(c["truth"])
        read = np.frombuffer(c["read"].encode(), dtype=np.uint8)
        truth = np.frombuffer(c["truth"].encode(), dtype=np.uint8)
        q = np.asarray(c["quals"], dtype=np.uint8)
        go = np.asarray(c["gap_open"], dtype=np.int8)
        ge = np.full(W, c["gap_extend"], dtype=np.int8)
        mask = np.zeros(W, dtype=np.uint8)
        prior = np.full(W, 100, dtype=np.int8)
        s0, s1 = C.c_int(0), C.c_int(0)
        rc = emul.emul_dp_pair(c["band"], L, P(read), P(q), P(read), P(q), P(truth), P(mask), P(prior), P(go), P(ge),
                               P(truth), P(mask), P(prior), P(go), P(ge), c["nuc_prior"], C.byref(s0), C.byref(s1))
        assert rc == 0 and s0.value == c["score"] and s1.value == c["score"], (c["suite"], c["index"])


def test_generic_align_with_traceback_matches_oracle(emul, coracle):
    rng = np.random.default_rng(12)
    for it in range(700):
        band = int(rng.choice([8, 16, 32, 64]))
        L = int(rng.integers(1, 120))
        nuc = int(rng.integers(0, 5))
        c = random_alignment_case(rng, band, L, read_n=(it % 5 == 0))
        W = len(c["truth"])
        lhs, rhs = int(rng.integers(0, W // 2 + 1)), int(rng.integers(0, W // 2 + 1))
        q8 = c["quals"].astype(np.int8)
        fp, fs, ms = C.c_int(0), C.c_int(0), C.c_int(0)
        args = (L, P(c["read"]), P(q8), P(c["truth"]), P(c["snv_mask"]), P(c["snv_prior"]), P(c["gap_open"]), P(c["gap_extend"]), nuc)
        s = emul.emul_generic(band, 0, *args, 0, 0, None, None, None)
        st = emul.emul_generic(band, 1, *args, lhs, rhs, C.byref(fp), C.byref(fs), C.byref(ms))
        t, r, m = c["truth"].tobytes(), c["read"].tobytes(), c["snv_mask"].tobytes()
        e = coracle.align(band, t, r, q8, c["gap_open"], c["gap_extend"], nuc, m, c["snv_prior"])
        es, efp, a1, a2 = coracle.align_tb(band, t, r, q8, c["gap_open"], c["gap_extend"], nuc, m, c["snv_prior"])
        efs, ems = coracle.flank_score(W, lhs, rhs, r, q8, m, c["snv_prior"], c["gap_open"], c["gap_extend"], nuc, efp, a1, a2)
        assert (s, st, fp.value, fs.value, ms.value) == (e, es, efp, efs, ems)


def test_pair_evaluation_logic_matches_oracle(emul, coracle):
    """Candidate slots → shortcut / DP / flank discount → min → mapping-quality mix, as the populate kernels run it."""
    rng = np.random.default_rng(5)
    acgt = np.frombuffer(b"ACGT", dtype=np.uint8)
    n_short = 0
    for it in range(1500):
        band = int(rng.choice([8, 16, 32]))
        L = int(rng.integers(6, 120))
        Lh = int(rng.integers(L + 2 * band - 4, L + 2 * band + 150))
        hap = acgt[rng.integers(0, 4, Lh)].copy()
        if rng.random() < 0.1:
            hap[rng.integers(0, Lh)] = ord("N")
        mask = np.roll(hap, 1)
        prior = rng.integers(1, 126, Lh).astype(np.int8)
        go = rng.integers(3, 46, Lh).astype(np.int8)
        ge = rng.integers(1, 11, Lh).astype(np.int8)
        p0 = int(rng.integers(0, max(1, Lh - L + 1)))
        read = hap[p0:p0 + L].copy()
        if len(read) < L:
            read = np.concatenate([read, acgt[rng.integers(0, 4, L - len(read))]])
        read[read == ord("N")] = ord("A")
        for _ in range(int(rng.choice([0, 0, 1, 1, 2, 3, 5]))):
            read[rng.integers(0, L)] = acgt[rng.integers(0, 4)]
        if rng.random() < 0.2:
            i = int(rng.integers(1, L - 1)); read = np.concatenate([read[:i], read[i + 1:], acgt[rng.integers(0, 4, 1)]])
        q = rng.integers(2, 42, L).astype(np.uint8)
        npos = int(rng.integers(0, 5))
        pos = np.array([min(max(0, p0 + int(rng.integers(-20, 21))), Lh) for _ in range(npos)], dtype=np.int32)
        if npos and rng.random() < 0.5:
            pos[rng.integers(0, npos)] = p0
        orig = max(0, p0 + int(rng.choice([0, 0, 0, -3, 4, -40, 40])))
        uf = int(rng.random() < 0.6)
        lhs, rhs = int(rng.integers(0, Lh // 2)), int(rng.integers(0, Lh // 2))
        mq = int(rng.choice([0, 10, 29, 60, 255]))
        usemq, trig, dpo = int(rng.random() < 0.8), int(rng.choice([-1, 40])), int(rng.random() < 0.3)
        out, ext = C.c_double(0), C.c_int(0)
        rc = emul.emul_pair_evaluate(band, P(hap), Lh, P(mask), P(prior), P(go), P(ge), P(read), P(q), L, uf, lhs, rhs,
                                     P(pos) if npos else None, npos, orig, usemq, mq, 120, trig, dpo, 2, C.byref(out), C.byref(ext))
        st, val, e = coracle.model_evaluate(band, hap.tobytes(), read.tobytes(), q, go, ge, mask.tobytes(), prior, pos.astype(np.int64), orig,
                                            mapping_quality=mq, flanks=(lhs, rhs) if uf else None, use_mapping_quality=bool(usemq),
                                            mapq_cap=120, mapq_cap_trigger=trig, dp_only=bool(dpo))
        assert rc == st
        if rc == 0:
            assert out.value == val
        else:
            assert ext.value == e
            n_short += 1
    assert n_short > 0


def test_flank_payload_dp_matches_traceback_flank_replay(emul, coracle):
    """dp_flank32 (no back-pointers: crossing cells carried as payload) == traceback + calculate_flank_score of the oracle:
    score, in-flank penalty and in-flank read bases, for every flank geometry incl. overlapping / empty flanks."""
    emul.emul_dp_flank32.argtypes = [C.c_int, C.c_int] + [vp] * 7 + [C.c_int, C.c_int, C.c_int, vp, vp, vp]
    rng = np.random.default_rng(21)
    n_routed = 0
    for it in range(1500):
        band = int(rng.choice([8, 16, 32]))
        L = int(rng.integers(1, 160))
        nuc = int(rng.integers(0, 5))
        c = random_alignment_case(rng, band, L, read_n=(it % 3 == 0))     # reads with 'N': the fifth cap of the 32-bit kernel
        W = len(c["truth"])
        mode = it % 4
        if mode == 0:
            lhs, rhs = int(rng.integers(0, W // 2 + 1)), int(rng.integers(0, W // 2 + 1))
        elif mode == 1:
            lhs, rhs = int(rng.integers(0, W + 1)), 0
        elif mode == 2:
            lhs, rhs = 0, int(rng.integers(0, W + 1))
        else:
            lhs, rhs = int(rng.integers(0, W + 1)), int(rng.integers(0, W + 1))
        sc, fl, ms = C.c_int(0), C.c_int(0), C.c_int(0)
        rc = emul.emul_dp_flank32(band, L, P(c["read"]), P(c["quals"]), P(c["truth"]), P(c["snv_mask"]), P(c["snv_prior"]), P(c["gap_open"]),
                                  P(c["gap_extend"]), nuc, lhs, rhs, C.byref(sc), C.byref(fl), C.byref(ms))
        # rc 2: an in-flank truth 'N' the DP may have charged less than the reference's replay re-adds (flank_replay_may_differ) —
        # the kernel hands such candidates to the exact traceback path; everything else must be identical
        assert rc in (0, 2)
        n_routed += rc == 2
        q8 = c["quals"].astype(np.int8)
        t, r, m = c["truth"].tobytes(), c["read"].tobytes(), c["snv_mask"].tobytes()
        es, efp, a1, a2 = coracle.align_tb(band, t, r, q8, c["gap_open"], c["gap_extend"], nuc, m, c["snv_prior"])
        efs, ems = coracle.flank_score(W, lhs, rhs, r, q8, m, c["snv_prior"], c["gap_open"], c["gap_extend"], nuc, efp, a1, a2)
        if rc == 0:
            assert (sc.value, fl.value, ms.value) == (es, efs, ems), (band, L, lhs, rhs)
        else:
            assert (sc.value, ms.value) == (es, ems) and fl.value <= efs, (band, L, lhs, rhs)
    assert n_routed < 40                     # rare with ordinary penalties (needs an in-flank 'N' column with an SNV prior of 1)


def test_lean_flank_dp_matches_traceback_flank_replay(emul, coracle):
    """dp_flank_acc (the in-flank penalty carried as an additive payload) == score and flank score of the oracle's traceback +
    replay wherever the kernel uses it: at least two read bases certain to lie outside the flanks (then the reference's
    `read_len - mask < 2` branch cannot fire), ACGT reads."""
    emul.emul_dp_flank_acc.argtypes = [C.c_int, C.c_int] + [vp] * 7 + [C.c_int, C.c_int, C.c_int, vp, vp]
    rng = np.random.default_rng(23)
    n_used = 0
    for it in range(2500):
        band = int(rng.choice([8, 16, 32]))
        L = int(rng.integers(1, 200))
        nuc = int(rng.integers(0, 5))
        c = random_alignment_case(rng, band, L, qmax=60 if it % 5 == 0 else 41)
        W = len(c["truth"])
        mode = it % 4
        if mode == 0:
            lhs, rhs = int(rng.integers(0, W // 3 + 1)), int(rng.integers(0, W // 3 + 1))
        elif mode == 1:
            lhs, rhs = int(rng.integers(0, W // 2 + 1)), 0
        elif mode == 2:
            lhs, rhs = 0, int(rng.integers(0, W // 2 + 1))
        else:
            lhs, rhs = int(rng.integers(0, W + 1)), int(rng.integers(0, W + 1))
        sc, fl = C.c_int(0), C.c_int(0)
        rc = emul.emul_dp_flank_acc(band, L, P(c["read"]), P(c["quals"]), P(c["truth"]), P(c["snv_mask"]), P(c["snv_prior"]), P(c["gap_open"]),
                                    P(c["gap_extend"]), nuc, lhs, rhs, C.byref(sc), C.byref(fl))
        assert rc in (0, 1, 2)
        if rc != 0:
            continue
        n_used += 1
        q8 = c["quals"].astype(np.int8)
        t, r, m = c["truth"].tobytes(), c["read"].tobytes(), c["snv_mask"].tobytes()
        es, efp, a1, a2 = coracle.align_tb(band, t, r, q8, c["gap_open"], c["gap_extend"], nuc, m, c["snv_prior"])
        efs, ems = coracle.flank_score(W, lhs, rhs, r, q8, m, c["snv_prior"], c["gap_open"], c["gap_extend"], nuc, efp, a1, a2)
        assert L - ems >= 2, (band, L, lhs, rhs, ems)          # the guarantee the kernel relies on
        assert (sc.value, fl.value) == (es, efs), (band, L, lhs, rhs)
    assert n_used > 800


def test_register_traceback_matches_oracle(emul, coracle):
    """dp_traceback_forward + traceback_walk (register-band forward pass writing one back-pointer word per cell, backward walk) ==
    the oracle's traceback: score, first_pos, both alignment strings, flank score and in-flank read bases; reads with 'N' included."""
    emul.emul_traceback.argtypes = [C.c_int, C.c_int] + [vp] * 7 + [C.c_int, C.c_int, C.c_int] + [vp] * 6
    rng = np.random.default_rng(29)
    for it in range(1500):
        band = int(rng.choice([8, 16, 32]))
        L = int(rng.integers(1, 180))
        nuc = int(rng.integers(0, 5))
        c = random_alignment_case(rng, band, L, read_n=(it % 4 == 0))
        W = len(c["truth"])
        lhs, rhs = (int(rng.integers(0, W + 1)), int(rng.integers(0, W + 1))) if it % 2 else (0, 0)
        sc, fp, fl, ms = C.c_int(0), C.c_int(0), C.c_int(0), C.c_int(0)
        n = 2 * (L + band) + 8
        a1, a2 = C.create_string_buffer(n), C.create_string_buffer(n)
        rc = emul.emul_traceback(band, L, P(c["read"]), P(c["quals"]), P(c["truth"]), P(c["snv_mask"]), P(c["snv_prior"]), P(c["gap_open"]),
                                 P(c["gap_extend"]), nuc, lhs, rhs, C.byref(sc), C.byref(fp), C.byref(fl), C.byref(ms), a1, a2)
        assert rc == 0
        q8 = c["quals"].astype(np.int8)
        t, r, m = c["truth"].tobytes(), c["read"].tobytes(), c["snv_mask"].tobytes()
        es, efp, e1, e2 = coracle.align_tb(band, t, r, q8, c["gap_open"], c["gap_extend"], nuc, m, c["snv_prior"])
        efs, ems = coracle.flank_score(W, lhs, rhs, r, q8, m, c["snv_prior"], c["gap_open"], c["gap_extend"], nuc, efp, e1, e2)
        assert (sc.value, fp.value, a1.value.decode(), a2.value.decode()) == (es, efp, e1, e2), (band, L)
        assert (fl.value, ms.value) == (efs, ems), (band, L, lhs, rhs)


def _fb_case(rng, band, L, it, qmax=41, ordered=False):
    c = random_alignment_case(rng, band, L, qmax=qmax, open_ge_extend=ordered)
    W = len(c["truth"])
    mode = it % 5
    if mode == 0:
        lhs, rhs = int(rng.integers(0, W // 2 + 1)), int(rng.integers(0, W // 2 + 1))
    elif mode == 1:
        lhs, rhs = int(rng.integers(1, W)), 0
    elif mode == 2:
        lhs, rhs = 0, int(rng.integers(1, W))
    elif mode == 3:
        lhs, rhs = int(rng.integers(0, W + 1)), int(rng.integers(0, W + 1))
    else:           # boundaries inside the first / last 2B columns (start cells beyond xl, ends before xr)
        lhs, rhs = int(rng.integers(0, 2 * band + 2)), int(rng.integers(0, 2 * band + 2))
    if W - rhs <= lhs or (lhs == 0 and rhs == 0):
        lhs, rhs = max(1, W // 4), 0
    return c, lhs, rhs


def test_forward_backward_flank_dp_matches_traceback_flank_replay(emul, coracle):
    """dp_flank_fb (packed forward pass to the flank boundary + packed backward pass from the window end; the crossing cell is the
    argmin of F + B): score, in-flank penalty and in-flank read bases equal the oracle's traceback + calculate_flank_score whenever
    the core does not report a tie — and ties (co-optimal paths that cross a boundary at different cells, which the kernel hands
    to the labelled DP) stay rare. Two alignments per call with independent flank geometries, as the kernel packs them."""
    emul.emul_dp_flank_fb.argtypes = [C.c_int, C.c_int] + [vp] * 14 + [C.c_int] * 5 + [vp, vp]
    rng = np.random.default_rng(29)
    n_used = n_tie = n_quirk = 0
    for it in range(1800):
        band = int(rng.choice([8, 16, 32], p=[0.4, 0.45, 0.15]))
        L = int(rng.integers(2 * band, 2 * band + 150))
        nuc = int(rng.integers(0, 5))
        same_geometry = it % 3 == 0
        ordered = it % 2 == 0          # gap_open >= gap_extend everywhere: the cores take the shorter (OGE) deletion update
        a, la, ra = _fb_case(rng, band, L, it, qmax=60 if it % 7 == 0 else 41, ordered=ordered)
        b, lb, rb = _fb_case(rng, band, L, it + 1, ordered=ordered)
        if same_geometry:
            lb, rb = la, ra
        o0, o1 = (C.c_int * 4)(), (C.c_int * 4)()
        emul.emul_force_form(0 if it % 4 == 0 else -1)     # the general form is valid for any penalties
        rc = emul.emul_dp_flank_fb(band, L, P(a["read"]), P(a["quals"]), P(b["read"]), P(b["quals"]),
                                   P(a["truth"]), P(a["snv_mask"]), P(a["snv_prior"]), P(a["gap_open"]), P(a["gap_extend"]),
                                   P(b["truth"]), P(b["snv_mask"]), P(b["snv_prior"]), P(b["gap_open"]), P(b["gap_extend"]),
                                   nuc, la, ra, lb, rb, o0, o1)
        emul.emul_force_form(-1)
        assert rc == 0, (rc, band, L, la, ra, lb, rb)
        for c, lhs, rhs, o in ((a, la, ra, o0), (b, lb, rb, o1)):
            W = len(c["truth"])
            q8 = c["quals"].astype(np.int8)
            t, r, m = c["truth"].tobytes(), c["read"].tobytes(), c["snv_mask"].tobytes()
            es, efp, a1, a2 = coracle.align_tb(band, t, r, q8, c["gap_open"], c["gap_extend"], nuc, m, c["snv_prior"])
            efs, ems = coracle.flank_score(W, lhs, rhs, r, q8, m, c["snv_prior"], c["gap_open"], c["gap_extend"], nuc, efp, a1, a2)
            n_used += 1
            assert o[0] == es, (band, L, lhs, rhs, o[0], es)
            if o[3]:
                n_tie += 1
                continue
            # the truth-'N' replay quirk (flank_replay_may_differ): the kernel sends those candidates to the traceback path
            has_n_prior_below_2 = bool(((c["truth"] == ord("N")) & (c["snv_prior"] < 2)).any())
            if (o[1], o[2]) != (efs, ems) and has_n_prior_below_2:
                n_quirk += 1
                assert o[2] == ems and o[1] <= efs
                continue
            assert (o[1], o[2]) == (efs, ems), (band, L, lhs, rhs, tuple(o), (es, efs, ems))
    assert n_used == 3600 and n_tie < 0.04 * n_used and n_quirk < 20, (n_used, n_tie, n_quirk)


def test_replay_quirk_test_from_prefix_counts_equals_the_column_scan(emul):
    """flank_replay_may_differ_pre (four loads of per-haplotype prefix counts of 'N'-like table columns) == flank_replay_may_differ
    (scan of the window's flank columns) for every window placement and flank geometry, N-rich haplotypes with SNV priors 0 / 1 / 2."""
    emul.emul_replay_prefix_check.argtypes = [C.c_int] + [vp] * 5 + [C.c_int] + [vp] * 5
    rng = np.random.default_rng(31)
    n_true = 0
    for it in range(60):
        hap_len = int(rng.integers(40, 400))
        truth = np.frombuffer(b"ACGT", np.uint8)[rng.integers(0, 4, hap_len)].copy()
        truth[rng.random(hap_len) < (0.0 if it % 4 == 0 else 0.03)] = ord("N")
        mask = np.frombuffer(b"ACGTN", np.uint8)[rng.integers(0, 5, hap_len)].copy()
        prior = rng.choice([0, 1, 2, 3, 30, 125], hap_len).astype(np.int8)
        go = rng.integers(3, 46, hap_len).astype(np.int8); ge = rng.integers(1, 11, hap_len).astype(np.int8)
        nq = 400
        W = rng.integers(1, hap_len + 1, nq).astype(np.int32)
        a = (rng.random(nq) * (hap_len - W + 1)).astype(np.int32)
        lhs = rng.integers(-5, W + 10).astype(np.int32); rhs = rng.integers(-5, W + 10).astype(np.int32)
        lhs[::3] = 0; rhs[1::3] = 0
        lowq = rng.integers(0, 2, nq).astype(np.int32)
        # the kernels only pass non-negative flank sizes (window_flanks)
        lhs = np.maximum(lhs, 0); rhs = np.maximum(rhs, 0)
        bad = emul.emul_replay_prefix_check(hap_len, P(truth), P(mask), P(prior), P(go), P(ge), nq, P(a), P(W), P(lhs), P(rhs), P(lowq))
        assert bad == 0, (it, bad)
