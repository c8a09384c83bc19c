"""ReadRealigner::realign on the GPU: the uncapped pair k-mer mapper (phmm_map_pairs) against the reference's map_query_to_target
with max_mapping_positions = the haplotype length, and phmm_realign_reads against the reference's composition
(read_realigner.cpp:128-129): that mapper, then HaplotypeLikelihoodModel::align at its positions. Where oracle/_ref was never built,
the C oracle's restatements of both stand in (tests/test_realign_oracle.py pins its mapper to the reference's)."""
import os
import subprocess
import tempfile

import numpy as np
import pytest

from exact import assert_mix_within_bound, assert_same_penalties, effective_mapq, penalties
from helpers import ACGT, random_region

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def oracle_map(refhmm, coracle, read, hap):
    cap = max(1, len(hap))
    if refhmm is not None:
        return refhmm.kmer_map(read, hap, cap)
    return list(coracle.kmer_map(read.tobytes().decode("latin1"), hap.tobytes().decode("latin1"), cap))


def oracle_align(refhmm, coracle, band_req, haps, reads, r, h, positions, flanks):
    """HaplotypeLikelihoodModel::align with mapping quality off. Returns (status, mapping_position, likelihood, cigar, extension)."""
    hp = haps.hap(h)
    b, q = reads.read(r)
    rev = bool(reads.reverse[r])
    hb = int(haps.begin[h]) if haps.begin is not None else 0
    if refhmm is not None:
        return refhmm.model_align(band_req, hp["seq"], b, q, hp["gap_open"], hp["gap_extend"], hp["snv_mask_fwd"], hp["snv_prior_fwd"],
                                  hp["snv_mask_rev"], hp["snv_prior_rev"], positions, hap_begin=hb, read_begin=int(reads.begin[r]),
                                  mapping_quality=int(reads.mapq[r]), reverse=rev, flanks=flanks, use_mapping_quality=False)
    band = next(x for x in (8, 16, 32, 64, 128, 256) if band_req <= x)
    return coracle.model_align(band, hp["seq"].tobytes(), b.tobytes(), q, hp["gap_open"], hp["gap_extend"],
                               hp["snv_mask_rev" if rev else "snv_mask_fwd"].tobytes(), hp["snv_prior_rev" if rev else "snv_prior_fwd"],
                               positions, int(reads.begin[r]) - hb, mapping_quality=int(reads.mapq[r]), flanks=flanks, use_mapping_quality=False)


def pack(seqs, reads, rng, begins=None, mapq=None, reverse=None):
    """Haplotype / read blocks with random penalties. seqs, reads: lists of uint8 arrays."""
    from octopus_b200.batch import pack_haplotypes, pack_reads
    haps = pack_haplotypes(seqs, [np.roll(s, 1) for s in seqs], [rng.integers(1, 126, len(s)).astype(np.int8) for s in seqs],
                           [np.roll(s, -1) for s in seqs], [rng.integers(1, 126, len(s)).astype(np.int8) for s in seqs],
                           [rng.integers(3, 46, len(s)).astype(np.int8) for s in seqs], [rng.integers(1, 11, len(s)).astype(np.int8) for s in seqs],
                           begin=np.zeros(len(seqs), np.int64))
    n = len(reads)
    rb = pack_reads(reads, [rng.integers(2, 42, len(b)).astype(np.uint8) for b in reads],
                    mapq=rng.choice([0, 10, 29, 60, 255], n).astype(np.uint8) if mapq is None else mapq,
                    reverse=(rng.random(n) < 0.5).astype(np.uint8) if reverse is None else reverse,
                    begin=np.zeros(n, np.int64) if begins is None else np.asarray(begins, np.int64))
    return haps, rb


def tandem(rng, length, unit_len=None):
    unit = ACGT[rng.integers(0, 4, unit_len or int(rng.integers(1, 7)))]
    return np.tile(unit, length // len(unit) + 1)[:length].copy()


def reads_from(rng, seqs, n, lengths, n_rate=0.0):
    out, begins = [], []
    for _ in range(n):
        s = seqs[int(rng.integers(0, len(seqs)))]
        L = int(rng.choice(lengths))
        p = int(rng.integers(0, max(1, len(s) - L + 1)))
        b = s[p:p + L].copy()
        if len(b) < L:
            b = np.concatenate([b, ACGT[rng.integers(0, 4, L - len(b))]])
        for _ in range(int(rng.integers(0, 3))):
            b[rng.integers(0, L)] = ACGT[rng.integers(0, 4)]
        if rng.random() < n_rate:
            b[rng.integers(0, L, int(rng.integers(1, 3)))] = ord("N")
        out.append(b)
        begins.append(p)
    return out, begins


def check_map(engine, refhmm, coracle, haps, reads, pairs, what):
    off, pos = engine.map_pairs(haps, reads, pairs)
    assert off[0] == 0 and len(off) == len(pairs) + 1 and len(pos) == off[-1], what
    counts = []
    for j, (r, h) in enumerate(pairs):
        want = oracle_map(refhmm, coracle, reads.read(int(r))[0], haps.hap(int(h))["seq"])
        got = pos[off[j]:off[j + 1]].tolist()
        assert got == want, (what, j, int(r), int(h), got[:12], want[:12], len(got), len(want))
        counts.append(len(want))
    return np.array(counts)


def all_pairs(R, H):
    return np.array([(r, h) for r in range(R) for h in range(H)], dtype=np.int32)


def test_map_pairs_random_and_repeat_rich(engine, refhmm, coracle):
    rng = np.random.default_rng(8101)
    haps, reads = random_region(rng, 16, n_haps=6, n_reads=60, hap_len=420, read_len_choices=[3, 5, 6, 40, 100, 150], read_n_rate=0.2)
    check_map(engine, refhmm, coracle, haps, reads, all_pairs(reads.n, haps.n), "random")
    # repeat-rich: tandem repeats and homopolymers (hundreds of tied diagonals), a haplotype and reads shorter than a k-mer, 'N's
    seqs = [tandem(rng, 600, 2), tandem(rng, 500, 3), np.full(520, ord("A"), np.uint8), tandem(rng, 450),
            ACGT[rng.integers(0, 4, 480)].copy(), ACGT[rng.integers(0, 4, 5)].copy(), ACGT[rng.integers(0, 4, 6)].copy()]
    seqs[4][100:260] = tandem(rng, 160, 4)
    rb, begins = reads_from(rng, seqs[:5], 50, [4, 30, 100, 150], n_rate=0.15)
    haps2, reads2 = pack(seqs, rb, rng, begins)
    n = check_map(engine, refhmm, coracle, haps2, reads2, all_pairs(reads2.n, haps2.n), "repeats")
    assert (n > 10).sum() > 30 and (n > 100).sum() > 20, (int((n > 10).sum()), int((n > 100).sum()))


def test_map_pairs_long_reads_and_tiles(engine, refhmm, coracle):
    rng = np.random.default_rng(8102)
    # reads over 260 bases: 16-bit vote counts; haplotypes over 2 053 bases: tiles of 2 048 diagonals, ties across tiles
    for hap_lens, read_lens in (((900, 700), (150, 300, 420)), ((2100, 2600, 5000), (150, 280)), ((2054, 4500), (60, 150))):
        seqs = [ACGT[rng.integers(0, 4, L)].copy() for L in hap_lens]
        seqs.append(tandem(rng, max(hap_lens), 2))
        seqs[0][-400:] = tandem(rng, 400, 3)
        rb, begins = reads_from(rng, seqs, 40, read_lens, n_rate=0.1)
        haps, reads = pack(seqs, rb, rng, begins)
        n = check_map(engine, refhmm, coracle, haps, reads, all_pairs(reads.n, haps.n), (hap_lens, read_lens))
        assert (n > 10).any()


def test_map_pairs_haplotypes_near_the_16_bit_limit(engine, refhmm, coracle):
    rng = np.random.default_rng(8103)
    big = ACGT[rng.integers(0, 4, 65535)].copy()
    big[30000:31000] = tandem(rng, 1000, 2)
    seqs = [big, tandem(rng, 65000, 3), big[:65534].copy()]
    rb, begins = reads_from(rng, [big], 40, [150, 300])
    rb += [tandem(rng, 120, 2), tandem(rng, 90, 3)]
    haps, reads = pack(seqs, rb, rng, begins + [0, 0])
    pairs = all_pairs(reads.n, haps.n)
    n = check_map(engine, refhmm, coracle, haps, reads, pairs, "65535")
    assert (n > 100).any()


def test_map_pairs_argument_checks(engine):
    from octopus_b200 import PhmmError
    rng = np.random.default_rng(8104)
    haps, reads = random_region(rng, 8, n_haps=2, n_reads=4, hap_len=200, read_len_choices=[50])
    for bad in ([[4, 0]], [[0, 2]], [[-1, 0]], [[0, -1]]):
        with pytest.raises(PhmmError) as ei:
            engine.map_pairs(haps, reads, np.array([[0, 0]] + bad, np.int32))
        assert ei.value.code == -1 and "out of range" in str(ei.value)
        with pytest.raises(PhmmError) as ei:
            engine.map_pairs(haps.to_device(), reads.to_device(), np.array([[0, 0]] + bad, np.int32))
        assert ei.value.code == -1 and "out of range" in str(ei.value)
        with pytest.raises(PhmmError) as ei:
            engine.realign_reads(_cfg(8, False), haps.to_device(), reads.to_device(), np.array([[0, 0]] + bad, np.int32))
        assert ei.value.code == -1 and "out of range" in str(ei.value)
    seqs = [ACGT[rng.integers(0, 4, 65536)].copy()]
    haps2, reads2 = pack(seqs, [seqs[0][100:250].copy()], rng)
    for call in (lambda: engine.map_pairs(haps2, reads2, [[0, 0]]), lambda: engine.realign_reads(_cfg(8, False), haps2, reads2, [[0, 0]])):
        with pytest.raises(PhmmError) as ei:
            call()
        assert ei.value.code == -1 and "65535" in str(ei.value)
    off, pos = engine.map_pairs(haps, reads, np.zeros((0, 2), np.int32))
    assert off.tolist() == [0] and len(pos) == 0
    mp, lk, cig, st = engine.realign_reads(_cfg(8, True), haps, reads, np.zeros((0, 2), np.int32))
    assert len(mp) == len(lk) == len(cig) == len(st) == 0


def _cfg(band_req, use_mq, trig=None, map_positions=True):
    from octopus_b200 import HaplotypeLikelihoodModel
    return HaplotypeLikelihoodModel.Config(max_indel_error=band_req, use_mapping_quality=use_mq, mapping_quality_cap_trigger=trig,
                                           map_positions=map_positions)


def realign_legs(engine, refhmm, coracle, band_req, haps, reads, pairs, flanks, trig=None, what=""):
    """phmm_realign_reads in both legs against the reference composition: mapping position and CIGAR equal, the likelihood bit-equal
    with mapping quality off and within 4 eps (1 + c|s| + c mapq) of the exact mix with it on; SHORT_HAP with the reference's
    extension. Returns the number of pairs with more than ten mapped positions."""
    res = {mq: engine.realign_reads(_cfg(band_req, mq, trig), haps, reads, pairs, flanks) for mq in (False, True)}
    lk_exact, lk_mixed, mq_eff = [], [], []
    many = n_short = 0
    for j, (r, h) in enumerate(pairs):
        r, h = int(r), int(h)
        positions = oracle_map(refhmm, coracle, reads.read(r)[0], haps.hap(h)["seq"])
        many += len(positions) > 10
        wst, wmp, wlk, wcig, wext = oracle_align(refhmm, coracle, band_req, haps, reads, r, h, positions, flanks)
        for mq in (False, True):
            mp, lk, cig, st = res[mq]
            if wst == 1:
                assert (st[j] & 0xFFFF) == 2 and (st[j] >> 16) == wext, (what, j, int(st[j]), wext)
                continue
            assert wst == 0 and st[j] == 0, (what, j, wst, int(st[j]))
            assert mp[j] == wmp and cig[j] == wcig, (what, j, mq, int(mp[j]), wmp, cig[j], wcig, positions[:12])
        n_short += wst == 1
        if wst == 0:
            lk_exact.append((res[False][1][j], wlk))
            lk_mixed.append(res[True][1][j])
            mq_eff.append(int(effective_mapq([reads.mapq[r]], 120, trig)[0]))
    got, want = np.array(lk_exact).T
    assert_same_penalties(got, want, None, np.zeros(len(got), np.int32), what)
    assert_mix_within_bound(np.array(lk_mixed), penalties(want), np.array(mq_eff), what)
    return many, n_short


@pytest.mark.parametrize("band_req", [8, 16, 32, 64])
def test_realign_reads_equals_reference_composition(engine, refhmm, coracle, band_req):
    rng = np.random.default_rng(8200 + band_req)
    many = 0
    for trial in range(3):
        flanks = (int(rng.integers(0, 80)), int(rng.integers(0, 80))) if trial % 2 else None
        trig = 40 if trial == 2 else None
        haps, reads = random_region(rng, band_req, n_haps=4, n_reads=40, hap_len=360, read_len_choices=[40, 76, 120], read_n_rate=0.1,
                                    edge_reads=(trial == 0))
        pairs = np.array([(r, int(rng.integers(0, haps.n))) for r in range(reads.n)], np.int32)
        realign_legs(engine, refhmm, coracle, band_req, haps, reads, pairs, flanks, trig, (band_req, trial))
        # repeat-rich haplotypes: reads tie on many diagonals, where a mapper capped at ten would choose differently
        L = 260 + 2 * band_req
        seqs = [ACGT[rng.integers(0, 4, L + 80)].copy() for _ in range(2)]
        seqs[0][60:60 + L - 100] = tandem(rng, L - 100, 2)
        seqs[1][40:40 + L - 120] = np.full(L - 120, ord("T"), np.uint8)
        rb, begins = reads_from(rng, seqs, 30, [40, 60, 100], n_rate=0.05)
        haps2, reads2 = pack(seqs, rb, rng, begins)
        pairs2 = all_pairs(reads2.n, haps2.n)
        m, _ = realign_legs(engine, refhmm, coracle, band_req, haps2, reads2, pairs2, flanks, trig, (band_req, trial, "repeats"))
        many += m
    assert many > 20


def test_realign_reads_short_haplotypes(engine, refhmm, coracle):
    rng = np.random.default_rng(8301)
    total_short = 0
    for band_req in (8, 16):
        base = ACGT[rng.integers(0, 4, 300)].copy()
        seqs = [base[20:80].copy(), base[0:64].copy(), base[:300].copy()]      # the first two: shorter than a read + 2 bands
        rb = [base[30:80].copy(), base[25:75].copy(), base[100:150].copy()]
        haps, reads = pack(seqs, rb, rng, [30, 25, 100])
        pairs = all_pairs(reads.n, haps.n)
        total_short += realign_legs(engine, refhmm, coracle, band_req, haps, reads, pairs, None, None, ("short", band_req))[1]
    assert total_short >= 4


def _c2_pairs(rng, n_reads=6000, n_haps=24):
    from octopus_b200 import synth
    haps, reads, band = synth.make_batch("C2", n_reads=n_reads, n_haps=n_haps)
    pairs = np.stack([np.arange(reads.n, dtype=np.int32), rng.integers(0, haps.n, reads.n).astype(np.int32)], axis=1)
    return haps, reads, band, pairs


def assert_same_alignments(got, want, what):
    """(mapping_position, likelihood, cigars, status) equal bit for bit."""
    assert np.array_equal(got[0], want[0]), what
    assert np.array_equal(got[1].view(np.int64), want[1].view(np.int64)), what
    assert got[2] == want[2], what
    assert np.array_equal(got[3], want[3]), what


def test_realign_reads_equals_align_reads_on_mapped_positions(engine):
    rng = np.random.default_rng(8401)
    haps, reads, band, pairs = _c2_pairs(rng)
    off, pos = engine.map_pairs(haps, reads, pairs)
    for flanks in (None, (30, 40)):
        for mq in (False, True):
            cfg = _cfg(band, mq)
            assert_same_alignments(engine.realign_reads(cfg, haps, reads, pairs, flanks),
                                   engine.align_reads(cfg, haps, reads, pairs, (off, pos), flanks), (flanks, mq))
            # map_positions = 0: the original position only, as align_reads without positions
            cfg0 = _cfg(band, mq, map_positions=False)
            assert_same_alignments(engine.realign_reads(cfg0, haps, reads, pairs, flanks),
                                   engine.align_reads(cfg0, haps, reads, pairs, None, flanks), (flanks, mq, "original only"))


def test_device_resident_inputs_equal_host_inputs(engine):
    import torch
    rng = np.random.default_rng(8501)
    haps, reads, band, pairs = _c2_pairs(rng, n_reads=3000)
    hd, rd = haps.to_device("cuda:0"), reads.to_device("cuda:0")
    off, pos = engine.map_pairs(haps, reads, pairs)
    doff, dpos = engine.map_pairs(hd, rd, torch.as_tensor(pairs, device="cuda:0"))
    assert doff.is_cuda and np.array_equal(doff.cpu().numpy(), off) and np.array_equal(dpos.cpu().numpy(), pos)
    cfg = _cfg(band, True)
    mp, lk, cig, st = engine.realign_reads(cfg, haps, reads, pairs, (20, 20))
    dmp, dlk, dcig, dst = engine.realign_reads(cfg, hd, rd, pairs, (20, 20))
    assert dmp.is_cuda and dlk.is_cuda and dst.is_cuda
    assert np.array_equal(dmp.cpu().numpy(), mp) and np.array_equal(dlk.cpu().numpy().view(np.int64), lk.view(np.int64))
    assert dcig == cig and np.array_equal(dst.cpu().numpy(), st)


def _groups(rng, n_groups, reads_per_group, read_len=150):
    """ReadAssignments-shaped input: per group 2 haplotypes of 400-800 bases (the second a variant of the first) and reads drawn
    from them; pairs (read, each haplotype of its group)."""
    from octopus_b200.batch import HaplotypeBlock, ReadBlock
    hl = rng.integers(400, 801, n_groups)
    hap_len = np.repeat(hl, 2)
    hoff = np.concatenate([[0], np.cumsum(hap_len)]).astype(np.int64)
    seq = ACGT[rng.integers(0, 4, int(hoff[-1]))]
    for g in range(0, n_groups):
        a, b = int(hoff[2 * g]), int(hoff[2 * g + 1])
        n = min(b - a, int(hoff[2 * g + 2]) - b)
        seq[b:b + n] = seq[a:a + n]
        seq[b + int(rng.integers(0, n))] = ACGT[rng.integers(0, 4)]
    T = int(hoff[-1])
    haps = HaplotypeBlock(hoff, seq, np.roll(seq, 1), rng.integers(1, 126, T).astype(np.int8), np.roll(seq, -1),
                          rng.integers(1, 126, T).astype(np.int8), rng.integers(3, 46, T).astype(np.int8), rng.integers(1, 11, T).astype(np.int8),
                          begin=np.zeros(2 * n_groups, np.int64))
    R = n_groups * reads_per_group
    grp = np.repeat(np.arange(n_groups), reads_per_group)
    src = 2 * grp + rng.integers(0, 2, R)
    start = (rng.random(R) * (hap_len[src] - read_len + 1)).astype(np.int64)
    bases = np.empty(R * read_len, np.uint8)
    for c in range(0, R, 100_000):
        idx = (hoff[src[c:c + 100_000]] + start[c:c + 100_000])[:, None] + np.arange(read_len)[None, :]
        bases[c * read_len:(c + len(idx)) * read_len] = seq[idx].reshape(-1)
    mut = rng.integers(0, R * read_len, R // 2)
    bases[mut] = ACGT[rng.integers(0, 4, len(mut))]
    reads = ReadBlock(np.arange(R + 1, dtype=np.int64) * read_len, bases, rng.integers(10, 41, R * read_len).astype(np.uint8),
                      rng.choice([20, 60], R).astype(np.uint8), (rng.random(R) < 0.5).astype(np.uint8), start)
    pairs = np.stack([np.repeat(np.arange(R, dtype=np.int32), 2), (2 * np.repeat(grp, 2) + np.tile([0, 1], R)).astype(np.int32)], axis=1)
    return haps, reads, pairs


def test_large_call_equals_its_two_halves(engine):
    rng = np.random.default_rng(8601)
    haps, reads, pairs = _groups(rng, n_groups=8000, reads_per_group=128)
    n = len(pairs)
    assert n >= 2_000_000
    cfg = _cfg(8, True)
    whole = engine.realign_reads(cfg, haps, reads, pairs, cigar_stride=96)
    halves = [engine.realign_reads(cfg, haps, reads, pairs[s], cigar_stride=96) for s in (slice(0, n // 2), slice(n // 2, n))]
    for k in (0, 3):
        assert np.array_equal(whole[k], np.concatenate([h[k] for h in halves]))
    assert np.array_equal(whole[1].view(np.int64), np.concatenate([h[1] for h in halves]).view(np.int64))
    assert whole[2] == halves[0][2] + halves[1][2]
    assert (whole[3] == 0).mean() > 0.99


CPP_SRC = os.path.join(ROOT, "tests", "cpp", "test_realign.cpp")


def test_cpp_realign_helper(refhmm, coracle):
    from octopus_b200 import build
    from octopus_b200.batch import pack_haplotypes, pack_reads
    build.build()
    exe = os.path.join(tempfile.mkdtemp(prefix="test_realign_"), "test_realign")     # the source tree may be read-only
    subprocess.run(["g++", "-std=c++14", "-O1", "-I", os.path.join(ROOT, "include"), "-I", os.path.join(ROOT, "octopus_b200", "cpp"),
                    CPP_SRC, "-o", exe, "-L", os.path.join(ROOT, "octopus_b200"), "-lphmm_b200",
                    "-Wl,-rpath," + os.path.join(ROOT, "octopus_b200")], check=True)
    out = subprocess.run([exe], capture_output=True, text=True, timeout=120)
    assert out.returncode == 0, out.stdout + out.stderr
    lines = [l.split() for l in out.stdout.strip().splitlines()]
    # the same blocks as the program builds
    h0 = b"ACGTTGCAAGCTTAGGCTAACGTTAGCATCGATCGGATCTAGCTAGGATCGATACGATCGATCGTAGCTAGCTAGTCGATCGATTTAGCGCGATATCGCGAT"
    rep = b"AC" * 60
    r1 = bytearray(h0[35:75]); r1[12] = ord("C") if r1[12] == ord("A") else ord("A")

    def block(seqs):
        a = [np.frombuffer(s, np.uint8) for s in seqs]
        return pack_haplotypes(a, a, [np.full(len(s), 50, np.int8) for s in a], a, [np.full(len(s), 50, np.int8) for s in a],
                               [np.full(len(s), 40, np.int8) for s in a], [np.full(len(s), 3, np.int8) for s in a], begin=np.zeros(len(a), np.int64))
    haps = block([h0, b"GGCT" + rep + b"TTGA"])
    rb = [np.frombuffer(x, np.uint8) for x in (h0[30:70], bytes(r1), rep[:40])]
    reads = pack_reads(rb, [np.full(40, q, np.uint8) for q in (30, 25, 35)], mapq=np.full(3, 60, np.uint8),
                       reverse=np.array([0, 1, 0], np.uint8), begin=np.array([30, 35, 10], np.int64))
    ra = [l for l in lines if l[0] == "RA"]
    assert len(ra) == 6
    for _, h, r, mp, cig, lk in ra:
        h, r = int(h), int(r)
        pos = oracle_map(refhmm, coracle, reads.read(r)[0], haps.hap(h)["seq"])
        wst, wmp, wlk, wcig, _ = oracle_align(refhmm, coracle, 8, haps, reads, r, h, pos, None)
        assert wst == 0 and (int(mp), cig, float(lk)) == (wmp, wcig, wlk), (h, r, mp, cig, lk, wmp, wcig, wlk)
    maps = [l for l in lines if l[0] == "MAP"]
    for l in maps:
        r, h = int(l[1]), int(l[2])
        assert [int(x) for x in l[3:]] == oracle_map(refhmm, coracle, reads.read(r)[0], haps.hap(h)["seq"])
    assert max(len(l) - 3 for l in maps) > 10
    short = block([h0[25:70]])
    first = None
    for r in range(reads.n):
        pos = oracle_map(refhmm, coracle, reads.read(r)[0], short.hap(0)["seq"])
        wst, _, _, _, ext = oracle_align(refhmm, coracle, 8, short, reads, r, 0, pos, None)
        if wst == 1:
            first = ext
            break
    assert first is not None
    assert [l for l in lines if l[0] == "SHORT"] == [["SHORT", "hap=0", "ext=%d" % first]]
