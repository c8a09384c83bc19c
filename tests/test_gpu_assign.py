"""compute_haplotype_support's scoring and choice on the GPU (phmm_assign_reads). Per pair the oracle is the reference's composition in
calculate_likelihoods (read_assigner.cpp:231-285): the uncapped map_query_to_target, then HaplotypeLikelihoodModel::evaluate at its
positions (the C oracle stands in where oracle/_ref was never built). The choice is checked against the C restatement of
find_map_haplotypes (tests/cpp/find_map_oracle.c, pinned in tests/test_assign_oracle.py)."""
import os
import subprocess
import tempfile

import numpy as np
import pytest

from exact import assert_mix_within_bound, assert_same_penalties, effective_mapq, penalties
from find_map_oracle import find_map, find_map_all
from helpers import ACGT

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
INF = float("inf")


def _cfg(band_req, use_mq, map_positions=True):
    from octopus_b200 import HaplotypeLikelihoodModel
    return HaplotypeLikelihoodModel.Config(max_indel_error=band_req, use_mapping_quality=use_mq, map_positions=map_positions)


def oracle_map(refhmm, coracle, read, hap):
    cap = max(1, len(hap))
    if refhmm is not None:
        return refhmm.kmer_map(read, hap, cap)
    return list(coracle.kmer_map(read.tobytes().decode("latin1"), hap.tobytes().decode("latin1"), cap))


def oracle_evaluate(refhmm, coracle, band_req, haps, reads, r, h, positions):
    """HaplotypeLikelihoodModel::evaluate(read, positions) with mapping quality off: (status, value, extension)."""
    hp = haps.hap(h)
    b, q = reads.read(r)
    rev = bool(reads.reverse[r])
    hb = int(haps.begin[h]) if haps.begin is not None else 0
    if refhmm is not None:
        return refhmm.model_evaluate(band_req, hp["seq"], b, q, hp["gap_open"], hp["gap_extend"], hp["snv_mask_fwd"], hp["snv_prior_fwd"],
                                     hp["snv_mask_rev"], hp["snv_prior_rev"], positions, hap_begin=hb, read_begin=int(reads.begin[r]),
                                     mapping_quality=int(reads.mapq[r]), reverse=rev, use_mapping_quality=False)
    band = next(x for x in (8, 16, 32, 64, 128, 256) if band_req <= x)
    return coracle.model_evaluate(band, hp["seq"].tobytes(), b.tobytes(), q, hp["gap_open"], hp["gap_extend"],
                                  hp["snv_mask_rev" if rev else "snv_mask_fwd"].tobytes(), hp["snv_prior_rev" if rev else "snv_prior_fwd"],
                                  positions, int(reads.begin[r]) - hb, mapping_quality=int(reads.mapq[r]), use_mapping_quality=False)


def group_block(rng, n_haps, n_reads, hap_len, read_len=150, repeat=False, duplicate=False):
    """One genotype: n_haps haplotypes (variants of one sequence; repeat=True puts a tandem repeat and a homopolymer in it; duplicate=True
    makes them identical, penalties included) and reads drawn from them."""
    from octopus_b200.batch import pack_haplotypes, pack_reads
    base = ACGT[rng.integers(0, 4, hap_len)].copy()
    if repeat:
        unit = ACGT[rng.integers(0, 4, int(rng.integers(1, 4)))]
        a = int(rng.integers(0, hap_len // 3))
        n = int(rng.integers(hap_len // 4, hap_len // 2))
        base[a:a + n] = np.tile(unit, n // len(unit) + 1)[:n]
        b = int(rng.integers(a + n, hap_len - 60))
        base[b:b + 60] = ACGT[rng.integers(0, 4)]
    seqs = []
    for k in range(n_haps):
        s = base.copy()
        if k and not duplicate:
            for _ in range(int(rng.integers(1, 4))):
                s[rng.integers(0, hap_len)] = ACGT[rng.integers(0, 4)]
            if rng.random() < 0.4:
                p = int(rng.integers(10, hap_len - 10)); s = np.concatenate([s[:p], s[p + int(rng.integers(1, 4)):]])
        seqs.append(s)
    pen = lambda lo, hi, s: rng.integers(lo, hi, len(s)).astype(np.int8)     # noqa: E731
    if duplicate:
        one = [pen(1, 126, base), pen(1, 126, base), pen(3, 46, base), pen(1, 11, base)]
        pf, pr, go, ge = ([x.copy() for _ in seqs] for x in one)
    else:
        pf, pr, go, ge = [pen(1, 126, s) for s in seqs], [pen(1, 126, s) for s in seqs], [pen(3, 46, s) for s in seqs], [pen(1, 11, s) for s in seqs]
    haps = pack_haplotypes(seqs, [np.roll(s, 1) for s in seqs], pf, [np.roll(s, -1) for s in seqs], pr, go, ge,
                           begin=np.zeros(n_haps, np.int64))
    bases, begins = [], []
    for _ in range(n_reads):
        s = seqs[int(rng.integers(0, n_haps))]
        p = int(rng.integers(0, max(1, len(s) - read_len + 1)))
        b = s[p:p + read_len].copy()
        if len(b) < read_len:
            b = np.concatenate([b, ACGT[rng.integers(0, 4, read_len - len(b))]])
        for _ in range(int(rng.integers(0, 4))):
            b[rng.integers(0, read_len)] = ACGT[rng.integers(0, 4)]
        bases.append(b)
        begins.append(p)
    reads = pack_reads(bases, [rng.integers(8, 41, read_len).astype(np.uint8) for _ in bases], mapq=rng.choice([0, 10, 29, 60, 255], n_reads).astype(np.uint8),
                       reverse=(rng.random(n_reads) < 0.5).astype(np.uint8), begin=np.asarray(begins, np.int64))
    return haps, reads


def filter_call(rng, n_groups, reads_range=(20, 60), repeat_every=3, **kw):
    """Filter-shaped groups back to back: (haps, reads, hap_first, read_first)."""
    from octopus_b200.batch import concat_blocks
    blocks = [group_block(rng, int(rng.integers(2, 4)), int(rng.integers(*reads_range)), int(rng.integers(400, 801)),
                          repeat=(g % repeat_every == 0), **kw) for g in range(n_groups)]
    return concat_blocks([b[0] for b in blocks], [b[1] for b in blocks])


def random_priors(rng, H, with_inf=True):
    pri = np.log(rng.dirichlet(np.ones(H)))
    if with_inf:
        pri[rng.random(H) < 0.15] = -INF
    return pri


def oracle_values(refhmm, coracle, band_req, haps, reads, hap_first, read_first):
    """Flat oracle values / statuses in the groups' slot order, and the number of pairs with more than 10 mapped positions."""
    vals, sts, many = [], [], 0
    for g in range(len(hap_first) - 1):
        for h in range(int(hap_first[g]), int(hap_first[g + 1])):
            for r in range(int(read_first[g]), int(read_first[g + 1])):
                pos = oracle_map(refhmm, coracle, reads.read(r)[0], haps.hap(h)["seq"])
                many += len(pos) > 10
                st, v, _ = oracle_evaluate(refhmm, coracle, band_req, haps, reads, r, h, pos)
                vals.append(v)
                sts.append(st)
    return np.array(vals), np.array(sts, np.int32), many


def slot_mapq(reads, hap_first, read_first):
    out = []
    for g in range(len(hap_first) - 1):
        nh = int(hap_first[g + 1] - hap_first[g])
        out.append(np.tile(reads.mapq[int(read_first[g]):int(read_first[g + 1])], nh))
    return np.concatenate(out)


@pytest.mark.parametrize("band_req", [8, 16, 32])
def test_assign_equals_reference_composition(engine, refhmm, coracle, band_req):
    rng = np.random.default_rng(9200 + band_req)
    haps, reads, hf, rf = filter_call(rng, 6)
    want, wst, _ = oracle_values(refhmm, coracle, band_req, haps, reads, hf, rf)
    assert (wst == 0).all()
    for trial in range(2):
        pri = random_priors(rng, haps.n) if trial else None
        top0, lnl0, st0 = engine.assign_reads(_cfg(band_req, False), haps, reads, hf, rf, pri, want_likelihoods=True, want_status=True)
        assert ((st0 & 0xFFFF) != 2).all()
        assert_same_penalties(lnl0, want, None, wst, (band_req, trial))
        assert np.array_equal(top0, find_map_all(want, hf, rf, pri)), (band_req, trial)
        top1, lnl1 = engine.assign_reads(_cfg(band_req, True), haps, reads, hf, rf, pri, want_likelihoods=True)
        assert_mix_within_bound(lnl1, penalties(want), effective_mapq(slot_mapq(reads, hf, rf)), (band_req, trial, "mapq"))
        assert np.array_equal(top1, find_map_all(lnl1, hf, rf, pri)), (band_req, trial, "mapq")
        # top alone (no matrix asked for) is the same
        assert np.array_equal(engine.assign_reads(_cfg(band_req, True), haps, reads, hf, rf, pri), top1)
    if pri is not None:
        assert np.isinf(pri).any()


def test_uncapped_positions_are_the_ones_used(engine, refhmm, coracle):
    """Repeat-rich groups where pairs have more than 10 positions: the values are the uncapped mapper's, and some differ from
    populate_regions with its mapper capped at 10."""
    rng = np.random.default_rng(9301)
    haps, reads, hf, rf = filter_call(rng, 5, reads_range=(15, 30), repeat_every=1)
    band = 16
    want, wst, many = oracle_values(refhmm, coracle, band, haps, reads, hf, rf)
    assert many > 50
    top, lnl = engine.assign_reads(_cfg(band, False), haps, reads, hf, rf, want_likelihoods=True)
    assert_same_penalties(lnl, want, None, wst, "repeats")
    capped, _ = engine.populate_regions(_cfg(band, False), haps, reads, hf, rf)
    assert (capped.view(np.int64) != lnl.view(np.int64)).sum() > 0
    assert np.array_equal(top, find_map_all(want, hf, rf))
    # map_positions = 0: the original position only, populate_regions' values and the choice applied to them
    pri = random_priors(rng, haps.n)
    for mq in (False, True):
        top0, lnl0 = engine.assign_reads(_cfg(band, mq, map_positions=False), haps, reads, hf, rf, pri, want_likelihoods=True)
        ref0, _ = engine.populate_regions(_cfg(band, mq, map_positions=False), haps, reads, hf, rf)
        assert np.array_equal(lnl0.view(np.int64), ref0.view(np.int64))
        assert np.array_equal(top0, find_map_all(ref0, hf, rf, pri))


def up(x, n):
    for _ in range(n):
        x = float(np.nextafter(x, INF))
    return x


def test_constructed_ties_on_the_device(engine):
    from octopus_b200.batch import concat_blocks
    rng = np.random.default_rng(9401)
    # duplicate haplotypes: equal values, every copy in the set
    blocks = [group_block(rng, int(rng.integers(2, 6)), int(rng.integers(5, 40)), 500, duplicate=True) for _ in range(8)]
    haps, reads, hf, rf = concat_blocks([b[0] for b in blocks], [b[1] for b in blocks])
    top, lnl = engine.assign_reads(_cfg(16, True), haps, reads, hf, rf, want_likelihoods=True)
    assert np.array_equal(top, find_map_all(lnl, hf, rf))
    nh = np.repeat(np.diff(hf), np.diff(rf))
    assert np.array_equal(top, ((1 << nh.astype(np.uint64)) - 1).astype(np.uint64))
    # single-read groups of three copies; the priors move the copies' sums to chosen ulp distances: the almost_equal boundary and the
    # maximum an almost-equal value does not raise
    blocks = [group_block(rng, 3, 1, 450, duplicate=True) for _ in range(40)]
    haps, reads, hf, rf = concat_blocks([b[0] for b in blocks], [b[1] for b in blocks])
    _, v = engine.assign_reads(_cfg(8, True), haps, reads, hf, rf, want_likelihoods=True)
    v = v[0::3]
    pri = np.zeros(haps.n)
    expect = {}
    for g in range(len(v)):
        x = float(v[g])
        n = 1
        while n < 64 and abs(up(x, n) - x) < 2.0 ** -52 * abs(up(x, n) + x):
            n += 1
        kind = g % 4
        steps = [(0, n - 1, 2 * (n - 1)), (0, n - 1, 0), (0, n, 0), (n, n - 1, 0)][kind]
        pri[3 * g:3 * g + 3] = [up(x, s) - x for s in steps]
        if x < -1e-3 and n < 64:
            expect[g] = [0b100, 0b111, 0b010, 0b011][kind] if 2 * (n - 1) >= n else None
    top = engine.assign_reads(_cfg(8, True), haps, reads, hf, rf, pri)
    sums = v.repeat(3) + pri
    for g in range(len(v)):
        assert int(top[g]) == find_map(sums[3 * g:3 * g + 3]), g
        if expect.get(g) is not None:
            assert int(top[g]) == expect[g], (g, float(v[g]), int(top[g]))
    assert sum(e is not None for e in expect.values()) >= 20


def _call(engine, cfg, haps, reads, hf, rf, pri):
    return engine.assign_reads(cfg, haps, reads, hf, rf, pri, want_likelihoods=True, want_status=True)


def _sub(haps, reads, hf, rf, g0, g1):
    """Groups [g0, g1) as blocks of their own."""
    from octopus_b200.batch import HaplotypeBlock, ReadBlock
    h0, h1, r0, r1 = int(hf[g0]), int(hf[g1]), int(rf[g0]), int(rf[g1])
    a, b = int(haps.off[h0]), int(haps.off[h1])
    hs = HaplotypeBlock(haps.off[h0:h1 + 1] - a, *[getattr(haps, f)[a:b] for f in HaplotypeBlock._fields[1:8]], haps.begin[h0:h1])
    c, d = int(reads.off[r0]), int(reads.off[r1])
    rs = ReadBlock(reads.off[r0:r1 + 1] - c, reads.bases[c:d], reads.quals[c:d], reads.mapq[r0:r1], reads.reverse[r0:r1], reads.begin[r0:r1])
    return hs, rs, (hf[g0:g1 + 1] - h0).astype(np.int32), (rf[g0:g1 + 1] - r0).astype(np.int32)


def test_many_groups_equal_one_call_per_group(engine):
    from octopus_b200.batch import concat_blocks
    rng = np.random.default_rng(9501)
    sizes = [(1, 30), (64, 12), (2, 1), (3, 1), (5, 25), (2, 300), (17, 4), (1, 1), (33, 9), (3, 150)]
    blocks = [group_block(rng, nh, nr, int(rng.integers(400, 801)), repeat=(i % 3 == 0)) for i, (nh, nr) in enumerate(sizes)]
    haps, reads, hf, rf = concat_blocks([b[0] for b in blocks], [b[1] for b in blocks])
    pri = random_priors(rng, haps.n)
    for cfg in (_cfg(16, True), _cfg(8, False), _cfg(32, True, map_positions=False)):
        whole = _call(engine, cfg, haps, reads, hf, rf, pri)
        parts = [_call(engine, cfg, *_sub(haps, reads, hf, rf, g, g + 1), pri[int(hf[g]):int(hf[g + 1])]) for g in range(len(sizes))]
        assert np.array_equal(whole[0], np.concatenate([p[0] for p in parts]))
        assert np.array_equal(whole[1].view(np.int64), np.concatenate([p[1] for p in parts]).view(np.int64))
        assert np.array_equal(whole[2], np.concatenate([p[2] for p in parts]))
        assert whole[0][int(rf[1]):int(rf[2])].max() >= 1 << 32          # the 64-haplotype group's upper bits are used
    # device-resident inputs and outputs equal host ones
    import torch
    hd, rd = haps.to_device("cuda:0"), reads.to_device("cuda:0")
    cfg = _cfg(16, True)
    host = _call(engine, cfg, haps, reads, hf, rf, pri)
    dev = engine.assign_reads(cfg, hd, rd, hf, rf, torch.as_tensor(pri, device="cuda:0"), want_likelihoods=True, want_status=True)
    assert all(t.is_cuda for t in dev)
    assert np.array_equal(dev[0].cpu().numpy().view(np.uint64), host[0])
    assert np.array_equal(dev[1].cpu().numpy().view(np.int64), host[1].view(np.int64))
    assert np.array_equal(dev[2].cpu().numpy(), host[2])
    assert np.array_equal(engine.assign_reads(cfg, hd, rd, hf, rf, pri).cpu().numpy().view(np.uint64), host[0])


def test_million_pair_call_equals_its_parts(engine):
    """Over 1 M pairs with one homopolymer group whose pairs have ~1 000 positions each: the position lists make populate's task lists
    long enough that the call runs in several tiles."""
    from octopus_b200.batch import concat_blocks, pack_haplotypes, pack_reads
    rng = np.random.default_rng(9601)
    haps, reads, hf, rf = filter_call(rng, 3300, reads_range=(100, 220), repeat_every=7)
    hp = np.full(1200, ord("T"), np.uint8)
    hb = pack_haplotypes([hp, hp.copy()], [hp, hp], [np.full(1200, 40, np.int8)] * 2, [hp, hp], [np.full(1200, 40, np.int8)] * 2,
                         [np.full(1200, 20, np.int8)] * 2, [np.full(1200, 3, np.int8)] * 2, begin=np.zeros(2, np.int64))
    rb = pack_reads([np.full(150, ord("T"), np.uint8)] * 4, [np.full(150, 30, np.uint8)] * 4, mapq=np.full(4, 60, np.uint8),
                    reverse=np.zeros(4, np.uint8), begin=np.full(4, 500, np.int64))
    from octopus_b200.batch import HaplotypeBlock, ReadBlock
    h2, r2, hf2, rf2 = _sub(haps, reads, hf, rf, 0, len(hf) - 1)
    haps, reads, hf_, rf_ = concat_blocks([hb, h2], [rb, r2])
    hf = np.concatenate([[0], 2 + hf2]).astype(np.int32)
    rf = np.concatenate([[0], 4 + rf2]).astype(np.int32)
    n_pairs = int((np.diff(hf).astype(np.int64) * np.diff(rf)).sum())
    assert n_pairs > 1_000_000
    pri = random_priors(rng, haps.n)
    cfg = _cfg(8, True)
    whole = _call(engine, cfg, haps, reads, hf, rf, pri)
    G = len(hf) - 1
    cuts = [0, 1, G // 3, 2 * G // 3, G]
    parts = [_call(engine, cfg, *_sub(haps, reads, hf, rf, a, b), pri[int(hf[a]):int(hf[b])]) for a, b in zip(cuts[:-1], cuts[1:])]
    assert np.array_equal(whole[0], np.concatenate([p[0] for p in parts]))
    assert np.array_equal(whole[1].view(np.int64), np.concatenate([p[1] for p in parts]).view(np.int64))
    assert np.array_equal(whole[2], np.concatenate([p[2] for p in parts]))
    assert (whole[2] == 0).mean() > 0.99


def test_argument_checks(engine, refhmm, coracle):
    from octopus_b200 import PhmmError, ShortHaplotypeError
    from octopus_b200.batch import concat_blocks, pack_haplotypes, pack_reads
    rng = np.random.default_rng(9701)
    cfg = _cfg(16, True)
    # 65 haplotypes in one group
    h65, r65 = group_block(rng, 65, 3, 400)
    with pytest.raises(PhmmError, match="64 haplotypes"):
        engine.assign_reads(cfg, h65, r65, [0, 65], [0, 3])
    # more than 4096 mapped positions for one pair: a 5 000-base homopolymer
    hp = np.full(5000, ord("A"), np.uint8)
    hb = pack_haplotypes([hp, hp], [hp, hp], [np.full(5000, 40, np.int8)] * 2, [hp, hp], [np.full(5000, 40, np.int8)] * 2,
                         [np.full(5000, 20, np.int8)] * 2, [np.full(5000, 3, np.int8)] * 2, begin=np.zeros(2, np.int64))
    rb = pack_reads([np.full(150, ord("A"), np.uint8)] * 2, [np.full(150, 30, np.uint8)] * 2, mapq=np.full(2, 60, np.uint8),
                    reverse=np.zeros(2, np.uint8), begin=np.zeros(2, np.int64))
    with pytest.raises(PhmmError, match="4096"):
        engine.assign_reads(cfg, hb, rb, [0, 2], [0, 2])
    # a haplotype over 65 535 bp with the mapper on
    hl = ACGT[rng.integers(0, 4, 70000)]
    hbig = pack_haplotypes([hl], [hl], [np.full(70000, 40, np.int8)], [hl], [np.full(70000, 40, np.int8)], [np.full(70000, 20, np.int8)],
                           [np.full(70000, 3, np.int8)], begin=np.zeros(1, np.int64))
    with pytest.raises(PhmmError, match="65535"):
        engine.assign_reads(cfg, hbig, rb, [0, 1], [0, 2])
    # group bounds
    haps, reads, hf, rf = filter_call(rng, 3)
    for bad_h, bad_r, msg in ((hf + [0, 0, 0, 1], rf, "cover"), (hf, rf - [0, 0, 0, 1], "cover"), ([0, 2, 2, hf[-1]], rf, "at least one"),
                              (hf, [0, rf[1], rf[1], rf[-1]], "at least one"), ([], [], "region list")):
        with pytest.raises(PhmmError, match=msg):
            engine.assign_reads(cfg, haps, reads, np.asarray(bad_h, np.int32), np.asarray(bad_r, np.int32))
    # a short haplotype: statuses and extensions equal phmm_populate's for that group, with the same return code
    g1 = group_block(rng, 2, 20, 500)
    base = ACGT[rng.integers(0, 4, 300)].copy()
    seqs = [base[20:80].copy(), base[:300].copy()]
    sh = pack_haplotypes(seqs, seqs, [np.full(len(s), 40, np.int8) for s in seqs], seqs, [np.full(len(s), 40, np.int8) for s in seqs],
                         [np.full(len(s), 20, np.int8) for s in seqs], [np.full(len(s), 3, np.int8) for s in seqs], begin=np.zeros(2, np.int64))
    sr = pack_reads([base[30:80].copy(), base[100:150].copy(), base[10:60].copy()], [np.full(50, 30, np.uint8)] * 3,
                    mapq=np.full(3, 60, np.uint8), reverse=np.array([0, 1, 0], np.uint8), begin=np.array([30, 100, 10], np.int64))
    haps, reads, hf, rf = concat_blocks([g1[0], sh], [g1[1], sr])
    with pytest.raises(ShortHaplotypeError):
        engine.assign_reads(cfg, haps, reads, hf, rf)
    _, lnl, st = engine.assign_reads(cfg, haps, reads, hf, rf, want_likelihoods=True, want_status=True)
    o = int(hf[1] * rf[1])
    assert (st[:o] == 0).all() and ((st[o:] & 0xFFFF) == 2).sum() >= 2
    off, pos = engine.map_pairs(sh, sr, np.array([(r, h) for h in range(2) for r in range(3)], np.int32))
    want = engine.populate(cfg, sh, sr, positions=(off, pos), want_status=True)
    assert np.array_equal(st[o:], want[1].reshape(-1))
    ok = want[1].reshape(-1) == 0
    assert np.array_equal(lnl[o:][ok].view(np.int64), want[0].reshape(-1)[ok].view(np.int64))


CPP_SRC = os.path.join(ROOT, "tests", "cpp", "test_assign.cpp")


def test_cpp_compute_haplotype_support(engine, refhmm, coracle):
    from octopus_b200 import build
    from octopus_b200.batch import concat_blocks
    build.build()
    exe = os.path.join(tempfile.mkdtemp(prefix="test_assign_"), "test_assign")
    subprocess.run(["g++", "-std=c++14", "-O1", "-I", os.path.join(ROOT, "include"), "-I", os.path.join(ROOT, "octopus_b200", "cpp"),
                    CPP_SRC, "-o", exe, "-L", os.path.join(ROOT, "octopus_b200"), "-lphmm_b200",
                    "-Wl,-rpath," + os.path.join(ROOT, "octopus_b200")], check=True)
    # the program reads the groups from a file the test writes: one haplotype / read per line
    rng = np.random.default_rng(9801)
    blocks = [group_block(rng, 2, 12, 420, duplicate=(g == 1)) for g in range(2)] + [group_block(rng, 3, 15, 450, repeat=True)]
    haps, reads, hf, rf = concat_blocks([b[0] for b in blocks], [b[1] for b in blocks])
    pri = random_priors(rng, haps.n, with_inf=False)
    pri[int(hf[1]):int(hf[2])] = pri[int(hf[1])]                # the duplicate group stays tied: ambiguous reads
    spec = os.path.join(os.path.dirname(exe), "groups.txt")
    with open(spec, "w") as f:
        f.write("%d %d %d\n" % (haps.n, reads.n, len(hf) - 1))
        for h in range(haps.n):
            hp = haps.hap(h)
            f.write("%s %s %s %s %s %s %s %r\n" % (hp["seq"].tobytes().decode(), hp["snv_mask_fwd"].tobytes().decode(),
                                                 ",".join(map(str, hp["snv_prior_fwd"])), hp["snv_mask_rev"].tobytes().decode(),
                                                 ",".join(map(str, hp["snv_prior_rev"])), ",".join(map(str, hp["gap_open"])),
                                                 ",".join(map(str, hp["gap_extend"])), float(pri[h])))
        for r in range(reads.n):
            b, q = reads.read(r)
            f.write("%s %s %d %d %d\n" % (b.tobytes().decode(), ",".join(map(str, q)), reads.mapq[r], reads.reverse[r], reads.begin[r]))
        f.write(" ".join(map(str, hf)) + "\n" + " ".join(map(str, rf)) + "\n")
    out = subprocess.run([exe, spec], capture_output=True, text=True, timeout=300)
    assert out.returncode == 0, out.stdout + out.stderr
    lines = [l.split() for l in out.stdout.strip().splitlines()]
    want, wst, _ = oracle_values(refhmm, coracle, 16, haps, reads, hf, rf)
    top = find_map_all(want, hf, rf, pri)
    for action in ("drop", "first", "all"):
        expect = []
        for g in range(len(hf) - 1):
            nh = int(hf[g + 1] - hf[g])
            for r in range(int(rf[g]), int(rf[g + 1])):
                ks = [k for k in range(nh) if int(top[r]) >> k & 1]
                chosen = ks if len(ks) == 1 or action == "all" else ks[:1] if action == "first" else []
                expect += [["SUP", action, str(g), str(k), str(r)] for k in chosen]
                if len(ks) > 1:
                    expect.append(["AMB", action, str(g), str(r)] + [str(k) for k in ks])
        got = [l for l in lines if l[1] == action and l[0] in ("SUP", "AMB")]
        assert sorted(got) == sorted(expect), action
    assert any(l[0] == "AMB" for l in lines)
    # the program appends a group of haplotype 0's first 60 bases with group 0's reads: ShortHaplotypeError for its first short pair
    from octopus_b200.batch import pack_haplotypes
    hp = haps.hap(0)
    sh = pack_haplotypes(*[[hp[k][:60]] for k in ("seq", "snv_mask_fwd", "snv_prior_fwd", "snv_mask_rev", "snv_prior_rev", "gap_open",
                                                   "gap_extend")], begin=np.zeros(1, np.int64))
    g0 = _sub(haps, reads, hf, rf, 0, 1)[1]
    _, st = engine.assign_reads(_cfg(16, False), sh, g0, [0, 1], [0, g0.n], want_status=True)
    first = next(int(x) for x in st if (x & 0xFFFF) == 2)
    assert [l for l in lines if l[0] == "SHORT"] == [["SHORT", "hap=%d" % haps.n, "ext=%d" % (first >> 16)]]
