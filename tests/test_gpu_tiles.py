"""populate across tile boundaries, and flank-state calls that hold reads of 6 400+ bases.

A populate call cuts its read lists into tiles when a per-tile scratch budget would be exceeded, and runs the whole kernel chain
once per tile over the same scratch (phmm_engine.cu, populate_impl). With H the most haplotypes any region has, a tile holds at most
- 8 Mi / (H * max_cand) reads with a flank state (traceback queue),
- 2^30 / (41 H) reads with the k-mer mapper (mapped positions),
- 160 Mi / (H * max_dp_per_pair) reads (task lists),
where max_cand / max_dp_per_pair are the longest candidate list + 2 / + 1 (12 / 11 with the mapper, 2 / 1 without a list).

Every call here crosses at least one budget, and each test checks that it did: its launch count must exceed that of the same mode
on a one-tile subset by at least the per-tile launches of the extra tiles. Every check runs in two legs: mapping quality off, values
and statuses bit-equal; on, values within the bound of the exact mix (tests/exact.py), statuses equal."""
import numpy as np
import pytest

from exact import assert_same_penalties, assert_sums_within_bound, penalties
from helpers import ACGT, random_region
from test_gpu_parity import mixed_within_bound, populate_legs

pytestmark = pytest.mark.gpu


def _band(band_req):
    from octopus_b200 import HaplotypeLikelihoodModel
    return HaplotypeLikelihoodModel(HaplotypeLikelihoodModel.Config(max_indel_error=band_req)).pad_requirement()


def _reads(rng, haps, specs, band):
    """specs: (length, quality, with 'N') per read; quality is a constant or an inclusive (lo, hi) range. Each read copies an in-range
    window of a random haplotype with a substitution per 50 bases."""
    from octopus_b200.batch import pack_reads
    bases, quals, begin = [], [], []
    for L, q, with_n in specs:
        src = haps.hap(int(rng.integers(0, haps.n)))["seq"]
        lo, hi = band, len(src) - L - band
        p = int(rng.integers(lo, max(lo, hi) + 1))
        b = src[p:p + L].copy()
        b[b == ord("N")] = ord("A")
        k = max(1, L // 50)
        b[rng.integers(0, L, k)] = ACGT[rng.integers(0, 4, k)]
        if with_n:
            b[rng.integers(0, L)] = ord("N")
        bases.append(b)
        quals.append(np.full(L, q, np.uint8) if np.isscalar(q) else rng.integers(q[0], q[1] + 1, L).astype(np.uint8))
        begin.append(p)
    n = len(specs)
    return pack_reads(bases, quals, mapq=rng.choice([0, 10, 29, 60, 255], n).astype(np.uint8),
                      reverse=(rng.random(n) < 0.5).astype(np.uint8), begin=np.asarray(begin, np.int64))


def _take(reads, idx):
    from octopus_b200.batch import pack_reads
    idx = np.asarray(idx)
    parts = [reads.read(int(r)) for r in idx]
    return pack_reads([b for b, _ in parts], [q for _, q in parts], reads.mapq[idx], reads.reverse[idx], reads.begin[idx])


def _slice(reads, a, b):
    from octopus_b200.batch import ReadBlock
    o0, o1 = int(reads.off[a]), int(reads.off[b])
    return ReadBlock(reads.off[a:b + 1] - o0, reads.bases[o0:o1], reads.quals[o0:o1], reads.mapq[a:b], reads.reverse[a:b], reads.begin[a:b])


def _cat_reads(blocks):
    from octopus_b200.batch import pack_reads
    parts = [blk.read(r) for blk in blocks for r in range(blk.n)]
    cat = lambda f: np.concatenate([getattr(blk, f) for blk in blocks])     # noqa: E731
    return pack_reads([b for b, _ in parts], [q for _, q in parts], cat("mapq"), cat("reverse"), cat("begin"))


def _reads_per_tile(H, max_cand=2, flanks=False, mapper=False):
    """populate_impl's tile size in reads (max_dp_per_pair = max_cand - 1)."""
    t = (160 << 20) // (H * (max_cand - 1))
    if mapper:
        t = min(t, (1 << 30) // (41 * H))
    if flanks:
        t = min(t, (8 << 20) // (H * max_cand))
    return max(2, t)


def _tile_guard(engine, full_launches, one_tile_call, n_pair_reads, per_tile, what):
    """The call that gave full_launches ran at least ceil(n_pair_reads / (tile size)) pair tiles; one_tile_call runs the same mode
    on a one-tile subset (with reads on the same lists). Every extra pair tile launches at least per_tile kernels (the DP kernel, and
    the classify pass unless in direct mode)."""
    rpt = n_pair_reads[1]
    tiles = -(-n_pair_reads[0] // (rpt + 2))
    one_tile_call()
    one = engine.launch_count()
    print("%s: %d pair-list reads, %d reads per tile: >= %d pair tiles; %d launches, %d on a one-tile subset" % (
        what, n_pair_reads[0], rpt, tiles, full_launches, one))
    assert tiles >= 2, what
    assert full_launches - one >= per_tile * (tiles - 1), (what, full_launches, one, tiles)


# ---------------------------------------------------------------------------------------------------------------------------------
# 1. A candidate list of 4 096 positions (max_cand 4 098): 63 reads per tile with a flank state, 1 279 without
# ---------------------------------------------------------------------------------------------------------------------------------

def _long_list_case(band, flanks):
    """H = 32 haplotypes of 4 400 bases. Pair (0, 0) lists 4 096 distinct in-range positions; about a third of the others list 1-3
    positions near the read's start. Reads: ACGT of 76 / 100 / 150 bases (odd counts), reads with 'N', reads shorter than 2B, reads
    of 1 024-1 500 bases (one with a quality sum above 27 648), and one read with a quality above 127. The first 24 reads hold one of
    each kind: the one-tile subset."""
    from octopus_b200.batch import pack_positions
    rng = np.random.default_rng(7000 + band + (1 if flanks else 0))
    haps, _ = random_region(rng, band, n_haps=32, n_reads=1, hap_len=4400, read_len_choices=[76], edge_reads=False)
    scale = 1 if flanks else 6
    short = max(4, 2 * band - 3)
    kinds = ([(150, (2, 41), False), (100, (2, 41), True), (short, (2, 41), False), (1100, 30, False), (1300, (2, 41), False),
              (150, (2, 41), False)] + [(int(rng.choice([76, 100, 150])), (2, 41), False) for _ in range(18)])
    body = ([(76, (2, 41), False)] * (61 * scale) + [(100, (2, 41), False)] * (73 * scale) + [(150, (2, 41), False)] * (87 * scale) +
            [(100, (2, 41), True)] * (9 * scale) + [(short, (2, 41), False)] * (5 * scale) + [(1500, (2, 41), False)])
    order = rng.permutation(len(body))
    specs = kinds + [body[i] for i in order]
    reads = _reads(rng, haps, specs, band)
    q = reads.quals.copy()
    q[reads.off[5] + 7] = 200
    reads.quals = q
    lists = []
    for h in range(haps.n):
        row = []
        for r in range(reads.n):
            top = haps.length(h) - reads.length(r) - band         # in range: the whole window lies on the haplotype
            if h == 0 and r == 0:
                row.append(list(range(band, band + 4096)))
            elif rng.random() < 0.35:
                p0 = int(reads.begin[r])
                row.append(sorted({int(np.clip(p0 + rng.integers(-12, 13), band, top)) for _ in range(int(rng.integers(1, 4)))}))
            else:
                row.append([])
        lists.append(row)
    n_pair = sum(1 for L, _, n in specs if L <= 1023 and not (n and band > 32)) - 1      # read 5: the generic list
    fl = (int(rng.integers(20, 90)), int(rng.integers(20, 90))) if flanks else None
    return haps, reads, (lambda idx: pack_positions([[row[i] for i in idx] for row in lists], haps.n, len(idx))), fl, n_pair


@pytest.mark.parametrize("band", [8, 16, 32, 64])
def test_long_candidate_list_across_tiles(engine, coracle, band):
    from octopus_b200 import HaplotypeLikelihoodModel
    for flanks in (True, False):
        haps, reads, positions_of, fl, n_pair = _long_list_case(band, flanks)
        for dp_only in (False, True):
            populate_legs(engine, coracle, band, haps, reads, positions_of(np.arange(reads.n)), fl, (band, flanks, dp_only),
                          dp_only=dp_only, max_indel_error=band)
            full = engine.launch_count()
            sub = np.arange(24)
            cfg = HaplotypeLikelihoodModel.Config(max_indel_error=band, disable_naive_shortcut=dp_only, map_positions=False)
            _tile_guard(engine, full, lambda: engine.populate(cfg, haps, _take(reads, sub), positions_of(sub), fl),
                        (n_pair, _reads_per_tile(haps.n, 4098, flanks)), 2, ("long list", band, flanks, dp_only))


# ---------------------------------------------------------------------------------------------------------------------------------
# 2. Production semantics: about 200 regions, Hmax 128, flank states, the mapper and the shortcut: 5 461 reads per tile
# ---------------------------------------------------------------------------------------------------------------------------------

def _many_regions():
    """Region 0: 128 haplotypes. Region 1: 3 haplotypes of 1 400 bases with a read of 1 100 bases and one with a quality above 127
    (the wide and generic lists). The others: 1-40 haplotypes, 40-80 reads. A flank state on four regions in five."""
    from octopus_b200.batch import concat_blocks
    rng = np.random.default_rng(4242)
    band = 16
    regions, flanks = [], []
    for g in range(200):
        if g == 1:
            haps, _ = random_region(rng, band, n_haps=3, n_reads=1, hap_len=1400, read_len_choices=[150])
            reads = _reads(rng, haps, [(1100, (2, 41), False), (150, 200, False)] + [(150, (2, 41), False)] * 9, band)
        else:
            haps, reads = random_region(rng, band, n_haps=128 if g == 0 else int(rng.integers(1, 41)), n_reads=int(rng.integers(40, 81)),
                                        hap_len=int(rng.choice([260, 300, 420])), read_len_choices=[40, 76, 100, 150], read_n_rate=0.05,
                                        edge_reads=(g % 3 == 0))
        regions.append((haps, reads))
        flanks.append((int(rng.integers(0, 90)), int(rng.integers(0, 90))) if g % 5 else None)
    cat = concat_blocks([h for h, _ in regions], [r for _, r in regions])
    return band, regions, flanks, cat


def test_many_regions_across_tiles(engine, coracle):
    from octopus_b200 import HaplotypeLikelihoodModel
    from octopus_b200.batch import concat_blocks
    band, regions, flanks, (bh, br, hf, rf) = _many_regions()
    R = br.n
    # groups of whole regions with at most 4 000 reads each: one tile per group
    groups, g0 = [], 0
    while g0 < len(regions):
        g1 = g0
        while g1 < len(regions) and rf[g1 + 1] - rf[g0] <= 4000:
            g1 += 1
        groups.append((g0, g1))
        g0 = g1
    assert len(groups) >= 3
    sample = [0, 1] + list(np.random.default_rng(5).choice(np.arange(2, len(regions)), 18, replace=False))
    oracle = {g: coracle.populate(band, *regions[g], None, flanks[g], use_mapping_quality=False, map_positions=True) for g in sample}
    for use_mq in (False, True):
        cfg = HaplotypeLikelihoodModel.Config(max_indel_error=band, use_mapping_quality=use_mq)
        flat, off, st = engine.populate_regions(cfg, bh, br, hf, rf, flanks, want_status=True)
        full = engine.launch_count()
        parts_v, parts_s = [], []
        for a, b in groups:
            sub_h, sub_r = np.asarray(hf[a:b + 1]) - hf[a], np.asarray(rf[a:b + 1]) - rf[a]
            gh, gr, _, _ = concat_blocks([regions[g][0] for g in range(a, b)], [regions[g][1] for g in range(a, b)])
            v, _, s = engine.populate_regions(cfg, gh, gr, sub_h, sub_r, flanks[a:b], want_status=True)
            parts_v.append(v); parts_s.append(s)
        assert np.array_equal(np.concatenate(parts_v).view(np.int64), flat.view(np.int64)), use_mq
        assert np.array_equal(np.concatenate(parts_s), st), use_mq
        vals, stats = engine.split_regions(flat, off, hf, rf), engine.split_regions(st, off, hf, rf)
        for g in sample:
            rc, want, wst = oracle[g]
            if not use_mq:
                assert_same_penalties(vals[g], want, stats[g], wst, ("region", g))
            else:
                assert np.array_equal(stats[g] != 0, (wst != 0) | (want == -1.7976931348623157e308)), g
                mixed_within_bound(vals[g], want, wst, regions[g][1].mapq[None, :], what=("region", g))
        if use_mq:
            a, b = groups[0]          # regions 0 and 1 among them: Hmax 128, reads on every list
            gh, gr, sh, sr = concat_blocks([regions[g][0] for g in range(a, b)], [regions[g][1] for g in range(a, b)])
            _tile_guard(engine, full, lambda: engine.populate_regions(cfg, gh, gr, sh, sr, flanks[a:b]),
                        (R - 2, _reads_per_tile(128, 12, True, True)), 2, "regions")


# ---------------------------------------------------------------------------------------------------------------------------------
# 3. Templates: H = 128, the mapper and a flank state, about 12 000 reads in pairs
# ---------------------------------------------------------------------------------------------------------------------------------

def test_templates_across_tiles(engine, coracle):
    from octopus_b200 import HaplotypeLikelihoodModel, synth
    rng = np.random.default_rng(31337)
    band = 16
    haps = synth.make_haplotypes(rng, 128, 1400)
    # template 0: a read of 1 100 bases and one with a quality above 127 (the wide and generic lists)
    head = _reads(rng, haps, [(1100, 30, False), (150, 200, False)], band)
    reads = _cat_reads([head, synth.make_reads(rng, haps, 12000, (100, 150), band, "empirical")])
    R = reads.n
    toff = np.arange(0, R + 1, 2, dtype=np.int64)
    T = len(toff) - 1
    fl = (300, 300)
    res = {}
    for use_mq in (False, True):
        cfg = HaplotypeLikelihoodModel.Config(max_indel_error=band, use_mapping_quality=use_mq)
        res[use_mq] = engine.populate_templates(cfg, haps, reads, toff, flank_state=fl)
        full = engine.launch_count()
        # template-aligned halves: each half is cut into tiles at other reads
        m = 2 * (T // 2 - 17)
        halves = [engine.populate_templates(cfg, haps, _slice(reads, 0, m), toff[:m // 2 + 1], flank_state=fl),
                  engine.populate_templates(cfg, haps, _slice(reads, m, R), toff[m // 2:] - m, flank_state=fl)]
        assert np.array_equal(np.concatenate(halves, axis=1).view(np.int64), res[use_mq].view(np.int64)), use_mq
        if use_mq:
            _tile_guard(engine, full, lambda: engine.populate_templates(cfg, haps, _slice(reads, 0, 2000), toff[:1001], flank_state=fl),
                        (R - 2, _reads_per_tile(128, 12, True, True)), 2, "templates")
    tsample = np.concatenate([[0], np.random.default_rng(6).choice(np.arange(1, T), 29, replace=False)])
    ridx = np.concatenate([np.arange(toff[t], toff[t + 1]) for t in tsample])
    sub = _take(reads, ridx)
    rc, per_read, wst = coracle.populate(band, haps, sub, None, fl, use_mapping_quality=False, map_positions=True)
    assert rc == 0 and (wst == 0).all()
    soff = np.arange(0, len(ridx) + 1, 2, dtype=np.int64)
    want = np.zeros((haps.n, len(tsample)))
    for j in range(len(tsample)):
        for r in range(soff[j], soff[j + 1]):
            want[:, j] = want[:, j] + per_read[:, r]
    assert np.array_equal(res[False][:, tsample], want)          # both sides add the reads' -ln10/10 * s in read order
    assert_sums_within_bound(res[True][:, tsample], penalties(per_read), sub.mapq[None, :], soff, "templates")


# ---------------------------------------------------------------------------------------------------------------------------------
# 4. Direct mode at two tiles: H = 1 024, 172 000 device-resident reads (163 840 reads per tile)
# ---------------------------------------------------------------------------------------------------------------------------------

def test_direct_mode_across_tiles(engine, coracle):
    import torch
    from octopus_b200 import HaplotypeLikelihoodModel, synth
    haps, reads, band = synth.make_batch("C5", n_reads=172000, n_haps=1024, read_lens=(76, 100, 150))
    rng = np.random.default_rng(11)
    with_n = np.sort(rng.choice(reads.n, 860, replace=False))
    bases = reads.bases.copy()
    for r in with_n:
        bases[reads.off[r] + int(rng.integers(0, reads.length(r)))] = ord("N")
    quals = reads.quals.copy()
    quals[reads.off[with_n[0] + 1] + 3] = 200                    # a read with a quality above 127: the generic list
    reads.bases, reads.quals = bases, quals
    reads.mapq = rng.choice([0, 10, 29, 60, 255], reads.n).astype(np.uint8)
    # test 1's call, before and after the direct-mode calls on the same engine: no state may carry over between calls of other budgets
    h1, r1, pos1, fl1, _ = _long_list_case(16, True)
    cfg1 = HaplotypeLikelihoodModel.Config(max_indel_error=16, use_mapping_quality=False)
    before = engine.populate(cfg1, h1, r1, pos1(np.arange(r1.n)), fl1, want_status=True)
    dh = haps.to_device("cuda:0")
    R, half = reads.n, reads.n // 2 + 123
    sample = np.concatenate([with_n[:6], [with_n[0] + 1], rng.choice(R, 23, replace=False)])
    res = {}
    for use_mq in (False, True):
        cfg = HaplotypeLikelihoodModel.Config(max_indel_error=band, use_mapping_quality=use_mq, disable_naive_shortcut=True,
                                              map_positions=False)
        dr = reads.to_device("cuda:0")
        out, st = engine.populate(cfg, dh, dr, want_status=True)
        full = engine.launch_count()
        del dr
        for a, b in ((0, half), (half, R)):
            part = _slice(reads, a, b).to_device("cuda:0")
            o2, s2 = engine.populate(cfg, dh, part, want_status=True)
            assert torch.equal(o2, out[:, a:b]) and torch.equal(s2, st[:, a:b]), (use_mq, a, b)
            del part, o2, s2
        cols = torch.as_tensor(sample, device=out.device)
        res[use_mq] = (out[:, cols].cpu().numpy(), st[:, cols].cpu().numpy())
        if use_mq:
            sub = _slice(reads, 0, 20000).to_device("cuda:0")
            n_pair = R - len(with_n) - 1
            _tile_guard(engine, full, lambda: engine.populate(cfg, dh, sub), (n_pair, _reads_per_tile(1024)), 1, "direct")
        del out, st
        torch.cuda.empty_cache()
    sub = _take(reads, sample)
    rc, want, wst = coracle.populate(band, haps, sub, None, None, use_mapping_quality=False, dp_only=True, map_positions=False)
    assert_same_penalties(res[False][0], want, res[False][1], wst, "direct")
    assert np.array_equal(res[True][1], res[False][1])
    mixed_within_bound(res[True][0], want, wst, sub.mapq[None, :], what="direct")
    after = engine.populate(cfg1, h1, r1, pos1(np.arange(r1.n)), fl1, want_status=True)
    assert np.array_equal(after[0].view(np.int64), before[0].view(np.int64)) and np.array_equal(after[1], before[1])


# ---------------------------------------------------------------------------------------------------------------------------------
# 5. Reads of 6 400+ bases in a flank-state call
# ---------------------------------------------------------------------------------------------------------------------------------

@pytest.mark.parametrize("longest", [6399, 6400])
@pytest.mark.parametrize("band", [16, 32])
def test_long_reads_keep_flank_candidates(engine, coracle, band, longest):
    """The wide list's flank kernels hold a warp's row entries of the call's longest read in shared memory: above 6 399 bases they
    do not run, and the classify pass must then send the wide list's near-flank candidates to the traceback queue. Haplotypes of
    7 000 bases with flanks of 3 000 on each side (most windows meet a flank). Reads: two of `longest` bases (quality 30 and quality 2,
    quality sum 12 800), four of 1 100-2 000 bases with quality sums at most 13 312, and 20 of 150 bases at quality 30; with and
    without int scores (every read on the wide list)."""
    rng = np.random.default_rng(64000 + band + longest)
    haps, _ = random_region(rng, band, n_haps=4, n_reads=1, hap_len=7000, read_len_choices=[150], edge_reads=False)
    specs = ([(longest, 30, False), (longest, 2, False), (1100, (2, 10), False), (1400, (2, 9), False), (1700, (2, 7), False),
              (2000, (2, 6), False)] + [(150, 30, False)] * 20)
    reads = _reads(rng, haps, specs, band)
    qsum = np.add.reduceat(reads.quals.astype(np.int64), reads.off[:-1])
    assert (qsum[1:6] <= 13312).all() and qsum[1] == 2 * longest
    for int_scores in (False, True):
        for dp_only in (False, True):             # dp_only: no candidate is settled by the shortcut, every one reaches a DP
            populate_legs(engine, coracle, band, haps, reads, None, (3000, 3000), (band, longest, int_scores, dp_only), dp_only=dp_only,
                          max_indel_error=band, use_int_scores=int_scores)
