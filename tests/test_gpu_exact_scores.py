"""Exact scores where the kernels' arithmetic changes, and the FP64 finish against a high-precision reference, on the GPU.

(a) Every mapping quality 0..255, penalties from 0 to about 27 000, five cap / trigger settings, through every finish: direct
    mode (k_mapq_terms + the DP kernel), the classify path (k_epilogue), reads with 'N' (k_list_slots), qualities above 127 (the
    generic kernel), align_reads and populate_templates; each held to 4 eps (1 + c|s| + c mapq) of the exact value.
(b) The routing thresholds, mapping quality off, bit-exact: quality sums 27 648 / 27 649 (kMaxScore16), 13 312 / 13 313
    (kMaxScoreFlank32), lengths 1 023 / 1 024 and 28 000 / 28 001, quality 127 / 128, on inputs built so that the 16-bit lanes
    carry the largest values they can meet (the optimum is the quality sum, intermediate values reach it + 254).
(c) dp_pair's first and last 2B columns (the ramps) in direct mode and align_scores, both deletion forms, G = 1, 2, 4."""
import numpy as np
import pytest

from exact import C, assert_same_penalties, assert_sums_within_bound, effective_mapq, penalties
from helpers import ACGT
from test_gpu_parity import _oracle_scores, align_reads_legs, populate_legs

pytestmark = pytest.mark.gpu

CAPS = [(120, None), (60, 40), (60, 60), (50, 200), (120, 0)]


def _haps(seqs, rng, go=None, ge=None, mask=None, prior=None):
    from octopus_b200.batch import pack_haplotypes
    n = [len(s) for s in seqs]
    return pack_haplotypes(seqs,
                           mask if mask is not None else [np.roll(s, 1) for s in seqs],
                           prior if prior is not None else [rng.integers(1, 126, k).astype(np.int8) for k in n],
                           mask if mask is not None else [np.roll(s, -1) for s in seqs],
                           prior if prior is not None else [rng.integers(1, 126, k).astype(np.int8) for k in n],
                           go if go is not None else [rng.integers(3, 46, k).astype(np.int8) for k in n],
                           ge if ge is not None else [rng.integers(1, 11, k).astype(np.int8) for k in n],
                           begin=np.zeros(len(seqs), np.int64))


# ------------------------------------------------------------------------------------------------------------------------------
# (a) the finish
# ------------------------------------------------------------------------------------------------------------------------------
def _finish_region(rng, band, n_reads=256, L=200, n_rate=0.0, qmax=127, hap_len=600, n_haps=6):
    """Reads at every mapping quality: copies of a haplotype with 0..k mismatches (penalties 0 up to a few thousand) and unrelated
    reads of high quality (beyond 10 000)."""
    from octopus_b200.batch import pack_reads
    base = ACGT[rng.integers(0, 4, hap_len)]
    seqs = []
    for h in range(n_haps):
        s = base.copy(); s[rng.integers(0, hap_len, h)] = ACGT[rng.integers(0, 4, h)]; seqs.append(s)
    bases, quals, begin = [], [], []
    for r in range(n_reads):
        p = int(rng.integers(band, hap_len - L - band))
        if r % 4 == 3:
            b = ACGT[rng.integers(0, 4, L)].copy()
            q = rng.integers(max(2, qmax - 10), qmax + 1, L)
        else:
            b = base[p:p + L].copy()
            k = int(rng.integers(0, 40)) if r % 4 else int(rng.integers(0, 3))
            b[rng.integers(0, L, k)] = ACGT[rng.integers(0, 4, k)]
            q = rng.integers(2, min(qmax, 60) + 1, L)
        if rng.random() < n_rate:
            b[rng.integers(0, L)] = ord("N")
        bases.append(b); quals.append(q.astype(np.uint8)); begin.append(p)
    reads = pack_reads(bases, quals, mapq=(np.arange(n_reads) % 256).astype(np.uint8), reverse=(rng.random(n_reads) < 0.5).astype(np.uint8),
                       begin=np.asarray(begin, np.int64))
    full = lambda v, d: [np.full(hap_len, v, d) for _ in seqs]     # gaps dearer than any mismatch: unrelated reads cost about their quality sum
    return _haps(seqs, rng, go=full(127, np.int8), ge=full(127, np.int8), mask=full(ord("N"), np.uint8), prior=full(127, np.int8)), reads


def test_finish_matches_high_precision_reference(engine, coracle):
    rng = np.random.default_rng(2024)
    worst = {}
    band = 16
    plain = _finish_region(rng, band)
    with_n = _finish_region(rng, band, n_rate=0.5)
    high_q = _finish_region(rng, band, n_reads=64, L=120, qmax=255)
    top = 0
    for cap, trig in CAPS:
        for name, (haps, reads), kw in (("direct", plain, dict(dp_only=True)), ("epilogue", plain, dict(map_positions=True)),
                                        ("n_slots", with_n, dict(dp_only=True)), ("generic", high_q, dict(dp_only=True))):
            rc, want, wst, w = populate_legs(engine, coracle, band, haps, reads, None, None, (name, cap, trig), cap=cap, trig=trig,
                                             max_indel_error=band, **kw)
            worst[name] = max(worst.get(name, 0.0), w)
            top = max(top, int(penalties(want[wst == 0]).max()))
    assert top > 10000
    assert (np.asarray(with_n[1].bases) == ord("N")).any()

    # align_reads (k_align_reads) at every mapping quality, the trigger rule applied
    haps, reads = plain
    pairs = np.array([(r, r % haps.n) for r in range(reads.n)], np.int32)
    positions = (np.arange(reads.n + 1, dtype=np.int64), reads.begin.astype(np.int32))
    for trig in (None, 40):
        align_reads_legs(engine, coracle, band, band, haps, reads, pairs, positions, positions[0], None, trig=trig, what=("align_reads", trig))

    # populate_templates: sums of mixed values, an additive bound
    from octopus_b200 import HaplotypeLikelihoodModel
    toff = np.arange(0, reads.n + 1, 3, dtype=np.int64)
    toff[-1] = reads.n
    rc, per_read, wst = coracle.populate(band, haps, reads, None, None, use_mapping_quality=False)
    for cap, trig in CAPS:
        got = engine.populate_templates(HaplotypeLikelihoodModel.Config(max_indel_error=band, mapping_quality_cap=cap,
                                                                        mapping_quality_cap_trigger=trig, map_positions=False), haps, reads, toff)
        w = assert_sums_within_bound(got, penalties(per_read), effective_mapq(reads.mapq, cap, trig)[None, :], toff, ("templates", cap, trig))
        worst["templates"] = max(worst.get("templates", 0.0), w)
    print("largest finish error on this GPU, in units of eps (1 + c|s| + c mapq) (templates: fraction of their bound): %s" % worst)


# ------------------------------------------------------------------------------------------------------------------------------
# (b) routing thresholds, worst case for the 16-bit lanes
# ------------------------------------------------------------------------------------------------------------------------------
def _worst_region(rng, band, reads_spec, n_haps):
    """Haplotypes of A / C only, reads of G / T only, SNV masks that never match, gap open / extend 127: every alignment's optimum
    is its quality sum. reads_spec: list of quality arrays; every read begins at `band` (its window starts at 0)."""
    from octopus_b200.batch import pack_reads
    hap_len = max(len(q) for q in reads_spec) + 2 * band + 8
    seqs = [ACGT[rng.integers(0, 2, hap_len)].copy() for _ in range(n_haps)]
    full = lambda v, d: [np.full(hap_len, v, d) for _ in seqs]
    haps = _haps(seqs, rng, go=full(127, np.int8), ge=full(127, np.int8), mask=full(ord("N"), np.uint8), prior=full(127, np.int8))
    bases = [ACGT[rng.integers(2, 4, len(q))].copy() for q in reads_spec]
    reads = pack_reads(bases, [np.asarray(q, np.uint8) for q in reads_spec], mapq=np.full(len(bases), 60, np.uint8),
                       begin=np.full(len(bases), band, np.int64))
    return haps, reads


def _q(L, q=127, tail=()):
    a = np.full(L, q, np.int64)
    for i, v in enumerate(tail):
        a[1 + 7 * i] = v
    return a


THRESHOLD_READS = {
    "qsum16": [_q(218, tail=[88]), _q(218, tail=[89]), _q(218, tail=[90])],                       # 27 647 / 27 648 / 27 649
    "qsum_flank": [_q(105, tail=[103]), _q(105, tail=[104]), _q(105, tail=[105])],                # 13 311 / 13 312 / 13 313
    "length_bins": [_q(1022, 20), _q(1023, 20), _q(1024, 20)],
    "quality_8bit": [_q(150), _q(150, tail=[128]), _q(150, tail=[128, 200, 255])],
}


@pytest.mark.parametrize("band", [8, 16, 32, 64])
def test_routing_thresholds_are_exact(engine, coracle, band):
    rng = np.random.default_rng(band)
    nuc = 127
    for name, spec in THRESHOLD_READS.items():
        for n_haps in ((5, 20) if band >= 32 else (5,)):
            haps, reads = _worst_region(rng, band, spec, n_haps)
            sums = np.array([int(q.sum()) for q in spec])
            flank_sets = [None, (band + 20, 30)] if name == "qsum_flank" else [None]
            for flanks in flank_sets:
                for kw in (dict(dp_only=True), dict(map_positions=True), dict(dp_only=True, use_int_scores=True)):
                    what = (band, name, n_haps, flanks, kw)
                    rc, want, wst = _legs_nuc(engine, coracle, band, haps, reads, flanks, what, nuc, kw)
                    if flanks is None and name != "quality_8bit":
                        assert np.array_equal(want, np.broadcast_to(-C * sums.astype(np.float64), want.shape)), what    # the construction
            tasks = np.array([(r, h, 0, 0) for r in range(reads.n) for h in range(haps.n)], np.int32)
            ref = _oracle_scores(coracle, haps, reads, band, tasks, nuc)
            if name != "quality_8bit":
                assert np.array_equal(ref, sums[tasks[:, 0]])
            for bits in (16, 32):
                got = engine.align_scores(band, haps, reads, tasks, nuc_prior=nuc, precision_bits=bits)
                assert np.array_equal(got, ref), (band, name, bits, got[got != ref][:5], ref[got != ref][:5])
            if name != "length_bins" or band <= 32:
                pairs = np.array([(r, h) for r in range(reads.n) for h in range(haps.n)], np.int32)
                positions = (np.arange(len(pairs) + 1, dtype=np.int64), np.full(len(pairs), band, np.int32))
                _align_reads_exact(engine, coracle, band, haps, reads, pairs, positions, nuc, (band, name))


def _legs_nuc(engine, coracle, band, haps, reads, flanks, what, nuc, kw):
    """The exact leg alone (mapping quality off) with a nuc_prior other than 2."""
    from octopus_b200 import HaplotypeLikelihoodModel
    dp_only, mapit = kw.get("dp_only", False), kw.get("map_positions", False)
    rc, want, wst = coracle.populate(band, haps, reads, None, flanks, use_mapping_quality=False, nuc_prior=nuc, dp_only=dp_only,
                                     map_positions=mapit)
    cfg = HaplotypeLikelihoodModel.Config(max_indel_error=band, use_mapping_quality=False, nuc_prior=nuc, disable_naive_shortcut=dp_only,
                                          map_positions=mapit, use_int_scores=kw.get("use_int_scores", False))
    got, st = engine.populate(cfg, haps, reads, None, flanks, want_status=True)
    assert_same_penalties(got, want, st, wst, what)
    return rc, want, wst


def _align_reads_exact(engine, coracle, band, haps, reads, pairs, positions, nuc, what):
    from octopus_b200 import HaplotypeLikelihoodModel
    cfg = HaplotypeLikelihoodModel.Config(max_indel_error=band, use_mapping_quality=False, nuc_prior=nuc)
    mp, lk, cig, st = engine.align_reads(cfg, haps, reads, pairs, positions)
    for j, (r, h) in enumerate(pairs):
        hp = haps.hap(int(h)); b, q = reads.read(int(r))
        wst, wmp, wlk, wcig, _ = coracle.model_align(band, hp["seq"].tobytes(), b.tobytes(), q, hp["gap_open"], hp["gap_extend"],
                                                     hp["snv_mask_fwd"].tobytes(), hp["snv_prior_fwd"], [band], band, nuc_prior=nuc,
                                                     use_mapping_quality=False)
        assert wst == 0 and st[j] == 0, (what, j)
        assert (mp[j], cig[j]) == (wmp, wcig) and lk[j] == wlk, (what, j, mp[j], wmp, lk[j], wlk)


def test_wide_kernel_length_limit_is_exact(engine, coracle):
    """Reads of 28 000 and 28 001 bases (the wide kernel's row limit), low quality so the penalty stays small."""
    rng = np.random.default_rng(28000)
    for band in (16, 64):
        haps, reads = _worst_region(rng, band, [_q(27999, 1), _q(28000, 1), _q(28001, 1)], 2)
        for kw in (dict(dp_only=True), dict(dp_only=True, use_int_scores=True)):
            rc, want, wst = _legs_nuc(engine, coracle, band, haps, reads, None, (band, kw), 127, kw)
            assert np.array_equal(want, np.broadcast_to(-C * np.array([27999.0, 28000.0, 28001.0]), want.shape))


# ------------------------------------------------------------------------------------------------------------------------------
# (c) the ramps of dp_pair on the GPU
# ------------------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("bands", [(8, 16), (32, 64)])
def test_ramp_columns_on_the_gpu(engine, coracle, bands):
    """test_emul_ramps's cases, each as a haplotype equal to its window plus one base and a read that begins at the band, so that
    the direct-mode window is the case's window: L = 1 .. 2B + 8 and 150, optima at the window's ends, indels within 2B of
    either end. Odd read counts at odd L (the pairing scheduler's pad partner). One call per form: gap_extend <= gap_open
    everywhere, and one haplotype with a single column where go < ge (the general form for the whole call)."""
    from octopus_b200 import HaplotypeLikelihoodModel
    from octopus_b200.batch import concat_blocks, pack_reads
    from test_emul_ramps import KINDS, _case
    for band in bands:
        rng = np.random.default_rng(7 * band)
        for H in (20, 12, 5):
            for general in (False, True):
                hap_blocks, read_blocks = [], []
                for L in list(range(1, 2 * band + 9)) + [150]:
                    cases = [_case(rng, band, L, KINDS[k % len(KINDS)]) for k in range(H)]
                    if general and L == 2 * band:
                        cases[0]["gap_open"][band] = 1; cases[0]["gap_extend"][band] = 10
                    ext = lambda a, v: np.concatenate([a, np.asarray([v], a.dtype)])
                    hap_blocks.append(_haps([ext(c["truth"], ord("A")) for c in cases], rng, go=[ext(c["gap_open"], 40) for c in cases],
                                            ge=[ext(c["gap_extend"], 3) for c in cases], mask=[ext(c["snv_mask"], ord("N")) for c in cases],
                                            prior=[ext(c["snv_prior"], 60) for c in cases]))
                    nr = H - (L % 2)
                    read_blocks.append(pack_reads([c["read"] for c in cases[:nr]], [c["quals"] for c in cases[:nr]],
                                                  mapq=np.full(nr, 60, np.uint8), begin=np.full(nr, band, np.int64)))
                haps, reads, hf, rf = concat_blocks(hap_blocks, read_blocks)
                cfg = HaplotypeLikelihoodModel.Config(max_indel_error=band, use_mapping_quality=False, disable_naive_shortcut=True,
                                                      map_positions=False)
                flat, off, st = engine.populate_regions(cfg, haps, reads, hf, rf, want_status=True)
                mats, sts = engine.split_regions(flat, off, hf, rf), engine.split_regions(st, off, hf, rf)
                for g, (h, r) in enumerate(zip(hap_blocks, read_blocks)):
                    rc, want, wst = coracle.populate(band, h, r, None, None, use_mapping_quality=False, dp_only=True, map_positions=False)
                    assert_same_penalties(mats[g], want, sts[g], wst, (band, H, general, g))
                tasks = np.array([(int(rf[g]) + j, int(hf[g]) + j, 0, 0) for g in range(len(hap_blocks)) for j in range(int(rf[g + 1] - rf[g]))], np.int32)
                want = _oracle_scores(coracle, haps, reads, band, tasks, 2)
                got = engine.align_scores(band, haps, reads, tasks, nuc_prior=2)
                assert np.array_equal(got, want), (band, H, general, np.nonzero(got != want)[0][:10])
