"""compute_haplotype_support over paired / linked templates on the GPU (phmm_assign_templates, phmm_batcher_assign_templates,
PairHMMEngine / PopulateBatcher.assign_templates, the C++ adapter's compute_haplotype_support(TemplateBlock, ...)). The oracle is
tests/test_gpu_assign.py's per read (the reference's evaluate at its uncapped mapped positions), then each template's sum in read order
from 0.0, then the C restatement of find_map_haplotypes over the template sums plus the priors."""
import ctypes as C
import os
import subprocess
import tempfile

import numpy as np
import pytest

from exact import assert_mix_within_bound, effective_mapq, penalties
from find_map_oracle import find_map, find_map_all
from test_gpu_assign import _sub, filter_call, group_block, oracle_values, random_priors, slot_mapq
from helpers import ACGT
from test_gpu_batcher_align import _homopolymer_request, _outcome, _same, assign_request, realign_request, through_batcher
from test_gpu_batcher_align import run as run_other

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _cfg(band_req, use_mq, map_positions=True):
    from octopus_b200 import HaplotypeLikelihoodModel
    return HaplotypeLikelihoodModel.Config(max_indel_error=band_req, use_mapping_quality=use_mq, map_positions=map_positions)


def make_templates(rng, rf, max_reads=3):
    """Each group's reads cut into templates of 1..max_reads reads: (template_off int64, template_first int32)."""
    toff, tf = [0], [0]
    for g in range(len(rf) - 1):
        r = int(rf[g])
        while r < int(rf[g + 1]):
            r = min(int(rf[g + 1]), r + int(rng.integers(1, max_reads + 1)))
            toff.append(r)
        tf.append(len(toff) - 1)
    return np.array(toff, np.int64), np.array(tf, np.int32)


def template_sums(values, hf, rf, toff, tf):
    """The groups' [H_g][T_g] template values from the flat per-read [H_g][R_g] values: each template's reads summed left to right
    from 0.0."""
    out, slot = [], 0
    for g in range(len(hf) - 1):
        nh, r0, nr = int(hf[g + 1] - hf[g]), int(rf[g]), int(rf[g + 1] - rf[g])
        m = values[slot:slot + nh * nr].reshape(nh, nr)
        for k in range(nh):
            for t in range(int(tf[g]), int(tf[g + 1])):
                acc = 0.0
                for r in range(int(toff[t]), int(toff[t + 1])):
                    acc += float(m[k, r - r0])
                out.append(acc)
        slot += nh * nr
    return np.array(out, np.float64)


def _bits(x):
    return np.ascontiguousarray(x).view(np.int64)


@pytest.mark.parametrize("band_req", [8, 16, 32])
def test_templates_equal_reference_composition(engine, refhmm, coracle, band_req):
    rng = np.random.default_rng(7100 + band_req)
    haps, reads, hf, rf = filter_call(rng, 5)
    toff, tf = make_templates(rng, rf)
    assert set(np.diff(toff)) == {1, 2, 3}
    want, wst, _ = oracle_values(refhmm, coracle, band_req, haps, reads, hf, rf)
    assert (wst == 0).all()
    sums = template_sums(want, hf, rf, toff, tf)
    for trial in range(2):
        pri = random_priors(rng, haps.n) if trial else None
        if pri is not None:
            pri[int(rng.integers(0, haps.n))] = -np.inf
        top, lnl, st = engine.assign_templates(_cfg(band_req, False), haps, reads, toff, hf, tf, pri, want_likelihoods=True, want_status=True)
        assert (st == 0).all() and st.shape == wst.shape
        assert np.array_equal(_bits(lnl), _bits(sums)), (band_req, trial)
        assert np.array_equal(top, find_map_all(sums, hf, tf, pri)), (band_req, trial)
        # mapping quality on: the per-read values within the existing bound, the template values their sums
        top1, lnl1 = engine.assign_templates(_cfg(band_req, True), haps, reads, toff, hf, tf, pri, want_likelihoods=True)
        _, per_read = engine.assign_reads(_cfg(band_req, True), haps, reads, hf, rf, pri, want_likelihoods=True)
        assert_mix_within_bound(per_read, penalties(want), effective_mapq(slot_mapq(reads, hf, rf)), (band_req, trial, "mapq"))
        assert np.array_equal(_bits(lnl1), _bits(template_sums(per_read, hf, rf, toff, tf)))
        assert np.array_equal(top1, find_map_all(lnl1, hf, tf, pri)), (band_req, trial, "mapq")
        assert np.array_equal(engine.assign_templates(_cfg(band_req, True), haps, reads, toff, hf, tf, pri), top1)


def test_single_read_templates_equal_assign_reads(engine):
    rng = np.random.default_rng(7201)
    haps, reads, hf, rf = filter_call(rng, 8)
    toff = np.arange(reads.n + 1, dtype=np.int64)
    pri = random_priors(rng, haps.n)
    for cfg in (_cfg(16, True), _cfg(8, False), _cfg(32, True, map_positions=False)):
        t = engine.assign_templates(cfg, haps, reads, toff, hf, rf, pri, want_likelihoods=True, want_status=True)
        r = engine.assign_reads(cfg, haps, reads, hf, rf, pri, want_likelihoods=True, want_status=True)
        assert t[0].tobytes() == r[0].tobytes()
        assert np.array_equal(t[2], r[2])
        assert (t[1] == r[1]).all()


def test_map_positions_off_equals_populate_templates(engine):
    rng = np.random.default_rng(7301)
    haps, reads = group_block(rng, 3, 120, 600)
    toff, tf = make_templates(rng, [0, reads.n])
    for mq in (False, True):
        cfg = _cfg(16, mq, map_positions=False)
        _, lnl = engine.assign_templates(cfg, haps, reads, toff, [0, haps.n], tf, want_likelihoods=True)
        want = engine.populate_templates(cfg, haps, reads, toff)
        assert np.array_equal(_bits(lnl), _bits(want.reshape(-1)))


def _tsub(haps, reads, hf, rf, toff, tf, g0, g1):
    """Groups [g0, g1) with their templates as a call of their own."""
    hs, rs, hf1, rf1 = _sub(haps, reads, hf, rf, g0, g1)
    t0, t1 = int(tf[g0]), int(tf[g1])
    return hs, rs, toff[t0:t1 + 1] - toff[t0], hf1, (tf[g0:g1 + 1] - t0).astype(np.int32)


def _tcall(engine, cfg, haps, reads, toff, hf, tf, pri):
    return engine.assign_templates(cfg, haps, reads, toff, hf, tf, pri, want_likelihoods=True, want_status=True)


def test_many_groups_equal_one_call_per_group_and_device_equals_host(engine):
    from octopus_b200.batch import concat_blocks
    rng = np.random.default_rng(7401)
    sizes = [(1, 30), (64, 12), (2, 1), (3, 2), (5, 25), (2, 300), (17, 4), (1, 1), (33, 9), (3, 150)]
    blocks = [group_block(rng, nh, nr, int(rng.integers(400, 801)), repeat=(i % 3 == 0)) for i, (nh, nr) in enumerate(sizes)]
    haps, reads, hf, rf = concat_blocks([b[0] for b in blocks], [b[1] for b in blocks])
    toff, tf = make_templates(rng, rf)
    pri = random_priors(rng, haps.n)
    for cfg in (_cfg(16, True), _cfg(8, False), _cfg(32, True, map_positions=False)):
        whole = _tcall(engine, cfg, haps, reads, toff, hf, tf, pri)
        parts = [_tcall(engine, cfg, *_tsub(haps, reads, hf, rf, toff, tf, g, g + 1), pri[int(hf[g]):int(hf[g + 1])]) for g in range(len(sizes))]
        for i in range(3):
            assert np.concatenate([p[i] for p in parts]).tobytes() == whole[i].tobytes(), (cfg.max_indel_error, i)
        assert whole[0][int(tf[1]):int(tf[2])].max() >= 1 << 32          # the 64-haplotype group's upper bits are used
    import torch
    hd, rd = haps.to_device("cuda:0"), reads.to_device("cuda:0")
    cfg = _cfg(16, True)
    host = _tcall(engine, cfg, haps, reads, toff, hf, tf, pri)
    dev = engine.assign_templates(cfg, hd, rd, torch.as_tensor(toff, device="cuda:0"), hf, tf, torch.as_tensor(pri, device="cuda:0"),
                                  want_likelihoods=True, want_status=True)
    assert all(t.is_cuda for t in dev)
    assert dev[0].cpu().numpy().tobytes() == host[0].tobytes()
    assert dev[1].cpu().numpy().tobytes() == host[1].tobytes()
    assert np.array_equal(dev[2].cpu().numpy(), host[2])
    assert engine.assign_templates(cfg, hd, rd, toff, hf, tf, pri).cpu().numpy().tobytes() == host[0].tobytes()


def test_one_large_group_spreads_over_the_grid(engine):
    """One genotype of 64 haplotypes with 2 000 templates next to small ones: the choice runs one thread per template, and every
    template of the large group gets its sums and its set."""
    from octopus_b200.batch import concat_blocks
    rng = np.random.default_rng(7451)
    blocks = [group_block(rng, 2, 7, 500), group_block(rng, 64, 4000, 600, duplicate=False), group_block(rng, 3, 5, 450)]
    haps, reads, hf, rf = concat_blocks([b[0] for b in blocks], [b[1] for b in blocks])
    toff, tf = make_templates(rng, rf)
    assert int(tf[2] - tf[1]) > 1500
    pri = random_priors(rng, haps.n)
    cfg = _cfg(8, True)
    top, lnl = engine.assign_templates(cfg, haps, reads, toff, hf, tf, pri, want_likelihoods=True)
    _, per_read = engine.assign_reads(cfg, haps, reads, hf, rf, pri, want_likelihoods=True)
    sums = template_sums(per_read, hf, rf, toff, tf)
    assert np.array_equal(_bits(lnl), _bits(sums))
    assert np.array_equal(top, find_map_all(sums, hf, tf, pri))


def up(x, n):
    for _ in range(n):
        x = float(np.nextafter(x, np.inf))
    return x


def test_constructed_ties(engine):
    from octopus_b200.batch import concat_blocks
    rng = np.random.default_rng(7501)
    # duplicate haplotypes: equal template sums, every copy in the set, with -inf priors leaving the set or emptying it
    blocks = [group_block(rng, int(rng.integers(2, 6)), int(rng.integers(5, 40)), 500, duplicate=True) for _ in range(8)]
    haps, reads, hf, rf = concat_blocks([b[0] for b in blocks], [b[1] for b in blocks])
    toff, tf = make_templates(rng, rf)
    top, lnl = engine.assign_templates(_cfg(16, True), haps, reads, toff, hf, tf, want_likelihoods=True)
    nh = np.repeat(np.diff(hf), np.diff(tf))
    assert np.array_equal(top, ((1 << nh.astype(np.uint64)) - 1).astype(np.uint64))
    pri = np.zeros(haps.n)
    pri[hf[:-1]] = -np.inf
    pri[hf[2]:hf[3]] = -np.inf                    # group 2: every prior -inf, an empty set becomes every haplotype
    top = engine.assign_templates(_cfg(16, True), haps, reads, toff, hf, tf, pri)
    assert np.array_equal(top, find_map_all(lnl, hf, tf, pri))
    assert np.array_equal(top[int(tf[2]):int(tf[3])], np.full(int(tf[3] - tf[2]), (1 << int(nh[tf[2]])) - 1, np.uint64))
    # two-read templates of three copies; the priors move the copies' sums to chosen ulp distances: both sides of the almost_equal
    # boundary and the maximum an almost-equal value does not raise
    blocks = [group_block(rng, 3, 2, 450, duplicate=True) for _ in range(40)]
    haps, reads, hf, rf = concat_blocks([b[0] for b in blocks], [b[1] for b in blocks])
    toff, tf = np.arange(0, reads.n + 1, 2, dtype=np.int64), np.arange(0, len(blocks) + 1, dtype=np.int32)
    _, v = engine.assign_templates(_cfg(8, True), haps, reads, toff, hf, tf, want_likelihoods=True)
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
    top = engine.assign_templates(_cfg(8, True), haps, reads, toff, hf, tf, pri)
    sums = v.repeat(3) + pri
    for g in range(len(v)):
        assert int(top[g]) == find_map(sums[3 * g:3 * g + 3]), g
        if expect.get(g) is not None:
            assert int(top[g]) == expect[g], (g, float(v[g]), int(top[g]))
    assert sum(e is not None for e in expect.values()) >= 20


def test_short_haplotype_as_assign_reads(engine):
    from octopus_b200 import ShortHaplotypeError
    from octopus_b200.batch import concat_blocks, pack_haplotypes, pack_reads
    rng = np.random.default_rng(7601)
    g1 = group_block(rng, 2, 20, 500)
    base = ACGT[rng.integers(0, 4, 300)].copy()
    seqs = [base[20:80].copy(), base[:300].copy()]
    sh = pack_haplotypes(seqs, seqs, [np.full(len(s), 40, np.int8) for s in seqs], seqs, [np.full(len(s), 40, np.int8) for s in seqs],
                         [np.full(len(s), 20, np.int8) for s in seqs], [np.full(len(s), 3, np.int8) for s in seqs], begin=np.zeros(2, np.int64))
    sr = pack_reads([base[30:80].copy(), base[100:150].copy(), base[10:60].copy()], [np.full(50, 30, np.uint8)] * 3,
                    mapq=np.full(3, 60, np.uint8), reverse=np.array([0, 1, 0], np.uint8), begin=np.array([30, 100, 10], np.int64))
    haps, reads, hf, rf = concat_blocks([g1[0], sh], [g1[1], sr])
    toff, tf = make_templates(rng, rf)
    cfg = _cfg(16, True)
    with pytest.raises(ShortHaplotypeError) as t_err:
        engine.assign_templates(cfg, haps, reads, toff, hf, tf)
    with pytest.raises(ShortHaplotypeError) as r_err:
        engine.assign_reads(cfg, haps, reads, hf, rf)
    assert t_err.value.code == r_err.value.code and str(t_err.value) == str(r_err.value)
    _, st = engine.assign_templates(cfg, haps, reads, toff, hf, tf, want_status=True)
    _, want = engine.assign_reads(cfg, haps, reads, hf, rf, want_status=True)
    assert np.array_equal(st, want) and ((st & 0xFFFF) == 2).sum() >= 2


def test_argument_checks(engine):
    """Every host check of phmm_assign_templates, with its message, through the C entry point."""
    from octopus_b200 import PhmmError
    from octopus_b200.api import _config, _regions
    rng = np.random.default_rng(7701)
    haps, reads, hf, rf = filter_call(rng, 3)
    toff, tf = make_templates(rng, rf)
    cfg = _cfg(16, True)
    top = np.zeros(len(toff) - 1, np.uint64)
    lib, h = engine._lib, engine._h

    def call(off, n, groups=(hf, rf), out=top):
        regs, _ = _regions(*groups)
        o = None if off is None else np.ascontiguousarray(off, np.int64)
        rc = lib.phmm_assign_templates(h, _config(cfg), C.byref(haps.c_struct()), C.byref(reads.c_struct()), C.byref(regs),
                                       None if o is None else o.ctypes.data, n, None, None if out is None else out.ctypes.data, None, None, 0)
        return rc, lib.phmm_last_error(h).decode()

    T = len(toff) - 1
    assert call(toff, T)[0] == 0
    bad = toff.copy(); bad[-1] += 1
    inc = toff.copy(); inc[1] = inc[0]
    dec = toff.copy(); dec[2], dec[1] = dec[1], dec[2]
    inside = np.delete(toff, int(tf[1]))            # the template at group 1's first read now starts in group 0
    for args, msg in (((None, T), "null / empty template offsets"), ((toff, 0), "null / empty template offsets"),
                      ((bad, T), "cover the reads exactly"), ((toff[:-1], T - 1), "cover the reads exactly"),
                      ((inc, T), "strictly increasing"), ((dec, T), "strictly increasing"),
                      ((inside, T - 1), "group boundary falls inside a template")):
        rc, err = call(*args)
        assert rc == -1 and msg in err, (msg, rc, err)
    assert call(toff, T, out=None) == (-1, "null config / output")
    assert call(toff, T, groups=(hf, rf - [0, 0, 0, 1]))[1].startswith("region ranges must cover")
    # through the Python method: template_first must index template_off
    with pytest.raises(ValueError):
        engine.assign_templates(cfg, haps, reads, toff, hf, [0, 1, T + 5, T])
    with pytest.raises(PhmmError, match="more than 64 haplotypes"):
        h65, r65 = group_block(rng, 65, 3, 400)
        engine.assign_templates(cfg, h65, r65, [0, 2, 3], [0, 65], [0, 2])


# ---------------------------------------------------------------------------------------------------------------------
# the shared engine
# ---------------------------------------------------------------------------------------------------------------------
def template_request(rng, cfg=None):
    """assign_request's genotypes with their reads cut into templates of 1-3 reads."""
    _, kw = assign_request(rng, cfg)
    toff, tf = make_templates(rng, kw.pop("read_first"))
    kw.update(template_off=toff, template_first=tf)
    return ("templates", kw)


def run(target, request):
    kind, kw = request
    if kind == "templates":
        return _outcome(lambda: target.assign_templates(**kw))
    return run_other(target, request)


def _each_alone(engine, requests, got):
    for i, (q, g) in enumerate(zip(requests, got)):
        want = run(engine, q)
        if q[0] == "populate":
            assert g[0] == want[0] == "ok", (i, g, want)
            ok = want[1][1] == 0
            assert _same(g[1][1], want[1][1]) and g[1][0][ok].tobytes() == want[1][0][ok].tobytes(), i
        elif q[0] in ("assign", "templates") and want[0] == "ok" and ((want[1][-1] & 0xFFFF) == 2).any():
            assert g[0] == "ok" and _same(g[1][-1], want[1][-1]), i
        else:
            assert _same(g, want), (i, q[0], g if g[0] != "ok" else "values differ", want if want[0] != "ok" else "")


@pytest.mark.parametrize("n_threads", [1, 8, 32])
def test_concurrent_template_requests_equal_one_engine_each(engine, n_threads, monkeypatch):
    import test_gpu_batcher_align
    from helpers import random_region
    monkeypatch.setattr(test_gpu_batcher_align, "run", run)       # through_batcher sends template requests too
    rng = np.random.default_rng(7800 + n_threads)
    requests = []
    for i in range(48):
        k = i % 6
        if k in (0, 1, 2):
            requests.append(template_request(rng))
        elif k == 3:
            requests.append(assign_request(rng))
        elif k == 4:
            requests.append(realign_request(rng))
        else:
            haps, reads = random_region(rng, 16, int(rng.integers(2, 8)), int(rng.integers(20, 80)), 300, [100, 150])
            requests.append(("populate", dict(config=_cfg(16, True), haps=haps, reads=reads, want_status=True)))
    # a template request with more than 4096 mapping positions for one pair fails alone, not its batch's other members
    _, kw = _homopolymer_request(requests[0][1]["config"])
    kw.pop("read_first")
    kw.update(template_off=np.array([0, 2], np.int64), template_first=[0, 1])
    requests[6] = ("templates", kw)
    got, stats, reruns = through_batcher(requests, n_threads)
    assert got[6][0] == "PhmmError" and "4096" in got[6][2], got[6]
    _each_alone(engine, requests, got)
    if n_threads > 1:
        assert stats["merged_calls"] > 0, stats


@pytest.mark.parametrize("with_reads", [False, True])
def test_merged_template_calls_succeed_without_reruns(engine, with_reads, monkeypatch):
    """Requests that cannot fail, at one config, from 8 threads: a merged call is rerun member by member when it returns
    PHMM_ERR_INVALID, which would hide a batch built wrong behind correct solo results. Here no call may be rerun, and calls of more
    than one request must happen. Template requests alone: every merged call is a template call. With plain assign requests mixed
    in: the two kinds still merge cleanly, each only with its own kind."""
    import test_gpu_batcher_align
    monkeypatch.setattr(test_gpu_batcher_align, "run", run)
    rng = np.random.default_rng(7900 + with_reads)
    cfg = _cfg(16, True)
    requests = [assign_request(rng, cfg) if with_reads and i % 3 == 2 else template_request(rng, cfg) for i in range(32)]
    wants = [run(engine, q) for q in requests]
    assert all(w[0] == "ok" and ((w[1][-1] & 0xFFFF) == 0).all() for w in wants)
    got, stats, reruns = through_batcher(requests, 8, max_wait_us=200000)
    for i, (g, w) in enumerate(zip(got, wants)):
        assert _same(g, w), (i, requests[i][0])
    assert reruns == 0, (stats, reruns)
    assert stats["merged_calls"] > 0 and stats["max_regions_per_call"] > 1, stats


CPP_SRC = os.path.join(ROOT, "tests", "cpp", "test_assign_templates.cpp")


def test_cpp_template_support_on_engine_and_shared_engine(engine):
    from octopus_b200 import build
    build.build()
    exe = os.path.join(tempfile.mkdtemp(prefix="test_assign_templates_"), "test_assign_templates")
    subprocess.run(["g++", "-std=c++14", "-O1", "-pthread", "-I", os.path.join(ROOT, "include"), "-I", os.path.join(ROOT, "octopus_b200", "cpp"),
                    CPP_SRC, "-o", exe, "-L", os.path.join(ROOT, "octopus_b200"), "-lphmm_b200",
                    "-Wl,-rpath," + os.path.join(ROOT, "octopus_b200")], check=True)
    out = subprocess.run([exe], capture_output=True, text=True, timeout=600)
    assert out.returncode == 0 and "TEMPLATE SUPPORT ok" in out.stdout, out.stdout + out.stderr
