"""Read assignment and realignment through the shared engine (phmm_batcher_assign_reads / phmm_batcher_realign_reads,
PopulateBatcher.assign_reads / realign_reads, the C++ adapter's compute_haplotype_support / realign on a SharedEngine): requests from
many threads merged into one assign or realign call, each with exactly the result it gets alone on an engine of its own."""
import os
import subprocess
import tempfile
import threading

import numpy as np
import pytest

from helpers import ACGT
from test_gpu_assign import group_block
from test_gpu_realign import pack

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _cfg(band, use_mq, map_positions=True, use_flank_state=False):
    from octopus_b200 import HaplotypeLikelihoodModel
    return HaplotypeLikelihoodModel.Config(max_indel_error=band, use_mapping_quality=use_mq, map_positions=map_positions,
                                           use_flank_state=use_flank_state)


def _outcome(call):
    """What a call returned, or the class, code and message of what it raised."""
    from octopus_b200 import PhmmError
    try:
        return ("ok", call())
    except PhmmError as e:
        return (type(e).__name__, e.code, str(e))


def _same(got, want):
    """Bit for bit: arrays by their bytes, CIGAR lists as lists, tuples member by member."""
    if isinstance(want, tuple):
        return isinstance(got, tuple) and len(got) == len(want) and all(_same(g, w) for g, w in zip(got, want))
    if isinstance(want, np.ndarray):
        return isinstance(got, np.ndarray) and got.dtype == want.dtype and got.shape == want.shape and got.tobytes() == want.tobytes()
    return got == want


# ---------------------------------------------------------------------------------------------------------------------
# requests: (kind, arguments); run(target, request) sends one through an engine or a batcher
# ---------------------------------------------------------------------------------------------------------------------
def assign_request(rng, cfg=None):
    """Genotypes of 2-4 haplotypes of 300-1 000 bp with 50-400 reads of 150 bp in all; band 8 or 16, mapping quality on or off,
    with and without priors and likelihoods."""
    from octopus_b200.batch import concat_blocks
    cfg = cfg or _cfg(int(rng.choice([8, 16])), bool(rng.integers(0, 2)))
    n_reads = int(rng.integers(50, 401))
    G = int(rng.integers(1, 4))
    sizes = np.diff(np.sort(np.concatenate([[0, n_reads], rng.choice(np.arange(1, n_reads), G - 1, replace=False)]))).astype(int)
    blocks = [group_block(rng, int(rng.integers(2, 5)), int(n), int(rng.integers(300, 1001)), duplicate=(rng.random() < 0.2)) for n in sizes]
    haps, reads, hf, rf = concat_blocks([b[0] for b in blocks], [b[1] for b in blocks])
    pri = np.log(rng.dirichlet(np.ones(haps.n))) if rng.random() < 0.5 else None
    return ("assign", dict(config=cfg, haps=haps, reads=reads, hap_first=hf, read_first=rf, log_priors=pri,
                           want_likelihoods=bool(rng.integers(0, 2)), want_status=True))


def realign_request(rng, cfg=None, lengths=(100, 150, 250, 300), long_read=False):
    """1-3 haplotypes of 300-1 000 bp (2 500 with long_read), 50-300 reads of a spread of lengths (one of 2 000 bp with long_read,
    over the register traceback's length cap), every read against one or two haplotypes, at the default or a random CIGAR stride."""
    cfg = cfg or _cfg(int(rng.choice([8, 16, 32])), bool(rng.integers(0, 2)), use_flank_state=bool(rng.integers(0, 2)))
    H = int(rng.integers(1, 4))
    hap_len = 2500 if long_read else int(rng.integers(300, 1001))
    base = ACGT[rng.integers(0, 4, hap_len)]
    seqs = []
    for _ in range(H):
        s = base.copy()
        s[rng.integers(0, hap_len, 3)] = ACGT[rng.integers(0, 4, 3)]
        seqs.append(s)
    R = int(rng.integers(50, 301))
    bases, begins = [], []
    for r in range(R):
        L = 2000 if long_read and r == 0 else 300 if long_read and r == 1 else min(int(rng.choice(lengths)), hap_len)
        p = int(rng.integers(0, hap_len - L + 1))
        b = base[p:p + L].copy()
        b[rng.integers(0, L, 2)] = ACGT[rng.integers(0, 4, 2)]
        bases.append(b)
        begins.append(p)
    haps, reads = pack(seqs, bases, rng, begins=begins)
    pairs = [(r, int(rng.integers(0, H))) for r in range(R)] + [(r, int(rng.integers(0, H))) for r in range(0, R, 3)]
    stride = None if rng.random() < 0.4 else int(rng.choice([8, 12, 24, 64, 200, 1300]))
    flank = (int(rng.integers(0, 40)), int(rng.integers(0, 40))) if rng.random() < 0.5 else None
    return ("realign", dict(config=cfg, haps=haps, reads=reads, pairs=np.array(pairs, np.int32), flank_state=flank, cigar_stride=stride))


def run(target, request):
    kind, kw = request
    if kind == "assign":
        return _outcome(lambda: target.assign_reads(**kw))
    if kind == "realign":
        return _outcome(lambda: target.realign_reads(**kw))
    if kind == "populate":
        return _outcome(lambda: target.populate(**kw))
    if kind == "mutation":
        return _outcome(lambda: target.mutation_prime(**kw))
    raise ValueError(kind)


def through_batcher(requests, n_threads, clients=None, max_wait_us=2000):
    """requests[i] on thread i % n_threads, all threads through one PopulateBatcher: (results, stats, reruns)."""
    from octopus_b200 import PopulateBatcher
    got = [None] * len(requests)
    errors = []
    with PopulateBatcher(0, clients=n_threads if clients is None else clients, max_wait_us=max_wait_us) as b:
        start = threading.Barrier(n_threads)

        def worker(k):
            try:
                start.wait()
                for i in range(k, len(requests), n_threads):
                    got[i] = run(b, requests[i])
            except Exception as e:          # noqa: BLE001 - reported below
                errors.append(repr(e))
        threads = [threading.Thread(target=worker, args=(k,)) for k in range(n_threads)]
        for t in threads:
            t.start()
        for t in threads:
            t.join()
        stats, reruns = b.stats(), b.reruns()
    assert not errors, errors
    return got, stats, reruns


def assert_each_alone(engine, requests, got):
    for i, (q, g) in enumerate(zip(requests, got)):
        want = run(engine, q)
        if q[0] == "assign" and want[0] == "ok" and ((want[1][-1] & 0xFFFF) == 2).any():
            assert g[0] == "ok" and _same(g[1][-1], want[1][-1]), i       # a short haplotype: only the statuses are specified
            continue
        assert _same(g, want), (i, q[0], g if g[0] != "ok" else "values differ", want if want[0] != "ok" else "")


# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("n_threads", [8, 32])
def test_concurrent_assign_requests_equal_one_engine_each(engine, n_threads):
    rng = np.random.default_rng(4100 + n_threads)
    requests = [assign_request(rng) for _ in range(3 * n_threads)]
    got, stats, reruns = through_batcher(requests, n_threads)
    assert_each_alone(engine, requests, got)
    assert stats["merged_calls"] > 0 and reruns == 0, stats


@pytest.mark.parametrize("n_threads", [8, 32])
def test_concurrent_realign_requests_equal_one_engine_each(engine, n_threads):
    rng = np.random.default_rng(4200 + n_threads)
    requests = [realign_request(rng) for _ in range(3 * n_threads)]
    # one request with a 300-bp read and a 2 000-bp read: its merged call crosses the register traceback's length cap
    requests[1] = realign_request(rng, cfg=requests[0][1]["config"], long_read=True)
    got, stats, reruns = through_batcher(requests, n_threads)
    assert_each_alone(engine, requests, got)
    assert stats["merged_calls"] > 0 and reruns == 0, stats
    assert any(g[0] == "ok" and ((g[1][3] & 0xFFFF) == 3).any() for g in got), "no request saw a truncated CIGAR"


def test_no_priors_and_zero_priors_choose_the_same(engine):
    rng = np.random.default_rng(4300)
    kind, kw = assign_request(rng, _cfg(16, True))
    kw.update(want_likelihoods=True, log_priors=None)
    without = engine.assign_reads(**kw)
    kw["log_priors"] = np.zeros(kw["haps"].n)
    zeros = engine.assign_reads(**kw)
    assert _same(without, zeros)


def _homopolymer_request(cfg):
    """A 150-base homopolymer read against a 5 000-base homopolymer haplotype: more than 4096 mapping positions for one pair."""
    from octopus_b200.batch import pack_haplotypes, pack_reads
    hp = np.full(5000, ord("A"), np.uint8)
    haps = pack_haplotypes([hp, hp], [hp, hp], [np.full(5000, 40, np.int8)] * 2, [hp, hp], [np.full(5000, 40, np.int8)] * 2,
                           [np.full(5000, 20, np.int8)] * 2, [np.full(5000, 3, np.int8)] * 2, begin=np.zeros(2, np.int64))
    reads = pack_reads([np.full(150, ord("A"), np.uint8)] * 2, [np.full(150, 30, np.uint8)] * 2, mapq=np.full(2, 60, np.uint8),
                       reverse=np.zeros(2, np.uint8), begin=np.zeros(2, np.int64))
    return ("assign", dict(config=cfg, haps=haps, reads=reads, hap_first=[0, 2], read_first=[0, 2], log_priors=None,
                           want_likelihoods=True, want_status=True))


def test_too_many_positions_fails_its_own_request_only(engine):
    rng = np.random.default_rng(4400)
    cfg = _cfg(16, True)
    requests = [assign_request(rng, cfg) for _ in range(8)]
    requests[3] = _homopolymer_request(cfg)
    got, stats, reruns = through_batcher(requests, 8, max_wait_us=500000)
    assert got[3][0] == "PhmmError" and "4096" in got[3][2], got[3]
    assert_each_alone(engine, requests, got)
    assert reruns >= 1 and stats["merged_calls"] > 0, (stats, reruns)


def test_short_haplotype_keeps_its_mates_top(engine):
    from octopus_b200.batch import concat_blocks
    rng = np.random.default_rng(4500)
    cfg = _cfg(8, False)
    requests = [assign_request(rng, cfg) for _ in range(6)]
    kw = dict(requests[2][1])
    h, r = group_block(rng, 2, 40, 400)
    short, _ = group_block(rng, 2, 1, 100)              # 100-bp haplotypes against 150-bp reads
    haps, reads, hf, rf = concat_blocks([h, short], [r, r])
    kw.update(haps=haps, reads=reads, hap_first=hf, read_first=rf, log_priors=None, want_status=False)
    requests[2] = ("assign", kw)
    got, stats, _ = through_batcher(requests, 6, max_wait_us=500000)
    assert got[2][0] == "ShortHaplotypeError", got[2]
    assert_each_alone(engine, requests, got)
    assert stats["merged_calls"] > 0, stats


def test_all_five_kinds_in_flight_at_once(engine):
    from octopus_b200 import ErrorModel, MutationModel
    from octopus_b200.batch import HaplotypeSequences
    from helpers import random_region
    rng = np.random.default_rng(4600)
    model = ErrorModel()
    o = np.full((11, 51), 1e-4, np.float32)
    e = np.full((11, 51, 50), 0.5, np.float32)
    mutation = MutationModel(1e-8, o, e)
    requests = []
    for i in range(40):
        k = i % 5
        if k == 0:
            requests.append(assign_request(rng, _cfg(16, True)))
        elif k == 1:
            requests.append(realign_request(rng, _cfg(16, True)))
        elif k in (2, 3):
            haps, reads = random_region(rng, 16, int(rng.integers(2, 8)), int(rng.integers(20, 80)), 300, [100, 150])
            kw = dict(config=_cfg(16, True), haps=haps, reads=reads, want_status=True)
            if k == 3:
                kw.update(haps=HaplotypeSequences.pack([haps.hap(h)["seq"].tobytes() for h in range(haps.n)], begin=haps.begin),
                          error_model=model)
            requests.append(("populate", kw))
        else:
            base = ACGT[rng.integers(0, 4, 200)]
            seqs = []
            for _ in range(int(rng.integers(2, 6))):
                s = base.copy()
                s[rng.integers(0, 200, 2)] = ACGT[rng.integers(0, 4, 2)]
                seqs.append(s.tobytes())
            requests.append(("mutation", dict(model=mutation, sequences=seqs)))
    got, stats, reruns = through_batcher(requests, 20)
    for i, (q, g) in enumerate(zip(requests, got)):
        want = run(engine, q)
        if q[0] == "populate":          # populate's values are specified at PHMM_STATUS_OK pairs
            assert g[0] == want[0] == "ok", (i, g, want)
            ok = want[1][1] == 0
            assert _same(g[1][1], want[1][1]) and g[1][0][ok].tobytes() == want[1][0][ok].tobytes(), i
        elif q[0] == "mutation":
            assert g[0] == want[0] == "ok", (i, g, want)
            keep = np.isin(want[1][1], [0, 1])
            assert _same(g[1][1], want[1][1]) and g[1][0][keep].tobytes() == want[1][0][keep].tobytes(), i
        else:
            assert _same(g, want), (i, q[0])
    assert stats["merged_calls"] > 0 and reruns == 0, stats


CPP_SRC = os.path.join(ROOT, "tests", "cpp", "test_batcher_align.cpp")


def test_cpp_shared_engine_support_and_realign_equal_an_engine_each(engine):
    from octopus_b200 import build
    build.build()
    exe = os.path.join(tempfile.mkdtemp(prefix="test_batcher_align_"), "test_batcher_align")
    subprocess.run(["g++", "-std=c++14", "-O1", "-pthread", "-I", os.path.join(ROOT, "include"), "-I", os.path.join(ROOT, "octopus_b200", "cpp"),
                    CPP_SRC, "-o", exe, "-L", os.path.join(ROOT, "octopus_b200"), "-lphmm_b200",
                    "-Wl,-rpath," + os.path.join(ROOT, "octopus_b200")], check=True)
    out = subprocess.run([exe], capture_output=True, text=True, timeout=600)
    assert out.returncode == 0 and "BATCHER ALIGN ok" in out.stdout, out.stdout + out.stderr
