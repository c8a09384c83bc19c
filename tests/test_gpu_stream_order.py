"""Ordering between the engine's stream and the caller's, for device-resident calls. Every call runs on the engine's own non-blocking
stream, so a call made while torch's current stream still has work queued must neither read an argument before the work that writes
it, nor write a block that queued work still reads. The API's own conversions, zero-fills and output allocations are that kind of
work, queued on torch's current stream right before the C call.

Each test queues a spin of about 0.2 s on the current stream, checks that it is still pending right before the call, puts the work
that produces the call's inputs behind it, and compares the result bit for bit with the host-space call on the final inputs (or, with
mapping quality off, with the oracle). Each call is warmed first at the same sizes with other valid content: no allocation inside it
then synchronises the device by accident, and whatever a lost ordering could expose is valid input the engine range-checks. The
tests avoid the API's host reads of device tensors (the default CIGAR stride, template offsets given as a tensor), which would drain
the stream first and hide a missing wait. Every test but the last runs on torch's default stream and on a side stream."""
import copy

import numpy as np
import pytest

from exact import assert_same_penalties
from helpers import random_region

pytestmark = pytest.mark.gpu

DEV = "cuda:0"
SPIN_CYCLES = 400_000_000           # about 0.2 s at the H100 SXM's 1.98 GHz boost clock; longer at lower clocks
BAND = 16


@pytest.fixture(params=["default stream", "side stream"])
def stream(request, engine):
    """Runs the test on torch's default stream, or on a stream of its own: the API must order after the current stream of the
    tensors' device, whichever it is."""
    import torch
    if request.param == "default stream":
        yield
    else:
        with torch.cuda.stream(torch.cuda.Stream(DEV)):
            yield
    torch.cuda.synchronize(DEV)


def busy():
    """Queue the spin on the current stream: work enqueued after it runs after the engine call has started."""
    import torch
    torch.cuda._sleep(SPIN_CYCLES)


def still_busy():
    import torch
    assert not torch.cuda.current_stream().query(), "the spin ended before the call, which then tests no ordering"


def _cfg(use_mq=True, map_positions=True):
    from octopus_b200 import HaplotypeLikelihoodModel
    return HaplotypeLikelihoodModel.Config(max_indel_error=BAND, use_mapping_quality=use_mq, map_positions=map_positions)


def _region(rng, n_haps=8, n_reads=64, hap_len=300):
    return random_region(rng, BAND, n_haps=n_haps, n_reads=n_reads, hap_len=hap_len, read_len_choices=[76, 100, 150], read_n_rate=0.05)


def _with_short_haplotype(haps, length=120):
    """The block with one more haplotype, a prefix of the first too short for the longer reads (status 2 for those pairs)."""
    from octopus_b200.batch import HaplotypeBlock, pack_haplotypes
    parts = [haps.hap(h) for h in range(haps.n)]
    parts.append({f: a[:length] for f, a in parts[0].items()})
    return pack_haplotypes(*[[p[f] for p in parts] for f in HaplotypeBlock._fields[1:8]], begin=np.zeros(haps.n + 1, np.int64))


PENALTIES = (("haps", "gap_open", 3, 46), ("haps", "snv_prior_fwd", 1, 126), ("reads", "quals", 2, 42))


def _repenalised(rng, haps, reads):
    """Copies of the blocks with other valid gap opens, forward SNV priors and base qualities (the same lengths)."""
    blocks = {"haps": copy.copy(haps), "reads": copy.copy(reads)}
    for b, f, lo, hi in PENALTIES:
        a = getattr(blocks[b], f)
        setattr(blocks[b], f, rng.integers(lo, hi, len(a)).astype(a.dtype))
    return blocks["haps"], blocks["reads"]


def _staged(haps, reads):
    """The arrays _repenalised changed, as device tensors: copied over a device block's own behind the spin, device to device."""
    import torch
    blocks = {"haps": haps, "reads": reads}
    return [(b, f, torch.as_tensor(getattr(blocks[b], f), device=DEV)) for b, f, _, _ in PENALTIES]


def _rewrite(dh, dr, staged):
    blocks = {"haps": dh, "reads": dr}
    for b, f, t in staged:
        getattr(blocks[b], f).copy_(t)


def _bits(x):
    x = x.cpu().numpy() if hasattr(x, "cpu") else np.asarray(x)
    return np.ascontiguousarray(x).view(np.uint8)


def _same(got, want):
    assert len(got) == len(want)
    for i, (g, w) in enumerate(zip(got, want)):
        if isinstance(w, list):
            assert g == w, i
        else:
            assert np.array_equal(_bits(g), _bits(w)), i


# -- A, B: realign_reads and map_pairs -----------------------------------------------------------------------------------
def _pairs_case(engine):
    """A realign input, its host-space results (map_pairs, realign_reads) and a permutation of its pairs to warm up with."""
    rng = np.random.default_rng(61)
    haps, reads = random_region(rng, BAND, n_haps=4, n_reads=48, hap_len=360, read_len_choices=[40, 76, 120], read_n_rate=0.1)
    pairs = np.array([(r, int(rng.integers(0, haps.n))) for r in range(reads.n)], np.int32)
    want = engine.realign_reads(_cfg(), haps, reads, pairs, REALIGN_FLANKS, REALIGN_STRIDE)
    assert any(want[2]) and (want[3] == 0).any()
    return haps, reads, pairs, pairs[rng.permutation(len(pairs))], engine.map_pairs(haps, reads, pairs), want


REALIGN_FLANKS, REALIGN_STRIDE = (20, 30), 4 * 120 + 64     # explicit: the default stride is a host read of the read offsets


@pytest.mark.parametrize("pair_dtype", ["int32", "int64"])
def test_realign_reads_orders_after_its_zero_fill_and_pair_conversion(engine, stream, pair_dtype):
    """The outputs' zero-fill must land before the engine writes them; int64 pairs, converted, before it reads them."""
    import torch
    haps, reads, pairs, warm, _, want = _pairs_case(engine)
    dh, dr = haps.to_device(DEV), reads.to_device(DEV)
    dp, dwarm = (torch.as_tensor(p, dtype=getattr(torch, pair_dtype), device=DEV) for p in (pairs, warm))
    engine.realign_reads(_cfg(), dh, dr, dwarm, REALIGN_FLANKS, REALIGN_STRIDE)
    busy()
    still_busy()
    _same(engine.realign_reads(_cfg(), dh, dr, dp, REALIGN_FLANKS, REALIGN_STRIDE), want)


def test_map_pairs_orders_after_the_pair_conversion(engine, stream):
    import torch
    haps, reads, pairs, warm, want, _ = _pairs_case(engine)
    dh, dr = haps.to_device(DEV), reads.to_device(DEV)
    dp, dwarm = (torch.as_tensor(p, dtype=torch.int64, device=DEV) for p in (pairs, warm))
    engine.map_pairs(dh, dr, dwarm)
    busy()
    still_busy()
    _same(engine.map_pairs(dh, dr, dp), want)


# -- C: populate and populate_regions read arguments rewritten behind queued work ----------------------------------------
@pytest.mark.parametrize("short", [False, True], ids=["dense", "short haplotype with statuses"])
def test_populate_reads_arguments_rewritten_behind_queued_work(engine, coracle, stream, short):
    """Qualities, gap opens and SNV priors rewritten in place behind the spin: populate allocates its result, so it must wait for
    them. Mapping quality off, against the oracle; with a short haplotype the statuses too."""
    rng = np.random.default_rng(62 + short)
    haps, reads = _region(rng)
    if short:
        haps = _with_short_haplotype(haps)
    final_h, final_r = _repenalised(rng, haps, reads)
    rc, want, wst = coracle.populate(BAND, final_h, final_r, None, None, use_mapping_quality=False)
    assert ((wst & 0xFFFF) == 2).any() == short and (wst == 0).any()
    cfg = _cfg(use_mq=False, map_positions=False)
    dh, dr = haps.to_device(DEV), reads.to_device(DEV)
    staged = _staged(final_h, final_r)
    engine.populate(cfg, dh, dr, want_status=short)
    busy()
    _rewrite(dh, dr, staged)
    still_busy()
    if short:
        got, st = engine.populate(cfg, dh, dr, want_status=True)
        assert_same_penalties(got.cpu().numpy(), want, st.cpu().numpy(), wst, "short")
    else:
        assert_same_penalties(engine.populate(cfg, dh, dr).cpu().numpy(), want, None, wst, "dense")


def test_populate_regions_reads_arguments_rewritten_behind_queued_work(engine, coracle, stream):
    from octopus_b200.batch import concat_blocks
    rng = np.random.default_rng(64)
    first = [_region(rng, n_haps=int(rng.integers(2, 6)), n_reads=int(rng.integers(20, 60))) for _ in range(3)]
    final = [_repenalised(rng, h, r) for h, r in first]
    flanks = [(20, 30), None, (5, 60)]
    haps, reads, hf, rf = concat_blocks([h for h, _ in first], [r for _, r in first])
    final_h, final_r, _, _ = concat_blocks([h for h, _ in final], [r for _, r in final])
    cfg = _cfg(use_mq=False, map_positions=False)
    dh, dr = haps.to_device(DEV), reads.to_device(DEV)
    staged = _staged(final_h, final_r)
    engine.populate_regions(cfg, dh, dr, hf, rf, flanks, want_status=True)
    busy()
    _rewrite(dh, dr, staged)
    still_busy()
    flat, off, st = engine.populate_regions(cfg, dh, dr, hf, rf, flanks, want_status=True)
    mats, sts = engine.split_regions(flat.cpu().numpy(), off, hf, rf), engine.split_regions(st.cpu().numpy(), off, hf, rf)
    for g, (h, r) in enumerate(final):
        rc, want, wst = coracle.populate(BAND, h, r, None, flanks[g], use_mapping_quality=False)
        assert_same_penalties(mats[g], want, sts[g], wst, g)


# -- D: an output block the caching allocator takes back from a tensor queued work still reads --------------------------
def test_populate_output_does_not_overwrite_a_block_queued_work_still_reads(engine, stream):
    rng = np.random.default_rng(65)
    haps, reads = _region(rng, n_reads=257)          # a result size of its own, so that the allocator hands the freed block back
    haps2, reads2 = _repenalised(rng, haps, reads)
    cfg = _cfg()
    dh, dr, dh2, dr2 = haps.to_device(DEV), reads.to_device(DEV), haps2.to_device(DEV), reads2.to_device(DEV)
    warm = engine.populate(cfg, dh2, dr2)            # kept: its block is not the one handed back
    prev = engine.populate(cfg, dh, dr)
    prev_host = prev.cpu().numpy()
    busy()
    pending = prev.clone()
    ptr = prev.data_ptr()
    del prev
    still_busy()
    got = engine.populate(cfg, dh2, dr2)
    assert got.data_ptr() == ptr, "the caching allocator did not hand the freed block back: nothing was tested"
    assert np.array_equal(_bits(pending), _bits(prev_host))
    assert np.array_equal(_bits(got), _bits(warm))


# -- E: a caller-supplied out, ordered by the caller with wait_event -----------------------------------------------------
def test_caller_out_window_is_ordered_with_wait_event(engine, stream):
    """The peer-ring pattern: the engine writes a column window of a matrix another stream fills first, ordered by an event."""
    import torch
    rng = np.random.default_rng(66)
    haps, reads = _region(rng)
    cfg = _cfg()
    want = engine.populate(cfg, haps, reads, None, (25, 40))
    dh, dr = haps.to_device(DEV), reads.to_device(DEV)
    H, R, a = haps.n, reads.n, 300
    engine.populate(cfg, dh, dr, None, (25, 40), out=torch.empty((H, R + 700), dtype=torch.float64, device=DEV)[:, a:a + R])
    busy()
    big = torch.full((H, R + 700), 7.0, dtype=torch.float64, device=DEV)
    ev = torch.cuda.Event()
    ev.record()
    engine.wait_event(ev)
    still_busy()
    engine.populate(cfg, dh, dr, None, (25, 40), out=big[:, a:a + R])
    whole = big.cpu().numpy()
    assert np.array_equal(_bits(whole[:, a:a + R]), _bits(want))
    assert (whole[:, :a] == 7.0).all() and (whole[:, a + R:] == 7.0).all()


# -- F: genotype_likelihoods converts the genotypes ----------------------------------------------------------------------
def test_genotype_likelihoods_order_after_the_genotype_conversion(engine, stream):
    import torch
    rng = np.random.default_rng(67)
    haps, reads = _region(rng)
    lnl = engine.populate(_cfg(), haps.to_device(DEV), reads.to_device(DEV))
    gts, warm = (rng.integers(0, haps.n, (300, 3)).astype(np.int64) for _ in range(2))
    want = engine.genotype_likelihoods(lnl.cpu().numpy(), gts)
    assert not np.array_equal(_bits(want), _bits(engine.genotype_likelihoods(lnl.cpu().numpy(), warm)))
    g, w = torch.as_tensor(gts, device=DEV), torch.as_tensor(warm, device=DEV)
    engine.genotype_likelihoods(lnl, w)
    busy()
    still_busy()
    assert np.array_equal(_bits(engine.genotype_likelihoods(lnl, g)), _bits(want))


# -- G: assign_reads and assign_templates convert the priors -------------------------------------------------------------
def test_assign_orders_after_the_prior_conversion(engine, stream):
    """float32 log priors: converted to float64 on torch's stream. Template offsets are given on the host (as a tensor they are
    moved there, which drains the stream)."""
    import torch
    from test_gpu_assign import filter_call, random_priors
    from test_gpu_assign_templates import make_templates
    rng = np.random.default_rng(68)
    haps, reads, hf, rf = filter_call(rng, 4)
    toff, tf = make_templates(rng, rf)
    pri, warm = random_priors(rng, haps.n).astype(np.float32), np.zeros(haps.n, np.float32)
    pri[hf[:-1]] = -np.inf                          # each group's first haplotype never chosen: the priors change the choice
    cfg = _cfg()
    calls = (lambda h, r, p: engine.assign_reads(cfg, h, r, hf, rf, p, want_likelihoods=True, want_status=True),
             lambda h, r, p: engine.assign_templates(cfg, h, r, toff, hf, tf, p, want_likelihoods=True, want_status=True))
    dh, dr = haps.to_device(DEV), reads.to_device(DEV)
    dpri, dwarm = torch.as_tensor(pri, device=DEV), torch.as_tensor(warm, device=DEV)
    for call in calls:
        want = call(haps, reads, pri)
        assert not np.array_equal(want[0], call(haps, reads, warm)[0])
        call(dh, dr, dwarm)
        busy()
        still_busy()
        _same(call(dh, dr, dpri), want)


# -- H: ErrorModel.reset_block on the engine -----------------------------------------------------------------------------
def test_reset_block_reads_a_sequence_rewritten_behind_queued_work(engine, stream):
    """reset_block reads the last offset on the host, which drains the stream before the call; this keeps the ordering checked
    should that read go away."""
    import torch
    from octopus_b200 import ErrorModel
    from octopus_b200.batch import pack_sequences
    from test_error_model import FIELDS, repeat_rich_sequence
    rng = np.random.default_rng(69)
    first = [repeat_rich_sequence(rng, 400) for _ in range(40)]
    final = [np.resize(repeat_rich_sequence(rng, len(s)), len(s)) for s in first]
    off, seq = pack_sequences(first)
    off2, seq2 = pack_sequences(final)
    assert np.array_equal(off, off2)
    m = ErrorModel("PCR.HiSeq-4000")
    want = m.reset_block(off, seq2)
    doff, dseq, dnew = (torch.as_tensor(a, device=DEV) for a in (off, seq, seq2))
    m.reset_block(doff, dseq, engine=engine)
    busy()
    dseq.copy_(dnew)
    still_busy()
    got = m.reset_block(doff, dseq, engine=engine)
    for f in FIELDS:
        assert np.array_equal(_bits(getattr(got, f)), _bits(getattr(want, f))), f


# -- I: align_scores converts the tasks ----------------------------------------------------------------------------------
def test_align_scores_orders_after_the_task_conversion(engine, stream):
    import torch
    rng = np.random.default_rng(70)
    haps, reads = random_region(rng, BAND, n_haps=6, n_reads=80, hap_len=300, read_len_choices=[50, 76, 100])
    tasks = []
    for _ in range(400):
        r, h = int(rng.integers(0, reads.n)), int(rng.integers(0, haps.n))
        tasks.append((r, h, int(rng.integers(0, haps.length(h) - reads.length(r) - 2 * BAND + 2)), int(rng.integers(0, 2))))
    tasks = np.array(tasks, np.int64)
    want = engine.align_scores(BAND, haps, reads, tasks.astype(np.int32))
    dh, dr = haps.to_device(DEV), reads.to_device(DEV)
    dt, dwarm = (torch.as_tensor(t, device=DEV) for t in (tasks, tasks[rng.permutation(len(tasks))]))
    engine.align_scores(BAND, dh, dr, dwarm)
    busy()
    still_busy()
    assert np.array_equal(engine.align_scores(BAND, dh, dr, dt).cpu().numpy(), want)


# -- K: the benchmark's and the peer ring's calls issue no wait ----------------------------------------------------------
def test_calls_over_caller_buffers_issue_no_wait(engine, monkeypatch):
    """Device blocks, out supplied, nothing converted: the caller orders with wait_event, and an unconditional wait would serialise
    a gather of the previous result with the next populate. A call that allocates its result or statuses waits once."""
    import torch
    from octopus_b200 import PairHMMEngine
    waits = []
    wait = PairHMMEngine.wait_event
    monkeypatch.setattr(PairHMMEngine, "wait_event", lambda self, ev: (waits.append(ev), wait(self, ev))[1])
    rng = np.random.default_rng(71)
    haps, reads = _region(rng)
    dh, dr = haps.to_device(DEV), reads.to_device(DEV)
    H, R, cfg = haps.n, reads.n, _cfg()
    out = torch.empty((H, R), dtype=torch.float64, device=DEV)
    wide = torch.empty((H, R + 100), dtype=torch.float64, device=DEV)
    engine.populate(cfg, dh, dr, flank_state=(20, 30), out=out)
    engine.populate(cfg, dh, dr, flank_state=(20, 30), out=wide[:, 50:50 + R])
    assert waits == []
    engine.populate(cfg, dh, dr)
    engine.populate(cfg, dh, dr, out=out, want_status=True)
    assert len(waits) == 2
