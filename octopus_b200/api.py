"""Host-side mirror of the reference interface for this path, over the C ABI (include/phmm_b200.h).

Names and argument meaning follow the reference:
  * ``PairHMMEngine.align_scores``            ↔ simd::PairHMM::align  (simd_pair_hmm.hpp:454-470), batched
  * ``HaplotypeLikelihoodModel.Config``       ↔ HaplotypeLikelihoodModel::Config (haplotype_likelihood_model.hpp:36-44)
  * ``HaplotypeLikelihoodArray.populate``     ↔ HaplotypeLikelihoodArray::populate (haplotype_likelihood_array.cpp:51-103)
  * ``ShortHaplotypeError``                   ↔ HaplotypeLikelihoodModel::ShortHaplotypeError (:123-139)
  * ``MutationModel`` + ``PairHMMEngine.mutation_prime`` ↔ DeNovoModel::prime / evaluate (core/models/mutation/denovo_model.cpp:64-84);
    ``mutation_prime_sets`` primes many regions' sets in one call, ``PopulateBatcher.mutation_prime`` from many threads on one engine
Every computing call goes through libphmm_b200.so to the GPU; nothing here computes likelihoods on the CPU.
"""
import ctypes as C

import numpy as np

from . import _lib
from .batch import HaplotypeBlock, HaplotypeSequences, ReadBlock, _ptr, _u8, concat_reads, pack_sequences


class PhmmError(RuntimeError):
    def __init__(self, code, message):
        super().__init__("phmm error %d: %s" % (code, message))
        self.code = code


class ShortHaplotypeError(PhmmError):
    """Haplotype is too short for alignment (reference: thrown out of populate, caller.cpp:1182-1188 skips the region)."""


class TooLargeBandSizeError(PhmmError):
    """Requested band > 256 (simd_pair_hmm_wrapper.hpp:45-61)."""


def _error(code, message):
    """The exception for a failed call's PHMM_ERR_* code."""
    cls = {_lib.PHMM_ERR_SHORT_HAPLOTYPE: ShortHaplotypeError, _lib.PHMM_ERR_BAND: TooLargeBandSizeError}.get(code, PhmmError)
    return cls(code, message)


def _is_torch(x):
    return hasattr(x, "data_ptr")


class _Space:
    """The memory space of one call: numpy arrays on the host, or torch tensors on one CUDA device."""
    __slots__ = ("device", "on_device", "flag", "enqueued")

    def __init__(self, device=None):
        self.device = device
        self.on_device = device is not None
        self.flag = _lib.SPACE_DEVICE if self.on_device else _lib.SPACE_HOST
        self.enqueued = False       # the call's own conversions, fills or allocations went to torch's current stream

    @classmethod
    def of(cls, haps, reads):
        assert haps.on_device == reads.on_device, "haplotypes and reads must live in the same memory space"
        return cls(haps.seq.device if haps.on_device else None)

    def dtype(self, dtype):
        if self.on_device:
            import torch
            return getattr(torch, np.dtype(dtype).name)
        return np.dtype(dtype)

    def empty(self, shape, dtype, zeroed=False):
        """An output array; zeroed where the call may leave entries unwritten."""
        if self.on_device:
            import torch
            self.enqueued = True
            return (torch.zeros if zeroed else torch.empty)(shape, dtype=self.dtype(dtype), device=self.device)
        return (np.zeros if zeroed else np.empty)(shape, dtype=dtype)

    def input(self, x, dtype):
        """x (a sequence, numpy array or torch tensor) as a contiguous array of `dtype` in this space."""
        if self.on_device:
            import torch
            t = x if _is_torch(x) else torch.as_tensor(np.ascontiguousarray(x, dtype=dtype), device=self.device)
            t = t.to(device=self.device, dtype=self.dtype(dtype)).contiguous()
            self.enqueued |= t is not x
            return t
        return np.ascontiguousarray(x, dtype=dtype)

    def order(self, engine):
        """Right before the C call: make the engine's stream wait for torch's current stream if this call put work there itself.
        The engine reads and writes on its own stream, so it must start after a conversion or a zero-fill, and after queued work
        still reading an output block the caching allocator handed back from a freed tensor. Buffers the caller supplies as they
        are take no wait; the caller orders those with engine.wait_event."""
        if self.enqueued:
            engine._wait_for_current_stream(self.device)

    ptr = staticmethod(_ptr)        # the data pointer of a numpy array or torch tensor, or None


_HOST = _Space()


def _ref(s):
    return None if s is None else C.byref(s)


def _config(config):
    """A HaplotypeLikelihoodModel.Config, or an already built _lib.Config, as the phmm_config argument."""
    return C.byref(config.c_struct() if hasattr(config, "c_struct") else config)


def _flank(flank_state):
    """(lhs_flank, rhs_flank) → phmm_flank_state; None → None."""
    return None if flank_state is None else _lib.FlankState(1, int(flank_state[0]), int(flank_state[1]))


def _positions(space, positions):
    """(off, pos) candidate positions → phmm_positions over arrays in the call's memory space (kept alive by the struct); None → None."""
    if positions is None:
        return None
    off, pos = space.input(positions[0], np.int64), space.input(positions[1], np.int32)
    s = _lib.Positions(space.ptr(off), space.ptr(pos))
    s.arrays = off, pos
    return s


def _regions(hap_first, read_first, flank_states=None):
    """Group bounds (and per-group flank states or None) → (phmm_regions, int64 offsets of the groups' [H_g, R_g] blocks in the flat
    result, whose last entry is its size)."""
    hf = np.ascontiguousarray(hap_first, dtype=np.int32)
    rf = np.ascontiguousarray(read_first, dtype=np.int32)
    G = len(hf) - 1
    sizes = np.diff(hf).astype(np.int64) * np.diff(rf).astype(np.int64)
    off = np.concatenate([[0], np.cumsum(sizes)]).astype(np.int64)
    fl = None
    if flank_states is not None:
        fl = (_lib.FlankState * G)()
        for g, f in enumerate(flank_states):
            if f is not None:
                fl[g] = _flank(f)
    regs = _lib.Regions(G, hf.ctypes.data, rf.ctypes.data, C.addressof(fl) if fl is not None else None)
    regs.arrays = hf, rf, fl
    return regs, off


def _haps(haps, error_model):
    """(haplotype block argument, model arguments): the plain call's HaplotypeBlock and (), or with an error model the _reset twin's
    HaplotypeSequences and (model handle,)."""
    if error_model is None:
        return C.byref(haps.c_struct()), ()
    if not isinstance(haps, HaplotypeSequences):
        raise TypeError("with error_model, haps must be a HaplotypeSequences block")
    return C.byref(haps.c_struct()), (error_model._h,)


def _call(lib, name, handle, config, haps, error_model, *rest):
    """lib.<name>(handle, config, haps, ...) or, with an error model, lib.<name>_reset(handle, config, model, sequences, ...)."""
    hs, model = _haps(haps, error_model)
    return getattr(lib, name + ("_reset" if model else ""))(handle, _config(config), *model, hs, *rest)


def _mutation_set(sequences):
    """One haplotype set → (off, seq, out, status): the packed block and its zeroed [H, H] outputs."""
    off, seq = pack_sequences(sequences)
    H = len(off) - 1
    return off, seq, np.zeros((H, H), dtype=np.float64), np.zeros((H, H), dtype=np.int32)


class _Alignments:
    """The outputs of n alignments: mapping position, likelihood, CIGAR text (n x stride bytes, NUL-terminated) and status, zeroed."""

    def __init__(self, space, reads, n, stride=None):
        self.n = n
        self.stride = 4 * int((reads.off[1:] - reads.off[:-1]).max()) + 64 if stride is None else stride
        self.mp, self.lk, self.st = space.empty(n, np.int64, True), space.empty(n, np.float64, True), space.empty(n, np.int32, True)
        self.cg = space.empty(n * self.stride, np.uint8, True)

    def pointers(self):
        """The (mapping_position, likelihood, cigar, cigar_stride, status) arguments of the aligning calls."""
        return _ptr(self.mp), _ptr(self.lk), _ptr(self.cg), self.stride, _ptr(self.st)

    def result(self):
        text = bytes(self.cg.cpu().numpy() if _is_torch(self.cg) else self.cg)
        s = self.stride
        return self.mp, self.lk, [text[j * s:(j + 1) * s].split(b"\0", 1)[0].decode() for j in range(self.n)], self.st


def _realign(call, owner, sp, config, haps, reads, pairs, flank_state, cigar_stride, *space):
    """One realign call (phmm_realign_reads or phmm_batcher_realign_reads on owner's handle; `space` the engine's trailing
    memory-space argument): (return code, the result PairHMMEngine.realign_reads returns)."""
    pr = sp.input(pairs, np.int32).reshape(-1, 2)
    n = pr.shape[0]
    res = _Alignments(sp, reads, n, cigar_stride)
    sp.order(owner)
    rc = call(owner._h, _config(config), C.byref(haps.c_struct()), C.byref(reads.c_struct()), sp.ptr(pr), n, _ref(_flank(flank_state)),
              *res.pointers(), *space)
    return rc, res.result()


def _template_groups(template_off, template_first):
    """Groups given in templates → (template offsets as host int64, the groups' read_first): group g's reads start at its first
    template's first read."""
    toff = np.ascontiguousarray(template_off.cpu().numpy() if _is_torch(template_off) else template_off, dtype=np.int64)
    tf = np.ascontiguousarray(template_first, dtype=np.int64)
    if toff.ndim != 1 or len(toff) < 2 or tf.ndim != 1 or len(tf) < 2 or tf.min() < 0 or tf.max() >= len(toff):
        raise ValueError("template_first must index template_off, which needs at least one template")
    return toff, toff[tf]


def _assign(call, owner, sp, config, haps, reads, hap_first, read_first, log_priors, want_likelihoods, want_status, *space,
            templates=None):
    """One assign call (phmm_assign_reads or phmm_batcher_assign_reads on owner's handle; with templates = (template_off,
    template_first), phmm_assign_templates or phmm_batcher_assign_templates; `space` the engine's trailing memory-space argument):
    (return code, the result PairHMMEngine.assign_reads / assign_templates returns)."""
    regs, off = _regions(hap_first, read_first)
    n_top, n_values, tmpl = reads.n, int(off[-1]), ()
    if templates is not None:
        toff, template_first = templates
        n_top = len(toff) - 1
        n_values = int(_regions(hap_first, template_first)[1][-1])
        tmpl = (toff.ctypes.data, n_top)
    top = sp.empty(n_top, np.int64 if sp.on_device else np.uint64)
    lnl = sp.empty(n_values, np.float64) if want_likelihoods else None
    status = sp.empty(int(off[-1]), np.int32) if want_status else None
    pri = None if log_priors is None else sp.input(log_priors, np.float64)
    if pri is not None and pri.shape[0] != haps.n:
        raise ValueError("log_priors needs one value per haplotype of the block")
    sp.order(owner)
    rc = call(owner._h, _config(config), C.byref(haps.c_struct()), C.byref(reads.c_struct()), C.byref(regs), *tmpl, sp.ptr(pri), sp.ptr(top),
              sp.ptr(lnl), sp.ptr(status), *space)
    out = (top,)
    if want_likelihoods:
        out += (lnl,)
    if want_status:
        out += (status,)
    return rc, out[0] if len(out) == 1 else out


def _grow(attempt, cap):
    """attempt(cap) → (size needed, result). Most calls fit the first guess; a second call takes the exact size."""
    while True:
        total, result = attempt(cap)
        if total <= cap:
            return result
        cap = total


class _Handle:
    """A library handle this object owns: freed by close(), at the end of a with block, or when the object is collected."""
    _h = None
    _destroy = None             # the phmm_*_destroy function's name

    def _create(self, create, *args):
        self._lib = _lib.load()
        h = C.c_void_p()
        rc = getattr(self._lib, create)(C.byref(h), *args)
        if rc != _lib.PHMM_OK:
            raise PhmmError(rc, self._last_error())
        self._h = h

    def _last_error(self):
        raise NotImplementedError

    def _raise(self, rc):
        """Raise the exception for a failed call's code, with this handle's last error message."""
        raise _error(rc, self._last_error())

    def _check(self, rc, tolerate_short=False):
        """Raise for a failed call. With tolerate_short (the caller asked for statuses) a short haplotype is no failure."""
        if rc != _lib.PHMM_OK and not (tolerate_short and rc == _lib.PHMM_ERR_SHORT_HAPLOTYPE):
            self._raise(rc)

    def close(self):
        if self._h:
            getattr(self._lib, self._destroy)(self._h)
            self._h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    def __enter__(self):
        return self

    def __exit__(self, *a):
        self.close()


class PairHMMEngine(_Handle):
    """One engine handle (not re-entrant; one per host thread, like the reference's per-thread model copies)."""
    _destroy = "phmm_destroy"
    _stream_event = None

    def __init__(self, device=-1):
        self._create("phmm_create", int(device))

    def _last_error(self):
        return self._lib.phmm_last_error(self._h).decode()

    # -- stream ordering -----------------------------------------------------------------------------------------
    def wait_event(self, event):
        """Make the engine's stream wait (on the device) for a CUDA event — a torch.cuda.Event or a raw cudaEvent_t — recorded
        after work on another stream that still writes a buffer the next call reads, or still reads one it will overwrite
        (phmm_wait_event). Every call runs on the engine's own stream. A device-space call that converts an argument or
        allocates an output or status tensor waits for torch's current stream itself, through this method. Device buffers the caller
        passes as they are (blocks, pairs, priors or ``out``, already in the right dtype and layout) are the caller's to order:
        record an event after the work that produces or still reads them and hand it here before the call."""
        handle = getattr(event, "cuda_event", event)
        self._check(self._lib.phmm_wait_event(self._h, C.c_void_p(int(handle))))

    def _wait_for_current_stream(self, device):
        """wait_event on an event recorded now on torch's current stream of `device`. One event per engine, recorded again each
        time: the wait takes the event's state when it is issued, and an engine serves one thread."""
        import torch
        if self._stream_event is None:
            self._stream_event = torch.cuda.Event()
        self._stream_event.record(torch.cuda.current_stream(device))
        self.wait_event(self._stream_event)

    def reserve_sms(self, n):
        """Keep the first n SMs free of persistent DP blocks, for a collective running beside the next call (phmm_reserve_sms)."""
        self._check(self._lib.phmm_reserve_sms(self._h, int(n)))

    def stream_handle(self):
        return int(self._lib.phmm_engine_stream(self._h) or 0)

    # -- statistics of the last call -------------------------------------------------------------------------
    def launch_count(self, total=False):
        return int(self._lib.phmm_launch_count(self._h, int(total)))

    def last_dp_kernel_ms(self):
        return float(self._lib.phmm_last_dp_kernel_ms(self._h))

    def last_dp_cells(self):
        return int(self._lib.phmm_last_dp_cells(self._h))

    # -- DeNovoModel::prime ------------------------------------------------------------------------------------
    def mutation_prime(self, model, sequences):
        """DeNovoModel::prime + evaluate for one haplotype set (phmm_mutation_prime): sequences (list of str / bytes) → (out, status),
        both [H, H] indexed [target, given]. out[t, g] = ln p(target | given) where status is MUT_HMM or MUT_SELF; the MUT_APPROX_*
        pairs need the reference's approximate path (Haplotype::difference) and MUT_OUT_OF_MODEL pairs have no defined value."""
        off, seq, out, status = _mutation_set(sequences)
        self._check(self._lib.phmm_mutation_prime(self._h, model._h, len(off) - 1, off.ctypes.data, seq.ctypes.data, out.ctypes.data,
                                                  status.ctypes.data))
        return out, status

    def mutation_prime_sets(self, model, sets):
        """DeNovoModel::prime for many haplotype sets in one call (phmm_mutation_prime_sets): sets (list of lists of sequences) → one
        (out, status) pair of [n_s, n_s] arrays per set, each what mutation_prime returns for that set alone. Empty sets are allowed."""
        sets = [list(s) for s in sets]
        sizes = np.array([len(s) for s in sets], dtype=np.int64)
        set_first = np.zeros(len(sets) + 1, dtype=np.int32)
        np.cumsum(sizes, out=set_first[1:])
        pair_first = np.zeros(len(sets) + 1, dtype=np.int64)
        np.cumsum(sizes * sizes, out=pair_first[1:])
        off, seq = pack_sequences([x for s in sets for x in s])
        out = np.zeros(int(pair_first[-1]), dtype=np.float64)
        status = np.zeros(int(pair_first[-1]), dtype=np.int32)
        self._check(self._lib.phmm_mutation_prime_sets(self._h, model._h, len(sets), set_first.ctypes.data, off.ctypes.data, seq.ctypes.data,
                                                       out.ctypes.data, status.ctypes.data))
        return [(out[a:b].reshape(n, n), status[a:b].reshape(n, n)) for a, b, n in zip(pair_first[:-1], pair_first[1:], sizes)]

    # -- raw kernel boundary -----------------------------------------------------------------------------------
    def align_scores(self, band, haps: HaplotypeBlock, reads: ReadBlock, tasks, nuc_prior=2, precision_bits=16):
        """tasks: (n, 4) int32 rows (read, hap, win_off, reverse). Returns the integer score of every task, i.e.
        reference ``hmm.align(hap_window, read, quals, L+2*band-1, L, snv_mask, snv_prior, gap_open, gap_extend, nuc_prior)``."""
        sp = _Space.of(haps, reads)
        t = sp.input(tasks, np.int32)
        if not sp.on_device:
            t = t.reshape(-1, 4)
        n = t.shape[0]
        out = sp.empty(n, np.int32)
        sp.order(self)
        self._check(self._lib.phmm_align_scores(self._h, int(band), int(precision_bits), int(nuc_prior), C.byref(haps.c_struct()),
                                                C.byref(reads.c_struct()), sp.ptr(t), n, sp.ptr(out), sp.flag))
        return out

    def align(self, band, truth, target, quals, gap_open, gap_extend, nuc_prior=2, snv_mask=None, snv_prior=None):
        """Per-call seam with traceback ↔ simd::PairHMM::align(..., first_pos, align1, align2) (simd_pair_hmm.hpp:472-509).
        Returns (score, first_pos, aligned_truth, aligned_target). gap_extend may be a scalar (the reference's scalar overload)."""
        t, r = _u8(truth).tobytes(), _u8(target).tobytes()
        q = np.ascontiguousarray(np.asarray(quals, dtype=np.int8))
        go = np.ascontiguousarray(np.asarray(gap_open, dtype=np.int8))
        if np.ndim(gap_extend) == 0:
            ge, gep, ges = None, None, int(gap_extend)
        else:
            ge = np.ascontiguousarray(np.asarray(gap_extend, dtype=np.int8)); gep, ges = ge.ctypes.data, 0
        if snv_mask is not None:
            m = _u8(snv_mask).tobytes()
            sp = np.ascontiguousarray(np.asarray(snv_prior, dtype=np.int8)); spp = sp.ctypes.data
        else:
            m, spp = None, None
        n = 2 * (len(r) + band) + 1
        a1, a2 = C.create_string_buffer(n + 8), C.create_string_buffer(n + 8)
        score, fp = C.c_int(0), C.c_int(0)
        self._check(self._lib.phmm_align_traceback(self._h, int(band), t, r, q.ctypes.data, len(t), len(r), m, spp, go.ctypes.data, gep, ges,
                                                   int(nuc_prior), C.byref(score), C.byref(fp), a1, a2))
        return score.value, fp.value, a1.value.decode(), a2.value.decode()

    def align_reads(self, config, haps: HaplotypeBlock, reads: ReadBlock, pairs, positions=None, flank_state=None, cigar_stride=None):
        """HaplotypeLikelihoodModel::align for explicit (read, haplotype) pairs (host blocks). pairs: (n, 2) int32 rows (read, hap);
        positions: None or (off[n+1], pos) CSR over the pair list. Returns (mapping_position[n], likelihood[n], cigars[list of str], status[n])."""
        assert not haps.on_device and not reads.on_device
        pr = np.ascontiguousarray(pairs, dtype=np.int32).reshape(-1, 2)
        n = pr.shape[0]
        res = _Alignments(_HOST, reads, n, cigar_stride)
        self._check(self._lib.phmm_align_reads(self._h, _config(config), C.byref(haps.c_struct()), C.byref(reads.c_struct()), pr.ctypes.data,
                                               n, _ref(_positions(_HOST, positions)), _ref(_flank(flank_state)), *res.pointers(),
                                               _lib.SPACE_HOST))
        return res.result()

    def align_pairs(self, config, truths: HaplotypeBlock, targets: ReadBlock, pairs, target_offsets, flank_state=None, cigar_stride=None):
        """hmm::align batched (phmm_align_pairs): pair j = (target pairs[j][0], truth pairs[j][1]) at target_offsets[j]. Host blocks.
        Returns (target_offset[n], likelihood[n], cigars, status[n])."""
        assert not truths.on_device and not targets.on_device
        pr = np.ascontiguousarray(pairs, dtype=np.int32).reshape(-1, 2)
        n = pr.shape[0]
        offs = np.ascontiguousarray(target_offsets, dtype=np.int32)
        assert len(offs) == n
        res = _Alignments(_HOST, targets, n, cigar_stride)
        self._check(self._lib.phmm_align_pairs(self._h, _config(config), C.byref(truths.c_struct()), C.byref(targets.c_struct()),
                                               pr.ctypes.data, offs.ctypes.data, n, _ref(_flank(flank_state)), *res.pointers(),
                                               _lib.SPACE_HOST))
        return res.result()

    def map_pairs(self, haps: HaplotypeBlock, reads: ReadBlock, pairs):
        """map_query_to_target(read, haplotype) uncapped, K = 6, for explicit (read, haplotype) pairs (phmm_map_pairs): every mapping
        begin at the pair's largest k-mer vote count, ascending — what ReadRealigner maps with. Returns the CSR (off[n+1] int64,
        pos int32) over the pair list: numpy for host blocks, torch CUDA tensors for device-resident ones."""
        sp = _Space.of(haps, reads)
        pr = sp.input(pairs, np.int32).reshape(-1, 2)
        n = pr.shape[0]
        hs, rs = C.byref(haps.c_struct()), C.byref(reads.c_struct())

        def attempt(cap):
            off, pos = sp.empty(n + 1, np.int64), sp.empty(cap, np.int32)
            sp.order(self)
            self._check(self._lib.phmm_map_pairs(self._h, hs, rs, sp.ptr(pr), n, sp.ptr(off), sp.ptr(pos), cap, sp.flag))
            total = int(off[-1])
            return total, (off, pos[:total])
        return _grow(attempt, 4 * n + 16)       # most pairs have one or a few maxima

    def realign_reads(self, config, haps: HaplotypeBlock, reads: ReadBlock, pairs, flank_state=None, cigar_stride=None):
        """ReadRealigner::realign for explicit (read, haplotype) pairs (phmm_realign_reads): HaplotypeLikelihoodModel::align at the
        positions of the uncapped k-mer mapper (map_pairs), mapped on the device (config.map_positions = False: the original position
        only). pairs: (n, 2) int32 rows (read, hap). Returns (mapping_position[n], likelihood[n], cigars[list of str], status[n]) as
        align_reads; for device-resident blocks the three arrays are torch CUDA tensors."""
        sp = _Space.of(haps, reads)
        rc, res = _realign(self._lib.phmm_realign_reads, self, sp, config, haps, reads, pairs, flank_state, cigar_stride, sp.flag)
        self._check(rc)
        return res

    def genotype_likelihoods(self, lnl, genotypes):
        """ConstantMixtureGenotypeLikelihoodModel::evaluate for every row of `genotypes` ((G, ploidy) haplotype indices) over the
        (H, R) matrix `lnl` (numpy on the host, or a torch CUDA tensor left where populate produced it). Returns G doubles."""
        sp = _Space(lnl.device if _is_torch(lnl) else None)
        m, gt = sp.input(lnl, np.float64), sp.input(genotypes, np.int32)
        out = sp.empty(gt.shape[0], np.float64)
        sp.order(self)
        self._check(self._lib.phmm_genotype_likelihoods(self._h, sp.ptr(m), m.shape[0], m.shape[1], sp.ptr(gt), gt.shape[0], gt.shape[1],
                                                        sp.ptr(out), sp.flag))
        return out

    def variational_bayes(self, lnl, genotypes, prior_alphas, genotype_log_priors, seeds, sample_off=None, epsilon=0.05,
                          max_iterations=1000):
        """run_variational_bayes (variational_bayes_mixture_model.hpp:653-669) of SubcloneModel::evaluate over the (H, R) matrix
        `lnl` (numpy on the host, or a torch CUDA tensor left where populate produced it), every seed in one call (phmm_variational_bayes).
        genotypes: (G, K) haplotype indices; prior_alphas: (S, K); genotype_log_priors: (G,); seeds: (n_seeds, G) initial log
        posteriors; sample_off: S + 1 column offsets of the samples (default: one sample over every column). Returns a VBResult;
        for a device matrix its arrays (and the two scalars, as 0-d tensors) stay on the device."""
        sp = _Space(lnl.device if _is_torch(lnl) else None)
        m, gt = sp.input(lnl, np.float64), sp.input(genotypes, np.int32)
        pa, lp, sd = sp.input(prior_alphas, np.float64), sp.input(genotype_log_priors, np.float64), sp.input(seeds, np.float64)
        if gt.ndim != 2 or pa.ndim != 2 or sd.ndim != 2 or m.ndim != 2:
            raise ValueError("lnl, genotypes, prior_alphas and seeds must be 2-dimensional")
        off = np.ascontiguousarray([0, m.shape[1]] if sample_off is None else sample_off, dtype=np.int64)
        G, K, S = gt.shape[0], gt.shape[1], len(off) - 1
        if pa.shape != (S, K) or lp.shape != (G,) or sd.shape[1] != G:
            raise ValueError("prior_alphas must be (S, K), genotype_log_priors (G,) and seeds (n_seeds, G)")
        post, lpost, wpost = sp.empty(G, np.float64), sp.empty(G, np.float64), sp.empty(G, np.float64)
        alphas, mev, ms = sp.empty((S, K), np.float64), sp.empty((), np.float64), sp.empty((), np.int32)
        sev, sit = sp.empty(sd.shape[0], np.float64), sp.empty(sd.shape[0], np.int32)
        sp.order(self)
        self._check(self._lib.phmm_variational_bayes(self._h, sp.ptr(m), m.shape[0], m.shape[1], off.ctypes.data, S, sp.ptr(gt), G, K,
                                                     sp.ptr(pa), sp.ptr(lp), sp.ptr(sd), sd.shape[0], float(epsilon), int(max_iterations),
                                                     sp.ptr(post), sp.ptr(lpost), sp.ptr(alphas), sp.ptr(wpost), sp.ptr(mev), sp.ptr(ms),
                                                     sp.ptr(sev), sp.ptr(sit), sp.flag))
        if not sp.on_device:
            mev, ms = float(mev), int(ms)
        return VBResult(post, lpost, alphas, mev, wpost, ms, sev, sit)

    def variational_bayes_mixture_mixture(self, lnl, group_sizes, combinations, genotype_log_priors, group_concentrations,
                                          mixture_concentrations, seeds, sample_off=None, group_priors=None, group_prior_mask=None,
                                          epsilon=0.05, max_iterations=1000):
        """VariationalBayesMixtureMixtureModel::evaluate (variational_bayes_mixture_mixture_model.cpp) of SingleCellModel over the
        (H, R) matrix `lnl` (numpy on the host, or a torch CUDA tensor left where populate produced it), every seed in one call
        (phmm_variational_bayes_mixture_mixture). group_sizes: the T groups' component counts K_t; combinations: (C, sum K_t)
        haplotype indices, group t's components at columns [koff_t, koff_t + K_t); genotype_log_priors: (C,); seeds: (n_seeds, C)
        initial log posteriors; sample_off: S + 1 column offsets of the samples (default: one sample over every column).
        group_concentrations: a scalar or (T,); mixture_concentrations: a scalar, one per sample (S,), or (S, sum K_t), expanded as
        the reference's scalar overloads expand them. group_priors: None, or (S, T) probabilities for the samples group_prior_mask
        selects (default: all). Returns a VBMixtureMixtureResult; for a device matrix its arrays (and the two scalars, as 0-d
        tensors) stay on the device."""
        sp = _Space(lnl.device if _is_torch(lnl) else None)
        sizes = np.ascontiguousarray(group_sizes, dtype=np.int32).ravel()
        T, K = len(sizes), int(sizes.sum()) if len(sizes) else 0
        m, gt = sp.input(lnl, np.float64), sp.input(combinations, np.int32)
        lp, sd = sp.input(genotype_log_priors, np.float64), sp.input(seeds, np.float64)
        if gt.ndim != 2 or sd.ndim != 2 or m.ndim != 2:
            raise ValueError("lnl, combinations and seeds must be 2-dimensional")
        off = np.ascontiguousarray([0, m.shape[1]] if sample_off is None else sample_off, dtype=np.int64)
        Cn, S = gt.shape[0], len(off) - 1
        if gt.shape[1] != K or lp.shape != (Cn,) or sd.shape[1] != Cn:
            raise ValueError("combinations must be (C, sum of group_sizes), genotype_log_priors (C,) and seeds (n_seeds, C)")
        ndim = lambda v: v.dim() if _is_torch(v) else np.ndim(v)
        scalar_gc, per_sample_mc = ndim(group_concentrations) == 0, ndim(mixture_concentrations) < 2
        gc, mc = sp.input(group_concentrations, np.float64), sp.input(mixture_concentrations, np.float64)
        if scalar_gc:                    # one concentration for every group
            gc = gc.reshape(1).expand(T).contiguous() if sp.on_device else np.full(T, float(gc.ravel()[0]))
        if per_sample_mc:                # one concentration, or one per sample, for every component
            mc = mc.reshape(-1, 1).expand(S, K).contiguous() if sp.on_device else \
                np.repeat(np.broadcast_to(mc.ravel(), (S,))[:, None], K, axis=1)
        sp.enqueued |= sp.on_device and (scalar_gc or per_sample_mc)     # the expansion ran on torch's current stream
        if gc.shape != (T,) or mc.shape != (S, K):
            raise ValueError("group_concentrations must be (T,) and mixture_concentrations (S, sum of group_sizes)")
        gp, mask = None, None
        if group_priors is not None:
            gp = sp.input(group_priors, np.float64)
            if gp.shape != (S, T):
                raise ValueError("group_priors must be (S, T)")
            if group_prior_mask is not None:
                mask = np.ascontiguousarray(group_prior_mask, dtype=np.int32)
                if mask.shape != (S,):
                    raise ValueError("group_prior_mask must be (S,)")
        post, lpost, wpost = sp.empty(Cn, np.float64), sp.empty(Cn, np.float64), sp.empty(Cn, np.float64)
        gco, mco = sp.empty(T, np.float64), sp.empty((S, K), np.float64)
        sigma, wsigma = sp.empty((S, T), np.float64), sp.empty((S, T), np.float64)
        mev, ms = sp.empty((), np.float64), sp.empty((), np.int32)
        sev, sit = sp.empty(sd.shape[0], np.float64), sp.empty(sd.shape[0], np.int32)
        sp.order(self)
        self._check(self._lib.phmm_variational_bayes_mixture_mixture(
            self._h, sp.ptr(m), m.shape[0], m.shape[1], off.ctypes.data, S, sizes.ctypes.data, T, sp.ptr(gt), Cn, sp.ptr(lp),
            sp.ptr(gp), None if mask is None else mask.ctypes.data, sp.ptr(gc), sp.ptr(mc), sp.ptr(sd), sd.shape[0], float(epsilon),
            int(max_iterations), sp.ptr(post), sp.ptr(lpost), sp.ptr(gco), sp.ptr(mco), sp.ptr(sigma), sp.ptr(wpost), sp.ptr(wsigma),
            sp.ptr(mev), sp.ptr(ms), sp.ptr(sev), sp.ptr(sit), sp.flag))
        if not sp.on_device:
            mev, ms = float(mev), int(ms)
        return VBMixtureMixtureResult(post, lpost, gco, mco, sigma, mev, wpost, wsigma, ms, sev, sit)

    # -- batch boundary ----------------------------------------------------------------------------------------
    def populate_templates(self, config, haps: HaplotypeBlock, reads: ReadBlock, template_off, flank_state=None, error_model=None):
        """HaplotypeLikelihoodArray::populate(TemplateMap): host blocks; template t = reads [template_off[t], template_off[t+1]).
        Returns the (H, T) matrix: each entry the sum of the template's reads' ln-likelihoods. With ``error_model`` (an ErrorModel),
        haps is a HaplotypeSequences block whose penalty arrays the GPU derives in the same call (phmm_populate_templates_reset)."""
        assert not haps.on_device and not reads.on_device
        toff = np.ascontiguousarray(template_off, dtype=np.int64)
        T = len(toff) - 1
        out = np.empty((haps.n, T), dtype=np.float64)
        self._check(_call(self._lib, "phmm_populate_templates", self._h, config, haps, error_model, C.byref(reads.c_struct()),
                          toff.ctypes.data, T, None, _ref(_flank(flank_state)), out.ctypes.data, None, _lib.SPACE_HOST))
        return out

    def populate_regions(self, config, haps: HaplotypeBlock, reads: ReadBlock, hap_first, read_first, flank_states=None, out=None, want_status=False,
                         error_model=None):
        """Many regions in one call (phmm_populate_regions): region g owns haplotypes [hap_first[g], hap_first[g+1]) and reads
        [read_first[g], read_first[g+1]). Returns the flat result vector (the regions' [H_g, R_g] matrices back to back) and the
        per-region offsets into it; ``split_regions`` cuts it into matrices. flank_states: None or a list of (lhs, rhs) / None.
        With ``error_model``, haps is a HaplotypeSequences block (phmm_populate_regions_reset)."""
        sp = _Space.of(haps, reads)
        regs, off = _regions(hap_first, read_first, flank_states)
        total = int(off[-1])
        if out is None:
            out = sp.empty(total, np.float64)
        status = sp.empty(total, np.int32) if want_status else None
        sp.order(self)
        self._check(_call(self._lib, "phmm_populate_regions", self._h, config, haps, error_model, C.byref(reads.c_struct()), C.byref(regs),
                          sp.ptr(out), sp.ptr(status), sp.flag), want_status)
        return (out, off, status) if want_status else (out, off)

    def assign_reads(self, config, haps: HaplotypeBlock, reads: ReadBlock, hap_first, read_first, log_priors=None, want_likelihoods=False,
                     want_status=False):
        """compute_haplotype_support's scoring and choice for many genotypes in one call (phmm_assign_reads). Group g (one genotype)
        owns haplotypes [hap_first[g], hap_first[g+1]) in genotype order and reads [read_first[g], read_first[g+1]); at most 64
        haplotypes per group. config.map_positions: every pair at the positions of the uncapped k-mer mapper (map_pairs), else at the
        original position only. log_priors: None or [H] per haplotype of the block.
        Returns top ([R] uint64: bit k = group-local haplotype k is in the read's find_map_haplotypes set), plus the flat likelihood
        vector (the groups' [H_g, R_g] matrices back to back, as populate_regions) when want_likelihoods and the per-pair statuses when
        want_status: numpy for host blocks, torch CUDA tensors for device-resident ones (top then as int64 with the same bits). With want_status a short haplotype does not
        raise; its statuses carry the extension and top is unspecified."""
        sp = _Space.of(haps, reads)
        rc, res = _assign(self._lib.phmm_assign_reads, self, sp, config, haps, reads, hap_first, read_first, log_priors, want_likelihoods,
                          want_status, sp.flag)
        self._check(rc, want_status)
        return res

    def assign_templates(self, config, haps: HaplotypeBlock, reads: ReadBlock, template_off, hap_first, template_first, log_priors=None,
                         want_likelihoods=False, want_status=False):
        """compute_haplotype_support over paired / linked templates for many genotypes in one call (phmm_assign_templates). Template
        t owns reads [template_off[t], template_off[t+1]) (at least one; template_off is moved to the host). Group g owns haplotypes
        [hap_first[g], hap_first[g+1]) and templates [template_first[g], template_first[g+1]). Scoring as assign_reads; the choice is
        per template, over the sum of its reads' likelihoods in read order plus the log prior.
        Returns top ([T] uint64: bit k = group-local haplotype k is in the template's find_map_haplotypes set), plus the flat template
        likelihoods (the groups' [H_g, T_g] matrices back to back) when want_likelihoods and the per-READ statuses (the groups'
        [H_g, R_g] matrices) when want_status; numpy or torch CUDA tensors as assign_reads."""
        sp = _Space.of(haps, reads)
        toff, read_first = _template_groups(template_off, template_first)
        rc, res = _assign(self._lib.phmm_assign_templates, self, sp, config, haps, reads, hap_first, read_first, log_priors,
                          want_likelihoods, want_status, sp.flag, templates=(toff, template_first))
        self._check(rc, want_status)
        return res

    @staticmethod
    def split_regions(flat, off, hap_first, read_first):
        """The per-region [H_g, R_g] views of a populate_regions result."""
        return [flat[int(off[g]):int(off[g + 1])].reshape(int(hap_first[g + 1] - hap_first[g]), int(read_first[g + 1] - read_first[g]))
                for g in range(len(off) - 1)]

    def populate(self, config, haps: HaplotypeBlock, reads: ReadBlock, positions=None, flank_state=None, out=None,
                 want_status=False, error_model=None):
        """Returns the (H, R) matrix of ln-likelihoods (numpy float64, or a torch CUDA tensor for device-resident blocks).
        positions: None or (off[H*R+1] int64, pos int32) CSR in [H][R] order. flank_state: None or (lhs_flank, rhs_flank).
        With ``error_model`` (an ErrorModel), haps is a HaplotypeSequences block: the GPU runs the model's reset() for every
        haplotype in the same call (phmm_populate_reset), with the result of error_model.reset + populate.
        out: None, or a float64 [H, R] CUDA tensor (or a column window of a wider one) for device-resident blocks. Without it the
        call allocates the result and waits for torch's current stream first; with it, and without want_status or positions to
        convert, the call issues no wait, so work still reading ``out`` from an earlier step must be ordered with wait_event."""
        sp = _Space.of(haps, reads)
        H, R = haps.n, reads.n
        if out is None:
            out = sp.empty((H, R), np.float64)
        status = sp.empty((H, R), np.int32) if want_status else None
        if sp.on_device and (tuple(out.shape) != (H, R) or out.dtype != sp.dtype(np.float64) or (R > 1 and out.stride(1) != 1)):
            raise ValueError("out must be a float64 [H, R] tensor with unit column stride")
        if error_model is not None and sp.on_device and H > 1 and out.stride(0) != R:
            raise ValueError("populate with an error model writes a dense [H, R] matrix")
        pos = _ref(_positions(sp, positions))
        sp.order(self)
        if error_model is not None:
            self._check(_call(self._lib, "phmm_populate", self._h, config, haps, error_model, C.byref(reads.c_struct()), pos,
                              _ref(_flank(flank_state)), sp.ptr(out), sp.ptr(status), sp.flag), want_status)
            return (out, status) if want_status else out
        args = (self._h, _config(config), C.byref(haps.c_struct()), C.byref(reads.c_struct()), pos, _ref(_flank(flank_state)))
        if sp.on_device and H > 1 and out.stride(0) != R:
            # a column window of a wider matrix — possibly another GPU's (octopus_b200.peer): phmm_populate_ld
            rc = self._lib.phmm_populate_ld(*args, sp.ptr(out), int(out.stride(0)), sp.ptr(status))
        else:
            rc = self._lib.phmm_populate(*args, sp.ptr(out), sp.ptr(status), sp.flag)
        self._check(rc, want_status)
        return (out, status) if want_status else out


class PopulateBatcher(_Handle):
    """One engine shared by many host threads (phmm_batcher_*): the populate requests that concurrent threads have in flight run
    as one multi-region kernel chain, their mutation-prime requests as one multi-set call, their assign and realign requests as one
    assign / realign call. Calls are thread-safe and block; ctypes releases the GIL during them, so Python threads really do wait
    together. Each result equals what ``PairHMMEngine.populate`` / ``mutation_prime`` / ``assign_reads`` / ``realign_reads`` returns
    for the request alone. Host blocks only."""
    _destroy = "phmm_batcher_destroy"

    def __init__(self, device=-1, clients=0, max_wait_us=None):
        opt = None
        if clients or max_wait_us is not None:
            opt = _lib.BatcherOptions(int(clients), 500 if max_wait_us is None else int(max_wait_us))
        self._create("phmm_batcher_create", int(device), _ref(opt))

    def _last_error(self):
        return self._lib.phmm_batcher_last_error().decode()      # this thread's last failing request

    def stats(self):
        """Counters since creation: requests, gpu_calls, merged_calls, max_regions_per_call, dp_cells."""
        s = _lib.BatcherStats()
        rc = self._lib.phmm_batcher_stats_get(self._h, C.byref(s))
        if rc != _lib.PHMM_OK:
            raise PhmmError(rc, "stats")
        return {f: int(getattr(s, f)) for f, _ in _lib.BatcherStats._fields_}

    def reruns(self):
        """Merged assign / realign calls that failed with PHMM_ERR_INVALID (one request's more than 4096 mapping positions) and were
        rerun one request at a time, so that each request got its own result (phmm_batcher_reruns)."""
        return int(self._lib.phmm_batcher_reruns(self._h))

    def populate(self, config, haps: HaplotypeBlock, reads: ReadBlock, positions=None, flank_state=None, want_status=False, error_model=None):
        """As PairHMMEngine.populate for host blocks: the (H, R) matrix (and the status matrix with want_status). With
        ``error_model``, haps is a HaplotypeSequences block (phmm_batcher_populate_reset): concurrent requests under models equal by
        content run as one call that derives their penalty arrays on the GPU."""
        assert not haps.on_device and not reads.on_device, "the batcher takes host blocks"
        H, R = haps.n, reads.n
        out = _HOST.empty((H, R), np.float64)
        status = _HOST.empty((H, R), np.int32) if want_status else None
        self._check(_call(self._lib, "phmm_batcher_populate", self._h, config, haps, error_model, C.byref(reads.c_struct()),
                          _ref(_positions(_HOST, positions)), _ref(_flank(flank_state)), _ptr(out), _ptr(status)), want_status)
        return (out, status) if want_status else out

    def populate_templates(self, config, haps: HaplotypeBlock, reads: ReadBlock, template_off, flank_state=None, want_status=False,
                           error_model=None):
        """As PairHMMEngine.populate_templates: the (H, T) matrix (and the per-read (H, R) status matrix with want_status). With
        ``error_model``, haps is a HaplotypeSequences block (phmm_batcher_populate_templates_reset)."""
        assert not haps.on_device and not reads.on_device, "the batcher takes host blocks"
        toff = np.ascontiguousarray(template_off, dtype=np.int64)
        T = len(toff) - 1
        out = _HOST.empty((haps.n, T), np.float64)
        status = _HOST.empty((haps.n, reads.n), np.int32) if want_status else None
        self._check(_call(self._lib, "phmm_batcher_populate_templates", self._h, config, haps, error_model, C.byref(reads.c_struct()),
                          toff.ctypes.data, T, _ref(_flank(flank_state)), _ptr(out), _ptr(status)), want_status)
        return (out, status) if want_status else out

    def assign_reads(self, config, haps: HaplotypeBlock, reads: ReadBlock, hap_first, read_first, log_priors=None, want_likelihoods=False,
                     want_status=False):
        """As PairHMMEngine.assign_reads for host blocks (phmm_batcher_assign_reads): concurrent requests with equal configs run as one
        call, each with the top sets, likelihoods and statuses it gets alone."""
        assert not haps.on_device and not reads.on_device, "the batcher takes host blocks"
        rc, res = _assign(self._lib.phmm_batcher_assign_reads, self, _HOST, config, haps, reads, hap_first, read_first, log_priors,
                          want_likelihoods, want_status)
        self._check(rc, want_status)
        return res

    def assign_templates(self, config, haps: HaplotypeBlock, reads: ReadBlock, template_off, hap_first, template_first, log_priors=None,
                         want_likelihoods=False, want_status=False):
        """As PairHMMEngine.assign_templates for host blocks (phmm_batcher_assign_templates): concurrent template requests with equal
        configs run as one call, each with the top sets, template likelihoods and statuses it gets alone."""
        assert not haps.on_device and not reads.on_device, "the batcher takes host blocks"
        toff, read_first = _template_groups(template_off, template_first)
        rc, res = _assign(self._lib.phmm_batcher_assign_templates, self, _HOST, config, haps, reads, hap_first, read_first, log_priors,
                          want_likelihoods, want_status, templates=(toff, template_first))
        self._check(rc, want_status)
        return res

    def realign_reads(self, config, haps: HaplotypeBlock, reads: ReadBlock, pairs, flank_state=None, cigar_stride=None):
        """As PairHMMEngine.realign_reads for host blocks (phmm_batcher_realign_reads): concurrent requests with equal configs and
        flank states run as one call whatever their CIGAR strides, each with the result it gets alone at its own stride."""
        assert not haps.on_device and not reads.on_device, "the batcher takes host blocks"
        rc, res = _realign(self._lib.phmm_batcher_realign_reads, self, _HOST, config, haps, reads, pairs, flank_state, cigar_stride)
        self._check(rc)
        return res

    def mutation_prime(self, model, sequences):
        """As PairHMMEngine.mutation_prime, through the shared engine: concurrent requests whose models are equal by content run as
        one phmm_mutation_prime_sets call, each with the (out, status) it gets alone."""
        off, seq, out, status = _mutation_set(sequences)
        self._check(self._lib.phmm_batcher_mutation_prime(self._h, model._h, len(off) - 1, off.ctypes.data, seq.ctypes.data,
                                                          out.ctypes.data, status.ctypes.data))
        return out, status


class MutationModel(_Handle):
    """DeNovoModel's parameters (core/models/mutation/denovo_model.hpp: Parameters{snv_prior, indel_prior}) as the engine holds them:
    the SNV prior and IndelMutationModel's repeat table for the indel prior (indel_mutation_model.cpp:40-55), open [P+1, Q+1] and
    extend [P+1, Q+1, X] float32 probabilities. The caller computes the table (it is not part of this library); the reference's
    defaults are P = 10, Q = 50, X = 50. SomaticMutationModel uses the same model under the cancer caller's priors."""
    _destroy = "phmm_mutation_model_destroy"

    def __init__(self, snv_prior, open_table, extend_table):
        self._open = np.ascontiguousarray(open_table, dtype=np.float32)
        self._extend = np.ascontiguousarray(extend_table, dtype=np.float32)
        if self._open.ndim != 2 or self._extend.ndim != 3 or self._extend.shape[:2] != self._open.shape:
            raise ValueError("open must be [P+1, Q+1] and extend [P+1, Q+1, X]")
        P, Q, X = self._open.shape[0] - 1, self._open.shape[1] - 1, self._extend.shape[2]
        self._create("phmm_mutation_model_create", float(snv_prior), self._open.ctypes.data, self._extend.ctypes.data, P, Q, X)
        self.snv_prior = float(snv_prior)
        self.max_period, self.max_periodicity, self.max_indel_length = P, Q, X

    def _last_error(self):
        return self._lib.phmm_error_model_last_error().decode()

    def context(self, sequences, n_threads=0):
        """IndelMutationModel::evaluate per haplotype (host): (cell, open_penalty, extend_penalty), flat over the concatenated bases.
        cell = period * (max_periodicity + 1) + periods of the repeat-table cell each base takes its probabilities from."""
        off, seq = pack_sequences(sequences)
        total = int(off[-1])
        cell = np.empty(total, dtype=np.int32)
        op, ep = np.empty(total, dtype=np.int8), np.empty(total, dtype=np.int8)
        self._check(self._lib.phmm_mutation_context(self._h, len(off) - 1, off.ctypes.data, seq.ctypes.data, cell.ctypes.data, op.ctypes.data,
                                                    ep.ctypes.data, int(n_threads)))
        return cell, op, ep


class ErrorModel(_Handle):
    """The reference's sequencing-error models behind HaplotypeLikelihoodModel::reset (haplotype_likelihood_model.cpp:60-78):
    make_error_model(label) / make_error_model(file) (core/models/error/error_model_factory.cpp:531-589). ``reset`` turns
    haplotype sequences into the HaplotypeBlock the engine consumes (host C++ inside libphmm_b200.so, no GPU involved)."""
    _destroy = "phmm_error_model_destroy"

    def __init__(self, label=None, custom_model_text=None):
        if custom_model_text is not None:
            self._create("phmm_error_model_create_custom", custom_model_text.encode() if isinstance(custom_model_text, str) else custom_model_text)
        else:
            self._create("phmm_error_model_create", None if label is None else label.encode())

    def _last_error(self):
        return self._lib.phmm_error_model_last_error().decode()

    def tandem_repeats(self, sequence, min_period=1, max_period=5):
        """tandem::extract_exact_tandem_repeats (lib/tandem/tandem.hpp:504-521): (n, 3) uint32 rows (pos, length, period)."""
        s = _u8(sequence)

        def attempt(cap):
            out = np.zeros((cap, 3), dtype=np.uint32)
            n = self._lib.phmm_tandem_repeats(s.ctypes.data, len(s), int(min_period), int(max_period), out.ctypes.data, cap)
            if n < 0:
                self._raise(n)
            return n, out[:n]
        return _grow(attempt, 4 * len(s) + 16)

    def reset(self, sequences, begin=None, is_substitution=None, n_threads=0, engine=None):
        """HaplotypeLikelihoodModel::reset for every haplotype: sequences (list of str / bytes / uint8 arrays) → HaplotypeBlock
        with the SNV masks / priors and gap penalties the reference's models assign. ``is_substitution``: optional list of
        per-base flag arrays (bases that are substitutions in Haplotype::cigar()). ``engine``: a PairHMMEngine to compute them
        on its GPU (byte-identical to the host threads)."""
        off, seq = pack_sequences(sequences)
        return self.reset_block(off, seq, begin, None if is_substitution is None else
                                np.ascontiguousarray(np.concatenate([np.asarray(x, dtype=np.uint8) for x in is_substitution])), n_threads,
                                engine)

    def reset_block(self, off, seq, begin=None, is_substitution=None, n_threads=0, engine=None):
        """reset for a packed block (off[n + 1], seq). Without ``engine``: host threads, numpy in and out. With a PairHMMEngine: its
        GPU computes the arrays; numpy inputs give a host block, CUDA torch tensors (off, seq, is_substitution) a device block."""
        if engine is not None:
            return self._reset_on(engine, off, seq, begin, is_substitution)
        off = np.ascontiguousarray(off, dtype=np.int64)
        seq = np.ascontiguousarray(seq, dtype=np.uint8)
        total = int(off[-1])
        mf, mr = np.empty(total, dtype=np.uint8), np.empty(total, dtype=np.uint8)
        pf, pr, go, ge = (np.empty(total, dtype=np.int8) for _ in range(4))
        self._check(self._lib.phmm_reset_haplotypes(self._h, len(off) - 1, off.ctypes.data, seq.ctypes.data,
                                                    None if is_substitution is None else is_substitution.ctypes.data,
                                                    mf.ctypes.data, pf.ctypes.data, mr.ctypes.data, pr.ctypes.data, go.ctypes.data,
                                                    ge.ctypes.data, int(n_threads)))
        return HaplotypeBlock(off, seq, mf, pf, mr, pr, go, ge, begin)

    def _reset_on(self, engine, off, seq, begin, is_substitution):
        sp = _Space(seq.device if _is_torch(seq) else None)
        off, seq = sp.input(off, np.int64), sp.input(seq, np.uint8)
        sub = None if is_substitution is None else sp.input(is_substitution, np.uint8)
        total = int(off[-1])
        mf, mr = sp.empty(total, np.uint8), sp.empty(total, np.uint8)
        pf, pr, go, ge = (sp.empty(total, np.int8) for _ in range(4))
        sp.order(engine)
        engine._check(self._lib.phmm_engine_reset_haplotypes(engine._h, self._h, len(off) - 1, sp.ptr(off), sp.ptr(seq), sp.ptr(sub),
                                                             sp.ptr(mf), sp.ptr(pf), sp.ptr(mr), sp.ptr(pr), sp.ptr(go), sp.ptr(ge), sp.flag))
        if not sp.on_device:
            return HaplotypeBlock(off, seq, mf, pf, mr, pr, go, ge, begin)
        return HaplotypeBlock.of_device(off, seq, mf, pf, mr, pr, go, ge, begin)


class HaplotypeLikelihoodModel:
    """Configuration holder with the reference's names (the per-haplotype state lives in the HaplotypeBlock)."""

    class Config:
        def __init__(self, use_mapping_quality=True, mapping_quality_cap_trigger=None, mapping_quality_cap=120,
                     use_flank_state=True, max_indel_error=8, use_int_scores=False, nuc_prior=2,
                     disable_naive_shortcut=False, map_positions=True):
            self.use_mapping_quality = use_mapping_quality
            self.mapping_quality_cap_trigger = mapping_quality_cap_trigger
            self.mapping_quality_cap = mapping_quality_cap
            self.use_flank_state = use_flank_state
            self.max_indel_error = max_indel_error
            self.use_int_scores = use_int_scores
            self.nuc_prior = nuc_prior
            self.disable_naive_shortcut = disable_naive_shortcut
            self.map_positions = map_positions   # run the reference's k-mer mapper on the device when no positions are given

        def c_struct(self):
            trig = self.mapping_quality_cap_trigger
            # haplotype_likelihood_model.cpp:50-52: a trigger >= the cap is dropped
            if trig is not None and trig >= self.mapping_quality_cap:
                trig = None
            return _lib.Config(int(self.max_indel_error), int(self.use_int_scores), int(self.use_mapping_quality),
                               int(self.mapping_quality_cap), -1 if trig is None else int(trig),
                               int(self.use_flank_state), int(self.nuc_prior), int(self.disable_naive_shortcut),
                               int(self.map_positions))

    def __init__(self, config=None):
        self.config = config or HaplotypeLikelihoodModel.Config()

    def pad_requirement(self):
        """hmm_.band_size() (haplotype_likelihood_model.cpp:55-58): smallest of 8,16,...,256 >= max_indel_error."""
        b = 8
        while b < self.config.max_indel_error:
            b *= 2
        return b


class VBResult:
    """VBResultPacket (variational_bayes_mixture_model.hpp:645-651) of one variational_bayes call: the max-evidence seed's
    genotype_posteriors, genotype_log_posteriors and alphas ([S, K]), max_log_evidence, evidence_weighted_genotype_posteriors;
    and which seed that was (max_seed), every seed's final log evidence and its number of iterations."""
    __slots__ = ("genotype_posteriors", "genotype_log_posteriors", "alphas", "max_log_evidence",
                 "evidence_weighted_genotype_posteriors", "max_seed", "seed_log_evidences", "seed_iterations")

    def __init__(self, *values):
        for name, v in zip(self.__slots__, values):
            setattr(self, name, v)


class VBMixtureMixtureResult:
    """VariationalBayesMixtureMixtureModel::Inferences (variational_bayes_mixture_mixture_model.hpp:72-77) of one
    variational_bayes_mixture_mixture call, without the component responsibilities: the max-evidence seed's genotype_posteriors,
    genotype_log_posteriors, group_concentrations [T], mixture_concentrations [S, sum K_t] and group_responsibilities [S, T],
    its approx_log_evidence (max_log_evidence); the weighted_genotype_posteriors and weighted_group_responsibilities; and which
    seed that was (max_seed), every seed's final log evidence and its number of iterations."""
    __slots__ = ("genotype_posteriors", "genotype_log_posteriors", "group_concentrations", "mixture_concentrations",
                 "group_responsibilities", "max_log_evidence", "weighted_genotype_posteriors", "weighted_group_responsibilities",
                 "max_seed", "seed_log_evidences", "seed_iterations")

    def __init__(self, *values):
        for name, v in zip(self.__slots__, values):
            setattr(self, name, v)


class HaplotypeLikelihoodArray:
    """likelihoods_[haplotype][sample][read or template] (haplotype_likelihood_array.hpp:34-175).

    All samples of a populate() go to the GPU as one batch: their reads are concatenated, one engine call fills one
    [H, R_total] matrix and a sample is a column range of it (views, no copies)."""

    mapperKmerSize = 6          # haplotype_likelihood_array.hpp:103
    maxMappingPositions = 10    # :104

    def __init__(self, likelihood_model=None, engine=None, error_model=None):
        self.likelihood_model = likelihood_model or HaplotypeLikelihoodModel()
        self._engine = engine
        self.error_model = error_model    # an ErrorModel: populate takes HaplotypeSequences and runs reset() on the GPU
        self.likelihoods = None     # [H, sum of the samples' widths]
        self._samples = []
        self._off = [0]
        self._primed = None

    @property
    def engine(self):
        if self._engine is None:
            self._engine = PairHMMEngine()
        return self._engine

    def _with_model(self):
        return {} if self.error_model is None else {"error_model": self.error_model}

    def _set_samples(self, names, widths):
        self._samples = list(names)
        self._off = [0]
        for w in widths:
            self._off.append(self._off[-1] + int(w))
        self._primed = None

    def populate(self, reads, haplotypes: HaplotypeBlock, flank_state=None, positions=None):
        """populate(ReadMap, haplotypes, flank_state) (haplotype_likelihood_array.cpp:51-103). ``reads``: a dict
        {sample: ReadBlock} in sample order, or one ReadBlock (a single unnamed sample, left primed)."""
        if isinstance(reads, ReadBlock):
            self._set_samples([""], [reads.n])
            self.likelihoods = self.engine.populate(self.likelihood_model.config, haplotypes, reads, positions, flank_state,
                                                    **self._with_model())
            self._primed = 0
            return self
        names = list(reads.keys())
        blocks = [reads[k] for k in names]
        self._set_samples(names, [b.n for b in blocks])
        self.likelihoods = self.engine.populate(self.likelihood_model.config, haplotypes, concat_reads(blocks), positions, flank_state,
                                                **self._with_model())
        return self

    def populate_templates(self, templates, haplotypes: HaplotypeBlock, flank_state=None):
        """populate(TemplateMap, ...) (:105-199). ``templates``: {sample: (ReadBlock, template_off)} — template t of the sample
        owns its reads [template_off[t], template_off[t+1]); one value per (haplotype, template)."""
        names = list(templates.keys())
        blocks, toff, base = [], [np.zeros(1, dtype=np.int64)], 0
        for k in names:
            rb, off = templates[k]
            off = np.asarray(off, dtype=np.int64)
            assert off[0] == 0 and off[-1] == rb.n, "template offsets must cover the sample's reads"
            blocks.append(rb)
            toff.append(off[1:] + base)
            base += rb.n
        self._set_samples(names, [len(templates[k][1]) - 1 for k in names])
        self.likelihoods = self.engine.populate_templates(self.likelihood_model.config, haplotypes, concat_reads(blocks),
                                                          np.concatenate(toff), flank_state, **self._with_model())
        return self

    # -- accessors (haplotype_likelihood_array.cpp:200-291) ----------------------------------------------------
    def samples(self):
        return list(self._samples)

    def _sample_index(self, sample):
        try:
            return self._samples.index(sample)
        except ValueError:
            raise KeyError(sample) from None      # the reference's unordered_map::at

    def num_likelihoods(self, sample=None):
        s = self._primed_index() if sample is None else self._sample_index(sample)
        return self._off[s + 1] - self._off[s]

    def __call__(self, sample, haplotype_index):
        s = self._sample_index(sample)
        return self.likelihoods[haplotype_index, self._off[s]:self._off[s + 1]]

    def __getitem__(self, haplotype_index):
        """likelihoods_[haplotype][primed sample] (:224-236)."""
        s = self._primed_index()
        return self.likelihoods[haplotype_index, self._off[s]:self._off[s + 1]]

    def extract_sample(self, sample):
        s = self._sample_index(sample)
        return self.likelihoods[:, self._off[s]:self._off[s + 1]]

    def is_empty(self):
        return self.likelihoods is None

    def clear(self):
        self.likelihoods = None
        self._set_samples([], [])

    def is_primed(self):
        return self._primed is not None

    def prime(self, sample):
        self._primed = self._sample_index(sample)

    def unprime(self):
        self._primed = None

    def _primed_index(self):
        if self._primed is None:
            raise RuntimeError("HaplotypeLikelihoodArray is not primed")      # an assert in the reference
        return self._primed

    def reset(self, haplotypes_to_keep):
        """reset(haplotypes) (:331-360): keep a subset of the haplotypes, given by their ascending old indices."""
        keep = [int(h) for h in haplotypes_to_keep]
        if not keep:
            self.clear()
            return
        assert all(a < b for a, b in zip(keep, keep[1:])) and 0 <= keep[0] and keep[-1] < self.likelihoods.shape[0]
        self.likelihoods = self.likelihoods[keep]

    def _columns(self, samples):
        """The matrix and column offsets of these samples in the given order: the array's own when they are its samples in its
        order, and gathered back to back otherwise."""
        idx = [self._sample_index(s) for s in samples]
        if idx == list(range(len(self._samples))):
            return self.likelihoods, self._off
        parts = [self.likelihoods[:, self._off[s]:self._off[s + 1]] for s in idx]
        if isinstance(self.likelihoods, np.ndarray):
            lnl = np.concatenate(parts, axis=1)
        else:
            import torch
            lnl = torch.cat(parts, dim=1)
        return lnl, np.concatenate([[0], np.cumsum([self._off[s + 1] - self._off[s] for s in idx])])

    def variational_bayes(self, samples, genotypes, prior_alphas, genotype_log_priors, seeds, epsilon=0.05, max_iterations=1000):
        """SubcloneModel::evaluate's inference (PairHMMEngine.variational_bayes) over these samples' columns, in the given order;
        prior_alphas[i] belongs to samples[i]. The samples' column ranges are passed as they are when they are the array's samples
        in its order, and gathered back to back otherwise."""
        lnl, off = self._columns(samples)
        return self.engine.variational_bayes(lnl, genotypes, prior_alphas, genotype_log_priors, seeds, off, epsilon, max_iterations)

    def variational_bayes_mixture_mixture(self, samples, group_sizes, combinations, genotype_log_priors, group_concentrations,
                                          mixture_concentrations, seeds, group_priors=None, group_prior_mask=None, epsilon=0.05,
                                          max_iterations=1000):
        """SingleCellModel's inference (PairHMMEngine.variational_bayes_mixture_mixture) over these samples' columns, in the given
        order; row i of the per-sample inputs belongs to samples[i]."""
        lnl, off = self._columns(samples)
        return self.engine.variational_bayes_mixture_mixture(lnl, group_sizes, combinations, genotype_log_priors, group_concentrations,
                                                             mixture_concentrations, seeds, off, group_priors, group_prior_mask,
                                                             epsilon, max_iterations)

    def merge_samples(self, samples=None, new_sample=None):
        """merge_samples (:362-409): a one-sample array holding the chosen samples' likelihoods back to back; primed."""
        samples = self.samples() if samples is None else list(samples)
        idx = [self._sample_index(s) for s in samples]
        out = HaplotypeLikelihoodArray(self.likelihood_model, self._engine, self.error_model)
        parts = [self.likelihoods[:, self._off[s]:self._off[s + 1]] for s in idx]
        if isinstance(self.likelihoods, np.ndarray):
            out.likelihoods = np.concatenate(parts, axis=1)
        else:                                                   # device-resident matrix (torch tensor)
            import torch
            out.likelihoods = torch.cat(parts, dim=1)
        out._set_samples(["".join(samples) if new_sample is None else new_sample], [out.likelihoods.shape[1]])
        out._primed = 0
        return out
