"""Checkers of the mutation model (DeNovoModel, phmm_mutation_*):

* ``RefMutation`` — the UNMODIFIED reference IndelMutationModel / DeNovoModel compiled into ``oracle/_ref/libref_mutation.so``
  (``oracle/ref_mutation_driver.cpp``, ``oracle/mutation.mk``; only where the reference checkout exists).
* ``recalculate`` — the plain-C restatement of recalculate_log_probability (tests/cpp/mutation_oracle.c), compiled on first use into a
  temporary directory so that the tree stays untouched.
* ``log_table`` — the per-cell table of logf(calculate_indel_probability), restated in numpy float32.
"""
import ctypes as C
import ctypes.util as ctypes_util
import os
import subprocess
import tempfile

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SRC = os.path.join(ROOT, "tests", "cpp", "mutation_oracle.c")
REF_LIB = os.path.join(ROOT, "oracle", "_ref", "libref_mutation.so")

# the reference's default priors (config/option_parser.cpp:614-620, 661-667: float options, widened to double): trio de novo SNV / indel,
# and the somatic ones of the cancer caller
TRIO_PRIORS = (float(np.float32(1.3e-8)), float(np.float32(1e-9)))
SOMATIC_PRIORS = (float(np.float32(1e-4)), float(np.float32(1e-6)))

_c = None


def _clib():
    global _c
    if _c is None:
        out = os.path.join(tempfile.mkdtemp(prefix="mutation_oracle_"), "libmutation_oracle.so")
        subprocess.run([os.environ.get("CC", "cc"), "-std=c11", "-O2", "-ffp-contract=off", "-fPIC", "-shared", "-Wall", "-o", out, SRC, "-lm"],
                       check=True)
        lib = C.CDLL(out)
        lib.oracle_recalculate.restype = C.c_int
        lib.oracle_recalculate.argtypes = [C.c_char_p, C.c_void_p, C.c_int64, C.c_void_p, C.c_int32, C.c_double, C.POINTER(C.c_double)]
        lib.oracle_recalculate_batch.restype = None
        lib.oracle_recalculate_batch.argtypes = [C.c_int64, C.c_void_p, C.c_int32, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_int32,
                                                 C.c_double, C.c_void_p, C.c_void_p]
        _c = lib
    return _c


def log_table(open_table, extend_table):
    """logp[cell, k] = logf(open * extend[1] * ... * extend[k]) accumulated left to right in float32 (calculate_indel_probability), the
    log taken by the C library's logf as std::log(float) does."""
    o = np.asarray(open_table, dtype=np.float32).reshape(-1)
    e = np.asarray(extend_table, dtype=np.float32).reshape(o.size, -1)
    prod = np.empty_like(e)
    acc = o.copy()
    for k in range(e.shape[1]):
        if k > 0:
            acc = (acc * e[:, k]).astype(np.float32)
        prod[:, k] = acc
    logf = C.CDLL(ctypes_util.find_library("m")).logf
    logf.restype, logf.argtypes = C.c_float, [C.c_float]
    return np.array([logf(float(x)) for x in prod.reshape(-1)], dtype=np.float32).reshape(prod.shape)


def recalculate_batch(cigars, stride, given, off, cell, logp, snv_prior):
    """cigars: bytes buffer of n * stride CIGAR texts; given[j]: the given haplotype of alignment j. Returns (values, status)."""
    n = len(given)
    given = np.ascontiguousarray(given, dtype=np.int32)
    off = np.ascontiguousarray(off, dtype=np.int64)
    cell = np.ascontiguousarray(cell, dtype=np.int32)
    logp = np.ascontiguousarray(logp, dtype=np.float32)
    buf = np.frombuffer(cigars, dtype=np.uint8) if isinstance(cigars, (bytes, bytearray)) else np.ascontiguousarray(cigars).view(np.uint8)
    out = np.zeros(n, dtype=np.float64)
    st = np.zeros(n, dtype=np.int32)
    _clib().oracle_recalculate_batch(n, buf.ctypes.data, int(stride), given.ctypes.data, off.ctypes.data, cell.ctypes.data,
                                     logp.ctypes.data, logp.shape[1], float(np.log(snv_prior)), out.ctypes.data, st.ctypes.data)
    return out, st


def recalculate(cigar, cell, logp, snv_prior):
    """One alignment against one given haplotype (cell: its per-base cells). Returns (status, value)."""
    cell = np.ascontiguousarray(cell, dtype=np.int32)
    logp = np.ascontiguousarray(logp, dtype=np.float32)
    v = C.c_double(0)
    st = _clib().oracle_recalculate(cigar.encode(), cell.ctypes.data, len(cell), logp.ctypes.data, logp.shape[1], float(np.log(snv_prior)), C.byref(v))
    return st, v.value


class RefMutation:
    """The reference's IndelMutationModel and DeNovoModel, unmodified (oracle/_ref/libref_mutation.so)."""

    @staticmethod
    def available():
        return os.path.exists(REF_LIB)

    def __init__(self):
        self.lib = L = C.CDLL(REF_LIB)
        L.ref_mutation_table.restype = C.c_int
        L.ref_mutation_table.argtypes = [C.c_double, C.c_void_p, C.c_void_p, C.c_void_p]
        L.ref_mutation_context.restype = C.c_int
        L.ref_mutation_context.argtypes = [C.c_double, C.c_char_p, C.c_int, C.c_void_p, C.c_void_p]
        L.ref_mutation_prime.restype = C.c_int
        L.ref_mutation_prime.argtypes = [C.c_double, C.c_double, C.c_int, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p]

    def table(self, indel_prior):
        """IndelMutationModel's repeat table: open [P+1, Q+1], extend [P+1, Q+1, X] (float32)."""
        dims = np.zeros(3, dtype=np.int32)
        self.lib.ref_mutation_table(float(indel_prior), dims.ctypes.data, None, None)
        P, Q, X = (int(x) for x in dims)
        o = np.zeros((P + 1, Q + 1), dtype=np.float32)
        e = np.zeros((P + 1, Q + 1, X), dtype=np.float32)
        self.lib.ref_mutation_table(float(indel_prior), dims.ctypes.data, o.ctypes.data, e.ctypes.data)
        return o, e

    def context(self, indel_prior, seq, max_indel_length=50):
        """IndelMutationModel::evaluate: (gap_open [n], gap_extend [n, X]) float32."""
        s = seq.encode() if isinstance(seq, str) else bytes(seq)
        go = np.zeros(len(s), dtype=np.float32)
        ge = np.zeros((len(s), max_indel_length), dtype=np.float32)
        assert self.lib.ref_mutation_context(float(indel_prior), s, len(s), go.ctypes.data, ge.ctypes.data) == 0
        return go, ge

    def prime(self, snv_prior, indel_prior, sequences):
        """DeNovoModel::prime + evaluate over every ordered pair: (out [H, H], approx [H, H] bool: Haplotype::difference was called)."""
        parts = [s.encode() if isinstance(s, str) else bytes(s) for s in sequences]
        off = np.zeros(len(parts) + 1, dtype=np.int64)
        np.cumsum([len(p) for p in parts], out=off[1:])
        seq = np.frombuffer(b"".join(parts) + b"\0", dtype=np.uint8)
        H = len(parts)
        out = np.zeros((H, H), dtype=np.float64)
        approx = np.zeros((H, H), dtype=np.int32)
        self.lib.ref_mutation_prime(float(snv_prior), float(indel_prior), H, off.ctypes.data, seq.ctypes.data, out.ctypes.data, approx.ctypes.data)
        return out, approx.astype(bool)


ACGT = "ACGT"


def repeat_sequence(rng, max_len=300, n_runs=True):
    """Random haplotype with injected exact tandem repeats (period 1..5, up to 70 periods, so some exceed the table's 50), the odd 'N'
    inside a motif and, optionally, N runs."""
    s = "".join(rng.choice(list(ACGT), int(rng.integers(1, max_len))))
    for _ in range(int(rng.integers(0, 4))):
        p = int(rng.integers(1, 6))
        motif = "".join(rng.choice(list("ACGTN" if rng.random() < 0.1 else ACGT), p))
        at = int(rng.integers(0, len(s) + 1))
        s = s[:at] + motif * int(rng.integers(2, 70)) + s[at:]
    if n_runs and rng.random() < 0.3:
        at = int(rng.integers(0, len(s) + 1))
        s = s[:at] + "N" * int(rng.integers(1, 8)) + s[at:]
    return s


def mutate(rng, s, n_events):
    """s with n_events SNVs and 1-20 bp indels (some inside repeats: a period-sized insertion copies the bases before it)."""
    s = list(s)
    for _ in range(n_events):
        at = int(rng.integers(0, len(s) + 1))
        r = rng.random()
        if r < 0.5 and at < len(s):
            s[at] = rng.choice([b for b in ACGT if b != s[at]])
        elif r < 0.75:
            k = int(rng.integers(1, 21))
            ins = s[max(0, at - k):at] if rng.random() < 0.5 and at >= k else list(rng.choice(list(ACGT), k))
            s[at:at] = ins
        elif len(s) > 21:
            k = int(rng.integers(1, 21))
            del s[at:at + k]
    return "".join(s) if s else "A"


def haplotype_set(rng, n, max_len=300, n_events=(0, 6)):
    """n haplotypes of one region: a repeat-rich base haplotype and mutated copies of it (trio-shaped sets)."""
    base = repeat_sequence(rng, max_len)
    return [base] + [mutate(rng, base, int(rng.integers(n_events[0], n_events[1] + 1))) for _ in range(n - 1)]


def penalty(p):
    """probability_to_penalty (denovo_model.cpp:23-27): std::round is half away from zero."""
    return int(max(min(np.floor(np.log(p) / -0.230258509299404568401799145468436420760110148862877297603 + 0.5), 127.0), 1.0))


def align_pairs_recipe(engine, model, open_table, extend_table, sequences):
    """DeNovoModel::prime the way it had to be assembled before phmm_mutation_prime: the library's host context model, padded truths
    and penalty arrays built here, phmm_align_pairs over the pairs within the band, every CIGAR copied back and re-scored on the host
    (the C restatement). Returns (out [H, H], status [H, H]) in phmm_mutation_prime's convention."""
    from octopus_b200 import HaplotypeLikelihoodModel, _lib
    from octopus_b200.batch import HaplotypeBlock, ReadBlock
    H = len(sequences)
    lens = np.array([len(s) for s in sequences], dtype=np.int64)
    off = np.zeros(H + 1, dtype=np.int64)
    np.cumsum(lens, out=off[1:])
    seq = np.frombuffer("".join(sequences).encode(), dtype=np.uint8)
    cell, op, ep = model.context(sequences)
    Lp = int(lens.max()) + 64
    tseq = np.full((H, Lp), ord("N"), np.uint8)
    tgo = np.full((H, Lp), 60, np.int8)
    tge = np.full((H, Lp), 60, np.int8)
    for h in range(H):
        tseq[h, 32:32 + lens[h]] = seq[off[h]:off[h + 1]]
        tgo[h, 32:32 + lens[h]] = op[off[h]:off[h + 1]]
        tge[h, 32:32 + lens[h]] = ep[off[h]:off[h + 1]]
    zeros = np.zeros(H * Lp, np.uint8)
    truths = HaplotypeBlock(np.arange(H + 1, dtype=np.int64) * Lp, tseq.reshape(-1), zeros, zeros.view(np.int8), zeros, zeros.view(np.int8),
                            tgo.reshape(-1), tge.reshape(-1))
    targets = ReadBlock(off, seq, np.full(len(seq), penalty(model.snv_prior), np.uint8), np.zeros(H, np.uint8))
    t, g = np.meshgrid(np.arange(H), np.arange(H), indexing="ij")
    t, g = t.reshape(-1), g.reshape(-1)
    listed = (t != g) & (np.abs(lens[t] - lens[g]) < 32)
    pairs = np.ascontiguousarray(np.stack([t[listed], g[listed]], axis=1), dtype=np.int32)
    n = len(pairs)
    stride = 4 * int(lens.max()) + 160
    cfg = HaplotypeLikelihoodModel.Config(max_indel_error=32, use_mapping_quality=False, use_flank_state=False, map_positions=False)
    toff, lk, st = np.zeros(n, np.int64), np.zeros(n, np.float64), np.zeros(n, np.int32)
    cg = np.zeros(n * stride, np.uint8)
    offs = np.full(n, 32, np.int32)
    hs, rs, cs = truths.c_struct(), targets.c_struct(), cfg.c_struct()
    rc = engine._lib.phmm_align_pairs(engine._h, C.byref(cs), C.byref(hs), C.byref(rs), pairs.ctypes.data, offs.ctypes.data, n, None,
                                      toff.ctypes.data, lk.ctypes.data, cg.ctypes.data, stride, st.ctypes.data, _lib.SPACE_HOST)
    if rc != 0:
        engine._raise(rc)
    values, rst = recalculate_batch(cg, stride, pairs[:, 1], off, cell, log_table(open_table, extend_table), model.snv_prior)
    out = np.zeros(H * H, np.float64)
    status = np.full(H * H, _lib.MUT_APPROX_LENGTH, np.int32)
    status[t == g] = _lib.MUT_SELF
    idx = t[listed] * H + g[listed]
    s = np.where(st == 4, _lib.MUT_APPROX_OVERFLOW,                                       # PHMM_STATUS_HMM_OVERFLOW
                 np.where(toff != 32, _lib.MUT_APPROX_OFFSET, np.where(rst != 0, _lib.MUT_OUT_OF_MODEL, _lib.MUT_HMM)))
    status[idx] = s
    out[idx] = np.where(s == _lib.MUT_HMM, values, 0.0)
    return out.reshape(H, H), status.reshape(H, H)
