"""TEST INFRASTRUCTURE ONLY — ctypes loaders for the two CPU oracles.

* ``RefKernel``  — the UNMODIFIED reference SIMD kernel compiled into ``oracle/_ref/libref_phmm_<isa>.so``
  (``oracle/ref_driver.cpp``, built by ``oracle/Makefile`` from the reference checkout, see ``REFERENCE``).
* ``RefHMM``     — the UNMODIFIED reference layer above the kernel (``hmm::evaluate`` / ``hmm::align`` / band choice) compiled
  into ``oracle/_ref/libref_hmm.so`` (``oracle/ref_hmm_driver.cpp``).
* ``COracle``    — the plain-C restatement ``oracle/liboctopus_oracle.so`` (``oracle/phmm_oracle.c``).

Only ``tests/``, ``__graft_entry__.smoke()`` and ``bench.py``'s cpu_baseline / ``--impl reference`` legs may
import this module. The product package ``octopus_b200`` never does.
"""
import ctypes as C
import os
import subprocess

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
REF_DIR = os.path.join(_HERE, "_ref")
# A source checkout of luntergroup/octopus: OCTOPUS_REFERENCE, else the build environment's standard location of it. Only where
# one exists are the reference oracles compiled into oracle/_ref/; elsewhere the tests use what oracle/_ref/ already holds and the
# fixtures under tests/golden/.
REFERENCE = os.environ.get("OCTOPUS_REFERENCE") or "/root/reference"


def have_reference():
    return bool(REFERENCE) and os.path.isdir(os.path.join(REFERENCE, "src", "core", "models", "pairhmm"))

_i8p = C.POINTER(C.c_int8)
_i32p = C.POINTER(C.c_int32)
_i64p = C.POINTER(C.c_int64)


def cpu_flags():
    try:
        with open("/proc/cpuinfo") as f:
            for line in f:
                if line.startswith("flags"):
                    return set(line.split(":", 1)[1].split())
    except OSError:
        pass
    return set()


def available_ref_isas():
    """ISA builds of the reference kernel this host can execute, best first."""
    flags = cpu_flags()
    out = []
    if {"avx512f", "avx512bw", "avx512vl", "avx512dq"} <= flags:
        out.append("avx512")
    if "avx2" in flags:
        out.append("avx2")
    if "sse4_1" in flags:
        out.append("sse")
    return [i for i in out if os.path.exists(os.path.join(REF_DIR, "libref_phmm_%s.so" % i))]


def build(ref=None, quiet=True):
    """(Re)build the oracle libraries. The reference build only happens where the reference checkout exists."""
    ref = have_reference() if ref is None else ref and have_reference()
    target = ["all", "REF=" + REFERENCE] if ref else ["liboctopus_oracle.so"]
    subprocess.run(["make", "-C", _HERE] + target, check=True,
                   stdout=subprocess.DEVNULL if quiet else None)


def _b(x):
    """bytes / str / uint8-or-int8 ndarray → a ctypes char buffer that keeps its storage alive."""
    if isinstance(x, str):
        x = x.encode()
    if isinstance(x, (bytes, bytearray)):
        return C.create_string_buffer(bytes(x), len(x) + 1)
    a = np.ascontiguousarray(x)
    return C.create_string_buffer(a.tobytes(), a.nbytes + 1)


def _i8(x):
    a = np.ascontiguousarray(np.asarray(x, dtype=np.int8))
    return a, a.ctypes.data_as(_i8p)


class RefErrorModel:
    """The UNMODIFIED reference error models + lib/tandem (``oracle/_ref/libref_errmodel.so``, ``oracle/ref_errmodel_driver.cpp``):
    what HaplotypeLikelihoodModel::reset computes per haplotype. Checker for octopus_b200.ErrorModel."""
    PATH = os.path.join(REF_DIR, "libref_errmodel.so")

    @classmethod
    def available(cls):
        return os.path.exists(cls.PATH)

    def __init__(self):
        self.lib = C.CDLL(self.PATH)
        self.lib.ref_tandem_repeats.restype = C.c_int
        self.lib.ref_tandem_repeats.argtypes = [C.c_char_p, C.c_int, C.c_int, C.c_int, C.c_void_p, C.c_int]
        for name in ("ref_errmodel_reset", "ref_errmodel_reset_custom"):
            f = getattr(self.lib, name)
            f.restype = C.c_int
            f.argtypes = [C.c_char_p, C.c_char_p, C.c_int, C.c_void_p] + [C.c_void_p] * 6

    def tandem_repeats(self, seq, min_period, max_period):
        s = bytes(seq)
        cap = 4 * len(s) + 16
        out = np.zeros((cap, 3), dtype=np.uint32)
        n = self.lib.ref_tandem_repeats(s, len(s), min_period, max_period, out.ctypes.data, cap)
        assert 0 <= n <= cap
        return out[:n]

    def reset(self, seq, label="PCR-free.HiSeq-2500", is_substitution=None, custom_model_text=None):
        """One haplotype → dict of the six arrays (+ 'rc': 1 with an SNV model, 0 without, < 0 on a model error)."""
        s = bytes(seq)
        n = len(s)
        names = ("snv_mask_fwd", "snv_prior_fwd", "snv_mask_rev", "snv_prior_rev", "gap_open", "gap_extend")
        arrs = [np.zeros(n, dtype=np.uint8 if "mask" in k else np.int8) for k in names]
        sub = None if is_substitution is None else np.ascontiguousarray(is_substitution, dtype=np.uint8)
        ptrs = [a.ctypes.data for a in arrs]
        if custom_model_text is not None:
            rc = self.lib.ref_errmodel_reset_custom(custom_model_text.encode(), s, n, None if sub is None else sub.ctypes.data, *ptrs)
        else:
            rc = self.lib.ref_errmodel_reset(label.encode(), s, n, None if sub is None else sub.ctypes.data, *ptrs)
        out = dict(zip(names, arrs))
        out["rc"] = rc
        return out


class RefKernel:
    """The reference kernel for one ISA build ('sse' | 'avx2' | 'avx512'). isa_force_sse2 → SSE2 policy even in a wider build."""

    def __init__(self, isa=None):
        isas = available_ref_isas()
        if isa is None:
            if not isas:
                raise RuntimeError("no oracle/_ref library usable on this host (build with `make -C oracle REF=<octopus checkout>`)")
            isa = isas[0]
        elif isa not in isas:
            raise RuntimeError("reference ISA build %r not available on this host (have %s)" % (isa, isas))
        self.isa = isa
        self.lib = C.CDLL(os.path.join(REF_DIR, "libref_phmm_%s.so" % isa))
        L = self.lib
        L.ref_isa_name.restype = C.c_char_p
        L.ref_isa_name.argtypes = [C.c_int, C.c_int, C.c_int]
        L.ref_align.restype = C.c_int
        L.ref_align.argtypes = [C.c_int, C.c_int, C.c_int, C.c_char_p, C.c_char_p, _i8p, C.c_int, C.c_int,
                                C.c_char_p, _i8p, _i8p, _i8p, C.c_int, C.c_int]
        L.ref_align_tb.restype = C.c_int
        L.ref_align_tb.argtypes = L.ref_align.argtypes + [_i32p, C.c_char_p, C.c_char_p]
        L.ref_flank_score.restype = C.c_int
        L.ref_flank_score.argtypes = [C.c_int, C.c_int, C.c_int, C.c_int, C.c_int, C.c_int, C.c_char_p, _i8p,
                                      C.c_char_p, _i8p, _i8p, _i8p, C.c_int, C.c_int, C.c_int, C.c_char_p, C.c_char_p, _i32p]
        L.ref_align_batch.restype = C.c_int
        L.ref_align_batch.argtypes = [C.c_int, C.c_int, C.c_int, C.c_long,
                                      C.c_void_p, C.c_void_p, C.c_void_p,
                                      C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p,
                                      C.c_void_p, C.c_void_p, C.c_void_p, C.c_int, C.c_int, C.c_void_p]

    def name(self, band, bits=16, force_sse2=False):
        return self.lib.ref_isa_name(band, bits, int(force_sse2)).decode()

    def _args(self, band, bits, force_sse2, truth, read, quals, snv_mask, snv_prior, gap_open, gap_extend, nuc_prior):
        keep = []
        t, r = _b(truth), _b(read)
        q, qp = _i8(quals)
        go, gop = _i8(gap_open)
        keep += [t, r, q, go]
        if snv_mask is not None:
            m = _b(snv_mask)
            sp, spp = _i8(snv_prior)
            keep += [m, sp]
        else:
            m, spp = None, None
        if np.ndim(gap_extend) == 0:
            gep, ges = None, int(gap_extend)
        else:
            ge, gep = _i8(gap_extend)
            keep.append(ge)
            ges = 0
        W, L = len(t) - 1, len(r) - 1
        assert W == L + 2 * band - 1, "truth window must be L + 2*band - 1 long"
        return keep, [band, bits, int(force_sse2), t, r, qp, W, L, m, spp, gop, gep, ges, int(nuc_prior)]

    def align(self, band, truth, read, quals, gap_open, gap_extend, nuc_prior=2, snv_mask=None, snv_prior=None,
              bits=16, force_sse2=False):
        keep, a = self._args(band, bits, force_sse2, truth, read, quals, snv_mask, snv_prior, gap_open, gap_extend, nuc_prior)
        s = self.lib.ref_align(*a)
        if s == -1000000:
            raise ValueError("unsupported (band, bits)")
        return s

    def align_tb(self, band, truth, read, quals, gap_open, gap_extend, nuc_prior=2, snv_mask=None, snv_prior=None,
                 bits=16, force_sse2=False):
        keep, a = self._args(band, bits, force_sse2, truth, read, quals, snv_mask, snv_prior, gap_open, gap_extend, nuc_prior)
        n = 2 * (len(read) + band) + 1
        a1, a2 = C.create_string_buffer(n + 8), C.create_string_buffer(n + 8)
        fp = C.c_int32(-7)
        s = self.lib.ref_align_tb(*(a + [C.byref(fp), a1, a2]))
        if s == -1000000:
            raise ValueError("unsupported (band, bits)")
        return s, fp.value, a1.value.decode(), a2.value.decode()

    def flank_score(self, band, truth_len, lhs, rhs, read, quals, snv_mask, snv_prior, gap_open, gap_extend, nuc_prior,
                    first_pos, align1, align2, bits=16, force_sse2=False):
        r, m = _b(read), _b(snv_mask)
        q, qp = _i8(quals)
        sp, spp = _i8(snv_prior)
        go, gop = _i8(gap_open)
        if np.ndim(gap_extend) == 0:
            gep, ges = None, int(gap_extend)
        else:
            ge, gep = _i8(gap_extend)
            ges = 0
        ms = C.c_int32(0)
        s = self.lib.ref_flank_score(band, bits, int(force_sse2), truth_len, lhs, rhs, r, qp, m, spp, gop, gep, ges, int(nuc_prior),
                                     first_pos, _b(align1), _b(align2), C.byref(ms))
        return s, ms.value

    def align_batch(self, band, batch, read_idx, hap_idx, win_off, nuc_prior=2, nthreads=1, bits=16, force_sse2=False, strand_rev=False):
        """batch: dict of packed numpy arrays (see octopus_b200.synth.pack_*). Returns int32 scores."""
        read_idx = np.ascontiguousarray(read_idx, dtype=np.int32)
        hap_idx = np.ascontiguousarray(hap_idx, dtype=np.int32)
        win_off = np.ascontiguousarray(win_off, dtype=np.int32)
        n = len(read_idx)
        out = np.empty(n, dtype=np.int32)
        mask = batch["hap_mask_rev"] if strand_rev else batch["hap_mask_fwd"]
        prior = batch["hap_prior_rev"] if strand_rev else batch["hap_prior_fwd"]
        arrs = [batch["read_bases"], batch["read_quals"], batch["read_off"], batch["hap_seq"], mask, prior,
                batch["hap_gap_open"], batch["hap_gap_extend"], batch["hap_off"], read_idx, hap_idx, win_off]
        for a in (batch["read_off"], batch["hap_off"]):
            assert a.dtype == np.int64
        rc = self.lib.ref_align_batch(band, bits, int(force_sse2), n, *[a.ctypes.data for a in arrs[:12]],
                                      int(nuc_prior), int(nthreads), out.ctypes.data)
        if rc != 0:
            raise ValueError("unsupported (band, bits)")
        return out


class _ModelArgs(C.Structure):      # struct ModelArgs of oracle/ref_hmm_driver.cpp
    _fields_ = [("max_indel_error", C.c_int), ("use_int_scores", C.c_int), ("use_mapping_quality", C.c_int), ("mapq_cap", C.c_int),
                ("mapq_cap_trigger", C.c_int),
                ("hap", C.c_char_p), ("hap_len", C.c_int), ("hap_begin", C.c_longlong),
                ("mask_f", C.c_char_p), ("prior_f", _i8p), ("mask_r", C.c_char_p), ("prior_r", _i8p), ("gap_open", _i8p), ("gap_extend", _i8p),
                ("has_flank", C.c_int), ("lhs_flank", C.c_longlong), ("rhs_flank", C.c_longlong),
                ("read", C.c_char_p), ("quals", C.c_void_p), ("read_len", C.c_int), ("mapping_quality", C.c_int), ("reverse", C.c_int),
                ("read_begin", C.c_longlong),
                ("positions", C.POINTER(C.c_longlong)), ("n_positions", C.c_int), ("map_positions", C.c_int)]


class _ArrayArgs(C.Structure):      # struct ArrayArgs of oracle/ref_hmm_driver.cpp
    _fields_ = [("max_indel_error", C.c_int), ("use_int_scores", C.c_int), ("use_mapping_quality", C.c_int), ("mapq_cap", C.c_int),
                ("mapq_cap_trigger", C.c_int),
                ("H", C.c_int), ("hap_off", C.c_void_p), ("seq", C.c_void_p), ("mask_f", C.c_void_p), ("prior_f", C.c_void_p), ("mask_r", C.c_void_p),
                ("prior_r", C.c_void_p), ("gap_open", C.c_void_p), ("gap_extend", C.c_void_p), ("hap_begin", C.c_void_p),
                ("S", C.c_int), ("sample_off", C.c_void_p),
                ("R", C.c_int), ("read_off", C.c_void_p), ("bases", C.c_void_p), ("quals", C.c_void_p), ("mapq", C.c_void_p),
                ("reverse", C.c_void_p), ("read_begin", C.c_void_p),
                ("T", C.c_int), ("template_off", C.c_void_p),
                ("has_flank", C.c_int), ("lhs_flank", C.c_longlong), ("rhs_flank", C.c_longlong)]


class RefHMM:
    """The UNMODIFIED reference above the kernel, behind oracle/ref_hmm_driver.cpp (oracle/_ref/libref_hmm.so): hmm::evaluate,
    hmm::align, the band-choosing PairHMMWrapper (pair_hmm.hpp, simd_pair_hmm_wrapper.hpp), the k-mer mapper
    (utils/kmer_mapper.hpp) and HaplotypeLikelihoodModel::{reset, evaluate, align} (haplotype_likelihood_model.cpp)."""

    @staticmethod
    def available():
        return os.path.exists(os.path.join(REF_DIR, "libref_hmm.so")) and "sse4_1" in cpu_flags()

    def __init__(self):
        self.lib = C.CDLL(os.path.join(REF_DIR, "libref_hmm.so"))
        self.lib.ref_hmm_band.restype = C.c_int
        self.lib.ref_hmm_evaluate.restype = C.c_double
        self.lib.ref_hmm_align.restype = C.c_int
        self.lib.ref_model_evaluate.restype = C.c_int
        self.lib.ref_model_align.restype = C.c_int
        self.lib.ref_array_populate.restype = C.c_int

    def band(self, requested, int32=False):
        return self.lib.ref_hmm_band(int(requested), int(int32))

    def _model_args(self, band_request, hap, read, quals, gap_open, gap_extend, mask_f, prior_f, mask_r, prior_r, positions, hap_begin, read_begin,
                    mapping_quality, reverse, flanks, use_mapping_quality, mapq_cap, mapq_cap_trigger, int32):
        h, r, mf, mr = _b(hap), _b(read), _b(mask_f), _b(mask_r)
        q = np.ascontiguousarray(np.asarray(quals, dtype=np.uint8))
        go, gop = _i8(gap_open); ge, gep = _i8(gap_extend); pf, pfp = _i8(prior_f); pr, prp = _i8(prior_r)
        n = len(h) - 1
        assert len(go) == len(ge) == len(pf) == len(pr) == n == len(mf) - 1 == len(mr) - 1 and len(q) == len(r) - 1
        map_positions = positions is None
        pos = (C.c_longlong * max(1, 0 if map_positions else len(positions)))(*([] if map_positions else [int(x) for x in positions]))
        a = _ModelArgs(int(band_request), int(int32), int(use_mapping_quality), int(mapq_cap), int(mapq_cap_trigger),
                       C.cast(h, C.c_char_p), n, int(hap_begin), C.cast(mf, C.c_char_p), pfp, C.cast(mr, C.c_char_p), prp, gop, gep,
                       0 if flanks is None else 1, 0 if flanks is None else int(flanks[0]), 0 if flanks is None else int(flanks[1]),
                       C.cast(r, C.c_char_p), q.ctypes.data, len(r) - 1, int(mapping_quality), int(bool(reverse)), int(read_begin),
                       pos, 0 if map_positions else len(positions), int(map_positions))
        return a, (h, r, mf, mr, q, go, ge, pf, pr, pos)

    def model_evaluate(self, band_request, hap, read, quals, gap_open, gap_extend, mask_f, prior_f, mask_r, prior_r, positions, hap_begin=0,
                       read_begin=0, mapping_quality=60, reverse=False, flanks=None, use_mapping_quality=True, mapq_cap=120,
                       mapq_cap_trigger=-1, int32=False):
        """HaplotypeLikelihoodModel::reset + evaluate. positions=None → mapped by the reference's k-mer mapper as populate() does.
        Returns (status, value, required_extension); status 1 == ShortHaplotypeError."""
        a, keep = self._model_args(band_request, hap, read, quals, gap_open, gap_extend, mask_f, prior_f, mask_r, prior_r, positions, hap_begin,
                                   read_begin, mapping_quality, reverse, flanks, use_mapping_quality, mapq_cap, mapq_cap_trigger, int32)
        out, ext = C.c_double(0), C.c_int(0)
        st = self.lib.ref_model_evaluate(C.byref(a), C.byref(out), C.byref(ext))
        return st, out.value, ext.value

    def model_align(self, band_request, hap, read, quals, gap_open, gap_extend, mask_f, prior_f, mask_r, prior_r, positions, hap_begin=0,
                    read_begin=0, mapping_quality=60, reverse=False, flanks=None, use_mapping_quality=True, mapq_cap=120,
                    mapq_cap_trigger=-1, int32=False):
        """HaplotypeLikelihoodModel::reset + align. Returns (status, mapping_position, likelihood, cigar_text, required_extension)."""
        a, keep = self._model_args(band_request, hap, read, quals, gap_open, gap_extend, mask_f, prior_f, mask_r, prior_r, positions, hap_begin,
                                   read_begin, mapping_quality, reverse, flanks, use_mapping_quality, mapq_cap, mapq_cap_trigger, int32)
        mp_, lk, ext = C.c_longlong(0), C.c_double(0), C.c_int(0)
        cap = 8 * (a.read_len + 512) + 64
        cig = C.create_string_buffer(cap)
        st = self.lib.ref_model_align(C.byref(a), C.byref(mp_), C.byref(lk), cig, cap, C.byref(ext))
        return st, mp_.value, lk.value, cig.value.decode(), ext.value

    def array_populate(self, band_request, haps, reads, sample_off=None, template_off=None, flanks=None, use_mapping_quality=True,
                       mapq_cap=120, mapq_cap_trigger=-1, int32=False):
        """HaplotypeLikelihoodArray::populate (haplotype_likelihood_array.cpp, unmodified) on a HaplotypeBlock / ReadBlock pair.
        sample_off: boundaries of the samples over the reads (or over the templates when template_off is given); default one sample.
        Returns (status, matrix [H, reads or templates], required_extension); status 1 == ShortHaplotypeError."""
        p = lambda a: np.ascontiguousarray(a).ctypes.data
        keep = [np.ascontiguousarray(x) for x in (haps.off, haps.seq, haps.snv_mask_fwd, haps.snv_prior_fwd, haps.snv_mask_rev, haps.snv_prior_rev,
                                                  haps.gap_open, haps.gap_extend, haps.begin if haps.begin is not None else np.zeros(haps.n, np.int64),
                                                  reads.off, reads.bases, reads.quals, reads.mapq, reads.reverse, reads.begin)]
        n_items = reads.n if template_off is None else len(template_off) - 1
        so = np.ascontiguousarray([0, n_items] if sample_off is None else sample_off, dtype=np.int64)
        to = np.ascontiguousarray([0] if template_off is None else template_off, dtype=np.int64)
        a = _ArrayArgs(int(band_request), int(int32), int(use_mapping_quality), int(mapq_cap), int(mapq_cap_trigger),
                       haps.n, *[k.ctypes.data for k in keep[:9]], len(so) - 1, so.ctypes.data,
                       reads.n, *[k.ctypes.data for k in keep[9:]], 0 if template_off is None else len(to) - 1, to.ctypes.data,
                       0 if flanks is None else 1, 0 if flanks is None else int(flanks[0]), 0 if flanks is None else int(flanks[1]))
        out = np.zeros((haps.n, n_items), dtype=np.float64)
        ext = C.c_int(0)
        st = self.lib.ref_array_populate(C.byref(a), out.ctypes.data_as(C.c_void_p), C.byref(ext))
        return st, out, ext.value

    def kmer_map(self, query, target, max_positions=10):
        """utils/kmer_mapper.hpp as HaplotypeLikelihoodArray::populate calls it (K = 6, at most ``max_positions``)."""
        q, t = _b(query), _b(target)
        out = (C.c_longlong * max_positions)()
        n = self.lib.ref_kmer_map(q, len(q) - 1, t, len(t) - 1, int(max_positions), out)
        return [int(out[i]) for i in range(n)]

    @staticmethod
    def _common(truth, read, quals, gap_open, gap_extend, snv_mask, snv_prior):
        t, r, m = _b(truth), _b(read), _b(snv_mask)
        q = np.ascontiguousarray(np.asarray(quals, dtype=np.uint8))
        go, gop = _i8(gap_open)
        ge, gep = _i8(gap_extend)
        pr, prp = _i8(snv_prior)
        assert len(go) == len(ge) == len(pr) == len(t) - 1 == len(m) - 1 and len(q) == len(r) - 1
        return (t, len(t) - 1, r, len(r) - 1, q.ctypes.data_as(C.c_void_p)), (gop, gep, m, prp), (t, r, m, q, go, ge, pr)

    def evaluate(self, band, truth, read, quals, offset, gap_open, gap_extend, snv_mask, snv_prior, flanks=(0, 0), nuc_prior=2, int32=False):
        seqs, model, keep = self._common(truth, read, quals, gap_open, gap_extend, snv_mask, snv_prior)
        return self.lib.ref_hmm_evaluate(int(band), int(int32), *seqs, C.c_longlong(int(offset)), *model,
                                         C.c_longlong(int(flanks[0])), C.c_longlong(int(flanks[1])), int(nuc_prior))

    def align(self, band, truth, read, quals, offset, gap_open, gap_extend, snv_mask, snv_prior, flanks=(0, 0), nuc_prior=2, int32=False):
        """Returns (target_offset, likelihood, cigar_text)."""
        seqs, model, keep = self._common(truth, read, quals, gap_open, gap_extend, snv_mask, snv_prior)
        off, lk = C.c_longlong(0), C.c_double(0)
        cap = 8 * (seqs[3] + 2 * 256) + 64
        cig = C.create_string_buffer(cap)
        rc = self.lib.ref_hmm_align(int(band), int(int32), *seqs, C.c_longlong(int(offset)), *model,
                                    C.c_longlong(int(flanks[0])), C.c_longlong(int(flanks[1])), int(nuc_prior),
                                    C.byref(off), C.byref(lk), cig, cap)
        assert rc == 0
        return off.value, lk.value, cig.value.decode()


    def align_mutation_model(self, truth, target, mismatch, gap_open, gap_extend):
        """hmm::PairHMM<VariableGapExtendMutationModel, 32, int>::align(target, truth) (DeNovoModel's call). Returns (rc, target_offset, likelihood, cigar)."""
        t, r = _b(truth), _b(target)
        go, gop = _i8(gap_open)
        ge, gep = _i8(gap_extend)
        off, lk = C.c_longlong(0), C.c_double(0)
        cap = 8 * (len(r) + 128) + 64
        cig = C.create_string_buffer(cap)
        f = self.lib.ref_hmm_align_mutation_model
        f.restype = C.c_int
        f.argtypes = [C.c_char_p, C.c_int, C.c_char_p, C.c_int, C.c_int, _i8p, _i8p, C.POINTER(C.c_longlong), C.POINTER(C.c_double), C.c_char_p, C.c_int]
        rc = f(t, len(t) - 1, r, len(r) - 1, int(mismatch), gop, gep, C.byref(off), C.byref(lk), cig, cap)
        return rc, off.value, lk.value, cig.value.decode()


class _Model(C.Structure):
    _fields_ = [("snv_mask", C.c_char_p), ("snv_prior", _i8p), ("gap_open", _i8p), ("gap_extend", _i8p),
                ("gap_open_scalar", C.c_int), ("gap_extend_scalar", C.c_int), ("nuc_prior", C.c_int)]


LOWEST = -1.7976931348623157e308


class COracle:
    """The plain-C restatement (oracle/phmm_oracle.c)."""

    def __init__(self):
        path = os.path.join(_HERE, "liboctopus_oracle.so")
        if not os.path.exists(path):
            build(ref=False)
        self.lib = L = C.CDLL(path)
        mp = C.POINTER(_Model)
        L.oracle_align.restype = C.c_int
        L.oracle_align.argtypes = [C.c_int, C.c_char_p, C.c_char_p, _i8p, C.c_int, C.c_int, mp]
        L.oracle_align_tb.restype = C.c_int
        L.oracle_align_tb.argtypes = L.oracle_align.argtypes + [_i32p, C.c_char_p, C.c_char_p]
        L.oracle_flank_score.restype = C.c_int
        L.oracle_flank_score.argtypes = [C.c_int, C.c_int, C.c_int, C.c_char_p, _i8p, mp, C.c_int, C.c_char_p, C.c_char_p, _i32p]
        L.oracle_try_naive_evaluate.restype = C.c_int
        L.oracle_try_naive_evaluate.argtypes = [C.c_char_p, C.c_int, C.c_char_p, C.c_void_p, C.c_int, C.c_int, mp,
                                                C.c_int, C.c_int, C.c_int, _i32p]
        L.oracle_evaluate.restype = C.c_double
        L.oracle_evaluate.argtypes = [C.c_int, C.c_char_p, C.c_int, C.c_char_p, C.c_void_p, C.c_int, C.c_int, mp,
                                      C.c_int, C.c_int, C.c_int, C.c_int, _i32p, _i32p]
        L.oracle_model_evaluate.restype = C.c_int
        L.oracle_model_evaluate.argtypes = [C.c_int, C.c_char_p, C.c_int, C.c_char_p, C.c_void_p, C.c_int, mp,
                                            C.c_int, C.c_int, C.c_int, _i64p, C.c_int, C.c_int64,
                                            C.c_int, C.c_int, C.c_int, C.c_int, C.c_int, C.POINTER(C.c_double), _i32p]
        L.oracle_kmer_map.restype = C.c_int
        L.oracle_kmer_map.argtypes = [C.c_char_p, C.c_int, C.c_char_p, C.c_int, C.c_int, _i64p]
        L.oracle_model_align.restype = C.c_int
        L.oracle_model_align.argtypes = [C.c_int, C.c_char_p, C.c_int, C.c_char_p, C.c_void_p, C.c_int, mp, C.c_int, C.c_int, C.c_int,
                                         _i64p, C.c_int, C.c_int64, C.c_int, C.c_int, C.c_int, C.c_int,
                                         _i64p, C.POINTER(C.c_double), C.c_char_p, C.c_int, _i32p]
        L.oracle_genotype_likelihoods.restype = None
        L.oracle_genotype_likelihoods.argtypes = [C.c_void_p, C.c_int, C.c_int, C.c_void_p, C.c_int, C.c_int, C.c_void_p]
        L.oracle_populate.restype = C.c_int
        L.oracle_populate.argtypes = [C.c_int, C.c_int] + [C.c_void_p] * 9 + [C.c_int] + [C.c_void_p] * 8 + [C.c_int] * 9 + [C.c_void_p, C.c_void_p]

    @staticmethod
    def model(gap_open, gap_extend, nuc_prior=2, snv_mask=None, snv_prior=None):
        """Returns (struct, keepalive). gap_open / gap_extend may be arrays or scalars."""
        keep = []
        m = _Model()
        if snv_mask is not None:
            b = _b(snv_mask)
            sp, spp = _i8(snv_prior)
            keep += [b, sp]
            m.snv_mask = C.cast(b, C.c_char_p)
            m.snv_prior = spp
        if np.ndim(gap_open) == 0:
            m.gap_open_scalar = int(gap_open)
        else:
            a, p = _i8(gap_open)
            keep.append(a)
            m.gap_open = p
        if np.ndim(gap_extend) == 0:
            m.gap_extend_scalar = int(gap_extend)
        else:
            a, p = _i8(gap_extend)
            keep.append(a)
            m.gap_extend = p
        m.nuc_prior = int(nuc_prior)
        return m, keep

    def align(self, band, truth, read, quals, gap_open, gap_extend, nuc_prior=2, snv_mask=None, snv_prior=None):
        m, keep = self.model(gap_open, gap_extend, nuc_prior, snv_mask, snv_prior)
        t, r = _b(truth), _b(read)
        q, qp = _i8(quals)
        return self.lib.oracle_align(band, t, r, qp, len(t) - 1, len(r) - 1, C.byref(m))

    def align_tb(self, band, truth, read, quals, gap_open, gap_extend, nuc_prior=2, snv_mask=None, snv_prior=None):
        m, keep = self.model(gap_open, gap_extend, nuc_prior, snv_mask, snv_prior)
        t, r = _b(truth), _b(read)
        q, qp = _i8(quals)
        n = 2 * (len(r) - 1 + band) + 1
        a1, a2 = C.create_string_buffer(n + 8), C.create_string_buffer(n + 8)
        fp = C.c_int32(-7)
        s = self.lib.oracle_align_tb(band, t, r, qp, len(t) - 1, len(r) - 1, C.byref(m), C.byref(fp), a1, a2)
        return s, fp.value, a1.value.decode(), a2.value.decode()

    def flank_score(self, truth_len, lhs, rhs, read, quals, snv_mask, snv_prior, gap_open, gap_extend, nuc_prior,
                    first_pos, align1, align2):
        m, keep = self.model(gap_open, gap_extend, nuc_prior, snv_mask, snv_prior)
        q, qp = _i8(quals)
        ms = C.c_int32(0)
        s = self.lib.oracle_flank_score(truth_len, lhs, rhs, _b(read), qp, C.byref(m), first_pos, _b(align1), _b(align2), C.byref(ms))
        return s, ms.value

    def try_naive_evaluate(self, truth, read, quals, offset, gap_open, gap_extend, snv_mask=None, snv_prior=None,
                           flanks=None):
        m, keep = self.model(gap_open, gap_extend, 2, snv_mask, snv_prior)
        t, r = _b(truth), _b(read)
        q = np.ascontiguousarray(np.asarray(quals, dtype=np.uint8))
        ph = C.c_int32(0)
        uf, lhs, rhs = (0, 0, 0) if flanks is None else (1, flanks[0], flanks[1])
        hit = self.lib.oracle_try_naive_evaluate(t, len(t) - 1, r, q.ctypes.data, len(r) - 1, offset, C.byref(m), uf, lhs, rhs, C.byref(ph))
        return bool(hit), ph.value

    def evaluate(self, band, truth, read, quals, offset, gap_open, gap_extend, nuc_prior=2, snv_mask=None, snv_prior=None,
                 flanks=None, dp_only=False, details=False):
        m, keep = self.model(gap_open, gap_extend, nuc_prior, snv_mask, snv_prior)
        t, r = _b(truth), _b(read)
        q = np.ascontiguousarray(np.asarray(quals, dtype=np.uint8))
        used, raw = C.c_int32(0), C.c_int32(0)
        uf, lhs, rhs = (0, 0, 0) if flanks is None else (1, flanks[0], flanks[1])
        v = self.lib.oracle_evaluate(band, t, len(t) - 1, r, q.ctypes.data, len(r) - 1, offset, C.byref(m), uf, lhs, rhs,
                                     int(dp_only), C.byref(used), C.byref(raw))
        return (v, used.value, raw.value) if details else v

    def model_evaluate(self, band, hap, read, quals, gap_open, gap_extend, snv_mask, snv_prior, positions, original_pos,
                       mapping_quality=60, nuc_prior=2, flanks=None, use_mapping_quality=True, mapq_cap=120,
                       mapq_cap_trigger=-1, dp_only=False):
        """Returns (status, value, required_extension); status 1 == ShortHaplotypeError."""
        m, keep = self.model(gap_open, gap_extend, nuc_prior, snv_mask, snv_prior)
        h, r = _b(hap), _b(read)
        q = np.ascontiguousarray(np.asarray(quals, dtype=np.uint8))
        pos = np.ascontiguousarray(np.asarray(positions, dtype=np.int64))
        out, ext = C.c_double(0), C.c_int32(0)
        uf, lhs, rhs = (0, 0, 0) if flanks is None else (1, flanks[0], flanks[1])
        st = self.lib.oracle_model_evaluate(band, h, len(h) - 1, r, q.ctypes.data, len(r) - 1, C.byref(m), uf, lhs, rhs,
                                            pos.ctypes.data_as(_i64p), len(pos), int(original_pos), int(use_mapping_quality),
                                            int(mapping_quality), int(mapq_cap), int(mapq_cap_trigger), int(dp_only),
                                            C.byref(out), C.byref(ext))
        return st, out.value, ext.value

    def kmer_map(self, query, target, max_positions=10):
        qb, tb = _b(query), _b(target)
        out = np.zeros(max(1, max_positions), dtype=np.int64)
        n = self.lib.oracle_kmer_map(qb, len(qb) - 1, tb, len(tb) - 1, max_positions, out.ctypes.data_as(_i64p))
        return out[:n].tolist()

    def populate(self, band, haps, reads, positions=None, flanks=None, use_mapping_quality=True, mapq_cap=120,
                 mapq_cap_trigger=-1, nuc_prior=2, dp_only=False, map_positions=False):
        """haps / reads: host HaplotypeBlock / ReadBlock (octopus_b200.batch). Returns (any_short, out[H,R], status[H,R])."""
        H, R = haps.n, reads.n
        out = np.empty((H, R), dtype=np.float64)
        status = np.zeros((H, R), dtype=np.int32)
        p = lambda a: None if a is None else a.ctypes.data
        po, pv = (None, None) if positions is None else (np.ascontiguousarray(positions[0], dtype=np.int64), np.ascontiguousarray(positions[1], dtype=np.int32))
        uf, lhs, rhs = (0, 0, 0) if flanks is None else (1, int(flanks[0]), int(flanks[1]))
        rc = self.lib.oracle_populate(int(band), H, p(haps.off), p(haps.seq), p(haps.snv_mask_fwd), p(haps.snv_prior_fwd),
                                      p(haps.snv_mask_rev), p(haps.snv_prior_rev), p(haps.gap_open), p(haps.gap_extend), p(haps.begin),
                                      R, p(reads.off), p(reads.bases), p(reads.quals), p(reads.mapq), p(reads.reverse), p(reads.begin),
                                      p(po), p(pv), uf, lhs, rhs, int(use_mapping_quality), int(mapq_cap), int(mapq_cap_trigger),
                                      int(nuc_prior), int(dp_only), int(map_positions), out.ctypes.data, status.ctypes.data)
        return rc, out, status

    def model_align(self, band, hap, read, quals, gap_open, gap_extend, snv_mask, snv_prior, positions, original_pos,
                    mapping_quality=60, nuc_prior=2, flanks=None, use_mapping_quality=True, mapq_cap=120, mapq_cap_trigger=-1):
        """HaplotypeLikelihoodModel::align. Returns (status, mapping_position, likelihood, cigar_text, required_extension)."""
        m, keep = self.model(gap_open, gap_extend, nuc_prior, snv_mask, snv_prior)
        h, r = _b(hap), _b(read)
        q = np.ascontiguousarray(np.asarray(quals, dtype=np.uint8))
        pos = np.ascontiguousarray(np.asarray(positions, dtype=np.int64))
        mp_, lk, ext = C.c_int64(0), C.c_double(0), C.c_int32(0)
        cap = 4 * (len(r) + 2 * band) + 64
        cig = C.create_string_buffer(cap)
        uf, lhs, rhs = (0, 0, 0) if flanks is None else (1, flanks[0], flanks[1])
        st = self.lib.oracle_model_align(band, h, len(h) - 1, r, q.ctypes.data, len(r) - 1, C.byref(m), uf, lhs, rhs,
                                         pos.ctypes.data_as(_i64p), len(pos), int(original_pos), int(use_mapping_quality), int(mapping_quality),
                                         int(mapq_cap), int(mapq_cap_trigger), C.byref(mp_), C.byref(lk), cig, cap, C.byref(ext))
        return st, mp_.value, lk.value, cig.value.decode(), ext.value

    def genotype_likelihoods(self, lnl, genotypes):
        lnl = np.ascontiguousarray(lnl, dtype=np.float64)
        gt = np.ascontiguousarray(genotypes, dtype=np.int32)
        out = np.empty(gt.shape[0], dtype=np.float64)
        self.lib.oracle_genotype_likelihoods(lnl.ctypes.data, lnl.shape[0], lnl.shape[1], gt.ctypes.data, gt.shape[0], gt.shape[1], out.ctypes.data)
        return out
