"""The UNMODIFIED reference VariationalBayesMixtureMixtureModel (core/models/genotype/variational_bayes_mixture_mixture_model.cpp)
compiled into oracle/_ref/libref_vbmm.so (oracle/vbmm.mk, oracle/ref_vbmm_driver.cpp). It keeps its expanded likelihoods and the
component update's sum over combinations in float, so it agrees with the double computation only to float tolerance. Its
per-seed iteration count is the smallest max_iterations whose run ends in the same latents as the full run."""
import ctypes as C
import os

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
REF_LIB = os.path.join(ROOT, "oracle", "_ref", "libref_vbmm.so")


class RefVBMM:
    _lib = None

    @classmethod
    def available(cls):
        return os.path.exists(REF_LIB)

    def __init__(self):
        if RefVBMM._lib is None:
            lib = C.CDLL(REF_LIB)
            vp = C.c_void_p
            lib.ref_vbmm_run.restype = C.c_int
            lib.ref_vbmm_run.argtypes = [vp, C.c_int, C.c_int, vp, C.c_int, vp, C.c_int, vp, C.c_int] + [vp] * 6 + \
                                        [C.c_int, C.c_double, C.c_int] + [vp] * 11
            RefVBMM._lib = lib
        self.lib = RefVBMM._lib

    def run(self, lnl, sample_off, group_sizes, combinations, genotype_log_priors, group_concentrations, mixture_concentrations,
            seeds, group_priors=None, group_prior_mask=None, epsilon=0.05, max_iterations=1000, per_seed=True):
        """The Inferences; with per_seed also every seed's evidence and iteration count (several more runs of each seed)."""
        lnl = np.ascontiguousarray(lnl, dtype=np.float64)
        off = np.ascontiguousarray(sample_off, dtype=np.int64)
        sizes = np.ascontiguousarray(group_sizes, dtype=np.int32)
        gt = np.ascontiguousarray(combinations, dtype=np.int32)
        lp = np.ascontiguousarray(genotype_log_priors, dtype=np.float64)
        gc = np.ascontiguousarray(group_concentrations, dtype=np.float64)
        mc = np.ascontiguousarray(mixture_concentrations, dtype=np.float64)
        sd = np.ascontiguousarray(seeds, dtype=np.float64)
        gp = None if group_priors is None else np.ascontiguousarray(group_priors, dtype=np.float64)
        mask = None if group_prior_mask is None else np.ascontiguousarray(group_prior_mask, dtype=np.int32)
        Cn, K = gt.shape
        S, T, n = len(off) - 1, len(sizes), sd.shape[0]
        out = dict(posteriors=np.empty(Cn), log_posteriors=np.empty(Cn), group_concentrations=np.empty(T),
                   mixture_concentrations=np.empty((S, K)), group_responsibilities=np.empty((S, T)), weighted=np.empty(Cn),
                   weighted_group_responsibilities=np.empty((S, T)), max_log_evidence=np.empty(1), max_seed=np.empty(1, np.int32),
                   seed_log_evidences=np.empty(n), seed_iterations=np.empty(n, np.int32))
        ptr = lambda a: None if a is None else a.ctypes.data
        rc = self.lib.ref_vbmm_run(lnl.ctypes.data, lnl.shape[0], lnl.shape[1], off.ctypes.data, S, sizes.ctypes.data, T, gt.ctypes.data,
                                   Cn, lp.ctypes.data, ptr(gp), ptr(mask), gc.ctypes.data, mc.ctypes.data, sd.ctypes.data, n,
                                   float(epsilon), int(max_iterations),
                                   *(out[k].ctypes.data for k in ("posteriors", "log_posteriors", "group_concentrations",
                                                                  "mixture_concentrations", "group_responsibilities", "weighted",
                                                                  "weighted_group_responsibilities", "max_log_evidence", "max_seed",
                                                                  "seed_log_evidences")),
                                   out["seed_iterations"].ctypes.data if per_seed else None)
        assert rc == 0
        out["max_log_evidence"] = float(out["max_log_evidence"][0])
        out["max_seed"] = int(out["max_seed"][0]) if per_seed else None
        return out
