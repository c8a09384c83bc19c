"""The UNMODIFIED reference run_variational_bayes (core/models/genotype/variational_bayes_mixture_model.hpp) compiled into
oracle/_ref/libref_vb.so (oracle/vb.mk, oracle/ref_vb_driver.cpp), for K in REF_K. It keeps alphas, digamma differences and the
inverted likelihoods in float with fmath's fast_exp / fast_log, so it agrees with the double computation only to float tolerance.
Its per-seed iteration count is the smallest max_iterations whose run ends in the same latents as the full run."""
import ctypes as C
import os

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
REF_LIB = os.path.join(ROOT, "oracle", "_ref", "libref_vb.so")
REF_K = (1, 2, 3, 4, 8, 100)


class RefVB:
    _lib = None

    @classmethod
    def available(cls):
        return os.path.exists(REF_LIB)

    def __init__(self):
        if RefVB._lib is None:
            lib = C.CDLL(REF_LIB)
            vp = C.c_void_p
            lib.ref_vb_run.restype = C.c_int
            lib.ref_vb_run.argtypes = [C.c_int, vp, C.c_int, C.c_int, vp, C.c_int, vp, C.c_int, vp, vp, vp, C.c_int, C.c_double, C.c_int] + [vp] * 8
            RefVB._lib = lib
        self.lib = RefVB._lib

    def run(self, lnl, sample_off, genotypes, prior_alphas, genotype_log_priors, seeds, epsilon=0.05, max_iterations=1000, per_seed=True):
        """The VBResultPacket; with per_seed also every seed's evidence and iteration count (several more runs of each seed)."""
        lnl = np.ascontiguousarray(lnl, dtype=np.float64)
        off = np.ascontiguousarray(sample_off, dtype=np.int64)
        gt = np.ascontiguousarray(genotypes, dtype=np.int32)
        pa = np.ascontiguousarray(prior_alphas, dtype=np.float64)
        lp = np.ascontiguousarray(genotype_log_priors, dtype=np.float64)
        sd = np.ascontiguousarray(seeds, dtype=np.float64)
        G, K = gt.shape
        S, n = len(off) - 1, sd.shape[0]
        assert K in REF_K, K
        out = dict(posteriors=np.empty(G), log_posteriors=np.empty(G), alphas=np.empty((S, K)), weighted=np.empty(G),
                   max_log_evidence=np.empty(1), max_seed=np.empty(1, np.int32), seed_log_evidences=np.empty(n),
                   seed_iterations=np.empty(n, np.int32))
        rc = self.lib.ref_vb_run(K, lnl.ctypes.data, lnl.shape[0], lnl.shape[1], off.ctypes.data, S, gt.ctypes.data, G, pa.ctypes.data,
                                 lp.ctypes.data, sd.ctypes.data, n, float(epsilon), int(max_iterations),
                                 *(out[k].ctypes.data for k in ("posteriors", "log_posteriors", "alphas", "weighted", "max_log_evidence",
                                                                "max_seed", "seed_log_evidences")),
                                 out["seed_iterations"].ctypes.data if per_seed else None)
        assert rc == 0
        out["max_log_evidence"] = float(out["max_log_evidence"][0])
        out["max_seed"] = int(out["max_seed"][0]) if per_seed else None
        return out
