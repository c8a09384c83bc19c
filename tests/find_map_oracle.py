"""ctypes loader of tests/cpp/find_map_oracle.c, the C restatement of find_map_haplotypes (read_assigner.cpp:45-64). Compiled on first
use into a temporary directory, so that the tree stays untouched."""
import ctypes as C
import os
import subprocess
import tempfile

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SRC = os.path.join(ROOT, "tests", "cpp", "find_map_oracle.c")
_lib = None


def load():
    global _lib
    if _lib is None:
        out = os.path.join(tempfile.mkdtemp(prefix="find_map_oracle_"), "libfind_map_oracle.so")
        subprocess.run([os.environ.get("CC", "cc"), "-std=c11", "-O2", "-ffp-contract=off", "-fPIC", "-shared", "-Wall", "-o", out, SRC, "-lm"],
                       check=True)
        lib = C.CDLL(out)
        lib.oracle_find_map_haplotypes.restype = C.c_uint64
        lib.oracle_find_map_haplotypes.argtypes = [C.c_int, C.c_void_p, C.c_void_p]
        lib.oracle_find_map_group.restype = None
        lib.oracle_find_map_group.argtypes = [C.c_int, C.c_int, C.c_void_p, C.c_void_p, C.c_void_p]
        _lib = lib
    return _lib


def find_map(values, log_priors=None):
    """The set of one read as a mask (bit k = haplotype k). values: its likelihood per haplotype, in genotype order."""
    v = np.ascontiguousarray(values, dtype=np.float64)
    p = None if log_priors is None else np.ascontiguousarray(log_priors, dtype=np.float64)
    return int(load().oracle_find_map_haplotypes(len(v), v.ctypes.data, None if p is None else p.ctypes.data))


def find_map_group(lnl, log_priors=None):
    """Every read of one group: lnl is its (H_g, R_g) matrix. Returns R_g uint64 masks."""
    m = np.ascontiguousarray(lnl, dtype=np.float64)
    H, R = m.shape
    assert 1 <= H <= 64
    p = None if log_priors is None else np.ascontiguousarray(log_priors, dtype=np.float64)
    top = np.zeros(R, dtype=np.uint64)
    load().oracle_find_map_group(H, R, m.ctypes.data, None if p is None else p.ctypes.data, top.ctypes.data)
    return top


def find_map_all(lnl_flat, hap_first, read_first, log_priors=None):
    """find_map_group over the groups of a flat assign_reads result (the groups' matrices back to back). Returns [R] uint64."""
    out = []
    o = 0
    for g in range(len(hap_first) - 1):
        h0, h1, r0, r1 = int(hap_first[g]), int(hap_first[g + 1]), int(read_first[g]), int(read_first[g + 1])
        n = (h1 - h0) * (r1 - r0)
        pri = None if log_priors is None else np.asarray(log_priors)[h0:h1]
        out.append(find_map_group(np.asarray(lnl_flat[o:o + n]).reshape(h1 - h0, r1 - r0), pri))
        o += n
    return np.concatenate(out) if out else np.zeros(0, np.uint64)
