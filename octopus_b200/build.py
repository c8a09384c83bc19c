"""Builds the CUDA extension in-tree: octopus_b200/libphmm_b200.so (sm_90a only, nvcc cross-compiles without a GPU)."""
import os
import subprocess
import sys

_HERE = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(_HERE, "csrc")
LIB = os.path.join(_HERE, "libphmm_b200.so")
SOURCES = ["phmm_engine.cu", "phmm_error_model.cpp", "phmm_batcher.cpp", "phmm_batcher_reset.cpp", "phmm_batcher_align.cpp",
           "phmm_batcher_templates.cpp"]
DEPS = ["phmm_engine.cu", "phmm_kernels.cuh", "phmm_device.cuh", "phmm_checks.h", "phmm_mutation.h", "phmm_reset.cuh", "phmm_vb.cuh", "phmm_vb_mm.cuh", "phmm_error_model.cpp", "phmm_error_model_tables.inc",
        "phmm_batcher.cpp", "phmm_batcher_reset.cpp", "phmm_batcher_align.cpp", "phmm_batcher_templates.cpp", "phmm_batcher_seam.h", os.path.join("..", "..", "include", "phmm_b200.h")]
NVCC_FLAGS = ["-O3", "-std=c++17", "-gencode", "arch=compute_90a,code=sm_90a", "-lineinfo",
              "-Xcompiler", "-fPIC", "-shared"]


def _nvcc():
    for cand in (os.environ.get("NVCC"), "/usr/local/cuda/bin/nvcc", "nvcc"):
        if cand and (os.path.isabs(cand) and os.path.exists(cand) or not os.path.isabs(cand)):
            return cand
    return "nvcc"


def _stale(target, deps):
    if not os.path.exists(target):
        return True
    t = os.path.getmtime(target)
    return any(os.path.exists(d) and os.path.getmtime(d) > t for d in deps)


def build(force=False, verbose=False):
    deps = [os.path.join(CSRC, d) for d in DEPS] + [__file__]    # a change of the flags here rebuilds too
    if not force and not _stale(LIB, deps):
        return LIB
    if not all(os.path.exists(os.path.join(CSRC, s)) for s in SOURCES):
        raise RuntimeError("CUDA sources missing")
    cmd = [_nvcc()] + NVCC_FLAGS + ["-o", LIB] + [os.path.join(CSRC, s) for s in SOURCES]
    if verbose:
        print(" ".join(cmd), file=sys.stderr)
    subprocess.run(cmd, check=True)
    return LIB


def build_cpu_emulation(force=False):
    """tests/cpu_emul/libphmm_emul.so: the engine's __host__ __device__ DP cores compiled for the CPU (test helper)."""
    root = os.path.dirname(_HERE)
    src = os.path.join(root, "tests", "cpu_emul", "emul.cu")
    out = os.path.join(root, "tests", "cpu_emul", "libphmm_emul.so")
    if not force and not _stale(out, [src, os.path.join(CSRC, "phmm_device.cuh"), __file__]):
        return out
    subprocess.run([_nvcc(), "-O2", "-std=c++17", "-gencode", "arch=compute_90a,code=sm_90a", "-Xcompiler", "-fPIC",
                    "-shared", "-o", out, src], check=True)
    return out


def build_vb_emulation(force=False):
    """tests/cpu_emul/libvb_emul.so: the variational Bayes loop over the engine's __host__ __device__ VB arithmetic (test helper)."""
    root = os.path.dirname(_HERE)
    src = os.path.join(root, "tests", "cpu_emul", "vb_emul.cu")
    out = os.path.join(root, "tests", "cpu_emul", "libvb_emul.so")
    if not force and not _stale(out, [src, os.path.join(CSRC, "phmm_vb.cuh"), __file__]):
        return out
    subprocess.run([_nvcc(), "-O2", "-std=c++17", "-gencode", "arch=compute_90a,code=sm_90a", "-Xcompiler", "-fPIC",
                    "-shared", "-o", out, src], check=True)
    return out


def build_vbmm_emulation(force=False):
    """tests/cpu_emul/libvbmm_emul.so: the mixture-of-mixtures VB loop over the engine's __host__ __device__ arithmetic (test helper)."""
    root = os.path.dirname(_HERE)
    src = os.path.join(root, "tests", "cpu_emul", "vbmm_emul.cu")
    out = os.path.join(root, "tests", "cpu_emul", "libvbmm_emul.so")
    if not force and not _stale(out, [src, os.path.join(CSRC, "phmm_vb_mm.cuh"), os.path.join(CSRC, "phmm_vb.cuh"), __file__]):
        return out
    subprocess.run([_nvcc(), "-O2", "-std=c++17", "-gencode", "arch=compute_90a,code=sm_90a", "-Xcompiler", "-fPIC",
                    "-shared", "-o", out, src], check=True)
    return out


if __name__ == "__main__":
    print(build(force="--force" in sys.argv, verbose=True))
