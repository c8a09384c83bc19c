"""A plain C++ program (g++, no torch) drives the engine through the C ABI and the C++ adapter header."""
import os
import subprocess
import tempfile

import numpy as np
import pytest

from exact import assert_mix_within_bound, assert_same_penalties, penalties

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SRC = os.path.join(ROOT, "tests", "cpp", "test_cabi.cpp")


def _build():
    """Compile the program into a fresh temporary directory (the source tree may be read-only) and return its path."""
    from octopus_b200 import build
    build.build()
    exe = os.path.join(tempfile.mkdtemp(prefix="test_cabi_"), "test_cabi")
    subprocess.run(["g++", "-std=c++14", "-O1", "-I", os.path.join(ROOT, "include"), "-I", os.path.join(ROOT, "octopus_b200", "cpp"),
                    SRC, "-o", exe, "-L", os.path.join(ROOT, "octopus_b200"), "-lphmm_b200",
                    "-Wl,-rpath," + os.path.join(ROOT, "octopus_b200")], check=True)
    return exe


def test_cpp_adapter_compiles_against_the_abi():
    assert os.path.exists(_build())


@pytest.mark.gpu
def test_cpp_client_matches_oracle_exactly(coracle):
    exe = _build()
    out = subprocess.run([exe], capture_output=True, text=True, timeout=120)
    assert out.returncode == 0, out.stdout + out.stderr
    lines = dict((l.split()[0] + (l.split()[1] if l.startswith(("ROW", "EXACT")) else ""), l.split()) for l in out.stdout.strip().splitlines())
    assert lines["KAT"][1:] == ["84", "84", "0", "CCCCACGTATATATATATATATGGGGACGT", "CCCCACGT---------------GGGACGT"]
    h0 = "ACGTTGCAAGCTTAGGCTAACGTTAGCATCGATCGGATCTAGCTAGGATCGATACGATCGATCGTAGCTAGCTAGTCGATCGATTTAGCGCGATATCGCGAT"
    h1 = list(h0); h1[50] = "C" if h1[50] == "A" else "A"; h1 = "".join(h1)
    reads = [(h0[30:70], 30, 30), (h1[35:75], 25, 35)]
    n = len(h0)
    for hi, h in enumerate((h0, h1)):
        for ri, (r, q, p) in enumerate(reads):
            st, want, _ = coracle.model_evaluate(16, h, r, np.full(40, q, np.uint8), np.full(n, 40, np.int8), np.full(n, 3, np.int8), h.encode(),
                                                 np.full(n, 50, np.int8), [], p, use_mapping_quality=False)
            assert st == 0
            exact = np.array([float(lines["EXACT%d" % hi][2 + ri])])
            assert_same_penalties(exact, np.array([want]), None, np.zeros(1), (hi, ri))       # %.17g round-trips a double
            assert_mix_within_bound([float(lines["ROW%d" % hi][2 + ri])], penalties([want]), [60], (hi, ri))
    assert lines["SHORT"][1].startswith("hap=0")
    e2e = dict(kv.split("=") for kv in lines["E2E"][1:])
    assert e2e["same"] == "1" and float(e2e["pinned_ms"]) > 0 and float(e2e["pageable_ms"]) > 0
    assert e2e["gap_open_range"] != "45..45"          # reset() produced repeat-structured penalties (homopolymer / dinucleotide runs)
    print("C++ adapter e2e (64 x 40000 pairs, L=100): pinned %.2f ms, pageable %.2f ms per populate" % (float(e2e["pinned_ms"]), float(e2e["pageable_ms"])))
    assert lines["SAMPLES"][1:] == ["ok", "throws"]          # multi-sample / template container semantics of the C++ adapter


# ---------------------------------------------------------------------------------------------------------------------
# The reference's own hmm::evaluate / hmm::align templates instantiated over GpuPairHMM (tests/cpp/test_dropin.cpp)
# ---------------------------------------------------------------------------------------------------------------------
DROPIN_SRC = os.path.join(ROOT, "tests", "cpp", "test_dropin.cpp")
DROPIN_EXE = os.path.join(ROOT, "oracle", "_ref", "test_dropin")      # a reference binary: it lives beside the other oracle/_ref builds


def _build_dropin():
    """Compiled only where the reference checkout exists (oracle.REFERENCE); elsewhere an oracle/_ref build made earlier is used."""
    from oracle.oracle import REFERENCE, have_reference
    if not have_reference():
        return os.path.exists(DROPIN_EXE)
    from octopus_b200 import build
    build.build()
    newest = max(os.path.getmtime(p) for p in (DROPIN_SRC, os.path.join(ROOT, "octopus_b200", "cpp", "phmm_b200.hpp"), os.path.join(ROOT, "include", "phmm_b200.h")))
    if not os.path.exists(DROPIN_EXE) or os.path.getmtime(DROPIN_EXE) < newest:
        os.makedirs(os.path.dirname(DROPIN_EXE), exist_ok=True)
        subprocess.run(["g++", "-std=c++17", "-O1", "-msse4.1", "-include", "immintrin.h", "-Wno-ignored-attributes",
                        "-I", os.path.join(ROOT, "oracle", "ref_shim"), "-I", os.path.join(REFERENCE, "src"), "-I", os.path.join(REFERENCE, "lib"),
                        "-I", os.path.join(ROOT, "include"), "-I", os.path.join(ROOT, "octopus_b200", "cpp"),
                        DROPIN_SRC, "-o", DROPIN_EXE, "-L", os.path.join(ROOT, "octopus_b200"), "-lphmm_b200",
                        "-Wl,-rpath,$ORIGIN/../../octopus_b200"], check=True)      # relative: the tree may be moved after the build
    return True


def test_reference_templates_instantiate_over_the_gpu_pair_hmm():
    """hmm::evaluate / hmm::align (pair_hmm.hpp, unmodified) compile with octopus_b200::GpuPairHMM<Band> as their PairHMM: built here
    where the reference checkout is given, else the oracle/_ref build made from it earlier."""
    if not _build_dropin():
        pytest.skip("no reference checkout (oracle.REFERENCE) and no oracle/_ref/test_dropin built from one")
    with open(DROPIN_EXE, "rb") as f:
        assert b"libphmm_b200.so" in f.read()            # linked against the engine, not a stand-in


@pytest.mark.gpu
def test_reference_evaluate_and_align_over_gpu_pair_hmm_equal_simd_kernel():
    """The reference's evaluate / align code paths (naive shortcut, score-only, traceback + flank discount, CIGAR) driven by the GPU
    kernel give exactly the values they give over the reference's SIMD kernel: 620 seeded cases, bands 8 / 16 / 32."""
    if not _build_dropin():
        pytest.skip("oracle/_ref/test_dropin was never built (needs the reference checkout at build time)")
    out = subprocess.run([DROPIN_EXE], capture_output=True, text=True, timeout=300)
    assert out.returncode == 0 and "DROPIN ok" in out.stdout, out.stdout + out.stderr
    assert int(out.stdout.split("traceback_cases=")[1].split()[0]) > 100
