"""The C-ABI library builds for sm_90a without a GPU, loads, exports every symbol include/phmm_b200.h declares, and
refuses to compute without a GPU (no CPU fallback)."""
import ctypes as C
import os
import re
import subprocess

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def test_library_builds_and_exports_header_symbols():
    from octopus_b200 import _lib, build
    path = build.build()
    assert os.path.exists(path)
    header = open(os.path.join(ROOT, "include", "phmm_b200.h")).read()
    declared = sorted(set(re.findall(r"\b(phmm_[a-z_0-9]+)\s*\(", header)))
    assert set(declared) == set(_lib.EXPORTS), (declared, _lib.EXPORTS)
    lib = _lib.load()
    for name in declared:
        assert hasattr(lib, name), name
    assert lib.phmm_version().decode().startswith("octopus_b200")
    # the library contains sm_90a code only
    sass = subprocess.run(["cuobjdump", "-lelf", path], capture_output=True, text=True).stdout
    assert "sm_90a" in sass and "sm_100" not in sass and "sm_80" not in sass


def test_struct_layouts_match_header():
    from octopus_b200 import _lib
    assert C.sizeof(_lib.Config) == 36
    assert C.sizeof(_lib.Haplotypes) == 8 + 9 * 8
    assert C.sizeof(_lib.Reads) == 8 + 6 * 8
    assert C.sizeof(_lib.Positions) == 16
    assert C.sizeof(_lib.FlankState) == 24
    cfg = _lib.Config()
    _lib.load().phmm_default_config(C.byref(cfg))
    assert (cfg.max_indel_error, cfg.use_mapping_quality, cfg.mapping_quality_cap, cfg.mapping_quality_cap_trigger,
            cfg.use_flank_state, cfg.nuc_prior, cfg.use_int_scores, cfg.disable_naive_shortcut, cfg.map_positions) == (8, 1, 120, -1, 1, 2, 0, 0, 1)


def test_no_cpu_fallback_without_gpu():
    import torch
    if torch.cuda.is_available():
        pytest.skip("GPU present")
    from octopus_b200 import PairHMMEngine, PhmmError
    with pytest.raises(PhmmError) as ei:
        PairHMMEngine(0)
    assert ei.value.code == -2          # PHMM_ERR_CUDA


def test_product_package_never_touches_the_oracle():
    pkg = os.path.join(ROOT, "octopus_b200")
    for dirpath, _, files in os.walk(pkg):
        for f in files:
            if f.endswith((".py", ".cu", ".cuh", ".hpp", ".h", ".cpp")):
                text = open(os.path.join(dirpath, f)).read()
                hit = re.search(r"(from|import)\s+oracle|oracle[/\\.](?!$)|liboctopus_oracle|libref_phmm|phmm_oracle|ref_driver", text)
                assert hit is None, (os.path.join(dirpath, f), hit.group(0))
