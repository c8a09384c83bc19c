"""The request batcher (octopus_b200/csrc/phmm_batcher.cpp) without a GPU: compiled together with a CPU fake of the engine
(tests/cpp/fake_engine.cpp) and a driver of many std::threads (tests/cpp/test_batcher_cpu.cpp), once under ThreadSanitizer and once
under AddressSanitizer + UBSan. Needs g++ only: neither the CUDA library nor the reference checkout."""
import os
import subprocess

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SOURCES = [os.path.join(ROOT, "octopus_b200", "csrc", "phmm_batcher.cpp"), os.path.join(ROOT, "tests", "cpp", "fake_engine.cpp"),
           os.path.join(ROOT, "tests", "cpp", "test_batcher_cpu.cpp")]
SANITIZERS = {
    "thread": {"TSAN_OPTIONS": "halt_on_error=1"},
    "address,undefined": {"ASAN_OPTIONS": "halt_on_error=1", "UBSAN_OPTIONS": "halt_on_error=1:print_stacktrace=1"},
}


@pytest.fixture(params=sorted(SANITIZERS))
def driver(request, tmp_path):
    exe = str(tmp_path / "test_batcher_cpu")
    subprocess.run(["g++", "-std=c++17", "-O1", "-g", "-pthread", "-fsanitize=" + request.param, "-fno-sanitize-recover=all",
                    "-fno-omit-frame-pointer", "-I", os.path.join(ROOT, "include")] + SOURCES + ["-o", exe], check=True)
    return exe, dict(os.environ, **SANITIZERS[request.param])


def test_batcher_life_cycle_against_fake_engine(driver):
    exe, env = driver
    out = subprocess.run([exe], capture_output=True, text=True, timeout=600, env=env)
    report = out.stdout + out.stderr
    assert out.returncode == 0 and "BATCHER CPU ok" in out.stdout, report
    assert "Sanitizer" not in report and "runtime error" not in report, report
