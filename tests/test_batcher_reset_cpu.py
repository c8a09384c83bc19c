"""The request batcher's populate requests with an error model without a GPU: octopus_b200/csrc/phmm_batcher.cpp and
phmm_batcher_reset.cpp with the real error models (phmm_error_model.cpp), against the CPU fakes of the plain engine symbols
(tests/cpp/fake_engine.cpp) and of the _reset ones (tests/cpp/fake_engine_reset.cpp), driven by tests/cpp/test_batcher_reset_cpu.cpp,
once under ThreadSanitizer and once under AddressSanitizer + UBSan. Needs g++ only."""
import os
import subprocess

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CSRC = os.path.join(ROOT, "octopus_b200", "csrc")
SOURCES = [os.path.join(CSRC, "phmm_batcher.cpp"), os.path.join(CSRC, "phmm_batcher_reset.cpp"), os.path.join(CSRC, "phmm_error_model.cpp"),
           os.path.join(ROOT, "tests", "cpp", "fake_engine.cpp"), os.path.join(ROOT, "tests", "cpp", "fake_engine_reset.cpp"),
           os.path.join(ROOT, "tests", "cpp", "test_batcher_reset_cpu.cpp")]
SANITIZERS = {
    "thread": {"TSAN_OPTIONS": "halt_on_error=1"},
    "address,undefined": {"ASAN_OPTIONS": "halt_on_error=1", "UBSAN_OPTIONS": "halt_on_error=1:print_stacktrace=1"},
}


@pytest.fixture(params=sorted(SANITIZERS))
def driver(request, tmp_path):
    exe = str(tmp_path / "test_batcher_reset_cpu")
    subprocess.run(["g++", "-std=c++17", "-O1", "-g", "-pthread", "-fsanitize=" + request.param, "-fno-sanitize-recover=all",
                    "-fno-omit-frame-pointer", "-I", os.path.join(ROOT, "include")] + SOURCES + ["-o", exe], check=True)
    return exe, dict(os.environ, **SANITIZERS[request.param])


def test_batcher_reset_requests_against_fake_engine(driver):
    exe, env = driver
    out = subprocess.run([exe], capture_output=True, text=True, timeout=600, env=env)
    report = out.stdout + out.stderr
    assert out.returncode == 0 and "BATCHER RESET CPU ok" in out.stdout, report
    assert "Sanitizer" not in report and "runtime error" not in report, report
