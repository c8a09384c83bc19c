"""The request batcher's assign and realign requests without a GPU: octopus_b200/csrc/phmm_batcher.cpp and phmm_batcher_align.cpp
against the CPU fakes of the populate / mutation engine symbols (tests/cpp/fake_engine.cpp) and of the assign / realign ones
(tests/cpp/fake_engine_align.cpp), driven by tests/cpp/test_batcher_align_cpu.cpp, once under ThreadSanitizer and once under
AddressSanitizer + UBSan. The driver wraps phmm_host_alloc to measure the batcher's page-locked staging. Needs g++ only."""
import os
import subprocess

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CSRC = os.path.join(ROOT, "octopus_b200", "csrc")
SOURCES = [os.path.join(CSRC, "phmm_batcher.cpp"), os.path.join(CSRC, "phmm_batcher_align.cpp"),
           os.path.join(ROOT, "tests", "cpp", "fake_engine.cpp"), os.path.join(ROOT, "tests", "cpp", "fake_engine_align.cpp"),
           os.path.join(ROOT, "tests", "cpp", "test_batcher_align_cpu.cpp")]
SANITIZERS = {
    "thread": {"TSAN_OPTIONS": "halt_on_error=1"},
    "address,undefined": {"ASAN_OPTIONS": "halt_on_error=1", "UBSAN_OPTIONS": "halt_on_error=1:print_stacktrace=1"},
}


@pytest.fixture(params=sorted(SANITIZERS))
def driver(request, tmp_path):
    exe = str(tmp_path / "test_batcher_align_cpu")
    subprocess.run(["g++", "-std=c++17", "-O1", "-g", "-pthread", "-fsanitize=" + request.param, "-fno-sanitize-recover=all",
                    "-fno-omit-frame-pointer", "-I", os.path.join(ROOT, "include")] + SOURCES +
                   ["-Wl,--wrap=phmm_host_alloc", "-o", exe], check=True)
    return exe, dict(os.environ, **SANITIZERS[request.param])


def test_batcher_assign_and_realign_requests_against_fake_engine(driver):
    exe, env = driver
    out = subprocess.run([exe], capture_output=True, text=True, timeout=600, env=env)
    report = out.stdout + out.stderr
    assert out.returncode == 0 and "BATCHER ALIGN CPU ok" in out.stdout, report
    assert "Sanitizer" not in report and "runtime error" not in report, report
