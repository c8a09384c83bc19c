"""The request batcher's template assign requests without a GPU: octopus_b200/csrc/phmm_batcher.cpp, phmm_batcher_align.cpp and
phmm_batcher_templates.cpp against the CPU fakes of the engine (tests/cpp/fake_engine.cpp, fake_engine_align.cpp and
fake_engine_templates.cpp), driven from many threads by tests/cpp/test_batcher_templates_cpu.cpp, once under ThreadSanitizer and once
under AddressSanitizer + UBSan. Needs g++ only."""
import os
import subprocess

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CSRC = os.path.join(ROOT, "octopus_b200", "csrc")
CPP = os.path.join(ROOT, "tests", "cpp")
SOURCES = [os.path.join(CSRC, f) for f in ("phmm_batcher.cpp", "phmm_batcher_align.cpp", "phmm_batcher_templates.cpp")] + \
          [os.path.join(CPP, f) for f in ("fake_engine.cpp", "fake_engine_align.cpp", "fake_engine_templates.cpp", "test_batcher_templates_cpu.cpp")]
SANITIZERS = {
    "thread": {"TSAN_OPTIONS": "halt_on_error=1"},
    "address,undefined": {"ASAN_OPTIONS": "halt_on_error=1", "UBSAN_OPTIONS": "halt_on_error=1:print_stacktrace=1"},
}


@pytest.fixture(params=sorted(SANITIZERS))
def driver(request, tmp_path):
    exe = str(tmp_path / "test_batcher_templates_cpu")
    subprocess.run(["g++", "-std=c++17", "-O1", "-g", "-pthread", "-fsanitize=" + request.param, "-fno-sanitize-recover=all",
                    "-fno-omit-frame-pointer", "-I", os.path.join(ROOT, "include")] + SOURCES + ["-o", exe], check=True)
    return exe, dict(os.environ, **SANITIZERS[request.param])


def test_batcher_template_requests_against_fake_engine(driver):
    exe, env = driver
    out = subprocess.run([exe], capture_output=True, text=True, timeout=600, env=env)
    report = out.stdout + out.stderr
    assert out.returncode == 0 and "BATCHER TEMPLATES CPU ok" in out.stdout, report
    assert "Sanitizer" not in report and "runtime error" not in report, report
