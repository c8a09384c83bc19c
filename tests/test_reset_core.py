"""The reset core shared by the host and the device (octopus_b200/csrc/phmm_reset.cuh), compiled with g++: its restatement of
std::sort gives libstdc++'s permutation, and a run capacity that is too small is reported without writing past the buffers."""
import os
import subprocess

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def test_reset_core_sort_and_run_capacity(tmp_path):
    exe = str(tmp_path / "test_reset_core")
    subprocess.run(["g++", "-std=c++17", "-O2", "-Wall", "-I", os.path.join(ROOT, "octopus_b200", "csrc"),
                    os.path.join(ROOT, "tests", "cpp", "test_reset_core.cpp"), "-o", exe], check=True)
    out = subprocess.run([exe], capture_output=True, text=True, timeout=600)
    assert out.returncode == 0, out.stdout + out.stderr
    assert "SORT ok" in out.stdout and "CAP ok" in out.stdout, out.stdout
    print(out.stdout)
