import os
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs an H100 (run with `pytest -m gpu` on a GPU machine)")


@pytest.fixture(scope="session")
def coracle():
    from oracle.oracle import COracle, build
    build()
    return COracle()


@pytest.fixture(scope="session")
def refkernels():
    """All reference-kernel ISA builds this host can run ({} where oracle/_ref was never built)."""
    from oracle.oracle import RefKernel, available_ref_isas
    return {isa: RefKernel(isa) for isa in available_ref_isas()}


@pytest.fixture(scope="session")
def refhmm(coracle):
    """The reference's own hmm::evaluate / hmm::align / PairHMMWrapper (oracle/_ref/libref_hmm.so), or None where it was never built."""
    from oracle.oracle import RefHMM
    return RefHMM() if RefHMM.available() else None


@pytest.fixture(scope="session")
def kats():
    import json
    with open(os.path.join(ROOT, "tests", "golden", "pair_hmm_kats.json")) as f:
        return json.load(f)["cases"]


@pytest.fixture(scope="session")
def engine():
    import torch
    if not torch.cuda.is_available():
        pytest.skip("no GPU")
    from octopus_b200 import PairHMMEngine
    return PairHMMEngine(0)
