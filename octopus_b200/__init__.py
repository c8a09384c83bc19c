"""octopus_b200 — H100-native (sm_90a) engine for Octopus's pair-HMM haplotype-likelihood path.

The product is the C-ABI shared library ``libphmm_b200.so`` (include/phmm_b200.h, csrc/*.cu). This Python package is
the host-side mirror used by the tests and the benchmark: a ctypes binding (``_lib``), struct-of-arrays batch packing
(``batch``), the reference-shaped wrappers (``api``) and the synthetic workload generator (``synth``).
There is no CPU fallback: importing works anywhere, computing requires an H100.
"""
from .api import (ErrorModel, HaplotypeLikelihoodArray, HaplotypeLikelihoodModel, MutationModel, PairHMMEngine, PhmmError,  # noqa: F401
                  PopulateBatcher, ShortHaplotypeError)
from .batch import HaplotypeBlock, HaplotypeSequences, ReadBlock, pack_haplotypes, pack_reads  # noqa: F401

__version__ = "0.1.0"
