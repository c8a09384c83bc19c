"""SASS of the built library: dp_pair's epilogue cells (the last 2B-1 columns, which leave the unrolled sequence after the
row-L cell) stay at the cost of a steady cell plus the exit test. They keep that cost only because each exit branches through a
block of its own (PHMM_DISTINCT_PATH in phmm_device.cuh); when ptxas merges those blocks, the register copies of every exit land on
the path that falls through to the next cell and the cells grow to 35 instructions. No GPU needed: tools/sass_column_cost.py reads
the library through cuobjdump."""
import importlib.util
import os

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.fixture(scope="module")
def cost():
    from octopus_b200 import _lib
    _lib.load()
    spec = importlib.util.spec_from_file_location("sass_column_cost", os.path.join(ROOT, "tools", "sass_column_cost.py"))
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod, mod.listing(_lib.LIB_PATH)


@pytest.mark.parametrize("band", [8, 16])
@pytest.mark.parametrize("form", ["oge", "general"])
def test_epilogue_cells_cost_a_steady_cell_plus_the_exit_test(cost, band, form):
    mod, text = cost
    K = 2 * band
    _, ins = mod.function(text, band)
    g = mod.Cfg(mod.blocks_of(ins), K, form)
    cells = [g.b[i] for i in g.exit_chain]
    assert len(cells) == K - 1
    # the last cell (k = 1) always exits: its block holds that exit's register copies and runs once per call
    assert max(c.n for c in cells[:-1]) <= 12, [c.n for c in cells]
    assert sum(c.movs for c in cells[:-1]) <= 2, [c.movs for c in cells]
    # a call's epilogue columns, top and end included, against their cells at the steady columns' rate: 1.25-1.31 with the
    # separate exit blocks, 1.43-1.75 without them
    L = 150
    epi = sum(g.walk(x, L) for x in range(L + 1, L + K))
    steady = g.walk(K, L)
    assert epi <= 1.4 * steady * (K - 1) / 2, (epi, steady)
