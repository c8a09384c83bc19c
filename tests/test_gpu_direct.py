"""Direct mode of populate (one candidate position per pair, shortcut off, no flank state, 16-bit scores): the pair list runs without
the classify pass and the epilogue. Its values and status words must equal the classify path's (PHMM_NO_DIRECT=1, read once per
process, hence the second process) bit for bit, and the oracle's."""
import os
import subprocess
import sys

import numpy as np
import pytest

from exact import assert_same_penalties
from helpers import random_region

pytestmark = pytest.mark.gpu

HERE = os.path.dirname(os.path.abspath(__file__))


def _config(band_req, use_mq=True):
    from octopus_b200 import HaplotypeLikelihoodModel
    return HaplotypeLikelihoodModel.Config(max_indel_error=band_req, use_mapping_quality=use_mq, mapping_quality_cap=60,
                                           mapping_quality_cap_trigger=40, disable_naive_shortcut=True, map_positions=False)


def _band(band_req):
    from octopus_b200 import HaplotypeLikelihoodModel
    return HaplotypeLikelihoodModel(HaplotypeLikelihoodModel.Config(max_indel_error=band_req)).pad_requirement()


def _single_cases():
    """(name, band_req, haps, reads): odd read counts per length, reads over the haplotype ends and with 'N', H <= 16 (G = 2, 4),
    and haplotypes too short for some reads (status 2)."""
    cases = []
    for band_req in (8, 16):
        for H in (5, 12, 40):
            rng = np.random.default_rng(1000 * band_req + H)
            haps, reads = random_region(rng, _band(band_req), n_haps=H, n_reads=37, hap_len=260, read_len_choices=[40, 76, 100, 150],
                                        read_n_rate=0.15, edge_reads=True)
            cases.append(("b%d_h%d" % (band_req, H), band_req, haps, reads))
    rng = np.random.default_rng(77)
    haps, reads = random_region(rng, _band(16), n_haps=6, n_reads=25, hap_len=90, read_len_choices=[40, 76], read_n_rate=0.1, edge_reads=True)
    cases.append(("short", 16, haps, reads))
    return cases


def _region_case():
    from octopus_b200.batch import concat_blocks
    rng = np.random.default_rng(5)
    a = random_region(rng, _band(16), n_haps=3, n_reads=21, hap_len=200, read_len_choices=[40, 76, 100], read_n_rate=0.1)
    b = random_region(rng, _band(16), n_haps=20, n_reads=30, hap_len=300, read_len_choices=[76, 150], read_n_rate=0.1)
    c = random_region(rng, _band(16), n_haps=9, n_reads=11, hap_len=90, read_len_choices=[40, 76])
    return [a, b, c], concat_blocks([a[0], b[0], c[0]], [a[1], b[1], c[1]])


def compute():
    """Every case's values and status words, under whatever PHMM_NO_DIRECT this process was started with."""
    import torch
    from octopus_b200 import PairHMMEngine
    eng = PairHMMEngine(0)
    res = {}
    for name, band_req, haps, reads in _single_cases():
        for use_mq in (True, False):
            out, st = eng.populate(_config(band_req, use_mq), haps, reads, want_status=True)
            res["%s_mq%d_val" % (name, use_mq)], res["%s_mq%d_st" % (name, use_mq)] = out, st
    _, (bh, br, hf, rf) = _region_case()
    out, _, st = eng.populate_regions(_config(16), bh, br, hf, rf, want_status=True)
    res["regions_val"], res["regions_st"] = out, st
    # a column window of a wider device matrix (row stride R + 5): phmm_populate_ld
    _, band_req, haps, reads = _single_cases()[3]
    dh, dr = haps.to_device("cuda:0"), reads.to_device("cuda:0")
    wide = torch.full((haps.n, reads.n + 5), 7.0, dtype=torch.float64, device="cuda:0")
    eng.populate(_config(band_req), dh, dr, out=wide[:, 2:2 + reads.n])
    res["ld_val"] = wide.cpu().numpy()
    return res


def _dump(path):
    np.savez(path, **compute())


@pytest.fixture(scope="module")
def both(tmp_path_factory):
    path = str(tmp_path_factory.mktemp("direct") / "classify.npz")
    env = dict(os.environ, PHMM_NO_DIRECT="1")
    code = "import sys; sys.path[:0] = [%r, %r]; import test_gpu_direct as t; t._dump(%r)" % (HERE, os.path.dirname(HERE), path)
    subprocess.run([sys.executable, "-s", "-c", code], env=env, check=True)
    with np.load(path) as f:
        classify = {k: f[k] for k in f.files}
    return compute(), classify


def test_direct_mode_equals_classify_path(both):
    direct, classify = both
    assert sorted(direct) == sorted(classify)
    for k in direct:
        assert np.array_equal(direct[k], classify[k]), k
    assert (direct["short_mq1_st"] & 0xFFFF == 2).any() and (direct["short_mq1_st"] == 0).any()
    assert (direct["regions_st"] & 0xFFFF == 2).any()
    ld = direct["ld_val"]
    assert np.array_equal(ld[:, 2:-3], direct["b16_h5_mq1_val"]) and (ld[:, :2] == 7.0).all() and (ld[:, -3:] == 7.0).all()


def test_direct_mode_matches_oracle(both, coracle):
    """Mapping quality off: bit-equal to the oracle. On (cap 60, trigger 40): within the bound of the exact mix of those penalties."""
    from test_gpu_parity import mixed_within_bound
    direct, _ = both
    for name, band_req, haps, reads in _single_cases():
        rc, want, wst = coracle.populate(_band(band_req), haps, reads, None, None, use_mapping_quality=False, dp_only=True, map_positions=False)
        assert_same_penalties(direct["%s_mq0_val" % name], want, direct["%s_mq0_st" % name], wst, name)
        got, st = direct["%s_mq1_val" % name], direct["%s_mq1_st" % name]
        assert np.array_equal(st, direct["%s_mq0_st" % name]), name
        mixed_within_bound(got, want, wst, reads.mapq[None, :], 60, 40, name)
    regions, (_, _, hf, rf) = _region_case()
    off = 0
    for haps, reads in regions:
        rc, want, wst = coracle.populate(_band(16), haps, reads, None, None, use_mapping_quality=False, dp_only=True, map_positions=False)
        n = haps.n * reads.n
        st = direct["regions_st"][off:off + n].reshape(haps.n, reads.n)
        got = direct["regions_val"][off:off + n].reshape(haps.n, reads.n)
        assert np.array_equal(st != 0, (wst != 0) | (want == -1.7976931348623157e308)) and np.array_equal(st[wst != 0], wst[wst != 0])
        mixed_within_bound(got, want, wst, reads.mapq[None, :], 60, 40, "regions")
        off += n


def test_direct_mode_raises_short_haplotype_error(engine):
    from octopus_b200 import ShortHaplotypeError
    _, band_req, haps, reads = _single_cases()[-1]
    with pytest.raises(ShortHaplotypeError):
        engine.populate(_config(band_req), haps, reads)
