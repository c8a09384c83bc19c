"""phmm_genotype_likelihoods (PairHMMEngine.genotype_likelihoods) against the exact value (tests/genotype_exact.py): every result
within the kernel's derived bound, eps [(ceil(R/256) + 16) sum_r |t_r| + sum_r (|mx_r| + ln p + 2p + 4)], of the exact value, or
of its non-finite class; the reference-form oracle within the same bound with R-long sequential chains, on the same inputs. Host
and device space give the same bits. Also: ploidy 0, ploidy 65, G = 0, and out-of-range indices in both spaces."""
import numpy as np
import pytest

import genotype_exact as ge
from octopus_b200 import PhmmError, _lib

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def worst():
    """Largest |error| / bound per ploidy, for the kernel and the oracle; printed at the end of the module (pytest -s)."""
    w = {}
    yield w
    for key in sorted(w):
        print("genotype likelihoods, %s: largest |error| / bound %.3f" % (key, w[key]))


def _group(p):
    return "ploidy %d" % p if p <= 4 else "ploidy 5-64"


def _check(engine, coracle, worst, m, gts, what, m_dev=None):
    import torch
    gts = np.ascontiguousarray(gts, dtype=np.int32)
    got = engine.genotype_likelihoods(m, gts)
    dev = torch.as_tensor(m, device="cuda:0") if m_dev is None else m_dev
    got_dev = engine.genotype_likelihoods(dev, torch.as_tensor(gts, device="cuda:0"))
    assert isinstance(got_dev, torch.Tensor)
    got_dev = got_dev.cpu().numpy()
    assert got.view(np.int64).tolist() == got_dev.view(np.int64).tolist(), what
    ex = ge.exact_genotypes(m, gts)
    key = _group(gts.shape[1])
    wk = ge.assert_within_bound(got, ex, ge.kernel_chain(m.shape[1]), "kernel, " + what)
    wo = ge.assert_within_bound(coracle.genotype_likelihoods(m, gts), ex, m.shape[1], "oracle, " + what)
    worst["kernel, " + key] = max(worst.get("kernel, " + key, 0.0), wk)
    worst["oracle, " + key] = max(worst.get("oracle, " + key, 0.0), wo)


def test_synthetic_inputs(engine, coracle, worst):
    """Every ploidy at R = 1, 31, 255, 256, 257, 4000; lowest(), -inf, 0.0, spreads of 700-1000, equal values; every duplicate
    pattern of ploidy 3 and 4, sorted and unsorted; one heterozygous copy among 63; H = 1024 with uniform draws; G = 1."""
    for name, m, gts in ge.synthetic_cases():
        _check(engine, coracle, worst, m, gts, name)


def test_more_than_65535_genotypes(engine, coracle, worst):
    m, gts = ge.many_genotypes_case()
    _check(engine, coracle, worst, m, gts, "G 70000")


def test_populate_output(engine, coracle, worst):
    """The matrix populate leaves on the device (C2-shaped region, 4000 reads, 12 haplotypes), mapping quality off and on."""
    from octopus_b200 import HaplotypeLikelihoodModel, synth
    haps, reads, band = synth.make_batch("C2", n_reads=4000, n_haps=12)
    hd, rd = haps.to_device("cuda:0"), reads.to_device("cuda:0")
    for use_mq in (False, True):
        cfg = HaplotypeLikelihoodModel.Config(max_indel_error=band, use_mapping_quality=use_mq)
        m_dev = engine.populate(cfg, hd, rd)
        m = m_dev.cpu().numpy()
        rng = np.random.default_rng(40 + use_mq)
        for p in ge.PLOIDIES:
            _check(engine, coracle, worst, m, ge.uniform_genotypes(rng, 12, p, 16), "populate mapq %s ploidy %d" % (use_mq, p), m_dev)


def test_million_read_matrix(engine, coracle, worst):
    """A C3-sized matrix (1 000 000 reads, 128 haplotypes) left on the device by populate, mapping quality off and on: the
    strided partial sums run 3 907 deep."""
    import torch
    from octopus_b200 import HaplotypeLikelihoodModel, synth
    haps, reads, band = synth.make_batch("C3")
    hd, rd = haps.to_device("cuda:0"), reads.to_device("cuda:0")
    gts = np.array([[7, 7], [3, 90], [0, 127]], dtype=np.int32)
    for use_mq in (False, True):
        m_dev = engine.populate(HaplotypeLikelihoodModel.Config(max_indel_error=band, use_mapping_quality=use_mq), hd, rd)
        rows = np.unique(gts)            # only the rows the genotypes read come to the host
        m, local = m_dev[torch.as_tensor(rows, device=m_dev.device)].cpu().numpy(), np.searchsorted(rows, gts).astype(np.int32)
        got = engine.genotype_likelihoods(m_dev, gts)
        assert isinstance(got, torch.Tensor)
        ex = ge.exact_genotypes(m, local)
        wk = ge.assert_within_bound(got.cpu().numpy(), ex, ge.kernel_chain(m.shape[1]), "kernel, C3 mapq %s" % use_mq)
        wo = ge.assert_within_bound(coracle.genotype_likelihoods(m, local), ex, m.shape[1], "oracle, C3 mapq %s" % use_mq)
        worst["kernel, C3"] = max(worst.get("kernel, C3", 0.0), wk)
        worst["oracle, C3"] = max(worst.get("oracle, C3", 0.0), wo)
        del m_dev
        torch.cuda.empty_cache()


def test_nonfinite_reads(engine):
    """A read on which every value of a heterozygous genotype is -inf gives NaN (-inf - -inf in the max shift, as the
    reference's log_sum_exp gives), though the exact value is -inf; a homozygous genotype takes the plain sum: -inf."""
    m = np.array([[-1.0, -np.inf, -2.0], [-2.0, -np.inf, -1.0], [-3.0, -4.0, -5.0]])
    for p in (2, 3, 5, 64):
        het = np.zeros((1, p), np.int32)
        het[0, -1] = 1
        got = engine.genotype_likelihoods(m, np.concatenate([het, np.zeros((1, p), np.int32), np.full((1, p), 2, np.int32)]))
        assert np.isnan(got[0]) and got[1] == -np.inf and np.isfinite(got[2]), (p, got)


@pytest.mark.parametrize("device", [False, True])
def test_ploidy_zero_and_sizes(engine, device):
    import torch
    m = np.random.default_rng(1).uniform(-50, 0, size=(5, 300))
    x = torch.as_tensor(m, device="cuda:0") if device else m
    out = engine.genotype_likelihoods(x, np.zeros((7, 0), np.int32))
    out = out.cpu().numpy() if device else out
    assert out.shape == (7,) and out.view(np.int64).tolist() == [0] * 7
    assert engine.genotype_likelihoods(x, np.zeros((0, 3), np.int32)).shape == (0,)
    with pytest.raises(PhmmError, match="bad argument") as e:
        engine.genotype_likelihoods(x, np.zeros((2, 65), np.int32))
    assert e.value.code == _lib.PHMM_ERR_INVALID


@pytest.mark.parametrize("device", [False, True])
@pytest.mark.parametrize("bad_index", [5, -1, 1 << 30])
def test_out_of_range_index(engine, device, bad_index):
    import torch
    m = np.random.default_rng(2).uniform(-50, 0, size=(5, 300))
    gts = np.array([[0, 1], [2, bad_index], [3, 4]], dtype=np.int32)
    x, g = (torch.as_tensor(m, device="cuda:0"), torch.as_tensor(gts, device="cuda:0")) if device else (m, gts)
    with pytest.raises(PhmmError, match="haplotype index out of range") as e:
        engine.genotype_likelihoods(x, g)
    assert e.value.code == _lib.PHMM_ERR_INVALID
    ok = engine.genotype_likelihoods(x, g[[0, 2]])          # the engine is usable afterwards and the flag starts clear
    ok = ok.cpu().numpy() if device else ok
    ge.assert_within_bound(ok, ge.exact_genotypes(m, gts[[0, 2]]), ge.kernel_chain(300), "after the error")
