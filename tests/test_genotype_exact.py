"""The genotype-likelihood bound (tests/genotype_exact.py) on the CPU: the kernel's operation order stays within it on every
input the GPU tests use, the checker rejects subtly wrong versions of that order, and the reference-form oracle
(oracle_genotype_likelihoods) stays within its own, read-by-read, bound."""
import numpy as np
import pytest

import genotype_exact as ge


@pytest.fixture(scope="module")
def cases():
    return [(name, m, gts, ge.exact_genotypes(m, gts)) for name, m, gts in ge.synthetic_cases()]


@pytest.fixture(scope="module")
def populated(coracle):
    """Realistic populate output, as the GPU tests' populate cases (scaled down: 600 reads), mapping quality off and on."""
    from octopus_b200 import synth
    haps, reads, band = synth.make_batch("C2", n_reads=600, n_haps=12)
    out = []
    for use_mq in (False, True):
        rc, m, _ = coracle.populate(band, haps, reads, use_mapping_quality=use_mq)
        assert rc == 0
        rng = np.random.default_rng(11 + use_mq)
        for p in ge.PLOIDIES:
            gts = ge.uniform_genotypes(rng, 12, p, 6)
            out.append(("populate mapq %s ploidy %d" % (use_mq, p), m, gts, ge.exact_genotypes(m, gts)))
    return out


def test_kernel_order_stays_within_the_bound(cases, populated):
    for name, m, gts, ex in cases + populated:
        ge.assert_within_bound(ge.kernel_model(m, gts), ex, ge.kernel_chain(m.shape[1]), name)


def test_kernel_order_within_the_bound_with_many_genotypes():
    m, gts = ge.many_genotypes_case()
    ge.assert_within_bound(ge.kernel_model(m, gts), ge.exact_genotypes(m, gts), ge.kernel_chain(m.shape[1]), "G 70000")


def test_kernel_order_within_the_bound_with_many_reads():
    """The GPU tests' million-read matrix, scaled down to 60 000 reads: the strided partial sums run 235 deep."""
    rng = np.random.default_rng(5)
    m = ge.penalty_matrix(rng, 6, 60_000, s_max=150)
    gts = np.array([[0, 0], [1, 4], [2, 3]], dtype=np.int32)
    ge.assert_within_bound(ge.kernel_model(m, gts), ge.exact_genotypes(m, gts), ge.kernel_chain(m.shape[1]), "R 60000")


def _mutation_input(mutation):
    rng = np.random.default_rng(3)
    if mutation == "max_short":
        # the max of every read sits in the genotype's last haplotype, 800 above the others: e^(x - max) overflows without it
        m = np.full((4, 50), -800.0) - rng.uniform(0, 5, size=(4, 50))
        m[3] = -rng.uniform(0, 5, size=50)
        return m, np.array([[0, 1, 3], [0, 2, 3], [1, 2, 3]], dtype=np.int32)
    m = ge.penalty_matrix(rng, 16, 4000)
    return m, ge.uniform_genotypes(rng, 16, 3, 8, homozygous=False)


@pytest.mark.parametrize("mutation", ge.MUTATIONS)
def test_checker_rejects_a_mutated_kernel_order(mutation):
    m, gts = _mutation_input(mutation)
    ex = ge.exact_genotypes(m, gts)
    n_seq = ge.kernel_chain(m.shape[1])
    ge.assert_within_bound(ge.kernel_model(m, gts), ex, n_seq, "unmutated")
    with pytest.raises(AssertionError, match="outside"):
        ge.assert_within_bound(ge.kernel_model(m, gts, mutation), ex, n_seq, mutation)


def test_reference_form_oracle_within_the_sequential_bound(coracle, cases, populated):
    for name, m, gts, ex in cases + populated:
        ge.assert_within_bound(coracle.genotype_likelihoods(m, gts), ex, m.shape[1], name)


def test_reference_form_oracle_edges(coracle):
    """Ploidy 0 is 0; a read on which every value of a heterozygous genotype is -inf gives NaN (-inf - -inf inside
    log_sum_exp, as the reference computes it) though the exact value is -inf; homozygous genotypes of ploidy 1 to 4 take the
    plain sum (-inf), from ploidy 5 the reference's buffer form (NaN)."""
    m = np.array([[-1.0, -np.inf], [-2.0, -np.inf], [-3.0, -4.0]])
    assert coracle.genotype_likelihoods(m, np.zeros((3, 0), np.int32)).tolist() == [0.0, 0.0, 0.0]
    het = coracle.genotype_likelihoods(m, np.array([[0, 1], [0, 2]], np.int32))
    assert np.isnan(het[0]) and np.isfinite(het[1])
    assert ge.exact_genotypes(m, np.array([[0, 1]], np.int32)).cls == ["-inf"]
    for p in (1, 2, 3, 4, 5, 8):
        v = coracle.genotype_likelihoods(m, np.zeros((1, p), np.int32))[0]
        assert (v == -np.inf) if p <= 4 else np.isnan(v), p
