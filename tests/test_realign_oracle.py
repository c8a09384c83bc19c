"""The C oracle's k-mer mapper without the cap of 10 (max_positions >= the haplotype length) against the reference's own
map_query_to_target (utils/kmer_mapper.hpp, compiled from the reference checkout) with the same setting: the vector overload
ReadRealigner::realign maps with (utils/kmer_mapper.cpp:14-22), which lists every mapping begin at the maximum vote count."""
import numpy as np
import pytest

ACGT = np.frombuffer(b"ACGT", dtype=np.uint8)
FOREIGN = np.frombuffer(b"NnacgtX-*", dtype=np.uint8)      # all < 128: the reference indexes a 128-entry table with the byte


def mapper_case(rng, kind):
    """(query, target) as uint8 arrays. kind: 'tandem', 'homopolymer', 'foreign', 'short' or 'random'."""
    if kind == "tandem":
        unit = ACGT[rng.integers(0, 4, int(rng.integers(2, 7)))]
        tl = int(rng.integers(40, 700))
        target = np.tile(unit, tl // len(unit) + 1)[:tl].copy()
        for _ in range(int(rng.integers(0, 3))):
            target[rng.integers(0, tl)] = ACGT[rng.integers(0, 4)]
    elif kind == "homopolymer":
        tl = int(rng.integers(120, 600))
        target = np.full(tl, ACGT[rng.integers(0, 4)], dtype=np.uint8)
        if rng.random() < 0.5:
            target[: int(rng.integers(0, 10))] = ACGT[rng.integers(0, 4)]
    elif kind == "short":
        tl = int(rng.integers(0, 12))
        target = ACGT[rng.integers(0, 4, tl)].copy()
    else:
        tl = int(rng.integers(20, 500))
        target = ACGT[rng.integers(0, 4, tl)].copy()
    if kind == "foreign":
        target[rng.integers(0, tl, int(rng.integers(1, 6)))] = FOREIGN[rng.integers(0, len(FOREIGN), 1)]
    ql = int(rng.integers(0, 12)) if kind == "short" and rng.random() < 0.7 else int(rng.integers(6, 200))
    if tl > ql and rng.random() < 0.85:
        s = int(rng.integers(0, tl - ql + 1))
        query = target[s:s + ql].copy()
        for _ in range(int(rng.integers(0, 3)) if ql else 0):
            query[rng.integers(0, ql)] = ACGT[rng.integers(0, 4)]
    else:
        query = ACGT[rng.integers(0, 4, ql)].copy()
    if kind == "foreign" and ql > 0:
        query[rng.integers(0, ql, int(rng.integers(1, 4)))] = FOREIGN[rng.integers(0, len(FOREIGN), 1)]
    return query, target


def test_uncapped_c_mapper_matches_reference_mapper(coracle, refhmm):
    if refhmm is None:
        pytest.skip("oracle/_ref/libref_hmm.so not built")
    rng = np.random.default_rng(6101)
    seen = dict(over10=0, over100=0, homopolymer_over100=0, empty=0)
    for it in range(1500):
        kind = ("tandem", "homopolymer", "foreign", "short", "random")[it % 5]
        query, target = mapper_case(rng, kind)
        cap = max(1, len(target))
        want = refhmm.kmer_map(query, target, cap)
        got = coracle.kmer_map(query.tobytes().decode("latin1"), target.tobytes().decode("latin1"), cap)
        assert list(got) == want, (it, kind, query.tobytes(), target.tobytes(), got[:20], want[:20])
        assert want == sorted(set(want))
        seen["over10"] += len(want) > 10
        seen["over100"] += len(want) > 100
        seen["homopolymer_over100"] += kind == "homopolymer" and len(want) > 100
        seen["empty"] += (len(query) < 6 or len(target) < 6) and not want
    assert seen["over10"] > 200 and seen["over100"] > 100 and seen["homopolymer_over100"] > 50 and seen["empty"] > 100, seen
