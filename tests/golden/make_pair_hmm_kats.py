#!/usr/bin/env python
"""Extract the reference's own known-answer tests for the raw pair-HMM kernel into a JSON fixture.

Source (read at generation time only, never at test time):
    test/unit/core/models/pair_hmm_tests.cpp of the octopus tree
      TestCase  {target(=truth window), query(=read), base_qualities, gap_open[], gap_extend, nuc_prior}  (:22-28)
      Alignment {score, begin(=first_pos), target(=aligned truth), query(=aligned read)}                   (:30-35)
      sse2_band_size_{8,16,32}_check_alignments, avx2_check_alignments (band 16, short)                    (:203-712)
      band8_speed_test / band16_speed_test + expected alignments                                           (:104-199)

Run with OCTOPUS_REFERENCE naming an octopus checkout:
    python tests/golden/make_pair_hmm_kats.py > tests/golden/pair_hmm_kats.json
"""
import json
import os
import re
import sys

SRC = os.path.join(os.environ.get("OCTOPUS_REFERENCE", "."), "test", "unit", "core", "models", "pair_hmm_tests.cpp")


def _ints(body):
    return [int(x) for x in re.findall(r"-?\d+", body)]


def _parse_test(block):
    strs = re.findall(r'"([^"]*)"', block)
    lists = re.findall(r"\{([^{}]*)\}", block)
    tail = block[block.rfind("}") + 1:]
    scalars = _ints(tail)
    return {"truth": strs[0], "read": strs[1], "quals": _ints(lists[0]), "gap_open": _ints(lists[1]),
            "gap_extend": scalars[0], "nuc_prior": scalars[1]}


def _parse_expected(block):
    strs = re.findall(r'"([^"]*)"', block)
    nums = _ints(block[:block.find('"')])
    return {"score": nums[0], "first_pos": nums[1], "align_truth": strs[0], "align_read": strs[1]}


def _balanced(text, start):
    """Return the text inside the braces opening at text[start] == '{'."""
    depth, i = 0, start
    while True:
        if text[i] == "{":
            depth += 1
        elif text[i] == "}":
            depth -= 1
            if depth == 0:
                return text[start + 1:i], i + 1
        i += 1


def main():
    text = open(SRC).read()
    cases = []
    # 1. the check_alignments suites
    for m in re.finditer(r"BOOST_AUTO_TEST_CASE\((\w+check_alignments)\)", text):
        name = m.group(1)
        body, _ = _balanced(text, text.index("{", m.end()))
        band = int(re.search(r"PairHMM<(\d+),", body).group(1))
        isa = name.split("_")[0]
        precisions = sorted(set(re.findall(r"PairHMM<\d+,\s*(short|int)>", body)))
        pos, idx = 0, 0
        while True:
            t = body.find("test = {", pos)
            if t < 0:
                break
            tb, after = _balanced(body, body.index("{", t))
            e = body.index("expected_alignment = {", after)
            eb, pos = _balanced(body, body.index("{", e))
            idx += 1
            case = {"suite": name, "index": idx, "isa": isa, "band": band, "precisions": precisions}
            case.update(_parse_test(tb))
            case.update(_parse_expected(eb))
            cases.append(case)
    # 2. the two "speed test" inputs (same KAT form, long sequences)
    for band in (8, 16):
        t = text.index("TestCase band%d_speed_test = {" % band)
        tb, after = _balanced(text, text.index("{", t))
        # NB the reference's band-16 speed test checks against band8_speed_expected_alignment (:746-756);
        # both expected alignments are recorded here against their own input.
        e = text.index("Alignment band%d_speed_expected_alignment = {" % band)
        eb, _ = _balanced(text, text.index("{", e))
        case = {"suite": "band%d_speed_test" % band, "index": 1, "isa": "sse2", "band": band, "precisions": ["int", "short"]}
        case.update(_parse_test(tb))
        case.update(_parse_expected(eb))
        cases.append(case)
    for c in cases:
        assert len(c["truth"]) == len(c["read"]) + 2 * c["band"] - 1, c["suite"]
        assert len(c["quals"]) == len(c["read"]) and len(c["gap_open"]) == len(c["truth"]), c["suite"]
    json.dump({"source": "octopus v0.7.4 test/unit/core/models/pair_hmm_tests.cpp", "cases": cases}, sys.stdout, indent=1)
    sys.stdout.write("\n")


if __name__ == "__main__":
    main()
