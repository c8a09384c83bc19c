#!/usr/bin/env python
"""Generates tests/golden/error_model_golden.json from the UNMODIFIED reference error models + lib/tandem compiled here
(oracle/_ref/libref_errmodel.so). Run with OCTOPUS_REFERENCE set; the JSON is committed."""
import json
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

from oracle.oracle import RefErrorModel, build   # noqa: E402
from test_error_model import FIELDS, LABELS, repeat_rich_sequence   # noqa: E402

CUSTOM = "# example custom model\nA:50,50,45,40,30,20,10,5\nC:50,50,46,41,31,21,11\nAC:48,48,40,30,20\nN:44,44,35\nNN:43,43,33\nNNN:42,40\nA+:3,3,4,5\nNN+:2,2,3\n"


def main():
    build(ref=True)
    ref = RefErrorModel()
    rng = np.random.default_rng(0xE44)
    cases = []
    plan = [(lab, None) for lab in LABELS for _ in range(5)] + [("PCR-free.HiSeq-2500", CUSTOM)] * 12
    for label, custom in plan:
        s = repeat_rich_sequence(rng, 160)
        sub = (rng.random(len(s)) < 0.05).astype(np.uint8) if rng.random() < 0.4 else None
        r = ref.reset(s, label, sub, custom_model_text=custom)
        assert r["rc"] >= 0
        c = {"label": label, "custom": custom, "sequence": bytes(s).decode(), "substitutions": None if sub is None else sub.tolist(),
             "repeats_1_5": ref.tandem_repeats(s, 1, 5).reshape(-1).tolist()}
        for f in FIELDS:
            c[f] = bytes(r[f]).decode() if "mask" in f else r[f].tolist()
        cases.append(c)
    out = os.path.join(ROOT, "tests", "golden", "error_model_golden.json")
    with open(out, "w") as f:
        json.dump({"source": "oracle/_ref/libref_errmodel.so (reference error models + lib/tandem, compiled from the reference checkout)", "cases": cases}, f)
    print("wrote", out, len(cases), "cases")


if __name__ == "__main__":
    main()
