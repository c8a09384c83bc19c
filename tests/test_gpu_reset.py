"""HaplotypeLikelihoodModel::reset on the device (phmm_engine_reset_haplotypes): all six arrays byte-equal to the host call
(phmm_reset_haplotypes), and to the compiled reference models (oracle/_ref/libref_errmodel.so) where that build is present."""
import json
import os

import numpy as np
import pytest

from test_error_model import FIELDS, GOLDEN, LABELS, repeat_rich_sequence

pytestmark = pytest.mark.gpu
ACGT_CHOICE = np.frombuffer(b"ACGT", dtype=np.uint8)

CUSTOM_TEXTS = [
    "# motifs and N wildcards\nA:30,25,20,15,10\nC:28,22\nAC:26,20,14,9\nNN:24,18,12\nN:27,21,16\nNNN:22,15\nACG:25,19\nA+:4,3,2\nN+:5,4\n",
    "AT:40,30,20,10,5\nCAG:35,25,15\nT:33,29,25,21,17,13,9\nGGCC:20,10\n",
]


@pytest.fixture(scope="module")
def engine():
    import torch
    if not torch.cuda.is_available():
        pytest.skip("no GPU")
    from octopus_b200 import PairHMMEngine
    return PairHMMEngine(0)


@pytest.fixture(scope="module")
def ref():
    from oracle.oracle import RefErrorModel
    return RefErrorModel() if RefErrorModel.available() else None


def _blocks_equal(a, b, what):
    for f in FIELDS:
        x, y = getattr(a, f), getattr(b, f)
        x = x.cpu().numpy() if hasattr(x, "cpu") else x
        y = y.cpu().numpy() if hasattr(y, "cpu") else y
        assert np.array_equal(np.asarray(x).view(np.uint8), np.asarray(y).view(np.uint8)), (what, f)


def _check_model(model, engine, ref, seqs, subs, ref_kwargs, what, ref_count=150):
    host = model.reset(seqs, is_substitution=subs)
    dev = model.reset(seqs, is_substitution=subs, engine=engine)
    _blocks_equal(host, dev, what)
    if ref is not None:
        for h in range(min(ref_count, len(seqs))):
            if len(seqs[h]) == 0 or max(bytes(seqs[h])) >= 0x80:
                continue        # the reference reads before an empty haplotype, and its suffix sorter takes bytes as signed chars
            want = ref.reset(seqs[h], is_substitution=None if subs is None else subs[h], **ref_kwargs)
            got = dev.hap(h)
            for f in FIELDS:
                assert np.array_equal(got[f].view(np.uint8), want[f].view(np.uint8)), (what, f, bytes(seqs[h]))


def test_every_builtin_model_on_device_equals_host(engine, ref):
    from octopus_b200 import ErrorModel
    rng = np.random.default_rng(31)
    for label in LABELS:
        m = ErrorModel(label)
        seqs = [repeat_rich_sequence(rng, 600)[:600] for _ in range(2000)]
        subs = [(rng.random(len(s)) < 0.05).astype(np.uint8) for s in seqs]
        _check_model(m, engine, ref, seqs, subs, {"label": label}, label)


def test_custom_models_on_device_equal_host(engine, ref):
    from octopus_b200 import ErrorModel
    rng = np.random.default_rng(32)
    for text in CUSTOM_TEXTS:
        m = ErrorModel(custom_model_text=text)
        seqs = [repeat_rich_sequence(rng, 600)[:600] for _ in range(2000)]
        subs = [(rng.random(len(s)) < 0.05).astype(np.uint8) for s in seqs]
        _check_model(m, engine, ref, seqs, subs, {"custom_model_text": text}, text)


def test_golden_fixture_on_device(engine):
    from octopus_b200 import ErrorModel
    with open(GOLDEN) as f:
        cases = json.load(f)["cases"]
    models = {}
    for c in cases:
        key = (c["label"], c.get("custom"))
        if key not in models:
            models[key] = ErrorModel(c["label"], custom_model_text=c.get("custom"))
        sub = None if c["substitutions"] is None else [np.asarray(c["substitutions"], dtype=np.uint8)]
        got = models[key].reset([c["sequence"]], is_substitution=sub, engine=engine).hap(0)
        for f in FIELDS:
            want = np.frombuffer(c[f].encode(), dtype=np.uint8) if "mask" in f else np.asarray(c[f], dtype=np.int8).view(np.uint8)
            assert np.array_equal(got[f].view(np.uint8), want), (c["label"], f, c["sequence"])


def test_edge_inputs(engine, ref):
    from octopus_b200 import ErrorModel, PhmmError
    rng = np.random.default_rng(33)
    m = ErrorModel()
    odd = bytes(rng.integers(0, 256, 300, dtype=np.uint8))
    seqs = [b"", b"A", b"", b"ACGTTTTTACAC", b"N" * 400, b"A" * 5000, b"AC" * 2500, b"ACGTN" * 3 + b"acgtXYZ\x00\xff" * 20, b"acgtXYZ\x01" * 30, odd, b"G"]
    _check_model(m, engine, ref, seqs, None, {"label": "PCR-free.HiSeq-2500"}, "edge")
    _check_model(ErrorModel("PCR.PacBio"), engine, None, seqs, None, {}, "edge, no SNV model")
    # the longest haplotype the call takes, and one base more
    longest = repeat_rich_sequence(rng, 400)
    longest = np.tile(longest, 65535 // len(longest) + 1)[:65535]
    _check_model(m, engine, None, [longest, b"ACGT"], None, {}, "65535")
    with pytest.raises(PhmmError, match="65535"):
        m.reset([np.concatenate([longest, longest[:1]])], engine=engine)
    # n = 0
    empty = m.reset_block(np.zeros(1, dtype=np.int64), np.zeros(0, dtype=np.uint8), engine=engine)
    assert empty.n == 0


def test_one_hundred_thousand_haplotypes_in_one_call(engine):
    from octopus_b200 import ErrorModel
    from octopus_b200.batch import pack_sequences
    rng = np.random.default_rng(34)
    pool = [repeat_rich_sequence(rng, 300) for _ in range(1000)]
    seqs = [np.resize(pool[i % 1000], 300) for i in range(100000)]
    for i in range(0, 100000, 7):
        seqs[i] = seqs[i].copy()
        seqs[i][rng.integers(0, 300, 3)] = ACGT_CHOICE[rng.integers(0, 4, 3)]
    off, seq = pack_sequences(seqs)
    m = ErrorModel()
    host = m.reset_block(off, seq)
    dev = m.reset_block(off, seq, engine=engine)
    _blocks_equal(host, dev, "100000 x 300")


def test_host_and_device_space_give_the_same_arrays(engine):
    import torch
    from octopus_b200 import ErrorModel
    from octopus_b200.batch import pack_sequences
    rng = np.random.default_rng(35)
    seqs = [repeat_rich_sequence(rng, 600) for _ in range(500)]
    subs = np.concatenate([(rng.random(len(s)) < 0.05).astype(np.uint8) for s in seqs])
    off, seq = pack_sequences(seqs)
    m = ErrorModel("PCR.HiSeq-4000")
    on_host = m.reset_block(off, seq, is_substitution=subs, engine=engine)
    on_dev = m.reset_block(torch.as_tensor(off, device="cuda:0"), torch.as_tensor(seq, device="cuda:0"),
                           is_substitution=torch.as_tensor(subs, device="cuda:0"), engine=engine)
    assert on_dev.on_device and not on_host.on_device
    _blocks_equal(on_host, on_dev, "spaces")
    _blocks_equal(on_host, m.reset_block(off, seq, is_substitution=subs), "host threads")


def test_cpp_adapter_reset_on_engine_equals_host(engine, tmp_path):
    import subprocess
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    src = os.path.join(root, "tests", "cpp", "test_reset_engine.cpp")
    exe = str(tmp_path / "test_reset_engine")
    from octopus_b200 import build
    build.build()
    subprocess.run(["g++", "-std=c++14", "-O1", "-I", os.path.join(root, "include"), "-I", os.path.join(root, "octopus_b200", "cpp"),
                    src, "-o", exe, "-L", os.path.join(root, "octopus_b200"), "-lphmm_b200",
                    "-Wl,-rpath," + os.path.join(root, "octopus_b200")], check=True)
    out = subprocess.run([exe], capture_output=True, text=True, timeout=300)
    assert out.returncode == 0, out.stdout + out.stderr
    assert "same=1" in out.stdout, out.stdout
