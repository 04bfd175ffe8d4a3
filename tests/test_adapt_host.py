"""CPU: the host side of speaker adaptation.

* adapt.py's argument errors: one source, -a with -wav, -holdout / -eval_set / -transcripts with their source, held-out
  clips that are adaptation clips (by path, and by id through the set), frame_size other than 1;
* the crop index: every valid start of every long enough clip, short clips skipped and counted, the no-clip refusal;
* the seeded crop order: seed 0 is the training run's order, another seed another order; the full-batch schedule;
* the JSON report's schema;
* avc_rec_loss_varlen: header and binding agree, the descriptor's size is the C compiler's.
"""
import ctypes as C
import json
import os
import pickle
import subprocess
import sys
import tempfile

import numpy as np
import pytest
import yaml

import oracle.ae_oracle as orc
from adaptive_voice_conversion_b200 import _lib as L
from adaptive_voice_conversion_b200 import adapt as A
from adaptive_voice_conversion_b200 import data_utils as D

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def root_adapt():
    if ROOT not in sys.path:
        sys.path.insert(0, ROOT)
    import adapt
    return adapt


def write_config(tmp_path, frame_size=1):
    cfg = orc.default_config(80)
    cfg["data_loader"]["frame_size"] = frame_size
    path = tmp_path / "config.yaml"
    path.write_text(yaml.safe_dump(cfg))
    return str(path)


def run_error(argv, capsys):
    with pytest.raises(SystemExit) as e:
        root_adapt().main(argv)
    assert e.value.code == 2
    return capsys.readouterr().err


# ----------------------------------------------------------------------------- argument errors
def test_argument_errors(tmp_path, capsys):
    cfg = write_config(tmp_path)
    wavs = []
    for i in range(3):
        w = tmp_path / f"a{i}.wav"
        w.write_bytes(b"RIFF")
        wavs.append(str(w))
    base = ["-c", cfg, "-m", "base.ckpt", "-o", str(tmp_path / "out"), "-speaker", "alice"]
    cases = [
        ([], "either -wav"),
        (["-wav", wavs[0], "-d", str(tmp_path), "-set", "train", "-a", "attr.pkl"], "either -wav"),
        (["-wav", wavs[0]], "needs -a"),
        (["-wav", wavs[0], "-a", "attr.pkl", "-transcripts", str(tmp_path)], "go with -d"),
        (["-wav", wavs[0], "-a", "attr.pkl", "-eval_set", "in_test"], "go with -d"),
        (["-wav", wavs[0], wavs[1], "-a", "attr.pkl", "-holdout", wavs[2], wavs[1]], "also adaptation clips"),
        (["-wav", wavs[0], "-a", "attr.pkl", "-holdout", os.path.join(str(tmp_path), ".", "a0.wav")], "also adaptation"),
        (["-wav", str(tmp_path / "missing.wav"), "-a", "attr.pkl"], "is not a file"),
        (["-d", str(tmp_path)], "-d and -set go together"),
        (["-d", str(tmp_path), "-set", "train", "-holdout", wavs[0]], "-holdout goes with -wav"),
        (["-d", str(tmp_path), "-set", "train", "-transcripts", str(tmp_path)], "needs -eval_set"),
        (["-wav", wavs[0], "-a", "attr.pkl", "-steps", "0"], ">= 1"),
    ]
    for extra, msg in cases:
        assert msg in run_error(base + extra, capsys), extra
    d2 = tmp_path / "fs2"
    d2.mkdir()
    assert "frame_size 1 only" in run_error(["-c", write_config(d2, frame_size=2)] + base[2:] + ["-wav", wavs[0], "-a", "x"],
                                            capsys)


def test_heldout_set_overlap_by_id(tmp_path, capsys):
    """-set and -eval_set sharing utterances of the speaker are refused before the model is loaded."""
    cfg = write_config(tmp_path)
    m = np.zeros((200, 80), np.float32)
    with open(tmp_path / "train.pkl", "wb") as f:
        pickle.dump({"p225_001.wav": m, "p225_002.wav": m, "p226_001.wav": m}, f)
    with open(tmp_path / "test.pkl", "wb") as f:
        pickle.dump({"p225_002.wav": m, "p225_003.wav": m}, f)
    base = ["-c", cfg, "-m", "missing.ckpt", "-o", str(tmp_path / "out"), "-d", str(tmp_path), "-set", "train"]
    err = run_error(base + ["-speaker", "p225", "-eval_set", "test"], capsys)
    assert "1 held-out utterance(s) are also adaptation clips (e.g. p225_002.wav)" in err
    assert "has no utterance in train" in run_error(base + ["-speaker", "p999"], capsys)
    with pytest.raises(ValueError, match="also adaptation clips"):
        A.check_disjoint(["a", "b"], ["b"])
    A.check_disjoint(["a", "b"], ["c"])


# ----------------------------------------------------------------------------- crops
def test_crop_index_enumerates_every_valid_start():
    seg = 128
    lengths = {"u1": 128, "u0": 300, "short": 127, "u2": 129, "tiny": 3}
    index, used, skipped = A.crop_index(lengths, seg)
    assert used == ["u1", "u0", "u2"] and skipped == ["short", "tiny"]
    want = [("u1", 0)] + [("u0", t) for t in range(173)] + [("u2", 0), ("u2", 1)]
    assert index == want
    # every entry is a valid crop of the device corpus, and only those
    data = {u: np.zeros((T, 80), np.float32) for u, T in lengths.items() if u in used}
    starts, n_mels, total = D.validate_corpus(data, index, seg, 1, 80)
    assert len(starts) == 176 and total == 128 + 300 + 129
    assert starts[-1] + seg == total


def test_no_clip_long_enough_raises_before_any_launch():
    cfg = orc.default_config(80)
    with pytest.raises(ValueError, match="no adaptation clip has segment_size = 128 frames \\(2 shorter"):
        A.segments({"a": np.zeros((100, 80)), "b": np.zeros((127, 80))}, cfg, 4, 0, "cpu")
    cfg["data_loader"]["frame_size"] = 2
    with pytest.raises(ValueError, match="frame_size 1 only"):
        A.segments({"a": np.zeros((300, 80))}, cfg, 4, 0, "cpu")


def test_seeded_order():
    """seed 0 is the training run's order, bit for bit; another seed gives another permutation, reproducibly."""
    n = 1000
    s0 = D.SegmentSampler(n, 64)
    s0b = D.SegmentSampler(n, 64, seed=0)
    s7 = D.SegmentSampler(n, 64, seed=7)
    s7b = D.SegmentSampler(n, 64, seed=7)
    for epoch in (0, 3):
        ref = D.epoch_order(n, 0, epoch)
        assert bool((s0.order(epoch) == ref).all()) and bool((s0b.order(epoch) == ref).all())
        assert not bool((s7.order(epoch) == ref).all())
        assert bool((s7.order(epoch) == s7b.order(epoch)).all())
        assert sorted(s7.order(epoch).tolist()) == list(range(n))
    assert not bool((D.epoch_order(n, 0, 0, seed=1) == D.epoch_order(n, 0, 0, seed=2)).all())


def test_drop_last_schedule():
    """drop_last: every batch has B entries, an epoch is the first floor(n/B) * B entries of its order; the default
    schedule is unchanged."""
    n, B = 33, 16
    s = D.SegmentSampler(n, B, seed=3, drop_last=True)
    assert s.batches_per_epoch == 2
    for k in range(7):
        epoch, first, count = s.locate(k)
        assert (epoch, first, count) == (k // 2, (k % 2) * B, B)
        batch = next(s)
        assert bool((batch == s.order(epoch)[first:first + B]).all())
    plain = D.SegmentSampler(n, B, seed=3)
    assert plain.batches_per_epoch == 3 and plain.locate(2) == (0, 32, 1)
    with pytest.raises(ValueError, match="drop_last needs batch_size <= n"):
        D.SegmentSampler(5, 8, drop_last=True)


# ----------------------------------------------------------------------------- report
def test_report_schema():
    settings = {"steps": 3, "lr": 1e-4, "batch_size": 8, "seed": 0}
    losses = [{"step": 0, "loss_rec": 0.5, "grad_norm": 1.0}, {"step": 2, "loss_rec": 0.4, "grad_norm": 0.9}]
    rec = {"rec": 0.3, "n": 2, "n_skipped": 1, "skipped": ["h9"]}
    r = A.make_report("alice", settings, ["a0", "a1"], ["a2"], 345, losses, {"rec": rec}, {"rec": dict(rec, rec=0.2)})
    assert tuple(r) == A.REPORT_KEYS
    back = json.loads(json.dumps(r))
    assert back["format"] == A.FORMAT and back["speaker"] == "alice"
    assert back["clips"] == {"used": ["a0", "a1"], "skipped": ["a2"], "n_entries": 345}
    assert [e["step"] for e in back["losses"]] == [0, 2] and set(back["losses"][0]) == {"step", "loss_rec", "grad_norm"}
    assert back["heldout"]["before"]["rec"]["rec"] == 0.3 and back["heldout"]["after"]["rec"]["rec"] == 0.2
    assert A.make_report("alice", settings, ["a0"], [], 1, losses, {}, {})["heldout"] is None


# ----------------------------------------------------------------------------- C ABI
def test_rec_loss_varlen_abi():
    from test_cabi_symbols import header_functions
    assert "avc_rec_loss_varlen" in header_functions() and "avc_rec_loss_varlen" in L.PROTOTYPES
    prog = ('#include <stdio.h>\n#include <stddef.h>\n#include "avc_b200.h"\nint main(){printf("%zu %zu %zu %zu\\n", '
            'sizeof(avc_rec_varlen_desc), offsetof(avc_rec_varlen_desc, dec), offsetof(avc_rec_varlen_desc, lengths), '
            'offsetof(avc_rec_varlen_desc, out));return 0;}\n')
    with tempfile.TemporaryDirectory() as td:
        c = os.path.join(td, "s.c")
        with open(c, "w") as f:
            f.write(prog)
        exe = os.path.join(td, "s")
        subprocess.check_call(["gcc", "-I", os.path.join(ROOT, "include"), c, "-o", exe])
        sizes = [int(v) for v in subprocess.check_output([exe]).split()]
    D_ = L.RecVarlenDesc
    assert sizes == [C.sizeof(D_), D_.dec.offset, D_.lengths.offset, D_.out.offset]
