"""CPU: the host side of speaker-code fitting (adaptive_voice_conversion_b200/fit.py).

* speaker_bank.py's -fit_* argument errors;
* the wave schedule (consecutive chunks in bank order, a smaller last wave);
* a speaker's crop order depends on (seed, name) only: its rows of a wave's order table do not change when other
  speakers join or leave the run, and follow SegmentSampler(drop_last=True) across epochs;
* the unfitted rule (fewer than m crops, or no clip of segment_size frames);
* the report schema;
* the fitted record: saved, checked against the content encoder and decoder on load, and absent from an old bank file,
  which loads as before;
* the descriptors of avc_group_l1 and avc_code_adam: the header's layout against the ctypes mirrors.
"""
import ctypes as C
import os
import shutil
import subprocess
import sys

import numpy as np
import pytest
import torch

import oracle.ae_oracle as orc
from adaptive_voice_conversion_b200 import _lib as L
from adaptive_voice_conversion_b200 import fit as F
from adaptive_voice_conversion_b200 import speaker_bank as SB
from adaptive_voice_conversion_b200.data_utils import SegmentSampler

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def root_module(name):
    if ROOT not in sys.path:
        sys.path.insert(0, ROOT)
    return __import__(name)


def cpu_model(cfg, seed=0):
    from adaptive_voice_conversion_b200.model import AE
    m = AE(cfg)
    m.load_state_dict(orc.init_state(cfg, seed=seed))
    return m


# ----------------------------------------------------------------------------- CLI
def test_fit_argument_errors(tmp_path, capsys):
    cli = root_module("speaker_bank")
    wav = tmp_path / "a.wav"
    wav.write_bytes(b"")
    base = ["-m", "m.ckpt", "-o", "b.pt"]
    dset = base + ["-d", "data", "-set", "train"]
    wavs = base + ["-a", "x", "-wav", "al", str(wav)]
    for argv, msg in ((dset + ["-fit_lr", "0.1"], "go(es) with -fit_steps"),
                      (dset + ["-holdout_set", "in_test"], "go(es) with -fit_steps"),
                      (dset + ["-report", "r.json"], "go(es) with -fit_steps"),
                      (dset + ["-fit_steps", "0"], "must be >= 1"), (dset + ["-fit_steps", "5", "-fit_crops", "0"], ">= 1"),
                      (dset + ["-fit_steps", "5", "-fit_speakers", "0"], ">= 1"),
                      (dset + ["-fit_steps", "5", "-fit_lr", "0"], "-fit_lr must be > 0"),
                      (dset + ["-fit_steps", "5", "-transcripts", "txt"], "needs -holdout_set"),
                      (wavs + ["-fit_steps", "5", "-holdout_set", "in_test"], "goes with -d")):
        with pytest.raises(SystemExit):
            cli.main(argv)
        assert msg in capsys.readouterr().err, argv
    p = cli.parser()
    cli.check_args(p, p.parse_args(dset + ["-fit_steps", "5", "-holdout_set", "in_test", "-transcripts", "t", "-report", "r"]))
    cli.check_args(p, p.parse_args(wavs + ["-fit_steps", "5", "-fit_lr", "1e-3", "-fit_crops", "4", "-fit_speakers", "2"]))
    cli.check_args(p, p.parse_args(dset))


def test_heldout_overlap_refused(tmp_path):
    import pickle
    import types
    cli = root_module("speaker_bank")
    names = ["p300", "p301"]
    utts = [["p300_001", "p300_002"], ["p301_001"]]
    bank = SB.SpeakerBank(names, torch.zeros(2, 4), [2, 1], utts, "f" * 64)
    with open(tmp_path / "in_test.pkl", "wb") as f:
        pickle.dump({"p300_009": np.zeros((5, 4), np.float32), "p301_001": np.zeros((5, 4), np.float32)}, f)
    args = types.SimpleNamespace(data_dir=str(tmp_path), holdout_set="in_test")
    with pytest.raises(SystemExit, match="held-out utterance"):
        cli.holdout_mels(args, bank, lambda u: u.split("_")[0])
    with open(tmp_path / "in_test.pkl", "wb") as f:
        pickle.dump({"p300_009": np.zeros((5, 4), np.float32), "p399_001": np.zeros((5, 4), np.float32)}, f)
    _, held = cli.holdout_mels(args, bank, lambda u: u.split("_")[0])
    assert list(held) == ["p300"] and list(held["p300"]) == ["p300_009"]


# ----------------------------------------------------------------------------- schedule
def test_wave_schedule():
    sp = [f"p{300 + i}" for i in range(7)]
    assert F.plan_waves(sp, 3) == [sp[0:3], sp[3:6], sp[6:7]]
    assert F.plan_waves(sp, 7) == [sp]
    assert F.plan_waves(sp, 100) == [sp]
    assert F.plan_waves(sp, 1) == [[s] for s in sp]
    assert F.plan_waves([], 4) == []
    with pytest.raises(ValueError, match=">= 1"):
        F.plan_waves(sp, 0)


def test_crop_order_is_per_speaker():
    m, steps, seed = 4, 9, 3
    n = {"p300": 10, "p301": 7, "p302": 13}
    alone = {s: F.speaker_order(k, m, steps, seed, s) for s, k in n.items()}
    # SegmentSampler(drop_last=True) of the speaker's own seed, one batch per step, across epoch boundaries
    for s, k in n.items():
        smp = SegmentSampler(k, m, seed=F.speaker_seed(seed, s), drop_last=True)
        want = np.stack([next(smp).numpy() for _ in range(steps)])
        assert np.array_equal(alone[s], want), s
        assert steps > smp.batches_per_epoch                      # the run crosses an epoch boundary
    assert F.speaker_seed(seed, "p300") != F.speaker_seed(seed, "p301") != F.speaker_seed(seed + 1, "p301")
    for names in (["p300", "p301", "p302"], ["p301", "p300"], ["p302", "p301"], ["p301"]):
        counts = [n[s] for s in names]
        tab = F.order_table(counts, m, steps, seed, names)
        assert tab.dtype == np.int32 and tab.shape == (steps * len(names) * m,)
        t = tab.reshape(steps, len(names), m)
        off = np.concatenate([[0], np.cumsum(counts)[:-1]])
        for i, s in enumerate(names):
            assert np.array_equal(t[:, i] - off[i], alone[s]), (names, s)


def test_unfitted_rule():
    lengths = {"a_1": 130, "a_2": 100, "b_1": 129, "c_1": 50, "c_2": 127, "d_1": 200}
    per, unfitted = F.plan(["a", "b", "c", "d"], [["a_1", "a_2"], ["b_1"], ["c_1", "c_2"], ["d_1"]], lengths, 128, 3)
    assert per["a"] == {"index": [("a_1", 0), ("a_1", 1), ("a_1", 2)], "used": ["a_1"], "skipped": ["a_2"], "n_crops": 3}
    assert per["b"]["n_crops"] == 2 and per["c"]["n_crops"] == 0 and per["c"]["skipped"] == ["c_1", "c_2"]
    assert per["d"]["n_crops"] == 73
    assert unfitted == ["b", "c"]                 # two crops < m = 3; no clip of segment_size frames


def test_report_schema():
    settings = {"steps": 3, "precision": "tf32"}
    sp = {"p300": {"fitted": True, "wave": 0, "clips": {"used": ["u"], "skipped": [], "n_crops": 9},
                   "losses": [{"step": 0, "loss_rec": 1.0, "grad_norm": 0.5}], "heldout": None, "extra": 1}}
    r = F.make_report(settings, ["p301"], sp, 1, 42, None)
    assert tuple(r) == F.REPORT_KEYS
    assert r["format"] == F.FORMAT and r["precision"] == "tf32" and r["unfitted"] == ["p301"] and r["n_waves"] == 1
    assert tuple(r["speakers"]["p300"]) == F.SPEAKER_KEYS
    import json
    assert json.loads(json.dumps(r)) == r


# ----------------------------------------------------------------------------- the fitted record
def test_fitted_record_and_old_banks(tmp_path):
    cfg = orc.default_config(80)
    model = cpu_model(cfg)
    fp, mf = SB.fingerprint(model), F.model_fingerprint(model)
    assert mf == F.model_fingerprint(cpu_model(cfg)) and len(mf) == 64
    g = torch.Generator().manual_seed(0)
    codes = torch.randn((2, cfg["SpeakerEncoder"]["c_out"]), generator=g)
    args = (["p300", "p301"], codes, [1, 1], [["p300_001"], ["p301_001"]], fp)
    # an old (unfitted) bank: the file holds exactly the keys it held before, and loads against any decoder
    old = str(tmp_path / "old.pt")
    SB.SpeakerBank(*args).save(old)
    raw = torch.load(old, weights_only=True)
    assert sorted(raw) == sorted(["format", "speakers", "codes", "n_utts", "utterances", "fingerprint", "n_skipped"])
    assert raw["format"] == SB.FORMAT == "avc-speaker-bank-1"
    changed = cpu_model(cfg)
    with torch.no_grad():
        next(changed.decoder.parameters()).view(-1)[0] += 1e-6
    for m in (model, changed):
        b = SB.SpeakerBank.load(old, m)
        assert b.fitted is None and torch.equal(b.codes, codes)
    # a fitted bank: loads against its model only
    rec = {"steps": 5, "lr": 1e-3, "model_fingerprint": mf, "fitted": ["p300"]}
    new = str(tmp_path / "fitted.pt")
    SB.SpeakerBank(*args, fitted=rec).save(new)
    raw = torch.load(new, weights_only=True)
    assert raw["format"] == SB.FORMAT and raw["fitted"] == rec
    back = SB.SpeakerBank.load(new, model)
    assert back.fitted == rec and torch.equal(back.codes, codes)
    assert F.model_fingerprint(changed) != mf
    with pytest.raises(ValueError, match="fitted to a different content encoder or decoder"):
        SB.SpeakerBank.load(new, changed)
    content = cpu_model(cfg)
    with torch.no_grad():
        next(content.content_encoder.parameters()).view(-1)[0] += 1e-6
    with pytest.raises(ValueError, match="fitted to a different"):
        SB.SpeakerBank.load(new, content)
    spk = cpu_model(cfg)
    with torch.no_grad():
        next(spk.speaker_encoder.parameters()).view(-1)[0] += 1e-6
    assert F.model_fingerprint(spk) == mf      # the speaker encoder is the bank fingerprint's business
    with pytest.raises(ValueError, match="model_fingerprint"):
        SB.SpeakerBank(*args, fitted={"steps": 1})


# ----------------------------------------------------------------------------- descriptors
@pytest.mark.parametrize("name,desc", [("avc_group_l1_desc", "GroupL1Desc"), ("avc_code_adam_desc", "CodeAdamDesc")])
def test_fit_descs_match_header(tmp_path, name, desc):
    cc = shutil.which("gcc") or shutil.which("cc")
    if cc is None:
        pytest.skip("no C compiler")
    D = getattr(L, desc)
    fields = [f for f, _ in D._fields_]
    src = tmp_path / "sz.c"
    src.write_text('#include <stdio.h>\n#include <stddef.h>\n#include "avc_b200.h"\nint main(void) {\n'
                   f'  printf("%zu %d", sizeof({name}), AVC_CODE_MAX_C);\n'
                   + "".join(f'  printf(" %zu", offsetof({name}, {f}));\n' for f in fields)
                   + "  return 0;\n}\n")
    exe = tmp_path / "sz"
    subprocess.run([cc, "-I", os.path.join(ROOT, "include"), str(src), "-o", str(exe)], check=True)
    got = [int(v) for v in subprocess.run([str(exe)], capture_output=True, text=True, check=True).stdout.split()]
    assert got == [C.sizeof(D), L.CODE_MAX_C] + [getattr(D, f).offset for f in fields]
