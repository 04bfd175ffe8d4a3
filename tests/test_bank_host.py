"""CPU: the host side of speaker banks.

* target specs: parsing, and SpeakerBank.code against a float64 restatement (one speaker: the stored bits);
* save / load round trip and the fingerprint refusal, on a CPU-built model;
* the evaluator's refusal of a bank that pooled evaluated utterances;
* build_bank's order (speakers sorted, utterances sorted, short ones skipped) and packing, through a recording model;
* inference.py's @SPEC pairs fields (a real file named @x stays a file) and argument errors of both CLIs;
* avc_spk_identify_desc: the header's layout against the ctypes mirror.
"""
import ctypes as C
import os
import shutil
import subprocess
import sys
import types

import numpy as np
import pytest
import torch

import oracle.ae_oracle as orc
from adaptive_voice_conversion_b200 import _lib as L
from adaptive_voice_conversion_b200 import speaker_bank as SB
from adaptive_voice_conversion_b200.inference import PADDED_BATCH_MAX, padded_extent
from adaptive_voice_conversion_b200.mcd import min_frames

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def root_module(name):
    if ROOT not in sys.path:
        sys.path.insert(0, ROOT)
    return __import__(name)


def small_bank(S=4, D=8, seed=0):
    g = torch.Generator().manual_seed(seed)
    names = [f"p{300 + s}" for s in range(S)]
    utts = [[f"{n}_{k:03d}" for k in range(s + 1)] for s, n in enumerate(names)]
    return SB.SpeakerBank(names, torch.randn((S, D), generator=g), [len(u) for u in utts], utts, "f" * 64)


# ----------------------------------------------------------------------------- specs and mixing
def test_parse_spec():
    assert SB.parse_spec("p225") == [("p225", 1.0)]
    assert SB.parse_spec("p225:0.7,p226:0.3") == [("p225", 0.7), ("p226", 0.3)]
    assert SB.parse_spec("p225:2, p226") == [("p225", 2.0), ("p226", 1.0)]
    for bad, msg in (("", "expected"), ("p1,p1", "named twice"), ("p1:-1", ">= 0"), ("p1:0,p2:0", "sum to 0"),
                     ("p1:x", "not a number"), ("p1:nan", "finite"), (":1", "empty"), ("p1:inf", "finite")):
        with pytest.raises(ValueError, match=msg):
            SB.parse_spec(bad)


def test_code_mixing_against_float64():
    bank = small_bank()
    for s, name in enumerate(bank.speakers):
        assert bank.code(name).numpy().tobytes() == bank.codes[s].numpy().tobytes()
        assert bank.code(f"{name}:0.37").numpy().tobytes() == bank.codes[s].numpy().tobytes()
    c = bank.codes.double().numpy()
    for spec, parts in (("p300:0.7,p301:0.3", [(0, 0.7), (1, 0.3)]), ("p303:1,p300:3,p302:0.5", [(3, 1), (0, 3), (2, 0.5)]),
                        ("p301:1e-3,p302:0", [(1, 1e-3), (2, 0.0)])):
        acc = np.zeros(c.shape[1])
        for r, w in parts:
            acc = acc + w * c[r]
        want = (acc / sum(w for _, w in parts)).astype(np.float32)
        got = bank.code(spec)
        assert got.dtype == torch.float32 and got.numpy().tobytes() == want.tobytes(), spec
    for bad, msg in (("p999", "not in the bank"), ("p300,p300", "twice"), ("p300:-0.5,p301", ">= 0"),
                     ("p300:0", "sum to 0")):
        with pytest.raises(ValueError, match=msg):
            bank.code(bad)


# ----------------------------------------------------------------------------- files and fingerprints
def cpu_model(cfg, seed=0):
    from adaptive_voice_conversion_b200.model import AE
    m = AE(cfg)
    m.load_state_dict(orc.init_state(cfg, seed=seed))
    return m


def test_save_load_and_fingerprint(tmp_path):
    cfg = orc.default_config(80)
    model = cpu_model(cfg)
    fp = SB.fingerprint(model)
    assert fp == SB.fingerprint(cpu_model(cfg)) and len(fp) == 64
    bank = small_bank(D=cfg["SpeakerEncoder"]["c_out"])
    bank = SB.SpeakerBank(bank.speakers, bank.codes, bank.n_utts, bank.utterances, fp, n_skipped=3)
    path = str(tmp_path / "bank.pt")
    bank.save(path)
    assert isinstance(torch.load(path, weights_only=True), dict)
    back = SB.SpeakerBank.load(path, model)
    assert back.speakers == bank.speakers and back.n_utts == bank.n_utts and back.utterances == bank.utterances
    assert back.n_skipped == 3 and back.fingerprint == fp and torch.equal(back.codes, bank.codes)
    # another speaker encoder: a changed weight, or a changed config
    other = cpu_model(cfg)
    with torch.no_grad():
        other.speaker_encoder.output_layer.bias[0] += 1e-6
    with pytest.raises(ValueError, match="different speaker encoder"):
        SB.SpeakerBank.load(path, other)
    assert SB.fingerprint(cpu_model(cfg, seed=1)) != fp
    # the decoder and content encoder do not enter the fingerprint
    same = cpu_model(cfg)
    with torch.no_grad():
        next(same.decoder.parameters()).add_(1.0)
    assert SB.fingerprint(same) == fp
    torch.save({"speakers": []}, str(tmp_path / "other.pt"))
    with pytest.raises(ValueError, match="not a speaker bank"):
        SB.SpeakerBank.load(str(tmp_path / "other.pt"), model)


def test_overlap_refused_before_any_work():
    bank = small_bank()
    data = {"p300_000": np.zeros((40, 80), np.float32), "p301_001": np.zeros((40, 80), np.float32),
            "p900_000": np.zeros((40, 80), np.float32)}
    with pytest.raises(ValueError, match="pooled 2 of the evaluated"):
        SB.check_disjoint(bank, data)
    SB.check_disjoint(bank, {"p900_000": None})
    from adaptive_voice_conversion_b200.speaker_eval import evaluate_speakers
    n0 = L.launch_count()
    with pytest.raises(ValueError, match="pooled 2 of the evaluated"):
        evaluate_speakers(cpu_model(orc.default_config(80)), data, bank=bank)
    assert L.launch_count() == n0


# ----------------------------------------------------------------------------- build order and packing
class RecordingModel(torch.nn.Module):
    """get_speaker_sums returns, per row, (utterance marker, valid length) so that the table can be read back."""

    def __init__(self, cfg):
        super().__init__()
        self.config = cfg
        self.speaker_encoder = torch.nn.Linear(2, 2)
        self.batches, self.calls = [], []

    def get_speaker_sums(self, x, *, lengths):
        B, Cc, T = x.shape
        assert B <= PADDED_BATCH_MAX and T == padded_extent(int(lengths.max()))
        self.batches.append((B, T))
        sums = torch.zeros(B, self.config["SpeakerEncoder"]["c_h"])
        sums[:, 0] = x[:, 0, 0]
        sums[:, 1] = lengths.float()
        return sums, lengths.clone()

    def speaker_codes_from_sums(self, sums, counts, *, groups):
        self.calls.append((sums.clone(), counts.clone(), groups.clone()))
        return torch.zeros(groups.shape[0] - 1, self.config["SpeakerEncoder"]["c_out"])

    def engine(self, dev):
        return types.SimpleNamespace(check_tc_status=lambda: None)


def test_build_order_and_packing():
    cfg = orc.default_config(80)
    min_ref = min_frames(cfg)[1]
    rng = np.random.default_rng(0)
    ids = [f"p{s}_{k:03d}" for s in (310, 301, 305) for k in rng.permutation(90)[:70]] + ["p200_000"]
    lens = {u: int(rng.integers(min_ref, 700)) for u in ids}
    lens["p200_000"] = min_ref - 1
    lens[ids[3]] = 1
    order = sorted(ids)
    marker = {u: float(i + 1) for i, u in enumerate(order)}
    mels = {u: torch.full((lens[u], 80), marker[u]) for u in reversed(ids)}
    m = RecordingModel(cfg)
    bank = SB.build_bank(m, mels, device="cpu")
    kept = [u for u in order if lens[u] >= min_ref]
    assert bank.speakers == ["p301", "p305", "p310"] and bank.n_skipped == 2
    assert bank.utterances == [[u for u in kept if u.startswith(s)] for s in bank.speakers]
    assert bank.n_utts == [len(u) for u in bank.utterances] and sum(bank.n_utts) == len(kept)
    (sums, counts, groups), = m.calls
    assert sums[:, 0].tolist() == [marker[u] for u in kept]                 # row r is kept[r]
    assert counts.tolist() == [lens[u] for u in kept]
    assert groups.dtype == torch.int64 and groups.tolist() == [0] + np.cumsum(bank.n_utts).tolist()
    assert len(m.batches) == -(-len(kept) // PADDED_BATCH_MAX)              # packed across speakers
    with pytest.raises(ValueError, match="no utterance"):
        SB.build_bank(RecordingModel(cfg), {"p1_000": torch.zeros(min_ref - 1, 80)}, device="cpu")


# ----------------------------------------------------------------------------- inference.py
def test_pairs_bank_fields(tmp_path, monkeypatch):
    inf = root_module("inference")
    monkeypatch.chdir(tmp_path)
    for f in ("s.npy", "@x.npy", "t.npy"):
        (tmp_path / f).write_bytes(b"")
    (tmp_path / "p.txt").write_text("s.npy @p225 o1.npy\ns.npy @p225:0.5,p226:0.5\ns.npy @x.npy\ns.npy t.npy\n")
    pairs = inf.read_pairs("p.txt", bank=True)
    assert isinstance(pairs[0][2], inf.BankTarget) and pairs[0][2].spec == "p225"
    assert pairs[1][2].spec == "p225:0.5,p226:0.5" and pairs[1][3] == "s_to_p225-0.5+p226-0.5.wav"
    assert pairs[2][2] == "@x.npy" and not isinstance(pairs[2][2], inf.BankTarget)    # a real file named @x
    assert pairs[3][2] == "t.npy"
    (tmp_path / "bad.txt").write_text("s.npy @p1,p1\n")
    with pytest.raises(ValueError, match="line 1: .*twice"):
        inf.read_pairs("bad.txt", bank=True)
    # without -bank an @ field is read as a path, as before
    (tmp_path / "q.txt").write_text("s.npy @p225\n")
    with pytest.raises(ValueError, match="@p225 is not an existing"):
        inf.read_pairs("q.txt")
    assert inf.read_pairs("q.txt", bank=True)[0][2].spec == "p225"


def test_inference_cli_argument_errors(tmp_path):
    inf = root_module("inference")
    p = inf.parser()
    for argv, msg in ((["-s", "a", "-o", "b"], "exactly one"), (["-s", "a", "-t", "x", "-bank", "k", "-speaker", "p1"], "exactly one"),
                      (["-s", "a", "-speaker", "p1"], "needs -bank"), (["-pairs", "f", "-bank", "k", "-speaker", "p1"], "@SPEC")):
        with pytest.raises(SystemExit):
            inf.check_args(p, p.parse_args(argv))
    inf.check_args(p, p.parse_args(["-s", "a", "-bank", "k", "-speaker", "p1:1,p2:1", "-o", "b"]))
    inf.check_args(p, p.parse_args(["-s", "a", "-t", "x", "y", "-o", "b"]))
    inf.check_args(p, p.parse_args(["-pairs", "f", "-bank", "k", "-o", "d"]))


def test_speaker_bank_cli_argument_errors(tmp_path, capsys):
    cli = root_module("speaker_bank")
    wav = tmp_path / "a.wav"
    wav.write_bytes(b"")
    base = ["-m", "m.ckpt", "-o", "b.pt"]
    for argv, msg in ((base, "either"), (base + ["-d", "data"], "go together"),
                      (base + ["-d", "data", "-set", "train", "-wav", "al", str(wav)], "either"),
                      (base + ["-wav", "al", str(wav)], "needs -a"), (base + ["-a", "x", "-wav", "al"], "at least one"),
                      (base + ["-a", "x", "-wav", "al", str(tmp_path / "none.wav")], "not a file"),
                      (base + ["-a", "x", "-wav", "al", str(wav), "-wav", "al", str(wav)], "named twice"),
                      (base + ["-a", "x", "-wav", "al", str(wav), "-speakers", "p1"], "-speakers")):
        with pytest.raises(SystemExit):
            cli.main(argv)
        assert msg in capsys.readouterr().err, argv


# ----------------------------------------------------------------------------- the descriptor
def test_identify_desc_matches_header(tmp_path):
    cc = shutil.which("gcc") or shutil.which("cc")
    if cc is None:
        pytest.skip("no C compiler")
    src = tmp_path / "sz.c"
    fields = [f for f, _ in L.SpkIdentifyDesc._fields_]
    src.write_text('#include <stdio.h>\n#include <stddef.h>\n#include "avc_b200.h"\nint main(void) {\n'
                   '  printf("%zu", sizeof(avc_spk_identify_desc));\n'
                   + "".join(f'  printf(" %zu", offsetof(avc_spk_identify_desc, {f}));\n' for f in fields)
                   + "  return 0;\n}\n")
    exe = tmp_path / "sz"
    subprocess.run([cc, "-I", os.path.join(ROOT, "include"), str(src), "-o", str(exe)], check=True)
    got = [int(v) for v in subprocess.run([str(exe)], capture_output=True, text=True, check=True).stdout.split()]
    assert got == [C.sizeof(L.SpkIdentifyDesc)] + [getattr(L.SpkIdentifyDesc, f).offset for f in fields]
