"""CPU: the host side of the MCD-DTW evaluation.  The float64 reference DTW against brute force over all monotone
paths; text normalisation; transcript discovery on VCTK- and LibriTTS-like trees; triplet selection against a literal
restatement; the shortest utterances AE.inference accepts; the CLI's flags and its output without -mcd; the
descriptor layouts; and the argument errors of the wrappers and of the two entry points."""
import ctypes
import io
import itertools
import json
import os
import random
import subprocess
import sys
from contextlib import redirect_stdout

import numpy as np
import pytest
import torch

from _mcd_ref import dist_rows, dtw64
from adaptive_voice_conversion_b200 import _lib as L
from adaptive_voice_conversion_b200 import mcd as M
from adaptive_voice_conversion_b200.config import default_config
from conftest import ROOT


# ----------------------------------------------------------------------------- the reference DTW
def brute_force(X, Y):
    """{S of every monotone path (steps (1,1), (1,0), (0,1)) from (0,0) to the corner: [its lengths]}."""
    Tx, Ty = len(X), len(Y)
    d = np.array([[dist_rows(X[i:i + 1], Y[j:j + 1])[0] for j in range(Ty)] for i in range(Tx)])
    out = {}

    def walk(i, j, s, n):
        if (i, j) == (Tx - 1, Ty - 1):
            out.setdefault(s, []).append(n)
            return
        for di, dj in ((1, 1), (1, 0), (0, 1)):
            if i + di < Tx and j + dj < Ty:
                walk(i + di, j + dj, s + d[i + di, j + dj], n + 1)
    walk(0, 0, d[0, 0], 1)
    return out


@pytest.mark.parametrize("Tx, Ty", [(1, 1), (1, 4), (4, 1), (2, 3), (3, 3), (5, 4), (4, 6), (5, 6)])
def test_reference_dtw_is_the_best_monotone_path(Tx, Ty):
    rng = np.random.default_rng(Tx * 10 + Ty)
    for dims in (1, 3):
        X = rng.standard_normal((Tx, dims)).astype(np.float32)
        Y = rng.standard_normal((Ty, dims)).astype(np.float32)
        S, Ln = dtw64(X, Y)
        paths = brute_force(X, Y)
        best = min(paths)
        assert abs(S - best) <= 1e-12 * max(1.0, best)
        assert Ln in {n for s, ns in paths.items() if abs(s - best) <= 1e-12 * max(1.0, best) for n in ns}


def test_reference_dtw_breaks_ties_towards_the_diagonal():
    # every distance is 0: every path costs 0, the diagonal-first rule gives the shortest path, max(Tx, Ty) cells
    for Tx, Ty in [(3, 3), (2, 5), (5, 2)]:
        assert dtw64(np.zeros((Tx, 2), np.float32), np.zeros((Ty, 2), np.float32)) == (0.0, max(Tx, Ty))
    # a sequence against itself with every frame doubled: S = 0 and the path visits all 2T cells of the copy
    X = np.random.default_rng(0).standard_normal((7, 4)).astype(np.float32)
    assert dtw64(X, np.repeat(X, 2, axis=0)) == (0.0, 14)


# ----------------------------------------------------------------------------- transcripts
def test_normalize_text():
    assert M.normalize_text("Please call Stella.") == "please call stella"
    assert M.normalize_text("  It's 5 o'clock -- \"NOW\"!\n") == "it's 5 o'clock now"
    assert M.normalize_text("Ask her to bring these things\twith her from the store.") == \
        "ask her to bring these things with her from the store"
    assert M.normalize_text("...?!") == "" and M.normalize_text("") == ""
    assert M.normalize_text("Café-au-lait") == "caf au lait"


def write(path, text):
    os.makedirs(os.path.dirname(path), exist_ok=True)
    with open(path, "w") as f:
        f.write(text)


def test_read_transcripts_vctk_tree(tmp_path):
    root = tmp_path / "txt"
    write(root / "p225" / "p225_001.txt", "Please call Stella.\n")
    write(root / "p225" / "p225_002.txt", "Ask her to bring these things.\n")
    write(root / "p226" / "p226_001.txt", "PLEASE call Stella!\n")
    write(root / "p226" / "p226_003.txt", "   \n")                     # empty after normalisation: dropped
    write(root / "p227" / "p227_009.txt", "Not in the set.\n")
    write(root / "p226" / "notes.md", "ignored")
    keys = ["p225_001.wav", "p225_002.wav", "p226_001.wav", "p226_003.wav", "p315_001.wav"]
    got = M.read_transcripts(str(root), keys)
    assert got == {"p225_001.wav": "please call stella", "p225_002.wav": "ask her to bring these things",
                   "p226_001.wav": "please call stella"}


def test_read_transcripts_libritts_tree(tmp_path):
    root = tmp_path / "LibriTTS"
    base = root / "dev-clean" / "84" / "121123"
    write(base / "84_121123_000007_000001.normalized.txt", "Go, do you hear?")
    write(base / "84_121123_000007_000001.original.txt", "Go! do you hear?!! (different)")
    write(base / "84_121123_000008_000000.normalized.txt", "But in less than five minutes.")
    write(base / "84_121123.book.tsv", "84_121123_000007_000001\tGo, do you hear?\n")
    write(base / "84_121123.trans.tsv", "x")
    keys = ["84_121123_000007_000001.wav", "84_121123_000008_000000.wav"]
    got = M.read_transcripts(str(root), keys)
    assert got == {"84_121123_000007_000001.wav": "go do you hear", "84_121123_000008_000000.wav": "but in less than five minutes"}


def test_read_transcripts_rejects_conflicting_files(tmp_path):
    root = tmp_path / "txt"
    write(root / "a" / "p225_001.txt", "Please call Stella.")
    write(root / "b" / "p225_001.txt", "please, call stella")          # the same text: accepted
    assert M.read_transcripts(str(root), ["p225_001.wav"]) == {"p225_001.wav": "please call stella"}
    write(root / "c" / "p225_001.txt", "Something else.")
    with pytest.raises(ValueError) as e:
        M.read_transcripts(str(root), ["p225_001.wav"])
    assert os.path.join("a", "p225_001.txt") in str(e.value) and os.path.join("c", "p225_001.txt") in str(e.value)
    with pytest.raises(ValueError, match="does not exist"):
        M.read_transcripts(str(tmp_path / "nope"), ["p225_001.wav"])


# ----------------------------------------------------------------------------- triplets
def literal_triplets(utts, texts, lengths, seed, max_pairs, min_src, min_ref):
    rng = random.Random(seed)
    spk = lambda u: u.split("_")[0]
    utts = sorted(utts)
    groups = sorted({texts[u] for u in utts if texts.get(u)})
    trip, n_short = [], 0
    for t in groups:
        speakers = sorted({spk(u) for u in utts if texts.get(u) == t})
        if len(speakers) < 2:
            continue
        first = {s: min(u for u in utts if texts.get(u) == t and spk(u) == s) for s in speakers}
        for a, b in itertools.permutations(speakers, 2):
            cands = [u for u in utts if spk(u) == b and texts.get(u) != t]
            if not cands:
                continue
            ref = rng.choice(cands)
            if lengths[first[a]] < min_src or lengths[ref] < min_ref:
                n_short += 1
            else:
                trip.append((first[a], ref, first[b]))
    if max_pairs > 0 and len(trip) > max_pairs:
        trip = [trip[i] for i in sorted(rng.sample(range(len(trip)), max_pairs))]
    return trip, n_short


def random_set(seed, n_speakers=6, n_sent=8, p_read=0.6, p_text=0.9):
    rng = np.random.default_rng(seed)
    utts, texts, lengths = [], {}, {}
    for s in range(n_speakers):
        for k in range(n_sent + 3):
            if rng.random() > p_read:
                continue
            u = f"p{225 + s}_{k:03d}.wav"
            utts.append(u)
            lengths[u] = int(rng.integers(5, 60))
            if rng.random() < p_text:
                texts[u] = f"sentence {k % n_sent}" if k < n_sent else f"own line {s} {k}"
    return utts, texts, lengths


@pytest.mark.parametrize("seed", range(6))
@pytest.mark.parametrize("max_pairs", [0, 1, 7])
def test_triplets_match_a_literal_restatement(seed, max_pairs):
    utts, texts, lengths = random_set(seed)
    shuffled = list(utts)
    random.Random(seed).shuffle(shuffled)
    got = M.parallel_triplets(shuffled, texts, lengths, seed, max_pairs, 17, 9)
    assert got == literal_triplets(utts, texts, lengths, seed, max_pairs, 17, 9)
    assert got == M.parallel_triplets(utts, texts, lengths, seed, max_pairs, 17, 9)        # deterministic
    trip, n_short = got
    if max_pairs:
        assert len(trip) <= max_pairs
    for s, r, g in trip:
        assert s.split("_")[0] != g.split("_")[0] and r.split("_")[0] == g.split("_")[0]
        assert texts[s] == texts[g] and texts.get(r) != texts[g]
        assert lengths[s] >= 17 and lengths[r] >= 9


def test_triplet_rules_on_a_small_set():
    texts = {"p1_001.wav": "hello there", "p2_001.wav": "hello there", "p2_002.wav": "other",
             "p3_001.wav": "hello there", "p3_005.wav": "hello there"}
    utts = sorted(texts) + ["p1_009.wav"]          # p1_009 has no transcript: it may be p1's reference
    lengths = {u: 100 for u in utts}
    trip, n_short = M.parallel_triplets(utts, texts, lengths, 0, 0, 17, 9)
    # p3 has no utterance of another text: every pair with B = p3 is skipped; p3_001 (first id) is p3's source
    assert [(s, g) for s, _, g in trip] == [("p1_001.wav", "p2_001.wav"), ("p2_001.wav", "p1_001.wav"),
                                           ("p3_001.wav", "p1_001.wav"), ("p3_001.wav", "p2_001.wav")]
    assert [r for _, r, _ in trip] == ["p2_002.wav", "p1_009.wav", "p1_009.wav", "p2_002.wav"] and n_short == 0
    lengths["p1_009.wav"] = 8                      # a reference below 9 frames drops the two triplets that use it
    lengths["p3_001.wav"] = 16                     # a source below 17 frames too
    trip2, n_short2 = M.parallel_triplets(utts, texts, lengths, 0, 0, 17, 9)
    assert [(s, g) for s, _, g in trip2] == [("p1_001.wav", "p2_001.wav")] and n_short2 == 3
    assert M.parallel_triplets(["p1_001.wav", "p1_002.wav"], {"p1_001.wav": "a", "p1_002.wav": "a"},
                               {"p1_001.wav": 50, "p1_002.wav": 50}) == ([], 0)        # one speaker: no group


def test_min_frames_of_the_shipped_config():
    from adaptive_voice_conversion_b200.config import load_config
    assert M.min_frames(load_config(os.path.join(ROOT, "config.yaml"))) == (17, 9)
    assert M.min_frames(default_config(80)) == (17, 9)
    cfg = default_config(80)
    cfg["ContentEncoder"]["subsample"] = [1, 1, 1, 1, 1, 1]
    cfg["Decoder"]["upsample"] = [1, 1, 1, 1, 1, 1]
    assert M.min_frames(cfg)[0] == 5               # the bank's kernel of 8 pads 4 on the left


def test_dct_rows_are_orthonormal():
    D = M.dct_matrix(512, 64)
    assert np.allclose(D.T @ D, np.eye(64), atol=1e-12)
    assert np.allclose(D.sum(axis=0), 0.0, atol=1e-12)          # no c_0: a constant log-mel has no cepstrum


# ----------------------------------------------------------------------------- the CLI
def cli():
    sys.path.insert(0, ROOT)
    import evaluate as cli_mod
    return cli_mod


def test_cli_needs_transcripts_with_mcd(capsys):
    with pytest.raises(SystemExit):
        cli().main(["-m", "x.ckpt", "-d", "data", "-mcd"])
    assert "-transcripts" in capsys.readouterr().err


def fake_run(monkeypatch, argv):
    mod = cli()
    res = {"in_test": {"loss_rec": 0.25, "loss_kl": 1.5, "n": 3, "speakers": {"p1": {}, "p2": {}}},
           "out_test": {"loss_rec": 0.125, "loss_kl": 2.0, "n": 2, "speakers": {"p3": {}}}}
    calls = []

    class FakeModel:
        def to(self, dev):
            return self

        def load_state_dict(self, sd, strict):
            calls.append(("load", strict))

        def eval(self):
            calls.append("eval")

    class FakeHeld:
        def __init__(self, sets, data_dir, config, device=None):
            calls.append(("held", sets, data_dir))

        def evaluate(self, model, per_speaker=False):
            return json.loads(json.dumps(res))
    monkeypatch.setattr(mod, "AE", lambda cfg: FakeModel())
    monkeypatch.setattr(mod, "HeldOut", FakeHeld)
    monkeypatch.setattr(mod, "local_device", lambda: torch.device("cpu"))
    monkeypatch.setattr(mod.torch, "load", lambda path, map_location=None: {})
    out = io.StringIO()
    with redirect_stdout(out):
        got = mod.main(argv)
    return got, out.getvalue(), calls, res


def test_cli_output_without_mcd_is_unchanged(monkeypatch, tmp_path):
    o = tmp_path / "eval.json"
    got, text, calls, res = fake_run(monkeypatch, ["-c", os.path.join(ROOT, "config.yaml"), "-m", "m.ckpt", "-d", "data",
                                                    "-o", str(o)])
    assert text == ("in_test: n=3 loss_rec=0.250000 loss_kl=1.500000 (2 speakers)\n"
                    "out_test: n=2 loss_rec=0.125000 loss_kl=2.000000 (1 speakers)\n")
    assert got == res and json.loads(o.read_text()) == res
    assert o.read_text() == json.dumps(res, indent=1)
    assert ("held", ["in_test", "out_test"], "data") in calls and ("load", True) in calls


def test_cli_mcd_flags_reach_evaluate_mcd(monkeypatch, tmp_path):
    import pickle
    d = tmp_path / "data"
    d.mkdir()
    for s, u in (("in_test", "p1_001.wav"), ("out_test", "p1_002.wav")):
        with open(d / f"{s}.pkl", "wb") as f:
            pickle.dump({u: np.zeros((20, 4), np.float32)}, f)
    with open(tmp_path / "attr.pkl", "wb") as f:
        pickle.dump({"mean": np.zeros(4, np.float32), "std": np.ones(4, np.float32)}, f)
    write(tmp_path / "txt" / "p1" / "p1_001.txt", "Hello.")
    seen = []

    def fake_mcd(model, data, attr, texts, dims, max_pairs, seed, device):
        seen.append((sorted(data), sorted(attr), texts, dims, max_pairs, seed))
        if "p1_001.wav" in data:
            return {"n": 0, "n_short": 0, "dims": dims, "speakers": {}}
        return {"n": 2, "n_short": 1, "dims": dims, "mcd": 7.5, "mcd_source": 9.25, "speakers": {"p1": {}}}
    monkeypatch.setattr(M, "evaluate_mcd", fake_mcd)
    o = tmp_path / "eval.json"
    got, text, _, _ = fake_run(monkeypatch, ["-c", os.path.join(ROOT, "config.yaml"), "-m", "m.ckpt", "-d", str(d),
                                             "-mcd", "-transcripts", str(tmp_path / "txt"), "-attr", str(tmp_path / "attr.pkl"),
                                             "-mcd_dims", "13", "-max_pairs", "5", "-seed", "3", "-o", str(o)])
    lines = text.splitlines()
    assert lines[2] == "in_test: mcd n=0 n_short=0 (dims 13, 0 target speakers)"
    assert lines[3] == "out_test: mcd n=2 n_short=1 mcd=7.5000 mcd_source=9.2500 (dims 13, 1 target speakers)"
    assert seen[0] == (["p1_001.wav"], ["mean", "std"], {"p1_001.wav": "hello"}, 13, 5, 3)
    assert seen[1][2] == {}
    assert json.loads(o.read_text())["out_test"]["mcd"]["mcd"] == 7.5
    assert got["in_test"]["mcd"] == {"n": 0, "n_short": 0, "dims": 13, "speakers": {}}


# ----------------------------------------------------------------------------- the C ABI
def test_descriptor_layouts_match_the_header(tmp_path):
    c = tmp_path / "s.c"
    c.write_text('#include <stdio.h>\n#include <stddef.h>\n#include "avc_b200.h"\nint main(){printf("%zu %zu %zu %zu %zu %zu '
                 '%zu %zu %zu %d %d %d\\n", sizeof(avc_cepstrum_desc), offsetof(avc_cepstrum_desc, in), '
                 'offsetof(avc_cepstrum_desc, out), sizeof(avc_dtw_pair), offsetof(avc_dtw_pair, tx), sizeof(avc_dtw_desc), '
                 'offsetof(avc_dtw_desc, pairs), offsetof(avc_dtw_desc, out), offsetof(avc_cepstrum_desc, max_db), '
                 'AVC_CEPSTRUM_MAX_DIMS, AVC_CEPSTRUM_MAX_MELS, AVC_DTW_MAX_SHORT);return 0;}\n')
    subprocess.check_call(["gcc", "-I", os.path.join(ROOT, "include"), str(c), "-o", str(tmp_path / "s")])
    got = [int(v) for v in subprocess.check_output([str(tmp_path / "s")]).split()]
    assert got == [ctypes.sizeof(L.CepstrumDesc), L.CepstrumDesc.in_.offset, L.CepstrumDesc.out.offset,
                   ctypes.sizeof(L.DtwPair), L.DtwPair.tx.offset, ctypes.sizeof(L.DtwDesc), L.DtwDesc.pairs.offset,
                   L.DtwDesc.out.offset, L.CepstrumDesc.max_db.offset, L.CEPSTRUM_MAX_DIMS, L.CEPSTRUM_MAX_MELS,
                   L.DTW_MAX_SHORT]


def test_entry_points_reject_invalid_arguments_without_a_device():
    lib = L.load()
    fake = 0x10000     # never dereferenced: every case fails validation before a launch
    cep = dict(rows=10, n_mels=80, dims=24, max_db=100.0, ref_db=20.0, in_=fake, mean=fake, std=fake, dct=fake, out=fake)
    cases = [({"in_": None}, L.ERR_INVALID, "null pointer"), ({"mean": None}, L.ERR_INVALID, "null pointer"),
             ({"std": None}, L.ERR_INVALID, "null pointer"), ({"dct": None}, L.ERR_INVALID, "null pointer"),
             ({"out": None}, L.ERR_INVALID, "null pointer"), ({"rows": 0}, L.ERR_INVALID, "positive"),
             ({"n_mels": -1}, L.ERR_INVALID, "positive"), ({"dims": 0}, L.ERR_INVALID, "positive"),
             ({"dims": 65}, L.ERR_UNSUPPORTED, "dims 65"), ({"n_mels": 4097}, L.ERR_UNSUPPORTED, "n_mels 4097")]
    n0 = L.launch_count()
    for patch, rc, msg in cases:
        assert lib.avc_mel_cepstrum(L.CepstrumDesc(**{**cep, **patch}), None) == rc, patch
        assert msg in L.last_error(), (patch, L.last_error())
    dtw = dict(n_pairs=3, dims=24, max_short=100, pairs=fake, x=fake, y=fake, out=fake)
    cases = [({"pairs": None}, L.ERR_INVALID, "null pointer"), ({"x": None}, L.ERR_INVALID, "null pointer"),
             ({"y": None}, L.ERR_INVALID, "null pointer"), ({"out": None}, L.ERR_INVALID, "null pointer"),
             ({"n_pairs": 0}, L.ERR_INVALID, "positive"), ({"dims": 0}, L.ERR_INVALID, "positive"),
             ({"max_short": 0}, L.ERR_INVALID, "positive"), ({"dims": 65}, L.ERR_UNSUPPORTED, "dims 65"),
             ({"max_short": 4097}, L.ERR_UNSUPPORTED, "4097 frames")]
    for patch, rc, msg in cases:
        assert lib.avc_dtw(L.DtwDesc(**{**dtw, **patch}), None) == rc, patch
        assert msg in L.last_error(), (patch, L.last_error())
    assert lib.avc_mel_cepstrum(None, None) == L.ERR_INVALID and "null descriptor" in L.last_error()
    assert lib.avc_dtw(None, None) == L.ERR_INVALID and "null descriptor" in L.last_error()
    assert L.launch_count() == n0


def test_wrappers_reject_bad_arguments_before_a_launch():
    attr = {"mean": np.zeros(80, np.float32), "std": np.ones(80, np.float32)}
    x = torch.zeros(10, 80)
    with pytest.raises(ValueError, match="dims"):
        M.mel_cepstrum([x], attr, dims=0)
    with pytest.raises(ValueError, match="dims"):
        M.mel_cepstrum([x], attr, dims=65)
    with pytest.raises(ValueError, match="empty"):
        M.mel_cepstrum([], attr)
    with pytest.raises(ValueError, match="CUDA"):
        M.mel_cepstrum([x], attr)
    c = torch.zeros(10, 24)
    with pytest.raises(ValueError, match="equally long"):
        M.dtw([c], [])
    with pytest.raises(ValueError, match="dims"):
        M.dtw([torch.zeros(3, 65)], [torch.zeros(3, 65)])
    with pytest.raises(ValueError, match="CUDA"):
        M.dtw([c], [c])
    with pytest.raises(ValueError, match="float32"):
        M.dtw([c], [torch.zeros(10, 13)])
    from adaptive_voice_conversion_b200.model import AE
    cfg = default_config(80)
    cfg["data_loader"]["frame_size"] = 2
    with pytest.raises(ValueError, match="frame_size"):
        M.evaluate_mcd(AE(cfg), {}, attr, {})
