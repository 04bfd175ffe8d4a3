"""CPU: the host side of the speaker measures.  The EER restatement against brute force over every threshold (heavy
ties, all-equal scores, one speaker, two utterances), and the counting search the kernel runs against both; pooling
and scores against literal loops; the conversion-pair rules against a literal restatement; the CLI's -spk output and
its output without -spk; the descriptor layouts; and the argument errors of the wrappers and the entry points."""
import ctypes
import json
import math
import os
import subprocess

import numpy as np
import pytest
import torch

import _spk_ref as R
from adaptive_voice_conversion_b200 import _lib as L
from adaptive_voice_conversion_b200 import speaker_eval as S
from adaptive_voice_conversion_b200.config import default_config
from adaptive_voice_conversion_b200.evaluate import speaker_of
from conftest import ROOT
from test_mcd_host import fake_run


# ----------------------------------------------------------------------------- the EER
def score_cases():
    rng = np.random.default_rng(0)
    for it in range(300):
        n = int(rng.integers(2, 30))
        kind = it % 6
        if kind == 0:
            s = rng.standard_normal(n)
        elif kind == 1:                       # heavy ties
            s = rng.integers(-2, 3, n) / 2.0
        elif kind == 2:                       # all equal
            s = np.full(n, 0.25)
        elif kind == 3:                       # +0 and -0 are one score
            s = np.where(rng.random(n) < 0.5, -0.0, 0.0)
        elif kind == 4:                       # tiny and negative
            s = rng.integers(0, 3, n) * 1e-300 - 1e-300
        else:                                 # targets all below the non-targets
            s = np.arange(n, dtype=np.float64)
        t = rng.random(n) < (rng.random() if kind != 5 else 2.0)
        if kind == 5:
            t = np.arange(n) < n // 2
        yield s, t


def test_eer_restatement_is_brute_force_over_every_threshold():
    for s, t in score_cases():
        assert R.eer64(s, t) == R.eer_brute(s, t), (s, t)


def test_counting_search_is_the_restatement():
    for s, t in score_cases():
        assert R.eer_by_counting(s, t) == R.eer64(s, t), (s, t)


def test_eer_edge_cases():
    # one speaker: no non-target trial
    S1 = R.scores64(np.random.default_rng(1).standard_normal((5, 4)).astype(np.float32))
    assert R.eer64(*R.trials(S1, [7] * 5)) == {"eer": None, "threshold": None, "frr": None, "far": None,
                                               "n_target": 10, "n_nontarget": 0}
    # two utterances: one trial
    assert R.eer_brute([0.5], [True])["eer"] is None and R.eer_brute([0.5], [False])["n_nontarget"] == 1
    # perfect separation: EER 0 at the smallest target score
    r = R.eer64([0.9, 0.8, 0.1, 0.2], [True, True, False, False])
    assert r == R.eer_brute([0.9, 0.8, 0.1, 0.2], [True, True, False, False])
    assert r["eer"] == 0.0 and r["threshold"] == 0.8
    # all scores equal: FRR 0 and FAR 1 at that score, FRR 1 at +inf; the smaller threshold wins
    r = R.eer64([0.3] * 6, [True, False] * 3)
    assert r["eer"] == 1.0 and r["threshold"] == 0.3 and r["frr"] == 0.0 and r["far"] == 1.0


def test_score_keys_preserve_order():
    s = np.array([-np.inf, -1.0, -1e-300, -0.0, 0.0, 1e-300, 0.5, 1.0, np.inf])
    k = R.score_keys(s)
    assert (np.diff(k[[0, 1, 2, 4, 5, 6, 7, 8]].astype(object)) > 0).all() and k[3] == k[4]
    assert (R.key_scores(k)[[0, 1, 2, 4, 5, 6, 7, 8]] == s[[0, 1, 2, 4, 5, 6, 7, 8]]).all()


# ----------------------------------------------------------------------------- pooling and scores
def test_pooling_restatement_is_a_literal_loop():
    rng = np.random.default_rng(2)
    x = (rng.standard_normal((3, 11)) * 4 + 1).astype(np.float32)
    for L_ in (1, 2, 7, 11):
        got = R.pool64(x, L_)
        for c in range(3):
            s = 0.0
            for t in range(L_):
                s += float(x[c, t])
            mean = s / L_
            v = 0.0
            for t in range(L_):
                v += (float(x[c, t]) - mean) ** 2
            assert got[c] == np.float32(mean) and got[3 + c] == np.float32(math.sqrt(v / L_))
    # NaN past the length is never read
    xn = x.copy()
    xn[:, 7:] = np.nan
    assert (R.pool64(xn, 7) == R.pool64(x, 7)).all()


def test_score_restatement_is_a_literal_loop_and_symmetric():
    rng = np.random.default_rng(3)
    V = rng.standard_normal((6, 5)).astype(np.float32)
    V[2] = 0.0                         # zero vector: score 0
    V[4] = V[1]                        # duplicate
    S_ = R.scores64(V)
    for i in range(6):
        for j in range(6):
            dot = na = nb = 0.0
            for k in range(5):
                dot += float(V[i, k]) * float(V[j, k])
                na += float(V[i, k]) * float(V[i, k])
                nb += float(V[j, k]) * float(V[j, k])
            ref = 0.0 if na == 0 or nb == 0 else dot / (math.sqrt(na) * math.sqrt(nb))
            assert S_[i, j] == ref and S_[i, j] == S_[j, i]
    assert S_[1, 4] == S_[1, 1]
    # group mean: ascending v over the label, the excluded index skipped
    lab = [0, 1, 0, 1, 1, 0]
    got = R.group_mean64(V[0], 1, 3, V, lab)
    assert got == (S_[0, 1] + S_[0, 4]) / 2
    assert math.isnan(R.group_mean64(V[0], 2, -1, V, lab))


# ----------------------------------------------------------------------------- conversion pairs
def make_utts(rng, n_spk, lone=2):
    utts, lengths = [], {}
    for s in range(n_spk):
        for k in range(int(rng.integers(2, 7))):
            utts.append(f"p{300 + s}_{k:03d}.wav")
    for s in range(lone):                       # speakers with one utterance
        utts.append(f"p{400 + s}_001.wav")
    utts.append("p30_001.wav")                  # sorts between p300_* and p301_* keys, its own speaker
    for u in utts:
        lengths[u] = int(rng.choice([5, 12, 17, 40, 300]))
    return utts, lengths


@pytest.mark.parametrize("seed", [0, 1, 2, 7, 123])
def test_pairs_follow_the_literal_rules(seed):
    rng = np.random.default_rng(seed)
    utts, lengths = make_utts(rng, 5)
    rng.shuffle(utts)
    for max_pairs in (0, 3, 1000):
        for mins in ((1, 1, 1), (17, 9, 17), (40, 17, 40)):
            got = S.conversion_pairs(utts, lengths, seed, max_pairs, *mins)
            ref = R.pairs_literal(utts, lengths, seed, max_pairs, *mins, speaker_of)
            assert got == ref, (max_pairs, mins)
    pairs, n_short = S.conversion_pairs(utts, lengths, seed, 0, 17, 9, 17)
    for u, r in pairs:
        assert speaker_of(u) != speaker_of(r) and not speaker_of(u).startswith("p4")
    capped, _ = S.conversion_pairs(utts, lengths, seed, 3, 17, 9, 17)
    assert len(capped) == min(3, len(pairs)) and set(capped) <= set(pairs)


def test_pairs_of_one_speaker_or_none():
    one = ["p1_001.wav", "p1_002.wav", "p2_001.wav"]
    assert S.conversion_pairs(one, {u: 50 for u in one}) == ([], 0)
    assert S.conversion_pairs([], {}) == ([], 0)


# ----------------------------------------------------------------------------- the CLI
CLI_BASE = ["-c", os.path.join(ROOT, "config.yaml"), "-m", "m.ckpt"]


def test_cli_output_without_spk_is_unchanged(monkeypatch, tmp_path):
    o = tmp_path / "eval.json"
    got, text, _, res = fake_run(monkeypatch, CLI_BASE + ["-d", "data", "-o", str(o), "-seed", "4", "-max_pairs", "2"])
    assert text == ("in_test: n=3 loss_rec=0.250000 loss_kl=1.500000 (2 speakers)\n"
                    "out_test: n=2 loss_rec=0.125000 loss_kl=2.000000 (1 speakers)\n")
    assert got == res and o.read_text() == json.dumps(res, indent=1)


def test_cli_spk_flags_reach_evaluate_speakers(monkeypatch, tmp_path):
    import pickle
    d = tmp_path / "data"
    d.mkdir()
    for s, u in (("in_test", "p1_001.wav"), ("out_test", "p1_002.wav")):
        with open(d / f"{s}.pkl", "wb") as f:
            pickle.dump({u: np.zeros((20, 4), np.float32)}, f)
    seen = []
    null = {"eer": None, "threshold": None, "frr": None, "far": None, "n_target": 0, "n_nontarget": 0}

    def fake_spk(model, data, seed, max_pairs, device):
        seen.append((sorted(data), seed, max_pairs))
        if "p1_001.wav" in data:
            return {"eer": {k: null for k in S.REPRESENTATIONS}, "n_utts": 1, "n_short": 0,
                    "conversion": {"n": 0, "n_short": 0, "speakers": {}}}
        e = {"eer": 0.125, "threshold": 0.5, "frr": 0.125, "far": 0.0625, "n_target": 8, "n_nontarget": 16}
        return {"eer": {"speaker": e, "content": {**e, "eer": 0.4375}, "mel": {**e, "eer": 0.25}}, "n_utts": 7, "n_short": 1,
                "conversion": {"sim_target": 0.5, "sim_source": 0.25, "success": 0.75, "sim_target_source": -0.125, "n": 4,
                               "n_short": 2, "speakers": {"p1": {}, "p2": {}}}}
    monkeypatch.setattr(S, "evaluate_speakers", fake_spk)
    o = tmp_path / "eval.json"
    got, text, _, _ = fake_run(monkeypatch, CLI_BASE + ["-d", str(d), "-spk", "-max_pairs", "5", "-seed", "3", "-o", str(o)])
    lines = text.splitlines()
    assert lines[2:] == [
        "in_test: spk eer speaker=n/a content=n/a mel=n/a (n_utts=1 n_short=0)",
        "in_test: spk conversion n=0 n_short=0 (0 target speakers)",
        "out_test: spk eer speaker=0.1250 content=0.4375 mel=0.2500 (n_utts=7 n_short=1)",
        "out_test: spk conversion n=4 n_short=2 sim_target=0.5000 sim_source=0.2500 success=0.7500 "
        "sim_target_source=-0.1250 (2 target speakers)"]
    assert seen == [(["p1_001.wav"], 3, 5), (["p1_002.wav"], 3, 5)]
    saved = json.loads(o.read_text())
    assert saved["out_test"]["spk"]["eer"]["content"]["eer"] == 0.4375 and saved["in_test"]["spk"]["eer"]["mel"] == null
    assert got["out_test"]["spk"]["conversion"]["n"] == 4 and "mcd" not in got["out_test"]


def test_cli_help_names_spk(capsys):
    from test_mcd_host import cli
    with pytest.raises(SystemExit):
        cli().main(["-h"])
    out = " ".join(capsys.readouterr().out.split())
    assert "-spk" in out and "conversion pairs (-spk)" in out and "(-mcd, -spk)" in out


# ----------------------------------------------------------------------------- the C ABI
def test_descriptor_layouts_match_the_header(tmp_path):
    c = tmp_path / "s.c"
    c.write_text('#include <stdio.h>\n#include <stddef.h>\n#include "avc_b200.h"\nint main(){printf("%zu %zu %zu %zu %zu '
                 '%zu %d %d %d\\n", sizeof(avc_eer_result), offsetof(avc_eer_result, n_target), sizeof(avc_spk_group_desc), '
                 'offsetof(avc_spk_group_desc, queries), offsetof(avc_spk_group_desc, set), offsetof(avc_spk_group_desc, out), '
                 'AVC_SPK_MAX_N, AVC_SPK_MAX_DIMS, AVC_SPK_STATE_BYTES);return 0;}\n')
    subprocess.check_call(["gcc", "-I", os.path.join(ROOT, "include"), str(c), "-o", str(tmp_path / "s")])
    got = [int(v) for v in subprocess.check_output([str(tmp_path / "s")]).split()]
    assert got == [ctypes.sizeof(L.EerResult), L.EerResult.n_target.offset, ctypes.sizeof(L.SpkGroupDesc),
                   L.SpkGroupDesc.queries.offset, L.SpkGroupDesc.set.offset, L.SpkGroupDesc.out.offset,
                   L.SPK_MAX_N, L.SPK_MAX_DIMS, L.SPK_STATE_BYTES]


def test_workspace_bytes():
    lib = L.load()
    for n in (1, 64, 65, 8000, 32768):
        nt = -(-n // 64)
        assert lib.avc_spk_eer_workspace_bytes(n) == 65536 + -(-8 * n // 256) * 256 + nt * (nt + 1) // 2 * 4096 * 8
    assert lib.avc_spk_eer_workspace_bytes(0) == -1 and lib.avc_spk_eer_workspace_bytes(32769) == -1


def test_entry_points_reject_invalid_arguments_without_a_device():
    lib = L.load()
    fake = 0x10000     # never dereferenced: every case fails validation before a launch
    n0 = L.launch_count()
    cases = [((None, fake, 2, 3, 4, fake), "null pointer"), ((fake, None, 2, 3, 4, fake), "null pointer"),
             ((fake, fake, 2, 3, 4, None), "null pointer"), ((fake, fake, 0, 3, 4, fake), "positive"),
             ((fake, fake, 2, -3, 4, fake), "positive"), ((fake, fake, 2, 3, 0, fake), "positive")]
    for args, msg in cases:
        assert lib.avc_time_stats_varlen(*args, None) == L.ERR_INVALID, args
        assert msg in L.last_error(), (args, L.last_error())
    need = lib.avc_spk_eer_workspace_bytes(100)
    eer = dict(vecs=fake, labels=fake, n=100, dims=128, ws=fake * 256, wsb=need, out=fake)
    cases = [({"vecs": None}, L.ERR_INVALID, "null pointer"), ({"labels": None}, L.ERR_INVALID, "null pointer"),
             ({"ws": None}, L.ERR_INVALID, "null pointer"), ({"out": None}, L.ERR_INVALID, "null pointer"),
             ({"n": 0}, L.ERR_INVALID, "positive"), ({"dims": -1}, L.ERR_INVALID, "positive"),
             ({"n": 32769}, L.ERR_UNSUPPORTED, "n 32769"), ({"dims": 2049}, L.ERR_UNSUPPORTED, "dims 2049"),
             ({"wsb": need - 1}, L.ERR_INVALID, "workspace"), ({"ws": fake * 256 + 8}, L.ERR_INVALID, "aligned")]
    for patch, rc, msg in cases:
        a = {**eer, **patch}
        assert lib.avc_spk_eer(a["vecs"], a["labels"], a["n"], a["dims"], a["ws"], a["wsb"], a["out"], None) == rc, patch
        assert msg in L.last_error(), (patch, L.last_error())
    gm = dict(m=4, n=10, dims=128, queries=fake, q_labels=fake, q_exclude=fake, set=fake, labels=fake, out=fake)
    cases = [({k: None}, L.ERR_INVALID, "null pointer") for k in ("queries", "q_labels", "q_exclude", "set", "labels", "out")]
    cases += [({"m": 0}, L.ERR_INVALID, "positive"), ({"n": 0}, L.ERR_INVALID, "positive"),
              ({"dims": 0}, L.ERR_INVALID, "positive"), ({"n": 32769}, L.ERR_UNSUPPORTED, "n 32769"),
              ({"dims": 2049}, L.ERR_UNSUPPORTED, "dims 2049")]
    for patch, rc, msg in cases:
        assert lib.avc_spk_group_mean(L.SpkGroupDesc(**{**gm, **patch}), None) == rc, patch
        assert msg in L.last_error(), (patch, L.last_error())
    assert lib.avc_spk_group_mean(None, None) == L.ERR_INVALID and "null descriptor" in L.last_error()
    assert L.launch_count() == n0


def test_wrappers_reject_bad_arguments_before_a_launch():
    n0 = L.launch_count()
    with pytest.raises(ValueError, match="CUDA"):
        S.time_stats(torch.zeros(2, 3, 4), [4, 4])
    with pytest.raises(ValueError, match="CUDA"):
        S.eer(torch.zeros(5, 3), [0, 0, 1, 1, 2])
    with pytest.raises(ValueError, match="float32"):
        S.eer(torch.zeros(5, 3, dtype=torch.float64), [0] * 5)
    with pytest.raises(ValueError, match="CUDA"):
        S.group_means(torch.zeros(1, 3), [0], [-1], torch.zeros(5, 3), [0] * 5)
    with pytest.raises(ValueError, match="vectors"):
        S.eer_workspace(0, "cpu")
    with pytest.raises(ValueError, match="vectors"):
        S.eer_workspace(32769, "cpu")
    from adaptive_voice_conversion_b200.model import AE
    cfg = default_config(80)
    cfg["data_loader"]["frame_size"] = 2
    with pytest.raises(ValueError, match="frame_size"):
        S.evaluate_speakers(AE(cfg), {})
    assert L.launch_count() == n0
