"""CPU: the host side of the speaker probes.  Fit-utterance selection (deterministic, independent of the pickle's key
order), the counting of unseen and short utterances, the refusal of overlapping sets, evaluate.py's -probe arguments
and output, and the float64 restatement (tests/_probe_ref.py) against finite differences and literal loops."""
import json
import os
import pickle

import numpy as np
import pytest

import _probe_ref as R
from adaptive_voice_conversion_b200 import _lib as L
from adaptive_voice_conversion_b200 import speaker_probe as P
from adaptive_voice_conversion_b200.config import default_config
from conftest import ROOT
from test_mcd_host import cli, fake_run


# ----------------------------------------------------------------------------- selection and counting
def lengths_of(rng, n_spk=6):
    out = {}
    for s in range(n_spk):
        for k in range(int(rng.integers(1, 12))):
            out[f"p{300 + s}_{k:03d}.wav"] = int(rng.choice([5, 16, 17, 40, 300]))
    out["p30_001.wav"] = 50          # sorts between p300_* and p301_*, its own speaker
    return out


@pytest.mark.parametrize("seed", [0, 1, 5])
def test_selection_is_the_literal_rule_and_ignores_key_order(seed):
    rng = np.random.default_rng(seed)
    lens = lengths_of(rng)
    for k in (1, 3, 64):
        got = P.probe_utterances(lens, 17, k, seed)
        import random
        r = random.Random(seed)
        by = {}
        for u in sorted(lens):
            if lens[u] >= 17:
                by.setdefault(u.split("_")[0], []).append(u)
        ref = sorted(v for s in sorted(by) for v in r.sample(by[s], min(k, len(by[s]))))
        assert got == ref
        keys = list(lens)
        rng.shuffle(keys)
        assert P.probe_utterances({u: lens[u] for u in keys}, 17, k, seed) == got
        assert P.probe_utterances(lens, 17, k, seed) == got
        assert all(lens[u] >= 17 for u in got)
        per = {}
        for u in got:
            per[u.split("_")[0]] = per.get(u.split("_")[0], 0) + 1
        assert max(per.values()) <= k
    with pytest.raises(ValueError, match="per_speaker_utts"):
        P.probe_utterances(lens, 17, 0)


def test_unseen_and_short_counts():
    lens = {"p1_001.wav": 20, "p1_002.wav": 5, "p2_001.wav": 30, "p9_001.wav": 40, "p9_002.wav": 3, "p1_003.wav": 17}
    seen, n_unseen, n_short = P.split_set(lens, {"p1", "p2"}, 17)
    assert seen == ["p1_001.wav", "p1_003.wav", "p2_001.wav"] and n_unseen == 1 and n_short == 2
    assert P.split_set(lens, set(), 17) == ([], 4, 2)
    assert P.split_set({}, {"p1"}, 17) == ([], 0, 0)


def test_overlapping_sets_are_refused_before_any_work():
    from adaptive_voice_conversion_b200.model import AE
    P.check_disjoint(["a_1", "b_2"], ["a_3"])
    with pytest.raises(ValueError, match="shares 1 utterance.*a_1"):
        P.check_disjoint(["a_1", "b_2"], ["a_1", "c_1"], "train", "in_test")
    n0 = L.launch_count()
    fit = {"p1_001.wav": np.zeros((40, 80), np.float32)}
    with pytest.raises(ValueError, match="train shares 1 utterance.*in_test.*p1_001.wav"):
        P.evaluate_probe(AE(default_config(80)), fit, {"in_test": dict(fit)}, fit_name="train")
    cfg = default_config(80)
    cfg["data_loader"]["frame_size"] = 2
    with pytest.raises(ValueError, match="frame_size"):
        P.evaluate_probe(AE(cfg), fit, {"in_test": {}})
    assert L.launch_count() == n0


# ----------------------------------------------------------------------------- the CLI
CLI_BASE = ["-c", os.path.join(ROOT, "config.yaml"), "-m", "m.ckpt"]


def write_sets(d, names):
    d.mkdir(exist_ok=True)
    for k, s in enumerate(names):
        with open(d / f"{s}.pkl", "wb") as f:
            pickle.dump({f"p{k}_001.wav": np.zeros((20, 4), np.float32)}, f)


@pytest.mark.parametrize("argv,msg", [
    (["-probe", "-probe_set", "in_test"], "also one of -eval_sets"),
    (["-probe", "-probe_set", "nosuch"], "nosuch.pkl"),
    (["-probe", "-probe_utts", "0"], "-probe_utts must be >= 1"),
])
def test_cli_probe_argument_errors(capsys, tmp_path, argv, msg):
    write_sets(tmp_path / "data", ["train", "in_test", "out_test"])
    with pytest.raises(SystemExit):
        cli().main(CLI_BASE + ["-d", str(tmp_path / "data")] + argv)
    assert msg in capsys.readouterr().err


def test_cli_probe_output(monkeypatch, tmp_path):
    d = tmp_path / "data"
    write_sets(d, ["train", "in_test", "out_test"])
    seen = []

    def entry(n, acc):
        e = {k: {"acc": acc, "top5": acc, "per_speaker": {}, "fit_acc": 1.0, "fit_loss": 0.5}
             for k in P.REPRESENTATIONS}
        e["content_frames"]["frame_acc"] = acc
        return {"n": n, "n_unseen": 0 if n else 3, "n_short": 1, "speakers": 4, "chance": 0.25, "majority": None,
                "fit_set": "train", "n_fit": 12, **e}

    def fake_probe(model, fit_data, data, seed, per_speaker_utts, device, fit_name):
        seen.append((sorted(fit_data), sorted(data), seed, per_speaker_utts, fit_name))
        return {"in_test": entry(5, 0.75), "out_test": entry(0, None)}
    monkeypatch.setattr(P, "evaluate_probe", fake_probe)
    o = tmp_path / "eval.json"
    got, text, _, res = fake_run(monkeypatch, CLI_BASE + ["-d", str(d), "-probe", "-probe_utts", "7", "-seed", "3",
                                                          "-o", str(o)])
    lines = text.splitlines()
    assert lines[2:] == [
        "in_test: probe speaker=0.7500 content=0.7500 content_frames=0.7500 mel=0.7500 chance=0.2500 (n=5 n_unseen=0 "
        "n_short=1, 4 speakers, fit on train: 12 utterances)",
        "out_test: probe speaker=n/a content=n/a content_frames=n/a mel=n/a chance=0.2500 (n=0 n_unseen=3 n_short=1, "
        "4 speakers, fit on train: 12 utterances)"]
    assert seen == [(["p0_001.wav"], ["in_test", "out_test"], 3, 7, "train")]
    saved = json.loads(o.read_text())
    assert saved["in_test"]["probe"]["speaker"]["acc"] == 0.75
    # every other entry is what the run without -probe writes
    _, _, _, plain = fake_run(monkeypatch, CLI_BASE + ["-d", str(d)])
    assert {s: {k: v for k, v in r.items() if k != "probe"} for s, r in saved.items()} == json.loads(json.dumps(plain))


# ----------------------------------------------------------------------------- the restatement
def mlp(rng, D=6, H=5, S=4):
    return [rng.standard_normal((H, D)) * 0.5, rng.standard_normal(H) * 0.1, rng.standard_normal((H, H)) * 0.5,
            rng.standard_normal(H) * 0.1, rng.standard_normal((S, H)) * 0.5, rng.standard_normal(S) * 0.1]


def test_gradients_match_finite_differences():
    rng = np.random.default_rng(0)
    P_ = mlp(rng)
    x = rng.standard_normal((9, 6))
    y = rng.integers(0, 4, 9)
    G = R.grads64(P_, x, y)
    h = 1e-6
    for i, p in enumerate(P_):
        for j in range(p.size):
            up = [q.copy() for q in P_]
            dn = [q.copy() for q in P_]
            up[i].flat[j] += h
            dn[i].flat[j] -= h
            num = (R.loss64(up, x, y) - R.loss64(dn, x, y)) / (2 * h)
            assert abs(num - G[i].flat[j]) < 1e-7 + 1e-5 * abs(num), (i, j, num, G[i].flat[j])


def test_xent_and_vote_are_literal_loops():
    rng = np.random.default_rng(1)
    z = rng.standard_normal((7, 5)).astype(np.float32)
    z[3] = [1, 2, 2, 0, 2]                      # ties: lower class index wins
    y = np.array([0, 4, 2, 2, 1, 3, 0])
    loss, d, rank = R.xent64(z, y, 0.5)
    for r in range(7):
        zr = z[r].astype(np.float64)
        lse = np.log(np.sum(np.exp(zr - zr.max()))) + zr.max()
        assert abs(loss[r] - (lse - zr[y[r]])) < 1e-14
        p = np.exp(zr - lse)
        p[y[r]] -= 1
        assert np.allclose(d[r], 0.5 * p, rtol=0, atol=1e-15)
        assert rank[r] == sum(1 for j in range(5) if zr[j] > zr[y[r]] or (zr[j] == zr[y[r]] and j < y[r]))
    assert list(rank[[3]]) == [1]               # class 2 ties with 1 and 4: only class 1 ranks above
    off = [0, 1, 4, 7]
    scores, vr = R.vote64(z, off, [0, 2, 3])
    ls = R.log_softmax64(z)
    assert np.array_equal(scores[0], ls[0]) and np.allclose(scores[2], ls[4] + ls[5] + ls[6], rtol=0, atol=1e-14)
    assert vr[0] == R.rank_of(scores[0], 0)


def test_adam_and_moments_are_literal():
    rng = np.random.default_rng(2)
    p, g = [rng.standard_normal(4)], [rng.standard_normal(4)]
    P1, m, v = R.adam64(p, g, [np.zeros(4)], [np.zeros(4)], 1)
    # the first bias-corrected step moves every coordinate by lr * g / (|g| + eps)
    assert np.allclose(P1[0], p[0] - 1e-3 * g[0] / (np.abs(g[0]) + 1e-8), rtol=0, atol=1e-15)
    x = rng.standard_normal((10, 3))
    x[:, 1] = 2.5                                # constant column: std 1
    mean, std = R.moments64(x)
    assert np.allclose(mean, x.mean(0), rtol=1e-15) and std[1] == 1.0 and np.allclose(std[[0, 2]], x.std(0)[[0, 2]])
    lens = [3, 1]
    xb = rng.standard_normal((2, 4, 5)).astype(np.float32)
    rows = R.frames64(xb, lens, [1, 0], 4)
    assert np.array_equal(rows[1:], xb[0, :, :3].T) and np.array_equal(rows[0], xb[1, :, 0])


def test_init_is_nn_linear_bounds_and_seeded():
    a = P.init_params(10, 3, P.ProbeParams(hidden=8), 4)
    b = P.init_params(10, 3, P.ProbeParams(hidden=8), 4)
    assert a.numel() == 8 * 10 + 8 + 8 * 8 + 8 + 3 * 8 + 3 and bool((a == b).all())
    W1, b1, W2, b2, W3, b3 = P.unflatten(a, 10, 8, 3)
    assert float(W1.abs().max()) <= 10 ** -0.5 and float(b3.abs().max()) <= 8 ** -0.5
    assert not bool((P.init_params(10, 3, P.ProbeParams(hidden=8), 5) == a).all())
    assert P.epoch_order(10, 1, 2).tolist() == P.epoch_order(10, 1, 2).tolist() != P.epoch_order(10, 1, 3).tolist()


def test_chunk_bounds_keep_utterances_whole():
    off = [0, 3, 5, 12, 13, 20]
    for m in (1, 4, 7, 8, 100):
        b = P._chunk_bounds(off, m)
        assert b[0] == 0 and b[-1] == 20 and set(b) <= set(off)
        for a, c in zip(b[:-1], b[1:]):
            assert c - a <= m or off.index(c) - off.index(a) == 1


def test_entry_points_reject_invalid_arguments_without_a_device():
    lib = L.load()
    f = 0x10000     # never dereferenced: every case fails validation before a launch
    n0 = L.launch_count()
    cases = [
        (lambda: lib.avc_probe_frames(None, 2, 3, 4, f, f, f, None), L.ERR_INVALID, "null pointer"),
        (lambda: lib.avc_probe_frames(f, 0, 3, 4, f, f, f, None), L.ERR_INVALID, "positive"),
        (lambda: lib.avc_probe_frames(f, 65536, 3, 4, f, f, f, None), L.ERR_UNSUPPORTED, "65535"),
        (lambda: lib.avc_probe_moments(f, 10, 3, None, f, None), L.ERR_INVALID, "null pointer"),
        (lambda: lib.avc_probe_moments(f, 0, 3, f, f, None), L.ERR_INVALID, "positive"),
        (lambda: lib.avc_probe_standardize(f, None, 10, 0, f, f, f, None), L.ERR_INVALID, "positive"),
        (lambda: lib.avc_probe_standardize(f, None, 10, 3, f, f, None, None), L.ERR_INVALID, "null pointer"),
        (lambda: lib.avc_probe_xent(f, f, 4, 3, 1.0, f, None, None, None, None, None), L.ERR_INVALID, "null pointer"),
        (lambda: lib.avc_probe_xent(f, f, 4, 3, 1.0, f, None, f, f, None, None), L.ERR_INVALID, "together"),
        (lambda: lib.avc_probe_xent(f, f, 0, 3, 1.0, f, None, f, None, None, None), L.ERR_INVALID, "positive"),
        (lambda: lib.avc_probe_xent(f, f, 4, 4097, 1.0, f, None, f, None, None, None), L.ERR_UNSUPPORTED, "4097"),
        (lambda: lib.avc_probe_vote(f, 3, f, 2, f, f, None, None), L.ERR_INVALID, "null pointer"),
        (lambda: lib.avc_probe_vote(f, 3, f, 0, f, f, f, None), L.ERR_INVALID, "positive"),
        (lambda: lib.avc_probe_vote(f, 4097, f, 2, f, f, f, None), L.ERR_UNSUPPORTED, "4097"),
    ]
    for call, rc, msg in cases:
        assert call() == rc, msg
        assert msg in L.last_error(), (msg, L.last_error())
    assert L.launch_count() == n0


def test_descriptor_constants_match_the_header(tmp_path):
    import subprocess
    c = tmp_path / "s.c"
    c.write_text('#include <stdio.h>\n#include "avc_b200.h"\nint main(){printf("%d\\n", AVC_PROBE_MAX_CLASSES);return 0;}\n')
    subprocess.check_call(["gcc", "-I", os.path.join(ROOT, "include"), str(c), "-o", str(tmp_path / "s")])
    assert int(subprocess.check_output([str(tmp_path / "s")])) == L.PROBE_MAX_CLASSES >= 4096
