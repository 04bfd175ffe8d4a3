"""GPU: avc_yin against the float64 restatement (tests/_f0_ref.py) on ragged batches (harmonic signals, noise, silence,
the shortest accepted signal, a glide, a 60 s signal, and the parameter edges win = tau_max, tau_min = 1 and the span
cap), a signal's bits alone and in a shuffled batch, mel_to_wav = trim(mel_to_signal), and evaluate_f0 end to end at
c_in 80 and 512 (conversions bit for bit with inference_ragged, every number against the restatement on the device's
own tracks, two runs, n_refs 2) and through evaluate.py -f0 -spk."""
import json
import os
import pickle
import sys

import numpy as np
import pytest
import torch

import _f0_ref as R
from adaptive_voice_conversion_b200 import _lib as L
from adaptive_voice_conversion_b200 import f0 as F
from adaptive_voice_conversion_b200 import vocoder as V
from adaptive_voice_conversion_b200.config import default_config

pytestmark = pytest.mark.gpu

SR, HOP = 24000, 300
REL = 1e-12


def dev(a):
    return torch.from_numpy(np.ascontiguousarray(a, np.float32)).cuda()


def close(a, b, rel=REL):
    a, b = np.asarray(a, np.float64), np.asarray(b, np.float64)
    return a.shape == b.shape and bool(np.all(np.abs(a - b) <= rel * np.abs(b)))


def check_against_restatement(sigs, p, frames=None):
    """avc_yin of the batch against the restatement of each signal (all frames, or frames[i])."""
    outs = F.yin([dev(y) for y in sigs], SR, HOP, p)
    for i, (y, o) in enumerate(zip(sigs, outs)):
        got = [t.cpu().numpy() for t in o]
        fr = None if frames is None else frames[i]
        ref = R.yin(y, SR, HOP, win=p.win, fmin=p.fmin, fmax=p.fmax, threshold=p.threshold, frames=fr)
        if fr is not None:
            got = [g[fr] for g in got]
        assert len(got[0]) == len(ref["tau"]), i
        for g, k in zip(got, ("tau", "aperiodicity", "energy")):
            assert close(g, ref[k]), (i, k, np.max(np.abs(g - ref[k]) / np.maximum(np.abs(ref[k]), 1e-300)))
        assert np.all(np.abs(got[0] - ref["tau_star"]) <= 0.5), i
        v_dev = F.voicing(*got, SR, p)[1]
        v_ref = R.voicing(ref["tau"], ref["aperiodicity"], ref["energy"], SR, p.threshold, p.silence_db)[1]
        assert np.array_equal(v_dev, v_ref), i
    return outs


def test_yin_matches_the_restatement_on_a_ragged_batch():
    p = F.F0Params()
    sigs = [R.harmonic(f, 0.4, phase_seed=k) for k, f in enumerate([55.0, 110.0, 180.0, 260.0, 450.0])]
    sigs.append((np.random.default_rng(1).standard_normal(9000) * 0.3).astype(np.float32))
    sigs.append(np.zeros(7000, np.float32))
    sigs.append(R.harmonic(150.0, p.min_samples(SR) / SR)[:p.min_samples(SR)])     # the shortest accepted signal
    sigs.append(R.harmonic(lambda t: 100.0 + 400.0 * t, 0.5))
    assert len(sigs[-2]) == p.min_samples(SR)
    outs = check_against_restatement(sigs, p)
    for o in outs[:5]:                     # tracking itself, away from the reflected edges
        f0, voiced = F.voicing(*[t.cpu().numpy() for t in o], SR, p)
        assert voiced[3:-3].all()
    with pytest.raises(ValueError, match="samples"):
        F.yin([dev(sigs[-2][:-1])], SR, HOP, p)


def test_yin_on_a_60_second_signal():
    y = R.harmonic(lambda t: 120.0 + 60.0 * np.sin(2 * np.pi * t / 7.0), 60.0)
    n_frames = 1 + len(y) // HOP
    fr = sorted(set(range(0, 4)) | set(range(n_frames - 4, n_frames)) | set(range(0, n_frames, 97)))
    check_against_restatement([y], F.F0Params(), frames=[fr])


@pytest.mark.parametrize("params", [
    dict(win=480),                                       # win = tau_max
    dict(fmax=24000.0, win=600),                         # tau_min = 1
    dict(fmin=23.4375, win=2048),                        # win + tau_max = AVC_YIN_MAX_SPAN
    dict(fmin=80.0, fmax=400.0, win=512, threshold=0.3),
], ids=["win_eq_tau_max", "tau_min_1", "span_cap", "other"])
def test_yin_parameter_edges(params):
    p = F.F0Params(**params)
    if params.get("win") == 2048:
        assert p.win + p.tau_max(SR) == L.YIN_MAX_SPAN
    sigs = [R.harmonic(f, 0.3, phase_seed=k) for k, f in enumerate([90.0, 230.0])]
    sigs.append((np.random.default_rng(2).standard_normal(8000) * 0.1).astype(np.float32))
    sigs.append(R.harmonic(200.0, 1.0)[:p.min_samples(SR)])
    check_against_restatement(sigs, p)


def test_yin_rejects_the_span_cap_plus_one():
    y = dev(R.harmonic(100.0, 0.5))
    n0 = L.launch_count()
    with pytest.raises(L.AvcError, match="AVC_YIN_MAX_SPAN"):
        F.yin([y], SR, HOP, F.F0Params(fmin=23.4375, win=2049))
    assert L.launch_count() == n0


def test_bits_alone_equal_bits_in_a_shuffled_batch():
    rng = np.random.default_rng(3)
    sigs = [R.harmonic(float(rng.uniform(60, 400)), float(rng.uniform(0.05, 0.6)), phase_seed=k) for k in range(12)]
    sigs = [s if len(s) >= 753 else np.pad(s, (0, 753 - len(s))) for s in sigs]
    sigs.append(np.zeros(2000, np.float32))
    alone = [[t.cpu().numpy() for t in F.yin([dev(y)], SR, HOP)[0]] for y in sigs]
    perm = rng.permutation(len(sigs))
    batch = F.yin([dev(sigs[i]) for i in perm], SR, HOP)
    for j, i in enumerate(perm):
        for a, b in zip(alone[i], batch[j]):
            assert a.tobytes() == b.cpu().numpy().tobytes(), i


def test_mel_to_wav_is_trimmed_mel_to_signal():
    g = torch.Generator().manual_seed(5)
    for n_mels in (80, 512):
        voc = V.Vocoder(n_mels=n_mels)
        mels = [torch.rand((T, n_mels), generator=g).cuda() for T in (9, 40, 133)]
        for kw in ({}, {"momentum": 0.5}, {"init": "pghi"}):
            sig = voc.mel_to_signal(mels, n_iter=6, **kw)
            assert [s.numel() for s in sig] == [HOP * (m.shape[0] - 1) for m in mels]
            wav = voc.mel_to_wav(mels, n_iter=6, **kw)
            for a, b in zip(wav, V.trim(sig, voc.hp.out_top_db)):
                assert a.cpu().numpy().tobytes() == b.cpu().numpy().tobytes()


# ----------------------------------------------------------------------------- evaluate_f0 end to end
def make_set(n_mels, seed, n_speakers=4, n_utts=4, dur=(0.6, 1.6)):
    """Utterances copy-analysed from harmonic signals at a speaker-specific pitch with vibrato (wav_to_mel), attr from
    their statistics, attr-normalised; one speaker with a single utterance and one utterance too short to embed."""
    rng = np.random.default_rng(seed)
    voc = V.Vocoder(n_mels=n_mels)
    wavs, keys = [], []
    for s in range(n_speakers):
        base = 90.0 * 1.35 ** s
        for k in range(n_utts):
            seconds = float(rng.uniform(*dur))
            rate, depth = float(rng.uniform(3, 6)), float(rng.uniform(0.02, 0.08))
            wavs.append(R.harmonic(lambda t: base * (1 + depth * np.sin(2 * np.pi * rate * t)), seconds,
                                   phase_seed=len(keys)))
            keys.append(f"p{300 + s}_{k:03d}.wav")
    wavs.append(R.harmonic(300.0, 0.8))
    keys.append("p399_001.wav")
    mels = [m.cpu().numpy() for m, _ in voc.wav_to_mel([dev(w) for w in wavs])]
    allm = np.concatenate(mels)
    attr = {"mean": allm.mean(0).astype(np.float32), "std": (allm.std(0) + 1e-2).astype(np.float32)}
    data = {k: ((m - attr["mean"]) / attr["std"]).astype(np.float32) for k, m in zip(keys, mels)}
    data["p300_900.wav"] = data["p300_000.wav"][:12].copy()
    return data, attr


def make_model(c_in):
    from adaptive_voice_conversion_b200.model import AE
    torch.manual_seed(c_in)
    return AE(default_config(c_in)).cuda()


def stand_in(sources, refs):
    """Voiced stand-in conversions: pair i's source mel itself (even i) or its first reference tiled to the source's
    T frames (odd i).  The random-init model's conversions are unvoiced, so only these reach every scored value."""
    return [x if i % 2 == 0 else c.repeat(-(-x.shape[0] // c.shape[0]), 1)[: x.shape[0]]
            for i, (x, c) in enumerate(zip(sources, refs))]


def use_stand_in(monkeypatch):
    from adaptive_voice_conversion_b200 import mcd as M

    def converted(model, sources, refs, batch_max=64, codes=None):
        yield list(range(len(sources))), stand_in(sources, refs)
    monkeypatch.setattr(M, "converted", converted)


def device_tracks(model, data, attr, n_refs, hp, p, fake=False):
    """The tracks evaluate_f0 measures, recomputed from the public pieces: inference_ragged (or the pooled codes, or
    the stand-in), mel_to_signal, avc_yin, the voicing rule."""
    from adaptive_voice_conversion_b200.inference import Inferencer, embed_reference_sets
    from adaptive_voice_conversion_b200 import mcd as M
    model.eval()
    cfg = model.config
    utts, pairs, refs, _ = F.select_pairs(cfg, {u: len(v) for u, v in data.items()}, 0, 0, n_refs)
    devm = {u: dev(v) for u, v in data.items()}
    srcs = [devm[u] for u, _ in pairs]
    if fake:
        convs = stand_in(srcs, [devm[r[0]] for r in refs])
    elif n_refs == 1:
        inf = Inferencer.__new__(Inferencer)
        inf.config, inf.model, inf.attr = cfg, model, None
        convs = [o[: s.shape[0]] for o, s in zip(inf.inference_ragged(srcs, [devm[r[0]] for r in refs]), srcs)]
        seen = 0
        for idx, decs in M.converted(model, srcs, [devm[r[0]] for r in refs]):
            for i, d in zip(idx, decs):
                assert d.contiguous().cpu().numpy().tobytes() == convs[i].contiguous().cpu().numpy().tobytes()
                seen += 1
        assert seen == len(pairs)
    else:
        codes = embed_reference_sets(model, [[devm[v].t() for v in rs] for rs in refs])
        convs = [None] * len(pairs)
        for idx, decs in M.converted(model, srcs, [devm[r[0]] for r in refs], codes=codes):
            for i, d in zip(idx, decs):
                convs[i] = d
    mean, std = dev(attr["mean"]), dev(attr["std"])
    voc = V.Vocoder(n_mels=cfg["SpeakerEncoder"]["c_in"], hp=hp)
    sig = voc.mel_to_signal([devm[u] * std + mean for u in utts] + [c * std + mean for c in convs], hp.n_iter,
                            hp.momentum, hp.gl_init)
    raw = [[t.cpu().numpy() for t in o] for o in F.yin(sig, SR, HOP, p)]
    tracks = [F.voicing(*o, SR, p) for o in raw]
    return utts, pairs, refs, sig, raw, dict(zip(utts, tracks[:len(utts)])), tracks[len(utts):]


def check_numbers(res, pairs, refs, real, conv, n_refs):
    """Every number of evaluate_f0's result against the restatement on the device's tracks; returns the rows."""
    rows, n_unv, total, spk, prof = R.measure([(u, r) for (u, _), r in zip(pairs, refs)], real, conv)
    assert res["n_unvoiced"] == n_unv and res["n"] == len(rows) and res["n"] + n_unv == len(pairs)
    assert [r[:2] for r in res["pairs"]] == [[pairs[i][0], refs[i] if n_refs > 1 else refs[i][0]] for i in rows]
    for got, i in zip(res["pairs"], rows):
        assert got[2:] == pytest.approx(rows[i], rel=REL, abs=1e-15), got[:2]
    for k in R.METRICS:
        assert (res.get(k) is None and not rows) or res[k] == pytest.approx(total[k], rel=REL, abs=1e-15), k
    assert set(res["speakers"]) == set(spk)
    for s in spk:
        assert res["speakers"][s]["n"] == spk[s]["n"]
        for k in R.METRICS:
            assert res["speakers"][s][k] == pytest.approx(spk[s][k], rel=REL, abs=1e-15), (s, k)
    assert set(res["profiles"]) == set(prof)
    for s, pr in prof.items():
        got = res["profiles"][s]
        assert (got["voiced"], got["frames"]) == (pr["voiced"], pr["frames"]), s
        if pr["log2_mean"] is None:
            assert got["log2_mean"] is None
        else:
            assert got["log2_mean"] == pytest.approx(pr["log2_mean"], rel=REL)
            assert got["log2_std"] == pytest.approx(pr["log2_std"], rel=1e-9)
    return rows


@pytest.mark.parametrize("c_in", [80, 512])
def test_evaluate_f0_end_to_end(c_in, monkeypatch):
    data, attr = make_set(c_in, c_in)
    model = make_model(c_in)
    model.train()
    hp = V.AudioParams(n_iter=12)
    p = F.F0Params()
    res = F.evaluate_f0(model, data, attr, per_pair=True, hp=hp)
    assert model.training
    utts, pairs, refs, sig, raw, real, conv = device_tracks(model, data, attr, 1, hp, p)
    assert res["n"] + res["n_unvoiced"] == len(pairs) > 8 and res["n_short"] > 0
    # the device's tracks are the restatement's, on a few of the device's own signals
    for i in (0, len(utts) - 1, len(utts), len(sig) - 1):
        y = sig[i].cpu().numpy()
        ref = R.yin(y, SR, HOP)
        for g, k in zip(raw[i], ("tau", "aperiodicity", "energy")):
            assert close(g, ref[k]), (i, k)
        assert np.array_equal(F.voicing(*raw[i], SR, p)[1], R.voicing(ref["tau"], ref["aperiodicity"], ref["energy"], SR)[1])
    check_numbers(res, pairs, refs, real, conv, 1)
    if c_in == 512:      # at 80 mels much of the copy-synthesis tracks as unvoiced (DESIGN §4)
        assert all(res["profiles"][f"p{300 + s}"]["voiced"] > 0 for s in range(4))
    assert res["tracker"]["tau_min"] == 48 and res["tracker"]["tau_max"] == 480
    assert res["griffin_lim"] == {"n_iter": 12, "momentum": 0.0, "init": "zero"}
    # two runs, the same JSON
    assert json.dumps(F.evaluate_f0(model, data, attr, per_pair=True, hp=hp)) == json.dumps(res)
    # voiced stand-in conversions reach every scored value
    use_stand_in(monkeypatch)
    res = F.evaluate_f0(model, data, attr, per_pair=True, hp=hp)
    *_, real, conv = device_tracks(model, data, attr, 1, hp, p, fake=True)
    rows = check_numbers(res, pairs, refs, real, conv, 1)
    assert c_in == 80 or len(rows) > 4
    index = {u: i for i, (u, _) in enumerate(pairs)}
    same = [r for r in res["pairs"] if index[r[0]] % 2 == 0]      # converted into itself
    assert (same or c_in == 80) and all(r[2] == 1.0 and r[3] == pytest.approx(1.0) and r[7] == r[4] for r in same)


def test_evaluate_f0_with_two_references(monkeypatch):
    data, attr = make_set(512, 7)
    model = make_model(512)
    hp = V.AudioParams(n_iter=8, momentum=0.9)
    p = F.F0Params()
    res = F.evaluate_f0(model, data, attr, per_pair=True, hp=hp, n_refs=2)
    one = F.evaluate_f0(model, data, attr, hp=hp)
    assert res["n_refs"] == 2 and res["n"] + res["n_unvoiced"] + res["n_few"] == one["n"] + one["n_unvoiced"]
    utts, pairs, refs, sig, raw, real, conv = device_tracks(model, data, attr, 2, hp, p)
    assert all(len(r) == 2 for r in refs)
    check_numbers(res, pairs, refs, real, conv, 2)
    use_stand_in(monkeypatch)
    res = F.evaluate_f0(model, data, attr, per_pair=True, hp=hp, n_refs=2)
    *_, real, conv = device_tracks(model, data, attr, 2, hp, p, fake=True)
    rows = check_numbers(res, pairs, refs, real, conv, 2)
    assert len(rows) > 4
    # the target profile leaves out both references
    logs = {u: np.log2(f[v]) for u, (f, v) in real.items()}
    for row in res["pairs"]:
        u, rs = row[0], row[1]
        kept = [v for v in utts if v.split("_")[0] == rs[0].split("_")[0] and v not in rs]
        assert len(kept) == len([v for v in utts if v.split("_")[0] == rs[0].split("_")[0]]) - len(set(rs) & set(utts))
        tm = R.profile([logs[v] for v in kept])[0]
        ms = R.seq_sum(logs[u]) / len(logs[u])
        assert row[7] == pytest.approx(12 * abs(ms - tm), rel=REL)


def test_cli_f0_and_spk_score_the_same_pairs(tmp_path):
    import yaml
    import oracle.ae_oracle as orc
    from adaptive_voice_conversion_b200.model import AE
    from conftest import ROOT
    cfg = orc.default_config(80)
    (tmp_path / "config.yaml").write_text(yaml.safe_dump(cfg))
    m = AE(cfg)
    m.load_state_dict(orc.init_state(cfg, seed=0))
    torch.save(m.state_dict(), tmp_path / "model.ckpt")
    data, attr = make_set(80, 9, dur=(1.7, 2.0))
    with open(tmp_path / "in_test.pkl", "wb") as f:
        pickle.dump(data, f)
    with open(tmp_path / "in_test_samples_128.json", "w") as f:
        json.dump([[u, 0] for u in sorted(data) if len(data[u]) >= 128][:4], f)
    assert sum(len(v) >= 128 for v in data.values()) >= 4
    with open(tmp_path / "attr.pkl", "wb") as f:
        pickle.dump(attr, f)
    if ROOT not in sys.path:
        sys.path.insert(0, ROOT)
    import evaluate as cli
    base = ["-c", str(tmp_path / "config.yaml"), "-m", str(tmp_path / "model.ckpt"), "-d", str(tmp_path),
            "-eval_sets", "in_test", "-spk", "-max_pairs", "6", "-seed", "2"]
    cli.main(base + ["-o", str(tmp_path / "plain.json")])
    cli.main(base + ["-f0", "-gl_iters", "8", "-gl_init", "pghi", "-o", str(tmp_path / "f0.json")])
    plain, withf0 = (json.loads((tmp_path / n).read_text()) for n in ("plain.json", "f0.json"))
    f0 = withf0["in_test"].pop("f0")
    assert json.dumps(withf0, indent=1) == (tmp_path / "plain.json").read_text()
    assert "f0" not in plain["in_test"]
    assert f0["griffin_lim"] == {"n_iter": 8, "momentum": 0.0, "init": "pghi"}
    assert f0["n"] + f0["n_unvoiced"] == plain["in_test"]["spk"]["conversion"]["n"] == 6
    # the pairs themselves: evaluate_f0 with per_pair against evaluate_speakers with per_pair
    from adaptive_voice_conversion_b200.speaker_eval import evaluate_speakers
    model = AE(cfg).cuda()
    model.load_state_dict(torch.load(tmp_path / "model.ckpt"))
    spk = evaluate_speakers(model, data, seed=2, max_pairs=6, per_pair=True)["conversion"]["pairs"]
    _, pairs, _, _ = F.select_pairs(cfg, {u: len(v) for u, v in data.items()}, 2, 6)
    assert [list(p) for p in pairs] == [r[:2] for r in spk]
    got = F.evaluate_f0(model, data, attr, seed=2, max_pairs=6, per_pair=True, hp=V.AudioParams(n_iter=8, gl_init="pghi"))
    assert json.dumps({k: v for k, v in got.items() if k != "pairs"}) == json.dumps(f0)
    assert all(r[:2] in [x[:2] for x in spk] for r in got["pairs"])
