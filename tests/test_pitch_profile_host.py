"""CPU: the mean-and-variance log-F0 transform (f0.mv_shifts) against its float64 restatement (tests/_mv_ref.py) on
hand-built tracks; the target profiles of banked specs, mixes and morphs; the banks' pitch record through save, load
and its checks; per-frame semitones validation; and the refusals of -pitch_shift mv before any GPU work."""
import importlib.util
import os
import subprocess
import sys
import types

import numpy as np
import pytest
import torch

import _mv_ref as R
import oracle.ae_oracle as orc
from adaptive_voice_conversion_b200 import f0 as F
from adaptive_voice_conversion_b200 import speaker_bank as SB
from conftest import ROOT

nan = np.nan


def trk(f0s):
    f = np.asarray(f0s, np.float64)
    return f, ~np.isnan(f)


def check(track, target, **kw):
    """mv_shifts of one track against the restatement; returns (shifts, info)."""
    shifts, info = F.mv_shifts([track], [target], **kw)
    want, flags = R.mv(list(track[0]), list(track[1]), target, **({"limit": kw["limit"]} if kw else {}))
    assert shifts[0].dtype == np.float64 and len(shifts[0]) == len(track[1])
    assert np.allclose(shifts[0], want, rtol=0, atol=1e-12), (shifts[0], want)
    for k, v in flags.items():
        assert info[0][k] == v, (k, info[0], flags)
    assert info[0]["voiced_conv"] == int(track[1].sum())
    assert info[0]["mean_shift"] == pytest.approx(float(np.mean(want)), abs=1e-12)
    return shifts[0], info[0]


# ----------------------------------------------------------------------------- the transform
def test_voiced_frames_follow_the_affine_map():
    track = trk([100.0, 120.0, 150.0, 90.0, 200.0])
    mu_t, sd_t = np.log2(220.0), 0.4
    s, info = check(track, (mu_t, sd_t))
    assert not (info["mean_only"] or info["unmatched"]) and info["clamped_frames"] == 0
    # after the shift the log2 F0 has the target's mean and std
    l = np.log2(track[0]) + s / 12.0
    assert l.mean() == pytest.approx(mu_t, abs=1e-12) and l.std() == pytest.approx(sd_t, abs=1e-12)


def test_gaps_are_interpolated_and_ends_held():
    track = trk([nan, nan, 100.0, nan, nan, nan, 180.0, 140.0, nan, nan])
    s, _ = check(track, (np.log2(200.0), 0.1))
    assert s[0] == s[1] == s[2] and s[8] == s[9] == s[7]
    assert s[4] == pytest.approx((s[2] + s[6]) / 2, abs=1e-12)
    assert s[3] == pytest.approx(s[2] + (s[6] - s[2]) / 4, abs=1e-12)


def test_equal_sigma_gives_the_match_shift():
    track = trk([100.0, nan, 130.0, 160.0, nan, 110.0])
    l = np.log2(track[0][track[1]])
    mc, sc, _ = F.profile([l])
    ref = trk([230.0, 250.0])
    (match,), _ = F.shifts_from_tracks([track], [[ref]])
    s, _ = check(track, (F.track_profile([ref])[0], sc))
    assert np.allclose(s, match, rtol=0, atol=1e-12)


def test_fallbacks_to_the_mean_only_shift():
    for track in (trk([150.0, nan, 150.0, 150.0]),           # sigma_c = 0
                  trk([nan, 120.0, nan])):                    # one voiced frame
        s, info = check(track, (np.log2(240.0), 0.3))
        assert info["mean_only"] and not info["unmatched"]
        assert np.all(s == s[0]) and s[0] == pytest.approx(12 * (np.log2(240.0) - np.log2(track[0][track[1]][0])),
                                                           abs=1e-12)
    # per frame for a profile that varies
    mu = np.log2(np.array([200.0, 220.0, 240.0]))
    s, info = check(trk([nan, 120.0, nan]), (mu, np.full(3, 0.3)))
    assert info["mean_only"] and np.allclose(s, 12 * (mu - np.log2(120.0)), rtol=0, atol=1e-12)


def test_clamping_and_counting():
    track = trk([60.0, 70.0, nan, 400.0, 65.0])
    s, info = check(track, (np.log2(300.0), 2.0))
    assert np.all(np.abs(s) <= 24.0) and info["clamped_frames"] >= 1
    s, info = check(track, (np.log2(300.0), 2.0), limit=3.0)
    assert np.all(np.abs(s) <= 3.0) and info["clamped_frames"] >= 3
    s, info = check(trk([50.0, 50.0]), (np.log2(1600.0), 0.0))        # mean only: five octaves, every frame clamped
    assert info["mean_only"] and list(s) == [24.0, 24.0] and info["clamped_frames"] == 2


def test_unmatched_on_either_side():
    s, info = check(trk([nan, nan, nan]), (np.log2(200.0), 0.2))
    assert info["unmatched"] and list(s) == [0.0] * 3 and info["voiced_conv"] == 0
    s, info = check(trk([100.0, 120.0]), None)
    assert info["unmatched"] and list(s) == [0.0, 0.0]


def test_per_frame_targets():
    track = trk([100.0, nan, 130.0, 160.0, 110.0, nan, nan, 140.0])
    T = len(track[1])
    mu = np.log2(np.linspace(180.0, 260.0, T))
    sd = np.linspace(0.1, 0.5, T)
    check(track, (mu, sd))
    # constant arrays give the bits of the constant profile
    a, _ = F.mv_shifts([track], [(np.full(T, mu[0]), np.full(T, sd[0]))])
    b, _ = F.mv_shifts([track], [(float(mu[0]), float(sd[0]))])
    assert a[0].tobytes() == b[0].tobytes()


# ----------------------------------------------------------------------------- banked profiles
def pitched_bank(codes_dim=8, fitted=None):
    names = ["p300", "p301", "p302", "p303"]
    utts = [[f"{n}_{k:03d}" for k in range(2)] for n in names]
    pitch = {"log2_mean": [7.0, 7.8, None, 6.5], "log2_std": [0.1, 0.25, None, 0.0], "voiced": [40, 55, 0, 3],
             "frames": [90, 80, 70, 60], "tracker": F.F0Params().settings(24000, 300),
             "griffin_lim": {"n_iter": 100, "momentum": 0.0, "init": "zero"}}
    codes = torch.randn((4, codes_dim), generator=torch.Generator().manual_seed(0))
    return SB.SpeakerBank(names, codes, [2] * 4, utts, "f" * 64, fitted=fitted, pitch=pitch)


def test_spec_profiles_mix_in_spec_order():
    bank = pitched_bank()
    P = [(7.0, 0.1), (7.8, 0.25), None, (6.5, 0.0)]
    assert bank.pitch_profile("p300") == (7.0, 0.1)
    assert bank.pitch_profile("p301:0.37") == pytest.approx((7.8, 0.25), abs=1e-15)
    for spec, parts in (("p300:0.7,p301:0.3", [(0, 0.7), (1, 0.3)]), ("p303:1,p300:3", [(3, 1.0), (0, 3.0)]),
                        ("p301:1e-3,p302:0", [(1, 1e-3), (2, 0.0)])):
        assert bank.pitch_profile(spec) == R.mix([P[r] for r, _ in parts], [w for _, w in parts]), spec
    assert bank.pitch_profile("p302") is None
    assert bank.pitch_profile("p300:0.5,p302:0.5") is None
    with pytest.raises(ValueError, match="not in the bank"):
        bank.pitch_profile("p999")
    with pytest.raises(ValueError, match="speaker_bank.py -f0"):
        bank.with_pitch(None).pitch_profile("p300")


def test_morph_profiles_per_frame():
    bank = pitched_bank()
    keys = [("p300", 0.0), ("p300", 1.0), ("p301", 2.0), ("p300:0.5,p301:0.5", 3.0)]
    T, fps = 50, 10.0
    mu, sd = bank.morph_pitch_profile(keys, T, fps)
    names, w = SB.morph_weights(keys, T, fps)
    P = {"p300": (7.0, 0.1), "p301": (7.8, 0.25)}
    for f in range(T):
        want = R.mix([P[n] for n in names], [float(w[k, f]) for k in range(len(names))])
        assert (mu[f], sd[f]) == pytest.approx(want, abs=1e-15)
    assert mu[0] == 7.0 and sd[0] == 0.1 and mu[20] == 7.8 and sd[20] == 0.25
    assert bank.morph_pitch_profile([("p300", 0.0), ("p302", 1.0)], T, fps) is None
    zero = bank.morph_pitch_profile([("p300:1,p302:0", 0.0)], T, fps)      # an unvoiced speaker of weight 0 is skipped
    assert np.all(zero[0] == 7.0) and np.all(zero[1] == 0.1)


def test_a_one_hot_morph_equals_the_speaker_target_bit_for_bit():
    bank = pitched_bank()
    track = trk([100.0, nan, 130.0, 160.0, 110.0, nan, nan, 140.0, 125.0, nan])
    T = len(track[1])
    morph = bank.morph_pitch_profile([("p301", 0.0), ("p301", 0.5)], T, 10.0)
    one = bank.pitch_profile("p301")
    assert np.all(morph[0] == one[0]) and np.all(morph[1] == one[1])
    a, ia = F.mv_shifts([track], [morph])
    b, ib = F.mv_shifts([track], [one])
    assert a[0].tobytes() == b[0].tobytes() and ia == ib


# ----------------------------------------------------------------------------- the record in files
def cpu_model(cfg):
    from adaptive_voice_conversion_b200.model import AE
    m = AE(cfg)
    m.load_state_dict(orc.init_state(cfg, seed=0))
    return m


@pytest.fixture(scope="module")
def model80():
    return cpu_model(orc.default_config(80))


def test_save_and_load_with_and_without_the_record(tmp_path, model80):
    fp = SB.fingerprint(model80)
    b = pitched_bank(model80.config["SpeakerEncoder"]["c_out"])
    b = SB.SpeakerBank(b.speakers, b.codes, b.n_utts, b.utterances, fp, pitch=b.pitch)
    path = str(tmp_path / "pitched.pt")
    b.save(path)
    raw = torch.load(path, weights_only=True)
    assert raw["format"] == SB.FORMAT == "avc-speaker-bank-1" and raw["pitch"] == b.pitch
    back = SB.SpeakerBank.load(path, model80)
    assert back.pitch == b.pitch and torch.equal(back.codes, b.codes)
    assert back.pitch_profile("p300:0.7,p301:0.3") == b.pitch_profile("p300:0.7,p301:0.3")
    # without the record: no "pitch" key, and the file is that of a bank made before the record existed
    plain = b.with_pitch(None)
    plain.save(str(tmp_path / "plain.pt"))
    raw = torch.load(str(tmp_path / "plain.pt"), weights_only=True)
    assert "pitch" not in raw and SB.SpeakerBank.load(str(tmp_path / "plain.pt"), model80).pitch is None
    old = {"format": "avc-speaker-bank-1", "speakers": list(b.speakers), "codes": b.codes.clone(),
           "n_utts": list(b.n_utts), "utterances": [list(u) for u in b.utterances], "fingerprint": fp, "n_skipped": 2}
    torch.save(old, str(tmp_path / "old.pt"))
    back = SB.SpeakerBank.load(str(tmp_path / "old.pt"), model80)
    assert back.pitch is None and back.n_skipped == 2 and torch.equal(back.codes, b.codes)


def test_a_fitted_record_and_a_pitch_record_travel_together(tmp_path, monkeypatch, model80):
    from adaptive_voice_conversion_b200 import fit
    monkeypatch.setattr(fit, "model_fingerprint", lambda m: "m" * 64)
    b = pitched_bank(model80.config["SpeakerEncoder"]["c_out"], fitted={"model_fingerprint": "m" * 64, "steps": 3})
    b = SB.SpeakerBank(b.speakers, b.codes, b.n_utts, b.utterances, SB.fingerprint(model80), fitted=b.fitted,
                       pitch=b.pitch)
    b.save(str(tmp_path / "f.pt"))
    back = SB.SpeakerBank.load(str(tmp_path / "f.pt"), model80)
    assert back.fitted == b.fitted and back.pitch == b.pitch


@pytest.mark.parametrize("edit,msg", [
    (lambda p: p["log2_mean"].pop(), "log2_mean must list"),
    (lambda p: p.update(frames=p["frames"] + [1]), "frames must list"),
    (lambda p: p["log2_mean"].__setitem__(0, float("nan")), "finite"),
    (lambda p: p["log2_std"].__setitem__(1, float("inf")), "finite"),
    (lambda p: p["log2_std"].__setitem__(0, -0.1), "std >= 0"),
    (lambda p: p["log2_mean"].__setitem__(2, 7.0), "without a voiced frame"),
    (lambda p: p["voiced"].__setitem__(0, 0), "without a voiced frame"),
    (lambda p: p["voiced"].__setitem__(1, 81), "voiced <= frames"),
    (lambda p: p["voiced"].__setitem__(1, -1), "voiced <= frames"),
    (lambda p: p["log2_mean"].__setitem__(0, None), "finite floats"),
    (lambda p: p.pop("griffin_lim"), "griffin_lim"),
    (lambda p: p.pop("tracker"), "tracker"),
])
def test_malformed_records_are_refused(tmp_path, model80, edit, msg):
    b = pitched_bank(model80.config["SpeakerEncoder"]["c_out"])
    pitch = {k: (list(v) if isinstance(v, list) else v) for k, v in b.pitch.items()}
    edit(pitch)
    with pytest.raises(ValueError, match=msg):
        b.with_pitch(pitch)
    d = {"format": SB.FORMAT, "speakers": list(b.speakers), "codes": b.codes, "n_utts": list(b.n_utts),
         "utterances": [list(u) for u in b.utterances], "fingerprint": SB.fingerprint(model80), "n_skipped": 0,
         "pitch": pitch}
    path = str(tmp_path / "bad.pt")
    torch.save(d, path)
    with pytest.raises(ValueError, match=msg):
        SB.SpeakerBank.load(path, model80)


# ----------------------------------------------------------------------------- per-frame semitones
def test_per_frame_semitones_validation():
    from adaptive_voice_conversion_b200.vocoder import _semitones
    ramp = np.linspace(-6.0, 6.0, 5)
    got = _semitones([1.5, ramp, torch.tensor(ramp)], 3, "x", [7, 5, 5])
    assert got[0] == 1.5 and got[1].dtype == np.float64 and np.array_equal(got[1], ramp)
    assert np.array_equal(got[2], ramp)
    assert _semitones(np.zeros((2, 4)), 2, "x", [4, 4])[1].tolist() == [0.0] * 4
    assert _semitones(np.array([1.0, -2.0]), 2, "x", [4, 4]) == [1.0, -2.0]
    assert _semitones(torch.tensor(3.0), 2, "x", [4, 4]) == [3.0, 3.0]
    with pytest.raises(ValueError, match=r"utterance 1: \(4,\) per-frame shifts, expected 5 frames"):
        _semitones([0.0, np.zeros(4)], 2, "x", [5, 5])
    with pytest.raises(ValueError, match="utterance 0: .*expected one per utterance"):
        _semitones([np.zeros(4)], 1, "x")
    with pytest.raises(ValueError, match="utterance 1: .*frames"):
        _semitones([0.0, np.zeros((2, 2))], 2, "x", [4, 4])
    for bad in (24.5, -25.0, nan, np.inf):
        v = np.zeros(6)
        v[3] = bad
        with pytest.raises(ValueError, match=r"mel_to_signal: utterance 1: pitch shift must be finite .* at frame 3"):
            _semitones([0.0, v], 2, "mel_to_signal", [4, 6])
    ok = np.array([-24.0, 24.0, -0.0])
    assert np.array_equal(_semitones([ok], 1, "x", [3])[0], ok)


def test_per_frame_ratios_are_rounded_once_from_float64():
    from adaptive_voice_conversion_b200.vocoder import _ratio
    for v in (-24.0, -7.3, -0.0, 0.01, 5.0, 24.0):
        assert np.float32(_ratio(v)) == np.float32(2.0 ** (v / 12.0))
    assert _ratio(0.0) == 1.0


# ----------------------------------------------------------------------------- refusals before the GPU
def load_script(name):
    spec = importlib.util.spec_from_file_location(f"{name}_mvcli", os.path.join(ROOT, f"{name}.py"))
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod


def test_mv_arguments(capsys):
    inf = load_script("inference")

    def check_args(argv):
        p = inf.parser()
        args = p.parse_args(argv)
        inf.check_args(p, args)
        return args
    for argv in (["-s", "a.wav", "-t", "b.wav", "-o", "o.wav"], ["-s", "a.wav", "-t", "b.wav", "c.wav", "-o", "o.wav"],
                 ["-s", "a.wav", "-bank", "b.pt", "-speaker", "p1:0.5,p2:0.5", "-o", "o.wav"],
                 ["-s", "a.wav", "-bank", "b.pt", "-morph", "p1@0", "p2@1", "-o", "o.wav"],
                 ["-pairs", "p.txt", "-o", "d"]):
        assert check_args(argv + ["-pitch_shift", "mv"]).semitones == "mv"
    for argv in (["-s", "a.wav", "-t", "b.wav", "-o", "o.npy"], ["-s", "a.wav", "-bank", "b.pt", "-speaker", "p1",
                                                                 "-o", "o.npy"]):
        with pytest.raises(SystemExit):
            check_args(argv + ["-pitch_shift", "mv"])
        assert ".npy output" in capsys.readouterr().err


def plain_bank_file(path):
    torch.save({"format": SB.FORMAT, "speakers": ["p1", "p2"], "codes": torch.zeros(2, 4), "n_utts": [1, 1],
                "utterances": [["p1_0"], ["p2_0"]], "fingerprint": "f" * 64, "n_skipped": 0}, path)


@pytest.mark.parametrize("target", [["-speaker", "p1"], ["-speaker", "p1:0.5,p2:0.5"], ["-morph", "p1@0", "p2@1"]])
def test_a_bank_without_profiles_is_refused_before_anything_runs(tmp_path, target):
    bank = str(tmp_path / "bank.pt")
    plain_bank_file(bank)
    # no config, model or source exists: the refusal must come before any of them is read
    run = subprocess.run([sys.executable, os.path.join(ROOT, "inference.py"), "-c", str(tmp_path / "none.yaml"),
                          "-m", str(tmp_path / "none.ckpt"), "-s", str(tmp_path / "none.wav"), "-bank", bank, *target,
                          "-o", str(tmp_path / "o.wav"), "-pitch_shift", "mv"],
                         capture_output=True, text=True, env=dict(os.environ, PYTHONPATH=ROOT, CUDA_VISIBLE_DEVICES=""))
    assert run.returncode == 2, run.stderr
    assert "no pitch profiles" in run.stderr and "speaker_bank.py -f0" in run.stderr
    assert not (tmp_path / "o.wav").exists()


def test_pairs_mv_refuses_an_unprofiled_bank_before_the_gpu(tmp_path):
    inf = load_script("inference")
    for name in ("a.wav", "b.wav"):
        (tmp_path / name).write_bytes(b"")
    bank = str(tmp_path / "bank.pt")
    plain_bank_file(bank)
    pf = tmp_path / "pairs.txt"
    pf.write_text(f"{tmp_path / 'a.wav'} {tmp_path / 'b.wav'}\n{tmp_path / 'b.wav'} @p1:0.5,p2:0.5\n")
    args = types.SimpleNamespace(pairs=str(pf), bank=bank, semitones="mv", output=str(tmp_path / "out"))
    with pytest.raises(ValueError, match="no pitch profiles.*speaker_bank.py -f0"):
        inf.run_pairs(args, {})
    assert not (tmp_path / "out").exists()


def test_evaluate_and_bank_builder_arguments(tmp_path, capsys):
    ev = load_script("evaluate")
    with pytest.raises(SystemExit):
        ev.main(["-m", str(tmp_path / "none.ckpt"), "-d", str(tmp_path), "-pitch_shift", "mv"])
    assert "-pitch_shift needs -f0" in capsys.readouterr().err
    sb = load_script("speaker_bank")

    def check_args(argv):
        p = sb.parser()
        args = p.parse_args(["-m", "m.ckpt", "-o", "b.pt"] + argv)
        sb.check_args(p, args)
        return args
    (tmp_path / "attr.pkl").write_bytes(b"")
    src = ["-d", str(tmp_path), "-set", "train"]
    assert check_args(src + ["-f0", "-gl_iters", "8", "-gl_init", "pghi"]).f0
    assert not check_args(src).f0
    for argv, msg in ((src + ["-gl_iters", "8"], "copy-synthesis of -f0"),
                      (src + ["-gl_init", "pghi"], "copy-synthesis of -f0"),
                      (src + ["-f0", "-gl_momentum", "1.0"], "[0, 1)"),
                      (src + ["-f0", "-gl_iters", "-1"], ">= 0"),
                      (["-d", str(tmp_path / "nowhere"), "-set", "train", "-f0"], "mel statistics")):
        with pytest.raises(SystemExit):
            check_args(argv)
        assert msg in capsys.readouterr().err, argv


def test_mv_match_takes_references_or_a_profile_per_conversion():
    conv = [torch.zeros(20, 512)]
    for kw, msg in (({"ref_sets": [[conv[0]]], "profiles": [(7.0, 0.1)]}, "not both"),
                    ({"ref_sets": [(conv[0],)]}, "non-empty list"),
                    ({"ref_sets": [[]]}, "non-empty list"),
                    ({"profiles": [(7.0, 0.1), None]}, "one reference set or profile per conversion")):
        with pytest.raises(ValueError, match=msg):
            F.mv_match(None, conv, None, **kw)
