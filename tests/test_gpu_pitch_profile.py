"""GPU: per-frame semitones through the vocoder (constant arrays give the bits of the float, zeros launch nothing, a
ramp is followed); banked pitch profiles (build_pitch_profiles equals f0.profile of the same utterances synthesised and
tracked directly, a speaker's bits alone and among many, known tone pitches, a fitted bank keeps the record); the
mean-and-variance transform on vibrato tones; inference.py -pitch_shift mv end to end with -speaker, a mix, @SPEC
pairs lines, file targets and -morph, as subprocesses with the model's (unvoiced) conversions and in process with voiced
ones; and evaluate_f0(pitch_shift="mv")."""
import json
import os
import subprocess
import sys

import numpy as np
import pytest
import torch

from _pshift_ref import formant_tone
from adaptive_voice_conversion_b200 import _lib as L
from adaptive_voice_conversion_b200 import f0 as F
from adaptive_voice_conversion_b200 import speaker_bank as SB
from adaptive_voice_conversion_b200 import vocoder as V

pytestmark = pytest.mark.gpu

SR, HOP = 24000, 300
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def dev(a):
    return torch.from_numpy(np.ascontiguousarray(a, np.float32)).cuda()


def tone_mels(voc, specs):
    """wav_to_mel of formant tones (f0, seconds, vibrato) (unnormalised mels)."""
    return [m for m, _ in voc.wav_to_mel([dev(formant_tone(f, s, phase_seed=i, vibrato=v))
                                          for i, (f, s, v) in enumerate(specs)])]


def bits(ts):
    return [t.cpu().numpy().tobytes() for t in ts]


# ----------------------------------------------------------------------------- per-frame semitones
def test_constant_and_zero_per_frame_entries():
    voc = V.Vocoder(n_mels=512, hp=V.AudioParams(n_iter=8))
    mels = tone_mels(voc, [(120.0, 0.7, 0.0), (200.0, 0.5, 0.0), (150.0, 0.9, 0.0)])
    T = [m.shape[0] for m in mels]
    floats = voc.mel_to_signal(mels, semitones=[3.0, -5.5, 0.0])
    arrays = voc.mel_to_signal(mels, semitones=[np.full(T[0], 3.0), torch.full((T[1],), -5.5), np.zeros(T[2])])
    assert bits(floats) == bits(arrays)
    torch.cuda.synchronize()
    n0 = L.launch_count()
    plain = voc.mel_to_signal(mels)
    torch.cuda.synchronize()
    n1 = L.launch_count()
    zero = voc.mel_to_signal(mels, semitones=[np.zeros(t) for t in T])
    torch.cuda.synchronize()
    assert L.launch_count() - n1 == n1 - n0           # no avc_pitch_shift launch
    assert bits(zero) == bits(plain)
    assert bits(arrays)[2] == bits(plain)[2]          # an all-zero entry copies its utterance
    # a per-frame entry of equal values is the bits of the float in pitch_shift itself
    mags = voc.mel_to_mag(mels)
    assert bits(V.pitch_shift(mags, [np.full(t, 7.25) for t in T])) == bits(V.pitch_shift(mags, 7.25))


@pytest.mark.parametrize("init", ["zero", "pghi"])
def test_a_ramp_is_followed_frame_by_frame(init):
    voc = V.Vocoder(n_mels=512)
    mel = tone_mels(voc, [(150.0, 2.0, 0.0)])[0]
    T = mel.shape[0]
    ramp = np.linspace(-6.0, 6.0, T)
    a, b = voc.mel_to_signal([mel, mel], init=init, semitones=[0.0, ramp])
    (fa, va), (fb, vb) = F.track([a, b], SR, HOP)
    both = va & vb
    err = np.abs(fb[both] / fa[both] / 2.0 ** (ramp[both] / 12.0) - 1.0)
    print(f"ramp -6..+6 st ({init}): median |ratio error| {np.median(err):.5f}, {int(both.sum())}/{T} frames voiced "
          f"in both")
    assert both.sum() >= T // 4
    assert np.median(err) <= 0.01


# ----------------------------------------------------------------------------- profiles
def tone_set(speakers, n_mels=512):
    """{utterance: attr-normalised mel} of formant tones: speakers = {name: [(f0, seconds, vibrato), ...]}, and attr."""
    voc = V.Vocoder(n_mels=n_mels)
    keys, specs = [], []
    for s, utts in speakers.items():
        for k, spec in enumerate(utts):
            keys.append(f"{s}_{k:03d}")
            specs.append(spec)
    wavs = [dev(formant_tone(f, sec, phase_seed=i, vibrato=v)) for i, (f, sec, v) in enumerate(specs)]
    mels = [m for m, _ in voc.wav_to_mel(wavs)]
    allm = torch.cat(mels).cpu().numpy()
    attr = {"mean": allm.mean(0).astype(np.float32), "std": (allm.std(0) + 1e-2).astype(np.float32)}
    mean, std = dev(attr["mean"]), dev(attr["std"])
    return {k: (m - mean) / std for k, m in zip(keys, mels)}, attr


def bare_bank(mels):
    """A SpeakerBank of every utterance, grouped by the name before '_' (codes are not used by the profiles)."""
    speakers, utts, _ = SB.bank_order(list(mels), {u: 1 for u in mels}, 0, lambda u: u.split("_")[0])
    return SB.SpeakerBank(speakers, torch.zeros(len(speakers), 4, device="cuda"), [len(u) for u in utts], utts,
                          "f" * 64)


SPEAKERS = {"pa": [(110.0, 1.0, 0.0), (112.0, 0.8, 0.0)], "pb": [(180.0, 0.9, 0.0), (176.0, 1.1, 0.0)],
            "pc": [(260.0, 0.7, 0.0), (255.0, 1.0, 0.0), (265.0, 0.8, 0.0)]}


def test_profiles_equal_the_direct_track_and_do_not_depend_on_the_bank():
    mels, attr = tone_set(SPEAKERS)
    hp = V.AudioParams(n_iter=16)
    bank = bare_bank(mels)
    rec = SB.build_pitch_profiles(bank, mels, attr, hp)
    voc = V.Vocoder(n_mels=512, hp=hp)
    mean, std = dev(attr["mean"]), dev(attr["std"])
    for s, us in zip(bank.speakers, bank.utterances):
        sig = F.synthesize(voc, [mels[u] * std + mean for u in us], voc.hp)
        tr = F.track_chunks(sig, SR, HOP, F.F0Params())
        m, sd, nv = F.profile([np.log2(f[v]) for f, v in tr])
        i = bank.index(s)
        assert (rec["log2_mean"][i], rec["log2_std"][i], rec["voiced"][i]) == (m, sd, nv), s
        assert rec["frames"][i] == sum(len(v) for _, v in tr)
        alone = SB.build_pitch_profiles(bare_bank({u: mels[u] for u in us}), mels, attr, hp)
        assert [alone[k][0] for k in SB.PITCH_LISTS] == [rec[k][i] for k in SB.PITCH_LISTS], s
    assert rec["griffin_lim"] == {"n_iter": 16, "momentum": 0.0, "init": "zero"}
    assert rec["tracker"] == F.F0Params().settings(SR, HOP)


def test_known_tone_pitches():
    mels, attr = tone_set(SPEAKERS)
    bank = bare_bank(mels)
    rec = SB.build_pitch_profiles(bank, mels, attr)
    worst = 0.0
    for s, utts in SPEAKERS.items():
        i = bank.index(s)
        # frame-weighted log2 mean of the utterances' pitches (steady tones: frames ~ seconds)
        want = sum(np.log2(f) * sec for f, sec, _ in utts) / sum(sec for _, sec, _ in utts)
        err = abs(rec["log2_mean"][i] - want)
        worst = max(worst, err)
        print(f"{s}: log2_mean {rec['log2_mean'][i]:.5f} (want {want:.5f}, |err| {err:.2e}), log2_std "
              f"{rec['log2_std'][i]:.5f}, {rec['voiced'][i]}/{rec['frames'][i]} frames voiced")
        assert rec["voiced"][i] > rec["frames"][i] // 2
    assert worst <= 3e-5          # 1.0e-5 at worst measured on an H100 (pb)


def test_a_fitted_bank_keeps_the_record():
    import oracle.ae_oracle as orc
    from adaptive_voice_conversion_b200 import fit
    from adaptive_voice_conversion_b200.model import AE
    cfg = orc.default_config(80)
    model = AE(cfg)
    model.load_state_dict(orc.init_state(cfg, seed=0))
    model = model.cuda()
    mels, attr = tone_set({"pa": [(110.0, 2.0, 0.0)], "pb": [(200.0, 2.0, 0.0)]}, n_mels=80)
    bank = SB.build_bank(model, mels, speaker_of=lambda u: u.split("_")[0])
    bank = bank.with_pitch(SB.build_pitch_profiles(bank, mels, attr, V.AudioParams(n_iter=4)))
    fitted, _ = fit.fit_bank(model, bank, mels, 1, crops=2, speakers_per_wave=2)
    assert fitted.fitted is not None and fitted.pitch == bank.pitch


# ----------------------------------------------------------------------------- the transform on tones
def test_mv_moves_the_tracked_std_toward_the_target():
    voc = V.Vocoder(n_mels=512)
    conv, *refs = tone_mels(voc, [(150.0, 2.0, 0.01), (220.0, 1.5, 0.04), (225.0, 1.2, 0.04)])
    hp = voc.hp
    sig = F.synthesize(voc, [conv] + refs, hp)
    tracks = F.track_chunks(sig, SR, HOP, F.F0Params())
    target = F.track_profile(tracks[1:])
    shifts, info = F.mv_shifts(tracks[:1], [target])
    match, _ = F.shifts_from_tracks(tracks[:1], [tracks[1:]])
    out = F.track_chunks(voc.mel_to_signal([conv, conv], semitones=[shifts[0], match[0]]), SR, HOP, F.F0Params())
    before, after, matched = F.track_profile(tracks[:1]), F.track_profile(out[:1]), F.track_profile(out[1:])
    print(f"target mu {target[0]:.4f} sd {target[1]:.4f}; before mu {before[0]:.4f} sd {before[1]:.4f}; mv mu "
          f"{after[0]:.4f} sd {after[1]:.4f}; match mu {matched[0]:.4f} sd {matched[1]:.4f}; {info[0]}")
    assert not (info[0]["unmatched"] or info[0]["mean_only"])
    # measured on an H100: the std gap falls to 0.39 of what it was (mv overshoots sigma_t through the vocoder)
    assert abs(after[1] - target[1]) <= 0.5 * abs(before[1] - target[1])
    assert 12 * abs(after[0] - target[0]) <= max(0.2, 12 * abs(matched[0] - target[0]) + 0.05)


# ----------------------------------------------------------------------------- the command lines
GL_ITERS = 32


@pytest.fixture(scope="module")
def cli(tmp_path_factory):
    """A random-init 512-mel model, tone recordings of two voiced speakers and one of noise, and a bank with pitch
    profiles built by speaker_bank.py -wav -f0 (512 mels: at 80 mels these tones track no voiced frame, DESIGN §4)."""
    import oracle.ae_oracle as orc
    import pickle
    import yaml
    from scipy.io.wavfile import write
    from adaptive_voice_conversion_b200.model import AE
    tmp = tmp_path_factory.mktemp("mv_cli")
    cfg = orc.default_config(512)
    (tmp / "config.yaml").write_text(yaml.safe_dump(cfg))
    m = AE(cfg)
    m.load_state_dict(orc.init_state(cfg, seed=0))
    torch.save(m.state_dict(), tmp / "model.ckpt")
    files = {}
    for i, (name, f, secs) in enumerate((("lo", 110.0, 1.0), ("lo", 115.0, 0.9), ("hi", 230.0, 1.0),
                                         ("hi", 220.0, 0.8), ("src", 160.0, 1.6), ("src", 140.0, 1.2))):
        files.setdefault(name, []).append(str(tmp / f"{name}{i}.wav"))
        write(files[name][-1], SR, (formant_tone(f, secs, phase_seed=i, vibrato=0.02) * 32767).astype(np.int16))
    files["noise"] = [str(tmp / "noise.wav")]
    write(files["noise"][0], SR, (np.random.default_rng(0).standard_normal(SR) * 3000).astype(np.int16))
    attr = {"mean": np.full(512, -0.5, np.float32), "std": np.full(512, 0.3, np.float32)}
    with open(tmp / "attr.pkl", "wb") as fh:
        pickle.dump(attr, fh)
    env = dict(os.environ, PYTHONPATH=ROOT)
    base = [sys.executable, os.path.join(ROOT, "inference.py"), "-c", str(tmp / "config.yaml"), "-m",
            str(tmp / "model.ckpt"), "-a", str(tmp / "attr.pkl"), "-gl_iters", str(GL_ITERS)]
    wavs = sum(([["-wav", n] + files[n]] for n in ("lo", "hi", "noise")), [])
    subprocess.run([sys.executable, os.path.join(ROOT, "speaker_bank.py"), "-c", str(tmp / "config.yaml"), "-m",
                    str(tmp / "model.ckpt"), "-a", str(tmp / "attr.pkl"), *sum(wavs, []), "-o", str(tmp / "bank.pt"),
                    "-f0", "-gl_iters", str(GL_ITERS)], check=True, env=env, cwd=str(tmp))

    def run(*args):
        r = subprocess.run(base + list(args), check=True, env=env, cwd=str(tmp), capture_output=True, text=True)
        print(r.stdout)
        return r.stdout
    return {"tmp": tmp, "files": files, "run": run, "model": m, "attr": attr}


def expected_wav(mel_npy, target, voc):
    """mel_to_wav(semitones=mv_shifts(...)) of a saved denormalised conversion mel toward target."""
    m = dev(np.load(mel_npy))
    tr = F.track_chunks(F.synthesize(voc, [m], voc.hp), SR, HOP, F.F0Params())
    shifts, info = F.mv_shifts(tr, [target])
    return voc.mel_to_wav([m], semitones=shifts)[0].cpu().numpy(), info[0]


def load_cli_bank(c):
    return SB.SpeakerBank.load(str(c["tmp"] / "bank.pt"), c["model"].cuda())


def test_the_bank_builder_records_profiles(cli):
    bank = load_cli_bank(cli)
    p = bank.pitch
    assert bank.speakers == ["hi", "lo", "noise"] and p["griffin_lim"]["n_iter"] == GL_ITERS
    print(f"bank profiles: {p}")
    lo, hi = bank.pitch_profile("lo"), bank.pitch_profile("hi")
    assert lo is not None and hi is not None and hi[0] - lo[0] > 0.8


@pytest.mark.parametrize("target", [["-speaker", "hi"], ["-speaker", "hi:0.6,lo:0.4"],
                                    ["-morph", "lo@0", "hi@0.6", "hi:0.5,lo:0.5@1.2"]])
def test_single_conversions_to_banked_targets(cli, target):
    from scipy.io.wavfile import read
    t = cli["tmp"]
    src = cli["files"]["src"][0]
    tag = "_".join(target).replace("@", "at").replace(":", "-").replace(",", "+")
    cli["run"]("-s", src, "-bank", str(t / "bank.pt"), *target, "-o", str(t / f"{tag}.npy"))
    cli["run"]("-s", src, "-bank", str(t / "bank.pt"), *target, "-o", str(t / f"{tag}_plain.wav"))
    out = cli["run"]("-s", src, "-bank", str(t / "bank.pt"), *target, "-o", str(t / f"{tag}.wav"), "-pitch_shift", "mv")
    assert "pitch shift mv" in out and "note:" not in out
    bank = load_cli_bank(cli)
    voc = V.Vocoder(n_mels=512, hp=V.AudioParams(n_iter=GL_ITERS))
    mel = np.load(t / f"{tag}.npy")
    if target[0] == "-morph":
        prof = bank.morph_pitch_profile(SB_keyframes(target[1:]), mel.shape[0], SR / HOP)
    else:
        prof = bank.pitch_profile(target[1])
    want, info = expected_wav(t / f"{tag}.npy", prof, voc)
    got = read(t / f"{tag}.wav")[1]
    assert got.tobytes() == want.tobytes()
    if info["unmatched"]:
        assert got.tobytes() == read(t / f"{tag}_plain.wav")[1].tobytes()


def SB_keyframes(texts):
    return [SB.parse_keyframe(k) for k in texts]


def test_pairs_with_bank_lines_and_files(cli):
    from scipy.io.wavfile import read
    t, files = cli["tmp"], cli["files"]
    s0, s1 = files["src"]
    (t / "pairs.txt").write_text(f"{s0} @hi a.wav\n{s0} @hi a.npy\n{s1} @lo:0.3,hi:0.7 b.wav\n{s1} @lo:0.3,hi:0.7 b.npy\n"
                                 f"{s0} @noise c.wav\n{s0} @noise c.npy\n{s1} {files['hi'][0]} d.wav\n"
                                 f"{s1} {files['hi'][0]} d.npy\n")
    base = ["-bank", str(t / "bank.pt"), "-pairs", str(t / "pairs.txt")]
    cli["run"](*base, "-o", str(t / "plain"))
    out = cli["run"](*base, "-o", str(t / "mv"), "-pitch_shift", "mv")
    lines = dict(ln.split(": ", 1) for ln in out.splitlines() if "pitch shift mv" in ln)
    assert sorted(lines) == ["a.wav", "b.wav", "c.wav", "d.wav"]
    bank = load_cli_bank(cli)
    voc = V.Vocoder(n_mels=512, hp=V.AudioParams(n_iter=GL_ITERS))
    ref = [m for m, _ in voc.wav_to_mel([dev(V.load_wav(files["hi"][0], SR))])]
    ref_sig = F.synthesize(voc, ref, voc.hp)
    targets = {"a": bank.pitch_profile("hi"), "b": bank.pitch_profile("lo:0.3,hi:0.7"),
               "c": bank.pitch_profile("noise"), "d": F.track_profile(F.track_chunks(ref_sig, SR, HOP, F.F0Params()))}
    n_unmatched = 0
    for k, prof in targets.items():
        want, info = expected_wav(t / "mv" / f"{k}.npy", prof, voc)
        got = read(t / "mv" / f"{k}.wav")[1]
        assert got.tobytes() == want.tobytes(), k
        assert ("unmatched" in lines[f"{k}.wav"]) == info["unmatched"], k
        if info["unmatched"]:
            n_unmatched += 1
            assert got.tobytes() == read(t / "plain" / f"{k}.wav")[1].tobytes(), k
        assert np.load(t / "mv" / f"{k}.npy").tobytes() == np.load(t / "plain" / f"{k}.npy").tobytes()
    if bank.pitch["voiced"][bank.index("noise")] == 0:
        assert "unmatched" in lines["c.wav"]
    # the random-init model's conversions track no voiced frame on an H100, so these command lines check the
    # unmatched path end to end; the voiced path is checked in process below
    print(f"{n_unmatched} of 4 conversions unmatched")


# ----------------------------------------------------------------------------- the command lines, voiced
# The random-init model's conversions track no voiced frame, so the runs above only reach mv's unmatched path.  Here
# inference.py runs in process with the conversion replaced by the identity (each conversion is its tone source), so
# every banked, mixed, morphed and file target meets a voiced conversion, through the same argument handling, bank
# loading, target profiles and synthesis as the command line.
def inference_script():
    import importlib.util
    spec = importlib.util.spec_from_file_location("inference_mv_cli", os.path.join(ROOT, "inference.py"))
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod


@pytest.fixture
def identity(monkeypatch):
    from adaptive_voice_conversion_b200.inference import Inferencer
    monkeypatch.setattr(Inferencer, "inference_with_codes", lambda self, xs, codes, *a, **k: [x.clone() for x in xs])
    monkeypatch.setattr(Inferencer, "inference_morph", lambda self, xs, codes, weights, *a, **k: [x.clone() for x in xs])
    mod = inference_script()
    monkeypatch.setattr(mod, "convert_pairs", lambda inf, pairs, mels, bank=None: [mels[s].clone() for _, s, _, _ in pairs])
    return mod


def in_process(mod, capsys, cli, *args):
    t = cli["tmp"]
    argv = ["-c", str(t / "config.yaml"), "-m", str(t / "model.ckpt"), "-a", str(t / "attr.pkl"), "-gl_iters",
            str(GL_ITERS)] + list(args)
    if "-pairs" in args:      # the pairs mode exits 0 when done
        with pytest.raises(SystemExit) as e:
            mod.main(argv)
        assert e.value.code == 0
    else:
        mod.main(argv)
    out = capsys.readouterr().out
    print(out)
    return out


@pytest.mark.parametrize("target", [["-speaker", "hi"], ["-speaker", "lo:0.3,hi:0.7"],
                                    ["-morph", "lo@0", "hi@0.6", "hi:0.5,lo:0.5@1.2"]])
def test_voiced_single_conversions_to_banked_targets(cli, identity, capsys, target):
    from scipy.io.wavfile import read
    t = cli["tmp"]
    tag = "voiced_" + "_".join(target).replace("@", "at").replace(":", "-").replace(",", "+")
    common = ["-s", cli["files"]["src"][0], "-bank", str(t / "bank.pt"), *target]
    in_process(identity, capsys, cli, *common, "-o", str(t / f"{tag}.npy"))
    out = in_process(identity, capsys, cli, *common, "-o", str(t / f"{tag}.wav"), "-pitch_shift", "mv")
    assert "pitch shift mv" in out and "note:" not in out
    bank = load_cli_bank(cli)
    mel = np.load(t / f"{tag}.npy")
    if target[0] == "-morph":
        prof = bank.morph_pitch_profile(SB_keyframes(target[1:]), mel.shape[0], SR / HOP)
        assert prof[0].max() - prof[0].min() > 0.5          # the target moves over the conversion
    else:
        prof = bank.pitch_profile(target[1])
    want, info = expected_wav(t / f"{tag}.npy", prof, V.Vocoder(n_mels=512, hp=V.AudioParams(n_iter=GL_ITERS)))
    print(f"{target}: {info}")
    assert not info["unmatched"] and info["voiced_conv"] > 10
    assert read(t / f"{tag}.wav")[1].tobytes() == want.tobytes()
    # other Griffin-Lim settings than the bank's profiles were made with are noted
    identity.main(["-c", str(t / "config.yaml"), "-m", str(t / "model.ckpt"), "-a", str(t / "attr.pkl"),
                   "-gl_iters", "4", *common, "-o", str(t / f"{tag}_gl4.wav"), "-pitch_shift", "mv"])
    assert "note: the bank's pitch profiles were synthesised with" in capsys.readouterr().out


def test_voiced_pairs_with_bank_lines_and_files(cli, identity, capsys):
    from scipy.io.wavfile import read
    t, files = cli["tmp"], cli["files"]
    s0, s1 = files["src"]
    (t / "vpairs.txt").write_text(f"{s0} @hi a.wav\n{s0} @hi a.npy\n{s1} @lo:0.3,hi:0.7 b.wav\n"
                                  f"{s1} @lo:0.3,hi:0.7 b.npy\n{s0} @noise c.wav\n{s0} @noise c.npy\n"
                                  f"{s1} {files['hi'][0]} d.wav\n{s1} {files['hi'][0]} d.npy\n")
    base = ["-bank", str(t / "bank.pt"), "-pairs", str(t / "vpairs.txt")]
    in_process(identity, capsys, cli, *base, "-o", str(t / "vplain"))
    out = in_process(identity, capsys, cli, *base, "-o", str(t / "vmv"), "-pitch_shift", "mv")
    lines = dict(ln.split(": ", 1) for ln in out.splitlines() if "pitch shift mv" in ln)
    assert sorted(lines) == ["a.wav", "b.wav", "c.wav", "d.wav"] and "note:" not in out
    bank = load_cli_bank(cli)
    voc = V.Vocoder(n_mels=512, hp=V.AudioParams(n_iter=GL_ITERS))
    ref = [m for m, _ in voc.wav_to_mel([dev(V.load_wav(files["hi"][0], SR))])]
    targets = {"a": bank.pitch_profile("hi"), "b": bank.pitch_profile("lo:0.3,hi:0.7"),
               "c": bank.pitch_profile("noise"),
               "d": F.track_profile(F.track_chunks(F.synthesize(voc, ref, voc.hp), SR, HOP, F.F0Params()))}
    assert targets["c"] is None            # the noise speaker has no voiced frame
    for k, prof in targets.items():
        want, info = expected_wav(t / "vmv" / f"{k}.npy", prof, voc)
        print(f"{k}: {info}")
        got = read(t / "vmv" / f"{k}.wav")[1]
        assert got.tobytes() == want.tobytes(), k
        assert info["voiced_conv"] > 10, k
        assert info["unmatched"] == (k == "c") and ("unmatched" in lines[f"{k}.wav"]) == (k == "c"), k
        if k == "c":      # a voiced conversion toward an unvoiced target keeps the bits of a run without the flag
            assert got.tobytes() == read(t / "vplain" / f"{k}.wav")[1].tobytes()
        else:
            assert got.tobytes() != read(t / "vplain" / f"{k}.wav")[1].tobytes(), k


# ----------------------------------------------------------------------------- evaluation
def test_evaluate_f0_mv(monkeypatch):
    from adaptive_voice_conversion_b200 import mcd as M
    from adaptive_voice_conversion_b200.config import default_config
    from adaptive_voice_conversion_b200.model import AE

    def converted(model, sources, refs, batch_max=64, codes=None):     # the identity: each conversion is its source
        yield list(range(len(sources))), list(sources)
    monkeypatch.setattr(M, "converted", converted)
    spk = {"p500": [(110.0 * (1 + 0.03 * k), 0.8 + 0.1 * k, 0.01) for k in range(5)],
           "p501": [(200.0 * (1 + 0.03 * k), 0.8 + 0.1 * k, 0.04) for k in range(5)]}
    mels, attr = tone_set(spk)
    data = {f"{k}.wav": v.cpu().numpy() for k, v in mels.items()}
    torch.manual_seed(0)
    model = AE(default_config(512)).cuda()
    hp = V.AudioParams(n_iter=32)
    plain = F.evaluate_f0(model, data, attr, per_pair=True, hp=hp)
    res = F.evaluate_f0(model, data, attr, per_pair=True, hp=hp, pitch_shift="mv")
    assert json.dumps(res["unshifted"]) == json.dumps(plain)
    ps = res["pitch_shift"]
    print(f"evaluate_f0 mv: st_target {plain['st_target']:.4f} -> {res['st_target']:.4f}, {ps}")
    assert set(res) - set(plain) == {"pitch_shift", "unshifted"}
    assert set(ps) == {"mode", "mean_semitones", "mean_abs_semitones", "n_unmatched", "n_clamped", "n_mean_only",
                       "n_clamped_frames", "sd_target", "sd_target_unshifted"}
    assert ps["mode"] == "mv" and ps["n_unmatched"] == 0 and ps["mean_abs_semitones"] > 1
    assert res["st_target"] < plain["st_target"]
    assert ps["sd_target"] < ps["sd_target_unshifted"]
