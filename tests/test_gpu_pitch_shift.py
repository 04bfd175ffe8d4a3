"""GPU: avc_pitch_shift against the float64 restatement (tests/_pshift_ref.py) on mel pseudo-inverse magnitudes at 80 and
512 mels and all-zero rows, ratios across +-24 semitones and lifters 1, 40 and 1024; a row's bits alone and in a
shuffled ragged batch; argument errors with no launch; the unshifted synthesis unchanged; the tracked pitch of shifted
syntheses of formant-shaped harmonic tones at 512 mels (plain, momentum 0.99 and the PGHI start); formant preservation
against a tone generated at the shifted pitch; match_shifts; evaluate_f0(pitch_shift="match"); and
inference.py -pairs -pitch_shift match end to end (an unmatched pair keeps its bits)."""
import json
import os
import subprocess
import sys

import numpy as np
import pytest
import torch

import _pshift_ref as R
from _pshift_ref import formant_tone
from adaptive_voice_conversion_b200 import _lib as L
from adaptive_voice_conversion_b200 import f0 as F
from adaptive_voice_conversion_b200 import vocoder as V

pytestmark = pytest.mark.gpu

SR, HOP = 24000, 300
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def dev(a):
    return torch.from_numpy(np.ascontiguousarray(a, np.float32)).cuda()


def mel_mags(n_mels, seed=0):
    """Linear magnitudes of mel-to-linear (the synthesis's input) of a few formant tones at n_mels, per utterance."""
    voc = V.Vocoder(n_mels=n_mels)
    mels = [m for m, _ in voc.wav_to_mel([dev(formant_tone(f, 0.4, phase_seed=seed + i)) for i, f in
                                          enumerate((95.0, 160.0, 240.0))])]
    return voc.mel_to_mag(mels)


# ----------------------------------------------------------------------------- the kernel
@pytest.mark.parametrize("n_mels", [80, 512])
@pytest.mark.parametrize("lifter", [1, 40, 1024])
def test_kernel_matches_the_restatement(n_mels, lifter):
    mags = mel_mags(n_mels) + [torch.zeros(7, 1025, device="cuda")]
    chunks, shifts = [], []
    for m in mags:
        for j, s in enumerate((-24.0, -12.5, -3.0, 0.0, 0.01, 7.0, 24.0)):
            chunks.append(m[j::7].contiguous())
            shifts.append(s)
    hp = V.AudioParams(ps_lifter=lifter)
    outs = V.pitch_shift(chunks, shifts, hp)
    worst = 0.0
    for x, s, o in zip(chunks, shifts, outs):
        S = x.cpu().numpy()
        got = o.cpu().numpy()
        if s == 0.0:
            assert got.tobytes() == S.tobytes()
            continue
        alpha = float(np.float32(2.0 ** (s / 12.0)))
        ref = R.pitch_shift(S.astype(np.float64), alpha, lifter)
        assert np.all(got > 0) and np.all(np.isfinite(got))
        err = float(np.max(np.abs(np.log(got.astype(np.float64)) - np.log(ref))))
        worst = max(worst, err)
    assert worst <= 1e-3, worst
    print(f"n_mels {n_mels} lifter {lifter}: max |ln out - ln ref| = {worst:.3e}")


def test_bits_alone_equal_bits_in_a_shuffled_ragged_batch():
    mags = mel_mags(512, seed=3)
    pieces = [mags[0][:5], mags[1][3:40], mags[2][:1], mags[0][10:33], mags[1][:64]]
    shifts = [3.0, -7.5, 0.0, 12.0, -24.0]
    alone = [V.pitch_shift([p], [s])[0] for p, s in zip(pieces, shifts)]
    order = [3, 0, 4, 2, 1]
    batch = V.pitch_shift([pieces[i] for i in order], [shifts[i] for i in order])
    for j, i in enumerate(order):
        assert batch[j].cpu().numpy().tobytes() == alone[i].cpu().numpy().tobytes(), i
    assert alone[2].cpu().numpy().tobytes() == pieces[2].cpu().numpy().tobytes()


def test_argument_errors_raise_and_launch_nothing():
    x = mel_mags(80)[0]
    n0 = L.launch_count()
    for lifter in (0, 1025):
        with pytest.raises(L.AvcError, match="lifter"):
            V.pitch_shift([x], 5.0, V.AudioParams(ps_lifter=lifter))
    lib = L.load()
    out = torch.empty_like(x)
    r = torch.ones(x.shape[0], device="cuda")
    with pytest.raises(L.AvcError, match="null"):
        L.check(lib.avc_pitch_shift(None, r.data_ptr(), out.data_ptr(), x.shape[0], 1025, 40, None), "avc_pitch_shift")
    with pytest.raises(L.AvcError, match="overlaps"):
        L.check(lib.avc_pitch_shift(x.data_ptr(), r.data_ptr(), x.data_ptr(), x.shape[0], 1025, 40, None), "avc_pitch_shift")
    torch.cuda.synchronize()
    assert L.launch_count() == n0
    with pytest.raises(ValueError, match="pitch shift"):
        V.pitch_shift([x], 24.5)
    with pytest.raises(ValueError, match="pitch shift"):
        V.pitch_shift([x], float("nan"))
    assert L.launch_count() == n0


def test_invalid_ratios_give_nan_rows():
    x = mel_mags(80)[0][:4].contiguous()
    r = torch.tensor([float("nan"), 0.0, -1.0, float("inf")], device="cuda")
    out = torch.empty_like(x)
    L.check(L.load().avc_pitch_shift(x.data_ptr(), r.data_ptr(), out.data_ptr(), 4, 1025, 40, None), "avc_pitch_shift")
    assert torch.isnan(out).all()


# ----------------------------------------------------------------------------- the vocoder
def test_zero_shift_is_the_unchanged_path():
    voc = V.Vocoder(n_mels=512, hp=V.AudioParams(n_iter=8))
    mels = [m for m, _ in voc.wav_to_mel([dev(formant_tone(f, d, phase_seed=i)) for i, (f, d) in
                                          enumerate([(120.0, 0.7), (200.0, 0.5), (150.0, 0.9)])])]
    torch.cuda.synchronize()
    n0 = L.launch_count()
    before = V.deemphasis(V.griffin_lim(voc.mel_to_mag(mels), voc.hp), voc.hp.preemphasis)   # the pre-shift composition
    torch.cuda.synchronize()
    n1 = L.launch_count()
    now = voc.mel_to_signal(mels)
    torch.cuda.synchronize()
    n2 = L.launch_count()
    zero = voc.mel_to_signal(mels, semitones=[0.0, -0.0, 0.0])
    torch.cuda.synchronize()
    assert n2 - n1 == n1 - n0 == L.launch_count() - n2
    for a, b, c in zip(before, now, zero):
        assert a.cpu().numpy().tobytes() == b.cpu().numpy().tobytes() == c.cpu().numpy().tobytes()
    mixed = voc.mel_to_signal(mels, semitones=[0.0, 5.0, 0.0])
    for i in (0, 2):
        assert mixed[i].cpu().numpy().tobytes() == now[i].cpu().numpy().tobytes(), i
    assert mixed[1].numel() == now[1].numel() and not torch.equal(mixed[1], now[1])
    # hp.pitch_shift is the default, and mel_to_wav trims the same synthesis
    shifted = V.Vocoder(n_mels=512, hp=V.AudioParams(n_iter=8, pitch_shift=5.0))
    assert shifted.mel_to_signal([mels[1]])[0].cpu().numpy().tobytes() == mixed[1].cpu().numpy().tobytes()
    w = shifted.mel_to_wav([mels[1]])[0]
    assert w.cpu().numpy().tobytes() == V.trim([mixed[1]], shifted.hp.out_top_db)[0].cpu().numpy().tobytes()


def median_ratio(voc, mel, s, **kw):
    """median F0 of the synthesis shifted by s over the frames voiced in both, over that of the unshifted one."""
    a, b = voc.mel_to_signal([mel, mel], semitones=[0.0, s], **kw)
    (f0a, va), (f0b, vb) = F.track([a, b], SR, HOP)
    both = va & vb
    return float(np.median(f0b[both]) / np.median(f0a[both])), int(both.sum()), len(va)


@pytest.mark.parametrize("s,kw", [(-12.0, {}), (-5.0, {}), (4.0, {}),
                                  (7.0, {"momentum": 0.99}), (-7.0, {"init": "pghi"})])
def test_tracked_pitch_moves_by_the_ratio_at_512_mels(s, kw):
    voc = V.Vocoder(n_mels=512)
    mel = voc.wav_to_mel([dev(formant_tone(150.0, 1.5, vibrato=0.02))])[0][0]
    ratio, voiced, frames = median_ratio(voc, mel, s, **kw)
    print(f"shift {s:+g} {kw}: tracked ratio {ratio:.5f}, want {2 ** (s / 12):.5f}, {voiced}/{frames} frames voiced")
    assert voiced >= 10          # fewer frames track as voiced the larger the shift (DESIGN §4)
    assert abs(ratio / 2 ** (s / 12) - 1.0) <= 0.01


def test_the_shift_preserves_formants_better_than_a_whole_spectrum_warp():
    from adaptive_voice_conversion_b200.mcd import mel_cepstrum
    voc = V.Vocoder(n_mels=512)
    attr = {"mean": np.zeros(512, np.float32), "std": np.ones(512, np.float32)}
    worse = []
    for f0, s in ((140.0, 5.0), (220.0, -7.0)):
        alpha = 2 ** (s / 12)
        src, truth = [m for m, _ in voc.wav_to_mel([dev(formant_tone(f0, 1.0)), dev(formant_tone(alpha * f0, 1.0))])]
        T = min(src.shape[0], truth.shape[0])
        mag = voc.mel_to_mag([src[:T]])[0]
        shifted = V.pitch_shift([mag], s)[0]
        warped = dev(R.whole_warp(mag.cpu().numpy(), float(np.float32(alpha))))
        to_mel = lambda m: V._mel_project(m, voc.fb_t, L.MAG_TO_MEL, voc.hp)  # noqa: E731
        c_truth, c_shift, c_warp = mel_cepstrum([truth[:T], to_mel(shifted), to_mel(warped)], attr)
        d_shift = float((c_shift - c_truth).norm(dim=1).mean())
        d_warp = float((c_warp - c_truth).norm(dim=1).mean())
        print(f"f0 {f0} shift {s:+g}: cepstral distance to the tone at {alpha * f0:.1f} Hz: shifted {d_shift:.4f}, "
              f"whole-spectrum warp {d_warp:.4f}")
        worse.append(d_shift < d_warp)
    assert all(worse)


# ----------------------------------------------------------------------------- matching
def test_match_shifts_moves_a_150_hz_conversion_to_a_220_hz_reference_set():
    voc = V.Vocoder(n_mels=512)
    mels = [m for m, _ in voc.wav_to_mel([dev(formant_tone(150.0, 1.2, vibrato=0.02)),
                                          dev(formant_tone(220.0, 0.9, phase_seed=1, vibrato=0.02)),
                                          dev(formant_tone(220.0, 1.4, phase_seed=2, vibrato=0.02))])]
    hp = voc.hp
    shifts, info = F.match_shifts(voc, [mels[0]], [mels[1:]], hp)
    want = 12 * np.log2(220.0 / 150.0)
    print(f"match: {shifts[0]:.4f} semitones (want {want:.4f}), {info[0]}")
    assert abs(shifts[0] - want) <= 0.1
    assert not info[0]["unmatched"] and not info[0]["clamped"] and info[0]["voiced_conv"] > 0
    ratio, voiced, frames = median_ratio(voc, mels[0], shifts[0])
    print(f"re-synthesis: tracked ratio {ratio:.5f} ({150.0 * ratio:.1f} Hz at 150 Hz), {voiced}/{frames} frames voiced")
    assert voiced >= 10 and abs(ratio / 2 ** (shifts[0] / 12) - 1.0) <= 0.01
    # a reference set with no voiced frame leaves the conversion unmatched
    silent = torch.zeros_like(mels[1])
    shifts, info = F.match_shifts(voc, [mels[0]], [[silent]], hp)
    assert shifts == [0.0] and info[0]["unmatched"] and info[0]["voiced_refs"] == 0


def two_pitch_set(n_mels=512):
    """Two speakers at 110 and 200 Hz, five utterances each, copy-analysed and attr-normalised."""
    voc = V.Vocoder(n_mels=n_mels)
    wavs, keys = [], []
    for s, base in enumerate((110.0, 200.0)):
        for k in range(5):
            wavs.append(formant_tone(base * (1 + 0.03 * k), 0.8 + 0.1 * k, phase_seed=10 * s + k, vibrato=0.02))
            keys.append(f"p{500 + s}_{k:03d}.wav")
    mels = [m.cpu().numpy() for m, _ in voc.wav_to_mel([dev(w) for w in wavs])]
    allm = np.concatenate(mels)
    attr = {"mean": allm.mean(0).astype(np.float32), "std": (allm.std(0) + 1e-2).astype(np.float32)}
    return {k: ((m - attr["mean"]) / attr["std"]).astype(np.float32) for k, m in zip(keys, mels)}, attr


def test_evaluate_f0_match(monkeypatch):
    from adaptive_voice_conversion_b200 import mcd as M
    from adaptive_voice_conversion_b200.config import default_config
    from adaptive_voice_conversion_b200.model import AE

    def converted(model, sources, refs, batch_max=64, codes=None):     # the identity: each conversion is its source
        yield list(range(len(sources))), list(sources)
    monkeypatch.setattr(M, "converted", converted)
    data, attr = two_pitch_set()
    torch.manual_seed(0)
    model = AE(default_config(512)).cuda()
    hp = V.AudioParams(n_iter=32)
    plain = F.evaluate_f0(model, data, attr, per_pair=True, hp=hp)
    res = F.evaluate_f0(model, data, attr, per_pair=True, hp=hp, pitch_shift="match")
    assert json.dumps(res["unshifted"]) == json.dumps(plain)
    ps = res["pitch_shift"]
    print(f"evaluate_f0 match: st_target {plain['st_target']:.4f} -> {res['st_target']:.4f}, {ps}")
    assert ps["mode"] == "match" and ps["n_unmatched"] == 0 and ps["n_clamped"] == 0 and ps["mean_abs_semitones"] > 1
    assert plain["n"] > 4 and res["n"] > 4
    assert res["st_target"] < plain["st_target"]
    assert set(res) - set(plain) == {"pitch_shift", "unshifted"}


def test_pairs_cli_match_with_an_unvoiced_model_changes_no_bit(tmp_path):
    import oracle.ae_oracle as orc
    import yaml
    from scipy.io.wavfile import read, write
    from adaptive_voice_conversion_b200.model import AE
    cfg = orc.default_config(80)
    (tmp_path / "config.yaml").write_text(yaml.safe_dump(cfg))
    m = AE(cfg)
    m.load_state_dict(orc.init_state(cfg, seed=0))
    torch.save(m.state_dict(), tmp_path / "model.ckpt")
    wavs = []
    for i, (f, secs) in enumerate(((120.0, 0.8), (210.0, 1.1), (160.0, 0.9))):
        wavs.append(str(tmp_path / f"w{i}.wav"))
        write(wavs[-1], SR, (formant_tone(f, secs, phase_seed=i) * 32767).astype(np.int16))
    (tmp_path / "pairs.txt").write_text(f"{wavs[0]} {wavs[1]} a\n{wavs[1]} {wavs[2]},{wavs[0]} b\n"
                                        f"{wavs[2]} {wavs[0]} c.npy\n")
    env = dict(os.environ, PYTHONPATH=ROOT)
    base = [sys.executable, os.path.join(ROOT, "inference.py"), "-c", str(tmp_path / "config.yaml"), "-m",
            str(tmp_path / "model.ckpt"), "-gl_iters", "8", "-pairs", str(tmp_path / "pairs.txt")]
    subprocess.run(base + ["-o", str(tmp_path / "plain")], check=True, env=env, cwd=str(tmp_path))
    run = subprocess.run(base + ["-o", str(tmp_path / "match"), "-pitch_shift", "match"], check=True, env=env,
                         cwd=str(tmp_path), capture_output=True, text=True)
    lines = dict(ln.split(": ", 1) for ln in run.stdout.splitlines() if "pitch shift" in ln)
    assert sorted(lines) == ["a.wav", "b.wav"], run.stdout
    print(run.stdout)
    # a random-init model's conversions and the 80-mel copy-syntheses track mostly unvoiced: an unmatched pair gets
    # shift 0, and its wav must be the bits of the run without the flag
    unmatched = [n for n, ln in lines.items() if "unmatched" in ln]
    assert unmatched and all(lines[n].startswith("pitch shift +0.000 semitones") for n in unmatched)
    for name in unmatched:
        assert read(tmp_path / "plain" / name)[1].tobytes() == read(tmp_path / "match" / name)[1].tobytes(), name
    assert np.load(tmp_path / "plain" / "c.npy").tobytes() == np.load(tmp_path / "match" / "c.npy").tobytes()
