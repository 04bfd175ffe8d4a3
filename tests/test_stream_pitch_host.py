"""Host checks of the streamed pitch stage (adaptive_voice_conversion_b200/streaming.py): the causal shift rule against
hand-worked cases and the float64 restatement (tests/_stream_pitch_ref.py), tracked_latency_samples by brute force and
by simulation, the pitch settings open() accepts, and the CLI's -stream_pitch refusals."""
import math
import os
import subprocess
import sys

import numpy as np
import pytest
import torch

import _stream_pitch_ref as R
from adaptive_voice_conversion_b200 import streaming as S
from adaptive_voice_conversion_b200.f0 import F0Params

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
WIN, HOP, SR = 1200, 300, 24000
P = F0Params()
SPAN = P.win + P.tau_max(SR)      # 1504


def tracker(mode, mu, sd, warmup):
    return S.PitchTracker(mode, mu, sd, warmup, SR, P)


def both(mode, mu, sd, warmup, tau, ap, en):
    """PitchTracker's shifts (fed in two parts) and the restatement's, which must agree exactly here."""
    tau, ap, en = (np.asarray(v, np.float64) for v in (tau, ap, en))
    tr = tracker(mode, mu, sd, warmup)
    k = len(tau) // 2
    a, b = tr.update(tau[:k], ap[:k], en[:k]), tr.update(tau[k:], ap[k:], en[k:])
    got = [np.concatenate([x, y]) for x, y in zip(a, b)]
    ref = R.shifts(tau, ap, en, mode, mu, sd, warmup, SR, P.theta(), P.silence_db)
    assert np.array_equal(got[1], ref[1])
    np.testing.assert_allclose(got[2], ref[2], rtol=0, atol=1e-12)
    return got[2]


def test_warmup_then_range():
    # f0 100, 200, 400 Hz: l = a, a + 1, a + 2 with a = log2(100); warm-up of 3 voiced frames, target (8, 0.5)
    a = math.log2(100.0)
    s = both("mv", 8.0, 0.5, 3, [240.0, 120.0, 60.0], [0.01] * 3, [1.0] * 3)
    assert s[0] == pytest.approx(12 * (8 - a), abs=1e-12)
    assert s[1] == pytest.approx(12 * (8 - (a + 0.5)), abs=1e-12)
    sd_c = math.sqrt(2.0 / 3.0)                  # of a, a + 1, a + 2 about a + 1
    assert s[2] == pytest.approx(12 * (8 + 0.5 / sd_c * 1.0 - (a + 2)), abs=1e-12)
    # match never scales the range
    m = both("match", 8.0, 0.5, 3, [240.0, 120.0, 60.0], [0.01] * 3, [1.0] * 3)
    assert m[2] == pytest.approx(12 * (8 - (a + 1)), abs=1e-12)


def test_unvoiced_hold_and_zero_before_first_voiced():
    a = math.log2(200.0)
    # unvoiced (aperiodic), voiced, unvoiced (aperiodic), unvoiced (silent: energy 0), voiced
    s = both("match", 7.5, 0.2, 1, [120.0] * 5, [0.5, 0.01, 0.5, 0.01, 0.01], [1.0, 1.0, 1.0, 0.0, 1.0])
    assert s[0] == 0.0
    assert s[1] == pytest.approx(12 * (7.5 - a), abs=1e-12)
    assert s[2] == s[1] and s[3] == s[1]
    assert s[4] == pytest.approx(12 * (7.5 - a), abs=1e-12)


def test_running_silence_floor():
    # frame 0 is voiced against its own energy; frame 2 is 50 dB below the running maximum: unvoiced, held
    tr = tracker("match", 7.0, 0.1, 1)
    _, voiced, s = tr.update(np.array([120.0, 240.0, 60.0]), np.full(3, 0.01), np.array([1e-6, 1.0, 1e-5]))
    assert voiced.tolist() == [True, True, False]
    assert s[2] == s[1]


def test_clamp():
    s = both("match", 12.0, 0.1, 1, [240.0], [0.01], [1.0])      # 12 (12 - log2 100) = 64 semitones
    assert s[0] == 24.0
    s = both("match", 3.0, 0.1, 1, [240.0], [0.01], [1.0])
    assert s[0] == -24.0


def test_zero_sigma_is_mean_only():
    # every voiced l equal: sigma_c = 0 keeps mv on the mean shift past the warm-up
    a = math.log2(200.0)
    s = both("mv", 7.0, 0.3, 1, [120.0] * 6, [0.01] * 6, [1.0] * 6)
    np.testing.assert_allclose(s, 12 * (7.0 - a), rtol=0, atol=1e-12)


def test_random_tracks_match_restatement():
    rng = np.random.default_rng(0)
    for trial in range(20):
        T = int(rng.integers(1, 400))
        tau = rng.uniform(48, 480, T)
        ap = np.where(rng.random(T) < 0.7, rng.uniform(0, 0.09, T), rng.uniform(0.1, 1, T))
        en = rng.uniform(0, 1, T) ** 6 * (rng.random(T) < 0.95)
        mode = ("match", "mv")[trial % 2]
        mu, sd, warm = float(rng.uniform(6, 9)), float(rng.uniform(0, 0.5)), int(rng.integers(1, 60))
        ref = R.shifts(tau, ap, en, mode, mu, sd, warm, SR, P.theta(), P.silence_db)
        tr = tracker(mode, mu, sd, warm)
        cuts = np.sort(rng.integers(0, T + 1, 5))
        parts = [tr.update(tau[a:b], ap[a:b], en[a:b]) for a, b in zip([0, *cuts], [*cuts, T])]
        got = [np.concatenate(x) for x in zip(*parts)]
        assert np.array_equal(got[1], ref[1])
        np.testing.assert_array_equal(np.isnan(got[0]), np.isnan(ref[0]))
        assert np.abs(got[2] - ref[2]).max() <= 1e-9, trial


@pytest.mark.parametrize("pitch,want", [(None, None), (0, None), (0.0, None), (3, 3.0), (-24.0, -24.0),
                                        (("mv", 7.5, 0.2), ("mv", 7.5, 0.2)), (["match", 7, 0], ("match", 7.0, 0.0))])
def test_parse_pitch(pitch, want):
    assert S.parse_pitch(pitch) == want


@pytest.mark.parametrize("pitch", [24.5, float("nan"), float("inf"), True, "mv", ("mv", 7.0), ("up", 7.0, 0.1),
                                   ("mv", float("nan"), 0.1), ("mv", 7.0, -0.1), ("match", None, 0.1)])
def test_parse_pitch_refused(pitch):
    with pytest.raises(ValueError):
        S.parse_pitch(pitch)


def test_warmup_param_refused():
    with pytest.raises(ValueError):
        S.check_params(S.StreamParams(pitch_warmup=0), 128)


def test_yin_ready():
    half = SPAN // 2
    assert S.yin_ready(half, HOP, SPAN) == 0 and S.yin_ready(half + 1, HOP, SPAN) == 1   # frame 0 reflects to `half`
    for n in range(0, 5000, 7):
        want = sum(1 for t in range(40) if max(abs(t * HOP - half), t * HOP - half + SPAN - 1) < n)
        assert S.yin_ready(n, HOP, SPAN) == want, n


@pytest.mark.parametrize("H,LA,LAv,m", [(8, 8, 3, 24), (16, 8, 0, 24), (8, 0, 7, 24), (8, 16, 3, 64), (24, 8, 5, 24)])
def test_tracked_latency_brute_force(H, LA, LAv, m):
    p = S.StreamParams(hop=H, lookahead=LA, gl_lookahead=LAv)
    half = SPAN // 2

    def released_by(n):
        c = (n + WIN // 2) // HOP                 # n's last covering frame, committed once frame t enters
        t = c + LAv
        need = max(abs(t * HOP - half), t * HOP - half + SPAN - 1)
        c_sh = next(k for k in range(10 ** 6) if k * HOP - WIN // 2 > need)   # shadow frames committed to release it
        f = c_sh - 1 + LAv
        j = f // H
        return (max((j + 1) * H + LA, m) - 1) * HOP + WIN // 2 - 1

    worst = max(released_by(n) - n for n in range(0, (m + 8 * H + 30) * HOP, 3))
    assert S.tracked_latency_samples(p, WIN, HOP, m, SPAN) == worst
    if m <= H + LA:   # no start-up windows: untracked plus D = LAv + 4 frames
        assert worst == (H + LA + 2 * LAv + 4 - 1) * HOP + WIN - 1


@pytest.mark.parametrize("H,LA,LAv,m", [(8, 8, 3, 24), (16, 8, 0, 24), (8, 0, 7, 24), (8, 16, 3, 64)])
def test_tracked_latency_by_simulation(H, LA, LAv, m):
    """The pipeline simulated sample by sample from its rules: blocks emitted as their windows are analysed, the shadow
    committing a frame once LA_v later ones have entered and releasing the samples before c hop - win/2, a YIN frame
    tracked once every sample it reads (one reflection at 0) is released, the output entering tracked frames only."""
    p = S.StreamParams(hop=H, lookahead=LA, gl_lookahead=LAv)
    half = SPAN // 2
    n_in_max = (m + 10 * H + 30) * HOP
    released, block, tracked, arrival = 0, 0, 0, {}
    for N in range(1, n_in_max + 1):
        frames = 0 if N < WIN // 2 else (N - WIN // 2) // HOP + 1
        while max((block + 1) * H + LA, m) <= frames:
            block += 1
        entered = block * H
        sh = max(0, max(0, entered - LAv) * HOP - WIN // 2)          # shadow samples released
        while tracked < entered and max(abs(tracked * HOP - half), tracked * HOP - half + SPAN - 1) < sh:
            tracked += 1
        now = max(0, max(0, tracked - LAv) * HOP - WIN // 2)
        for n in range(released, now):
            arrival[n] = N - 1
        released = now
    n_check = released - 20 * HOP
    worst = max(arrival[n] - n for n in range(n_check))
    assert worst == S.tracked_latency_samples(p, WIN, HOP, m, SPAN)
    for n in range(0, n_check, 7):
        assert arrival[n] == S.tracked_release_sample(n, p, WIN, HOP, m, SPAN), n


def test_tracked_latency_defaults():
    p = S.StreamParams()
    # without start-up windows the tracking adds D = 7 frames, 2 100 samples, to the steady-state 6 599
    assert S.tracked_latency_samples(p, WIN, HOP, 16, SPAN) - S.latency_samples(p, WIN, HOP, 16) == 7 * HOP
    # with the shipped config (m = 24) the untracked worst case is start-up's 7 499; the tracked one is steady state's
    # 6 599 + 2 100 = 8 699 (0.362 s at 24 kHz): the first block's wait for m frames hides part of D
    assert S.latency_samples(p, WIN, HOP, 24) == 7499
    assert S.tracked_latency_samples(p, WIN, HOP, 24, SPAN) == 8699


def _cli(*args):
    return subprocess.run([sys.executable, os.path.join(ROOT, "inference.py"), *args], capture_output=True, text=True,
                          cwd=ROOT)


@pytest.mark.parametrize("extra,msg", [
    (["-t", "t.wav", "-stream_pitch", "mv"], "-stream_pitch needs -stream"),
    (["-t", "t.wav", "-stream", "-stream_pitch", "25"], "-stream_pitch"),
    (["-t", "t.wav", "-stream", "-stream_pitch", "nan"], "-stream_pitch"),
    (["-t", "t.wav", "-stream", "-stream_pitch", "up"], "-stream_pitch"),
    (["-t", "t.wav", "-stream", "-pitch_shift", "3"], "-stream_pitch"),
])
def test_cli_stream_pitch_refusals(extra, msg):
    r = _cli("-c", "config.yaml", "-s", "s.wav", "-o", "o.wav", *extra)
    assert r.returncode == 2 and msg in r.stderr, r.stderr


@pytest.mark.parametrize("mode", ["mv", "match"])
def test_cli_stream_pitch_needs_profiled_bank(tmp_path, mode):
    bank = tmp_path / "bank.pt"
    torch.save({"speakers": ["p1"], "codes": torch.zeros(1, 128)}, str(bank))
    r = _cli("-c", "config.yaml", "-s", "s.wav", "-o", "o.wav", "-bank", str(bank), "-speaker", "p1", "-stream",
             "-stream_pitch", mode)
    assert r.returncode == 2 and "pitch profiles" in r.stderr, r.stderr
    err = r.stderr.strip().splitlines()[-1]      # the error line, after argparse's usage text
    assert f"which -stream_pitch {mode} needs" in err and "-pitch_shift" not in err, err


def test_stream_profiles_refuses_short_reference():
    """A -t reference too short for the tracker is named before anything is synthesised."""
    import importlib.util
    import types
    from adaptive_voice_conversion_b200.vocoder import AudioParams
    spec = importlib.util.spec_from_file_location("inference_cli", os.path.join(ROOT, "inference.py"))
    cli = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(cli)
    hp = AudioParams()
    need = P.min_samples(hp.sr)
    T = 1 + need // hp.hop_length              # hop (T - 1) < need
    jobs = [(None, "s.wav", "short.wav", "o.wav")]
    with pytest.raises(ValueError, match=f"short.wav: .*{hp.hop_length * (T - 1)} samples.*at least {need}"):
        cli.stream_profiles(jobs, {"short.wav": torch.zeros(T, 80)}, None, types.SimpleNamespace(hp=hp),
                            S.StreamParams())
