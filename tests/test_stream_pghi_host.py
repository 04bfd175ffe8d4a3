"""The streamed PGHI start of RTISI-LA on the host: the float64 restatement (tests/_stream_pghi_ref.py) against offline
PGHI, the latency it adds, StreamParams.gl_init and the CLI, an RTISI-LA run from given spectra against the iSTFT, and
what the start buys on a synthetic signal."""
import os
import subprocess
import sys

import numpy as np
import pytest

import _pghi_ref as P
import _rtisi_ref as R
import _stream_pghi_ref as SP
import oracle.audio_oracle as ao
from adaptive_voice_conversion_b200 import streaming as S

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
WIN, HOP = 1200, 300


def _mags(T, seed=3, crescendo=False):
    y = R.harmonic(HOP * max(T - 1, 1), 24000, seed=seed)
    if crescendo:
        y = y * np.linspace(0.2, 1.0, len(y))
    return R.stft_mag(y, WIN, HOP)[:T]


@pytest.mark.parametrize("T", [1, 2, 5, 40])
def test_early_maximum_equals_offline(T):
    S_ = _mags(T, seed=T)
    S_[min(1, T - 1)] *= 4.0                      # the largest magnitude in frame 0 or 1
    phi, par = SP.stream_pghi(S_, hop=HOP, win=WIN)
    phi_o, par_o = P.pghi_heap(S_, hop=HOP, win=WIN)
    assert np.array_equal(par, par_o)
    d = np.abs(P.wrap(phi - phi_o))
    assert d.max() <= 1e-12, d.max()


def test_crescendo_differs_from_offline():
    S_ = _mags(40, crescendo=True)
    assert S_[:2].max() < S_.max()
    phi, par = SP.stream_pghi(S_, hop=HOP, win=WIN)
    phi_o, par_o = P.pghi_heap(S_, hop=HOP, win=WIN)
    assert not np.array_equal(par, par_o) or np.abs(P.wrap(phi - phi_o)).max() > 1e-6


def test_continued_stream_equals_whole():
    """A stream's frames from f on depend on the earlier ones only through s_max, phi(f-1) and rows f-1: the
    restatement run on all frames equals itself however its output is cut (one definition, no chunk dependence)."""
    S_ = _mags(24, crescendo=True)
    phi, par = SP.stream_pghi(S_, hop=HOP, win=WIN)
    phi2, par2 = SP.stream_pghi(S_[:10], hop=HOP, win=WIN)
    assert np.array_equal(par[:9], par2[:9]) and np.abs(P.wrap(phi[:9] - phi2[:9])).max() <= 1e-12


@pytest.mark.parametrize("H,LA,LAv,m", [(8, 8, 3, 24), (16, 8, 0, 24), (8, 0, 7, 24), (8, 16, 3, 64), (8, 8, 2, 16)])
def test_latency_brute_force(H, LA, LAv, m):
    p = S.StreamParams(hop=H, lookahead=LA, gl_lookahead=LAv, gl_init="pghi")

    def released_by(n):   # n's last covering frame waits for LA_v later frames in RTISI-LA, and its entry for one more
        j = ((n + WIN // 2) // HOP + LAv + 1) // H
        return (max((j + 1) * H + LA, m) - 1) * HOP + WIN // 2 - 1

    worst = max(released_by(n) - n for n in range(0, (m + 8 * H + 20) * HOP))
    assert S.latency_samples(p, WIN, HOP, m) == worst
    if m <= H + LA:
        assert worst == (H + LA + LAv) * HOP + WIN - 1


@pytest.mark.parametrize("H,LA,LAv,m", [(8, 8, 3, 24), (8, 0, 7, 24), (8, 16, 3, 64)])
def test_latency_by_simulation(H, LA, LAv, m):
    """The pipeline sample by sample from its rules: PGHI completes every frame it has but the newest, RTISI-LA commits
    a frame once LA_v later frames have entered it."""
    p = S.StreamParams(hop=H, lookahead=LA, gl_lookahead=LAv, gl_init="pghi")
    released, block, arrival = 0, 0, {}
    for N in range(1, (m + 10 * H + 20) * HOP + 1):
        frames = 0 if N < WIN // 2 else (N - WIN // 2) // HOP + 1
        while max((block + 1) * H + LA, m) <= frames:
            block += 1
        entered = max(0, block * H - 1)
        now = max(0, max(0, entered - LAv) * HOP - WIN // 2)
        for n in range(released, now):
            arrival[n] = N - 1
        released = now
    n_check = released - 20 * HOP
    assert max(arrival[n] - n for n in range(n_check)) == S.latency_samples(p, WIN, HOP, m)
    for n in range(0, n_check, 7):
        assert arrival[n] == S.release_sample(n, p, WIN, HOP, m), n


def test_latency_defaults():
    span = 1504                                   # the tracker's span at 24 kHz (F0Params defaults)
    est, pghi = S.StreamParams(), S.StreamParams(gl_init="pghi")
    assert S.latency_samples(est, WIN, HOP, 24) == S.latency_samples(pghi, WIN, HOP, 24) == 7499
    assert S.latency_samples(est, WIN, HOP, 16) == 6599
    assert S.latency_samples(pghi, WIN, HOP, 16) == 6899
    assert S.tracked_latency_samples(est, WIN, HOP, 24, span) == 8699
    assert S.tracked_latency_samples(pghi, WIN, HOP, 24, span) == 9299
    la2 = S.StreamParams(gl_init="pghi", gl_lookahead=2)
    assert S.latency_samples(la2, WIN, HOP, 16) == 6599
    assert S.tracked_latency_samples(la2, WIN, HOP, 24, span) == 8699


def test_tracked_latency_brute_force():
    """Every output sample's release: its frame c enters the output RTISI-LA at c + LA_v, once frame c + LA_v + 1 is
    shifted, i.e. tracked by YIN, i.e. once the shadow (same schedule and start) has released that frame's span."""
    span, m = 1504, 24
    p = S.StreamParams(gl_init="pghi")
    worst = 0
    for n in range(0, 60 * HOP):
        t = (n + WIN // 2) // HOP + p.gl_lookahead + 1
        last = max(t * HOP + span - span // 2 - 1, span // 2 - t * HOP)
        worst = max(worst, S.release_sample(last, p, WIN, HOP, m) - n)
    assert worst == S.tracked_latency_samples(p, WIN, HOP, m, span)


def test_params():
    S.check_params(S.StreamParams(gl_init="pghi"), 128)
    with pytest.raises(ValueError, match="gl_init"):
        S.check_params(S.StreamParams(gl_init="zero"), 128)
    with pytest.raises(ValueError, match="init"):
        S.Rtisi(None, init="zero")


def test_rtisi_pghi_refuses_past_int32_frames():
    rt = S.Rtisi.__new__(S.Rtisi)
    rt.hp, rt.la, rt.init, rt.host, rt.held = None, 3, "pghi", {"a": [S.RTISI_MAX_FRAMES - 5, 3]}, {"a": 1}
    with pytest.raises(ValueError, match="RTISI-LA limit"):
        rt.prepare({"a": np.zeros((1, 1025), np.float32)})
    assert rt.host["a"] == [S.RTISI_MAX_FRAMES - 5, 3] and rt.held["a"] == 1


def _cli(*args):
    return subprocess.run([sys.executable, os.path.join(ROOT, "inference.py"), *args], capture_output=True, text=True,
                          cwd=ROOT)


def test_cli():
    base = ("-c", "config.yaml", "-s", "s.wav", "-t", "t.wav", "-o", "o.wav")
    r = _cli(*base, "-stream_gl_init", "pghi")
    assert r.returncode == 2 and "-stream_gl_init needs -stream" in r.stderr, r.stderr
    r = _cli(*base, "-stream", "-stream_gl_init", "zero")
    assert r.returncode == 2 and "-stream_gl_init" in r.stderr, r.stderr
    r = _cli(*base, "-stream", "-gl_init", "pghi")
    assert r.returncode == 2 and "-gl_init: -stream synthesises with RTISI-LA" in r.stderr, r.stderr
    sys.path.insert(0, ROOT)
    import inference
    p = inference.parser()
    args = p.parse_args([*base, "-stream", "-stream_gl_init", "pghi"])
    inference.check_stream_args(p, args, [*base, "-stream", "-stream_gl_init", "pghi"])
    assert inference.stream_params(args).gl_init == "pghi"
    assert inference.stream_params(p.parse_args([*base, "-stream"])).gl_init == "estimate"


def test_rtisi_from_k0_is_istft():
    T = 12
    S_ = _mags(T, seed=5)
    X = SP.stream_X(S_, hop=HOP, win=WIN)
    y = SP.rtisi_from(X, S_, WIN, HOP, 3, 0)
    ref = ao.istft(X, hop=HOP, win=WIN)
    assert len(y) == HOP * (T - 1)
    # the restatement's Hann is the kernels' float32 one, the oracle's float64 (7e-8 of the peak apart here)
    assert np.abs(y - ref[:len(y)]).max() <= 1e-6 * np.abs(ref).max()


def _sc_table(n_mels, cases, T=160):
    y = R.harmonic(HOP * (T - 1), 24000, seed=3) * np.linspace(0.2, 1.0, HOP * (T - 1))
    A = R.stft_mag(y, WIN, HOP)
    fb = ao.mel_filterbank(n_mels=n_mels)
    S_ = np.maximum(fb @ A.T, 0).T @ np.linalg.pinv(fb).T
    S_ = np.maximum(S_, 0)
    X = SP.stream_X(S_, hop=HOP, win=WIN)
    out = {}
    for la, K in cases:
        out[("estimate", la, K)] = R.spectral_convergence(S_, R.rtisi(S_, WIN, HOP, la, K), WIN, HOP)
        out[("pghi", la, K)] = R.spectral_convergence(S_, SP.rtisi_from(X, S_, WIN, HOP, la, K), WIN, HOP)
    return out


def test_quality_ordering_512_mels():
    sc = _sc_table(512, [(3, 8), (0, 0)])
    print(sc)
    assert sc[("pghi", 3, 8)] < 0.75 * sc[("estimate", 3, 8)], sc
    assert sc[("pghi", 0, 0)] < 0.9 * sc[("estimate", 3, 8)], sc
