"""Host checks of streaming conversion (adaptive_voice_conversion_b200/streaming.py): the block schedule, its blend
weights, the latency formula by brute force, the float64 RTISI-LA restatement (tests/_rtisi_ref.py) and the CLI's
refusals."""
import os
import subprocess
import sys

import numpy as np
import pytest

import _rtisi_ref as R
from adaptive_voice_conversion_b200 import streaming as S

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
WIN, HOP = 1200, 300


def test_block_schedule_defaults():
    m = 24   # the shipped config's 17 source frames, rounded up to 8
    assert S.block_schedule(0, 128, 8, 8, m) == (0, 8, 0, 24)
    assert S.block_schedule(1, 128, 8, 8, m) == (8, 16, 0, 24)
    assert S.block_schedule(2, 128, 8, 8, m) == (16, 24, 0, 32)
    assert S.block_schedule(14, 128, 8, 8, m) == (112, 120, 0, 128)
    assert S.block_schedule(15, 128, 8, 8, m) == (120, 128, 8, 136)
    assert S.close_window(300, 128) == (172, 300)
    assert S.close_window(30, 128) == (0, 30)


@pytest.mark.parametrize("W,H,LA", [(128, 8, 8), (64, 16, 8), (128, 24, 0), (96, 8, 16)])
def test_schedule_covers_frames_once(W, H, LA):
    m = 24
    for j in range(40):
        b0, b1, w0, w1 = S.block_schedule(j, W, H, LA, m)
        assert b1 - b0 == H and w0 <= b0 and b1 <= w1 and w1 - w0 <= W
        assert w1 >= b1 + LA and w1 >= m
        assert w0 % 8 == 0 and w1 % 8 == 0
        if j:   # the previous window computed the blended frames in its look-ahead
            _, _, _, pe = S.block_schedule(j - 1, W, H, LA, m)
            assert pe >= b0 + min(LA, H)
    # start-up windows are at most W / 8 more lengths
    lens = {S.block_schedule(j, W, H, LA, m)[3] - S.block_schedule(j, W, H, LA, m)[2] for j in range(200)}
    assert len(lens) <= W // 8 + 1


def test_blend_weights():
    w = S.blend_weights(8, 8)
    assert w.dtype == np.float32 and len(w) == 8
    assert np.array_equal(w, np.float32(np.arange(1, 9)) / np.float32(9))
    assert len(S.blend_weights(16, 8)) == 8 and len(S.blend_weights(8, 16)) == 8     # X = min(LA, H)
    assert len(S.blend_weights(8, 0)) == 0


@pytest.mark.parametrize("kw", [dict(hop=12), dict(lookahead=4), dict(window=100), dict(hop=0), dict(window=16, hop=16),
                                dict(gl_lookahead=8), dict(gl_iters=-1)])
def test_params_refused(kw):
    p = S.StreamParams(**kw)
    with pytest.raises(ValueError):
        S.check_params(p, p.window if p.window is not None else 128)


def test_params_accepted_h_above_la():
    S.check_params(S.StreamParams(hop=16, lookahead=8), 128)
    S.check_params(S.StreamParams(hop=8, lookahead=0), 128)


@pytest.mark.parametrize("H,LA,LAv,m", [(8, 8, 3, 24), (16, 8, 0, 24), (8, 0, 7, 24), (8, 16, 3, 64), (24, 8, 5, 24)])
def test_latency_brute_force(H, LA, LAv, m):
    p = S.StreamParams(hop=H, lookahead=LA, gl_lookahead=LAv)

    def released_by(n):   # the frames covering n, the block each is emitted in, and its window's last frame
        c_last = (n + WIN // 2) // HOP
        f = c_last + LAv
        j = f // H
        e = max((j + 1) * H + LA, m)
        return (e - 1) * HOP + WIN // 2 - 1

    worst = max(released_by(n) - n for n in range(0, (m + 8 * H + 20) * HOP))
    assert S.latency_samples(p, WIN, HOP, m) == worst
    if m <= H + LA:   # no start-up windows: the closed form
        assert worst == (H + LA + LAv - 1) * HOP + WIN - 1


@pytest.mark.parametrize("H,LA,LAv,m", [(8, 8, 3, 24), (16, 8, 0, 24), (8, 0, 7, 24), (8, 16, 3, 64)])
def test_latency_by_simulation(H, LA, LAv, m):
    """The pipeline simulated sample by sample, from its rules rather than release_sample: frames analysed once their
    window's last non-zero sample arrives, blocks emitted when their window's frames are analysed, RTISI-LA committing
    a frame once LA_v later frames have entered, a commit of c frames releasing the samples before c hop - win/2.  The
    worst wait over every released sample is latency_samples, and release_sample gives each sample's arrival."""
    p = S.StreamParams(hop=H, lookahead=LA, gl_lookahead=LAv)
    n_in_max = (m + 10 * H + 20) * HOP
    released, block, arrival = 0, 0, {}
    for N in range(1, n_in_max + 1):            # sample N - 1 has just arrived
        frames = 0 if N < WIN // 2 else (N - WIN // 2) // HOP + 1
        while max((block + 1) * H + LA, m) <= frames:
            block += 1
        entered = block * H                     # frames handed to RTISI-LA
        committed = max(0, entered - LAv)
        now = max(0, committed * HOP - WIN // 2)
        for n in range(released, now):
            arrival[n] = N - 1
        released = now
    n_check = released - 20 * HOP                # samples far enough from the end of the simulated input
    worst = max(arrival[n] - n for n in range(n_check))
    assert worst == S.latency_samples(p, WIN, HOP, m)
    for n in range(0, n_check, 7):
        assert arrival[n] == S.release_sample(n, p, WIN, HOP, m), n


def test_latency_defaults():
    # start-up: block 0's window ends at frame m = 24, which its samples wait for
    p = S.StreamParams()
    lat = S.latency_samples(p, WIN, HOP, 24)
    assert lat == 7499, lat                         # 0.312 s at 24 kHz
    assert S.latency_samples(p, WIN, HOP, 16) == (8 + 8 + 3 - 1) * HOP + WIN - 1   # 6599: 0.275 s


def _mags(T=24, seed=0):
    y = R.harmonic(HOP * (T - 1), 24000, seed=seed)
    return R.stft_mag(y, WIN, HOP)[:T]


def test_rtisi_ref_grid_and_first_frame():
    S_ = _mags(12)
    assert len(R.rtisi(S_, WIN, HOP, 2, 3)) == HOP * (12 - 1)
    assert len(R.rtisi(S_[:1], WIN, HOP, 2, 3)) == 0
    # K = 0: frame 0 enters with phase 0 (a zero estimate), its frame is the zero-phase inverse times the window
    st = R.State(WIN, HOP, 3)
    assert len(R.step(st, S_[:1], False, 0)) == 0 and (st.c, st.nbuf) == (0, 1)
    off = (R.NFFT - WIN) // 2
    assert np.allclose(st.fr[0], np.fft.irfft(S_[0], R.NFFT)[off:off + WIN] * R.hann(WIN))
    # samples before 0 are dropped: commits of frames 0 and 1 release nothing, frame 2's the first hop samples
    st = R.State(WIN, HOP, 0)
    assert [len(R.step(st, S_[f:f + 1], False, 1)) for f in range(4)] == [0, 0, HOP, HOP]


def test_rtisi_ref_chunking_invariant():
    S_ = _mags(10, seed=1)
    a = R.rtisi(S_, WIN, HOP, 3, 2, 0.97)
    st = R.State(WIN, HOP, 3)
    parts = [R.step(st, S_[:1], False, 2, 0.97), R.step(st, S_[1:6], False, 2, 0.97), R.step(st, S_[6:], True, 2, 0.97)]
    assert np.array_equal(a, np.concatenate(parts))


def test_rtisi_ref_converges():
    T = 24
    S_ = _mags(T, seed=2)
    sc = {k: R.spectral_convergence(S_, R.rtisi(S_, WIN, HOP, 3, k), WIN, HOP) for k in (0, 8)}
    assert sc[8] < sc[0], sc
    # with a long look-ahead and many iterations it approaches the LSEE fixed point (a consistent spectrogram)
    sc_long = R.spectral_convergence(S_, R.rtisi(S_, WIN, HOP, 12, 24), WIN, HOP)
    assert sc_long < sc[8], (sc_long, sc)


def _cli(*args):
    return subprocess.run([sys.executable, os.path.join(ROOT, "inference.py"), *args], capture_output=True, text=True,
                          cwd=ROOT)


@pytest.mark.parametrize("extra,msg", [
    (["-bank", "b.pt", "-morph", "p1@0"], "-morph"),
    (["-t", "t.wav", "-pitch_shift", "2"], "-pitch_shift"),
    (["-t", "t.wav", "-gl_iters", "50"], "-gl_"),
    (["-t", "t.wav", "-gl_momentum", "0.9"], "-gl_"),
    (["-t", "t.wav", "-gl_init", "pghi"], "-gl_"),
    (["-t", "t.wav", "-stream_hop", "12"], "multiple of 8"),
    (["-t", "t.wav", "-stream_chunk_ms", "0"], "-stream_chunk_ms"),
])
def test_cli_stream_refusals(extra, msg):
    r = _cli("-c", "config.yaml", "-s", "s.wav", "-o", "o.wav", "-stream", *extra)
    assert r.returncode == 2 and msg in r.stderr, r.stderr


def test_cli_stream_needs_wav_output():
    r = _cli("-c", "config.yaml", "-s", "s.wav", "-t", "t.wav", "-o", "o.npy", "-stream")
    assert r.returncode == 2 and "-stream" in r.stderr, r.stderr


def _direct_estimate(st, n0, length, newest):
    """The estimate sample by sample, as the kernel's thread for sample n sums it."""
    win, hop, h = st.win, st.hop, st.win // 2
    w2 = R.hann(win) ** 2
    out = np.zeros(length)
    for i in range(length):
        n = n0 + i
        lo, hi = (n + h - win) // hop + 1, (n + h) // hop
        acc = st.num[n - st.c * hop + h] if 0 <= n - st.c * hop + h < win else 0.0
        for F in range(max(lo, st.c), min(hi, st.c + st.nbuf - 1) + 1):
            acc += st.fr[F][n - F * hop + h]
        wss = sum(w2[n - F * hop + h] for F in range(max(lo, 0), min(hi, newest) + 1))
        out[i] = acc / wss if wss > np.finfo(np.float32).tiny else acc
    return out


def _direct_release(st, n0, length, last, deemph):
    win, hop, h = st.win, st.hop, st.win // 2
    w2 = R.hann(win) ** 2
    out, carry = [], st.carry
    for i in range(length):
        n = n0 + i
        lo, hi = (n + h - win) // hop + 1, (n + h) // hop
        wss = sum(w2[n - F * hop + h] for F in range(max(lo, 0), min(hi, last) + 1))
        x = st.num[n - st.c * hop + h]
        x = x / wss if wss > np.finfo(np.float32).tiny else x
        if n >= 0:
            carry = x + deemph * carry
            out.append(carry)
    return np.asarray(out), carry


@pytest.mark.parametrize("win,hop", [(1200, 300), (2046, 1023), (64, 1)])
def test_rtisi_ref_vectorised_matches_direct_sums(win, hop):
    """The restatement's numpy estimate and release against per-sample sums written out here, on random states at
    the start of a stream (frames before 0 and samples before 0), far into one and past 2^31 samples."""
    rng = np.random.default_rng(win + hop)
    for la in (0, 3, 7):
        for c in (0, 1, 2, 5, 40, 2 ** 31 // hop + 3):
            for nbuf in sorted({0, 1, la, la + 1}):
                st = R.State(win, hop, la)
                st.c, st.nbuf, st.carry = c, nbuf, float(rng.standard_normal())
                st.num = rng.standard_normal(win)
                st.fr = {F: rng.standard_normal(win) for F in range(c, c + nbuf)}
                h = win // 2
                for n0, length, newest in [(c * hop - h, max(nbuf - 1, 0) * hop + win, c + nbuf - 1),
                                           ((c + nbuf) * hop - h, win, c + nbuf - 1)]:
                    got, want = R.estimate(st, n0, length, newest), _direct_estimate(st, n0, length, newest)
                    assert np.allclose(got, want, rtol=1e-12, atol=1e-12 * np.abs(want).max()), (la, c, nbuf, n0)
                for n0, length, last in [(c * hop - h, hop, c), (c * hop - h, max(0, h - hop), c - 1)]:
                    want, carry = _direct_release(st, n0, length, last, 0.97)
                    s2 = st.copy()
                    out = []
                    R._release(s2, n0, length, last, 0.97, out)
                    assert len(out) == len(want) and np.allclose(out, want, rtol=1e-12, atol=1e-12), (la, c, nbuf, n0)
                    assert s2.carry == carry or abs(s2.carry - carry) <= 1e-12 * abs(carry), (s2.carry, carry)


def test_rtisi_refuses_past_int32_frames():
    """avc_rtisi_la's frame counts are int32: an update that would take a stream past 2^31 - 1 frames is refused before
    any count moves (no device is touched: the check precedes the launch's tables)."""
    rt = S.Rtisi.__new__(S.Rtisi)
    rt.hp, rt.la, rt.host = None, 3, {"a": [S.RTISI_MAX_FRAMES - 5, 3]}
    with pytest.raises(ValueError, match="RTISI-LA limit"):
        rt.prepare({"a": np.zeros((3, 1025), np.float32)})
    assert rt.host["a"] == [S.RTISI_MAX_FRAMES - 5, 3]
