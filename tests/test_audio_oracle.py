"""CPU: the float64 vocoder oracle (oracle/audio_oracle.py) pinned on scipy and on librosa's published constants.

The reference's own DSP needs librosa and tensorflow, so no fixture can come from it; these identities are what
ties the oracle to the reference's definitions."""
import numpy as np
import pytest
import scipy.signal as ss

import oracle.audio_oracle as ao


def signal(n, seed=0):
    return np.random.default_rng(seed).standard_normal(n)


@pytest.mark.parametrize("n,hop,win", [(24000 + 137, 300, 1200), (2048, 300, 1200), (5000, 256, 2048), (4800, 300, 600)])
def test_stft_equals_scipy(n, hop, win):
    """scipy's 'even' boundary extension is numpy 'reflect'; scipy scales by 1 / window.sum() (and refuses signals
    shorter than the window)."""
    y = signal(n)
    w = ao.window(2048, win)
    X = ao.stft(y, 2048, hop, win)
    _, _, Z = ss.stft(y, window=w, nperseg=2048, noverlap=2048 - hop, boundary="even", padded=False)
    Z = Z.T * w.sum()
    assert X.shape == (1 + n // hop, 1025)
    assert np.abs(X - Z[:X.shape[0]]).max() <= 1e-12 * np.abs(X).max()


@pytest.mark.parametrize("n,hop,win", [(24000 + 137, 300, 1200), (1025, 300, 1200), (7001, 512, 2048), (3000, 150, 300)])
def test_istft_of_stft_is_identity_including_the_ends(n, hop, win):
    y = signal(n, 1)
    z = ao.istft(ao.stft(y, 2048, hop, win), 2048, hop, win)
    m = hop * (1 + n // hop - 1)
    assert len(z) == m
    assert np.abs(z - y[:m]).max() < 1e-10


def test_window_is_periodic_hann_centred():
    w = ao.window(2048, 1200)
    nz = np.flatnonzero(w)
    assert nz[0] == 425 and nz[-1] == 1623 and w[424] == 0.0     # w[0] of the Hann is 0, so offset 424 is zero
    assert abs(w[424 + 600] - 1.0) < 1e-15


def test_mel_scale_anchors():
    assert abs(float(ao.hz_to_mel(60.0)) - 0.9) < 1e-12
    assert abs(float(ao.hz_to_mel(1000.0)) - 15.0) < 1e-12
    assert abs(float(ao.hz_to_mel(6400.0)) - 42.0) < 1e-12
    f = np.array([0.0, 500.0, 1000.0, 4000.0, 12000.0])
    assert np.allclose(ao.mel_to_hz(ao.hz_to_mel(f)), f, rtol=1e-13, atol=1e-12)


@pytest.mark.parametrize("n_mels", [80, 512])
def test_mel_filterbank_shape_and_peaks(n_mels):
    fb = ao.mel_filterbank(24000, 2048, n_mels)
    assert fb.shape == (n_mels, 1025) and (fb >= 0).all()
    mel_f = ao.mel_to_hz(np.linspace(ao.hz_to_mel(0.0), ao.hz_to_mel(12000.0), n_mels + 2))
    peak = 2.0 / (mel_f[2:] - mel_f[:-2])
    assert (fb.max(axis=1) <= peak * (1 + 1e-12)).all()
    # the narrowest triangle (13.3 Hz wide at 512 mels) is wider than the 11.7 Hz bin spacing: no filter is empty
    assert (fb.max(axis=1) > 0).all()


def test_mel_to_linear_matrix_keeps_the_colsum_of_empty_filters():
    fb = ao.mel_filterbank(24000, 2048, 512)
    M = ao.mel_to_linear_matrix(fb)
    cs = (fb @ fb.T).sum(axis=0)
    assert M.shape == (1025, 512)
    full = np.abs(cs) > 1e-8
    assert np.allclose(M[:, full], fb.T[:, full] / cs[full], rtol=1e-12, atol=0)
    assert np.array_equal(M[:, ~full], fb.T[:, ~full] * cs[~full])


@pytest.mark.parametrize("onset,top_db", [(12345, 15), (12800, 15), (12345, 60)])
def test_trim_finds_burst_edges(onset, top_db):
    """Frame f is centred on sample 512 f and spans 1024 either side.  The kept range starts at the first frame
    that hears enough of the burst: on the 512 grid, at most one hop before the first frame that reaches the onset
    and never after the onset; the end mirrors it."""
    sr = 24000
    burst = 0.5 * np.sin(2 * np.pi * 440 * np.arange(sr) / sr)
    n = onset + sr + 20000
    y = np.zeros(n)
    y[onset:onset + sr] = burst
    y += 1e-6 * signal(n, 2)
    z = ao.trim(y, top_db)
    s, e = ao.trim_bounds(ao.frame_power(y), len(y), top_db)
    assert np.array_equal(z, y[s:e])
    first_reach = (onset - 1024) // 512 * 512 + 512          # first grid point whose frame covers the onset
    assert s % 512 == 0 and first_reach - 512 <= s <= onset
    last_reach = (onset + sr + 1024 - 1) // 512 * 512 + 512  # end of the last frame that covers the burst's last sample
    assert onset + sr <= e <= last_reach and (e - (onset + sr)) <= 1024 + 512


def test_trim_bounds_all_silent_and_one_frame():
    assert ao.trim_bounds(np.zeros(5), 2500, 60) == (0, 2500)   # power == max everywhere: nothing is below it
    p = np.full(10, 1e-12)
    p[4] = 1.0
    assert ao.trim_bounds(p, 5000, 15) == (4 * 512, 5 * 512)


def test_deemphasis_equals_lfilter_and_inverts_preemphasis():
    x = signal(20000, 3)
    assert np.abs(ao.deemphasis(x) - ss.lfilter([1.0], [1.0, -0.97], x)).max() < 1e-11
    assert np.abs(ao.deemphasis(ao.preemphasis(x)) - x).max() < 1e-11


@pytest.mark.parametrize("coef", [0.0, 0.5, 0.999, 1.0, -0.97])
def test_deemphasis_equals_lfilter_at_other_coefficients(coef):
    """tests/test_gpu_vocoder_kernels.py checks avc_deemphasis against lfilter at these coefficients."""
    x = signal(20000, 4)
    ref = ss.lfilter([1.0], [1.0, -coef], x)
    assert np.abs(ao.deemphasis(x, coef) - ref).max() <= 1e-11 * max(1.0, np.abs(ref).max())


def test_too_short_is_rejected():
    with pytest.raises(ValueError, match="n_fft/2"):
        ao.stft(np.zeros(1024))
    ao.stft(np.zeros(1025))


def test_griffin_lim_reduces_spectral_convergence():
    y = np.sin(2 * np.pi * 220 * np.arange(6000) / 24000) * np.hanning(6000)
    S = np.abs(ao.stft(y))
    sc0 = ao.spectral_convergence(S, ao.griffin_lim(S, 0))
    sc = ao.spectral_convergence(S, ao.griffin_lim(S, 20))
    assert sc < 0.5 * sc0
