"""float64 numpy / scipy restatement of the reference's vocoder DSP (preprocess/tacotron/utils.py get_spectrograms,
melspectrogram2wav and the librosa 0.6/0.7 functions they call), written from the definitions: periodic Hann window
centred in n_fft, center=True reflect-padded STFT, window-sum-square normalised iSTFT, Griffin-Lim, the Slaney mel
filterbank (htk=False, norm=1), its pseudo-inverse as the reference builds it, and librosa's effects.trim.

Pure CPU; used by the tests as the reference the CUDA kernels are checked against.
"""
from __future__ import annotations

import numpy as np

N_FFT, HOP, WIN, SR = 2048, 300, 1200, 24000
TINY = np.finfo(np.float32).tiny


def window(n_fft=N_FFT, win=WIN):
    """Periodic Hann of length win, zero-padded and centred in n_fft."""
    w = np.zeros(n_fft)
    off = (n_fft - win) // 2
    w[off:off + win] = 0.5 - 0.5 * np.cos(2 * np.pi * np.arange(win) / win)
    return w


def _check_len(n, n_fft, what):
    if n < n_fft // 2 + 1:
        raise ValueError(f"{what}: {n} samples, need at least n_fft/2 + 1 = {n_fft // 2 + 1}")


def stft(y, n_fft=N_FFT, hop=HOP, win=WIN):
    """[1 + len(y)//hop, n_fft/2 + 1] complex."""
    y = np.asarray(y, np.float64)
    _check_len(len(y), n_fft, "stft")
    yp = np.pad(y, n_fft // 2, mode="reflect")
    n = 1 + len(y) // hop
    idx = np.arange(n)[:, None] * hop + np.arange(n_fft)[None]
    return np.fft.rfft(yp[idx] * window(n_fft, win), axis=1)


def window_sumsquare(n_frames, n_fft=N_FFT, hop=HOP, win=WIN):
    w2 = window(n_fft, win) ** 2
    ws = np.zeros(n_fft + hop * (n_frames - 1))
    for f in range(n_frames):
        ws[f * hop:f * hop + n_fft] += w2
    return ws


def istft(X, n_fft=N_FFT, hop=HOP, win=WIN):
    """[hop * (n_frames - 1)] samples."""
    X = np.asarray(X)
    n = X.shape[0]
    fr = np.fft.irfft(X, n=n_fft, axis=1) * window(n_fft, win)
    y = np.zeros(n_fft + hop * (n - 1))
    for f in range(n):
        y[f * hop:f * hop + n_fft] += fr[f]
    ws = window_sumsquare(n, n_fft, hop, win)
    nz = ws > TINY
    y[nz] /= ws[nz]
    return y[n_fft // 2:len(y) - n_fft // 2]


def griffin_lim_iteration(X, S, n_fft=N_FFT, hop=HOP, win=WIN):
    E = stft(istft(X, n_fft, hop, win), n_fft, hop, win)
    return S * E / np.maximum(1e-8, np.abs(E))


def griffin_lim(S, n_iter=100, n_fft=N_FFT, hop=HOP, win=WIN):
    S = np.asarray(S, np.float64)
    X = S.astype(np.complex128)
    for _ in range(n_iter):
        X = griffin_lim_iteration(X, S, n_fft, hop, win)
    return istft(X, n_fft, hop, win)


def spectral_convergence(S, y, n_fft=N_FFT, hop=HOP, win=WIN):
    return float(np.linalg.norm(S - np.abs(stft(y, n_fft, hop, win))) / np.linalg.norm(S))


def hz_to_mel(f):
    """Slaney scale: linear below 1 kHz, logarithmic above."""
    f = np.asarray(f, np.float64)
    lin = f / (200.0 / 3)
    return np.where(f >= 1000.0, 15.0 + np.log(np.maximum(f, 1e-300) / 1000.0) / (np.log(6.4) / 27.0), lin)


def mel_to_hz(m):
    m = np.asarray(m, np.float64)
    return np.where(m >= 15.0, 1000.0 * np.exp((np.log(6.4) / 27.0) * (m - 15.0)), (200.0 / 3) * m)


def mel_filterbank(sr=SR, n_fft=N_FFT, n_mels=512):
    """librosa.filters.mel(sr, n_fft, n_mels) with htk=False, norm=1, fmin=0, fmax=sr/2: [n_mels, n_fft/2+1]."""
    fft_f = np.linspace(0, sr / 2, 1 + n_fft // 2)
    mel_f = mel_to_hz(np.linspace(hz_to_mel(0.0), hz_to_mel(sr / 2.0), n_mels + 2))
    fdiff = np.diff(mel_f)
    ramps = mel_f[:, None] - fft_f[None, :]
    w = np.zeros((n_mels, 1 + n_fft // 2))
    for i in range(n_mels):
        lower = -ramps[i] / fdiff[i]
        upper = ramps[i + 2] / fdiff[i + 1]
        w[i] = np.maximum(0, np.minimum(lower, upper))
    w *= (2.0 / (mel_f[2:n_mels + 2] - mel_f[:n_mels]))[:, None]
    return w


def mel_to_linear_matrix(m):
    """M = m^T diag(d), d_j = 1 / colsum_j(m m^T), the colsum itself where |colsum| <= 1e-8: [bins, n_mels]."""
    cs = (m @ m.T).sum(axis=0)
    d = np.array([1.0 / x if np.abs(x) > 1e-8 else x for x in cs])
    return m.T @ np.diag(d)


def frame_power(y, frame=2048, hop=512):
    yp = np.pad(np.asarray(y, np.float64), frame // 2, mode="reflect")
    n = 1 + len(y) // hop
    idx = np.arange(n)[:, None] * hop + np.arange(frame)[None]
    return np.mean(yp[idx] ** 2, axis=1)


def trim_bounds(power, n_samples, top_db, hop=512):
    """[start, end) kept by librosa.effects.trim(ref=max) given the frame powers; (0, 0) when all is silent."""
    db = 10 * np.log10(np.maximum(1e-10, power))
    ref = 10 * np.log10(max(1e-10, float(np.max(power))))
    nz = np.flatnonzero(db - ref > -top_db)
    if nz.size == 0:
        return 0, 0
    return int(nz[0]) * hop, min(n_samples, (int(nz[-1]) + 1) * hop)


def trim(y, top_db, frame=2048, hop=512):
    y = np.asarray(y, np.float64)
    _check_len(len(y), frame, "trim")
    s, e = trim_bounds(frame_power(y, frame, hop), len(y), top_db, hop)
    return y[s:e]


def preemphasis(y, coef=0.97):
    y = np.asarray(y, np.float64)
    return np.append(y[0], y[1:] - coef * y[:-1])


def deemphasis(x, coef=0.97):
    y = np.empty(len(x))
    c = 0.0
    for n, v in enumerate(np.asarray(x, np.float64)):
        c = v + coef * c
        y[n] = c
    return y


def normalize_db(a, max_db=100.0, ref_db=20.0):
    db = 20 * np.log10(np.maximum(1e-5, a))
    return np.clip((db - ref_db + max_db) / max_db, 1e-8, 1)


def get_spectrograms(y, n_mels=512, top_db=15, preemph=0.97, max_db=100.0, ref_db=20.0,
                     sr=SR, n_fft=N_FFT, hop=HOP, win=WIN):
    """y: the loaded signal at sr.  Returns (mel [T, n_mels], mag [T, n_fft/2+1]), normalised."""
    y = trim(y, top_db)
    mag = np.abs(stft(preemphasis(y, preemph), n_fft, hop, win))
    mel = mag @ mel_filterbank(sr, n_fft, n_mels).T
    return normalize_db(mel, max_db, ref_db), normalize_db(mag, max_db, ref_db)


def mel_to_mag(mel, n_mels=None, max_db=100.0, ref_db=20.0, sr=SR, n_fft=N_FFT):
    mel = np.asarray(mel, np.float64)
    amp = 10.0 ** ((np.clip(mel, 0, 1) * max_db - max_db + ref_db) / 20.0)
    M = mel_to_linear_matrix(mel_filterbank(sr, n_fft, n_mels or mel.shape[1]))
    return amp @ M.T


def melspectrogram2wav(mel, n_iter=100, preemph=0.97, max_db=100.0, ref_db=20.0, top_db=60,
                       sr=SR, n_fft=N_FFT, hop=HOP, win=WIN):
    """mel [T, n_mels] normalised -> trimmed waveform (float64)."""
    mag = mel_to_mag(mel, None, max_db, ref_db, sr, n_fft)
    y = deemphasis(griffin_lim(mag, n_iter, n_fft, hop, win), preemph)
    return trim(y, top_db)
