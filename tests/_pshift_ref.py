"""float64 restatement of the formant-preserving pitch shift (avc_pitch_shift, include/avc_b200.h), numpy only.

Per row S of n_bins = 1025 linear magnitudes, N = 2 (n_bins - 1), Q = lifter, alpha = ratio:
  l = ln max(S, 1e-5); c[q] = (1/N) (l[0] + (-1)^q l[-1] + 2 sum_{k=1}^{n_bins-2} l[k] cos(pi q k / (n_bins-1))), q < Q;
  E[k] = c[0] + 2 sum_{q=1}^{Q-1} c[q] cos(pi q k / (n_bins-1)); F = l - E;
  out[k] = exp(E[k] + F~(p)), p = min(float32(k) / float32(alpha) rounded to float32, n_bins - 1), F~ the linear
  interpolation of F at p (F[-1] at p = n_bins - 1).
alpha == 1 gives S itself; alpha not finite or <= 0 gives NaN.  The position p is the kernel's correctly rounded float32
quotient, so the two interpolate at the same point and differ only by the kernel's float32 arithmetic.
"""
import numpy as np

FLOOR = 1e-5
FORMANTS = ((500.0, 120.0, 1.0), (1500.0, 150.0, 0.6), (2600.0, 200.0, 0.35), (3800.0, 250.0, 0.2))


def cos_matrix(Q, n_bins):
    q = np.arange(Q)[:, None]
    k = np.arange(n_bins)[None, :]
    return np.cos(np.pi * ((q * k) % (2 * (n_bins - 1))) / (n_bins - 1))


def cepstrum(ell, Q):
    """c[q], q < Q, of the even extension of each row of ell [rows, n_bins] (float64)."""
    ell = np.atleast_2d(np.asarray(ell, np.float64))
    n_bins = ell.shape[1]
    N = 2 * (n_bins - 1)
    cm = cos_matrix(Q, n_bins)
    sign = (-1.0) ** np.arange(Q)
    return (ell[:, :1] + sign[None, :] * ell[:, -1:] + 2.0 * ell[:, 1:-1] @ cm[:, 1:-1].T) / N


def envelope(c, n_bins):
    c = np.atleast_2d(np.asarray(c, np.float64))
    cm = cos_matrix(c.shape[1], n_bins)
    return c[:, :1] + 2.0 * c[:, 1:] @ cm[1:]


def positions(alpha, n_bins):
    """(i0, frac) of p = min(fl32(k / alpha), n_bins - 1) for every bin k."""
    k = np.arange(n_bins, dtype=np.float32)
    p = np.minimum(k / np.float32(alpha), np.float32(n_bins - 1)).astype(np.float64)
    i0 = np.floor(p).astype(np.int64)
    return i0, p - i0


def interpolate(F, alpha):
    n_bins = F.shape[-1]
    i0, fr = positions(alpha, n_bins)
    i1 = np.minimum(i0 + 1, n_bins - 1)
    return F[..., i0] + fr * (F[..., i1] - F[..., i0])


def split(S, lifter):
    """(l, E, F) of each row of S [rows, n_bins]."""
    ell = np.log(np.maximum(np.atleast_2d(np.asarray(S, np.float64)), FLOOR))
    E = envelope(cepstrum(ell, lifter), ell.shape[1])
    return ell, E, ell - E


def pitch_shift(S, ratio, lifter=40):
    """out [rows, n_bins] float64 of S [rows, n_bins] with per-row ratios (a scalar applies to every row)."""
    S = np.atleast_2d(np.asarray(S, np.float64))
    ratio = np.broadcast_to(np.asarray(ratio, np.float64), (S.shape[0],))
    ell, E, F = split(S, lifter)
    out = np.empty_like(S)
    for r, a in enumerate(ratio):
        if a == 1.0:
            out[r] = S[r]
        elif not np.isfinite(a) or a <= 0:
            out[r] = np.nan
        else:
            out[r] = np.exp(E[r] + interpolate(F[r], a))
    return out


def whole_warp(S, ratio):
    """S[k / alpha] linearly interpolated, no envelope split: the spectrum warp a formant-preserving shift improves on."""
    S = np.atleast_2d(np.asarray(S, np.float64))
    return interpolate(S, ratio)


def formant_tone(f0, seconds, phase_seed=0, vibrato=0.0, sr=24000):
    """Harmonics of f0 (Hz, with an optional 5 Hz vibrato of relative depth `vibrato`) up to 8 kHz whose amplitudes
    follow a fixed envelope in Hz (four resonances over a floor): the formants do not depend on f0.  float32."""
    t = np.arange(int(round(seconds * sr))) / sr
    inst = f0 * (1.0 + vibrato * np.sin(2 * np.pi * 5.0 * t))
    phi = np.concatenate([[0.0], np.cumsum((inst[1:] + inst[:-1]) / 2.0) / sr])
    rng = np.random.default_rng(phase_seed)
    y = np.zeros_like(t)
    for k in range(1, int(8000.0 // (f0 * (1 + vibrato))) + 1):
        f = k * inst
        amp = 0.02 + sum(g / (1.0 + ((f - c) / b) ** 2) for c, b, g in FORMANTS)
        y += amp * np.sin(2 * np.pi * k * phi + rng.uniform(0, 2 * np.pi))
    return (0.5 * y / np.abs(y).max()).astype(np.float32)
