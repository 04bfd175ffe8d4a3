"""float64 restatement of the MCD-DTW definition (adaptive_voice_conversion_b200/mcd.py, include/avc_b200.h): the
cepstrum from its formula, and the DTW as an anti-diagonal numpy loop that adds in exactly the order the kernel does."""
import math

import numpy as np

MCD_SCALE = 10.0 * math.sqrt(2.0) / math.log(10.0)


def cepstrum64(x, mean, std, dims, max_db=100.0, ref_db=20.0):
    """[T, n_mels] float32 attr-normalised frames -> [T, dims] float64."""
    x = np.asarray(x, np.float32)
    a = np.clip(x * np.asarray(std, np.float32) + np.asarray(mean, np.float32), 0.0, 1.0)     # float32, like the vocoder
    ell = (a.astype(np.float64) * max_db - max_db + ref_db) * (math.log(10.0) / 20.0)
    N = x.shape[1]
    m = np.arange(N, dtype=np.float64)
    c = np.empty((x.shape[0], dims))
    for k in range(1, dims + 1):
        c[:, k - 1] = (ell * (math.sqrt(2.0 / N) * np.cos(math.pi * k * (2.0 * m + 1.0) / (2.0 * N)))).sum(axis=1)
    return c


def dist_rows(X, Y):
    """d between matched rows of X and Y (float32 -> float64), terms added in ascending k, one at a time."""
    X, Y = np.asarray(X, np.float64), np.asarray(Y, np.float64)
    acc = np.zeros(X.shape[0])
    for k in range(X.shape[1]):
        t = X[:, k] - Y[:, k]
        acc = acc + t * t
    return np.sqrt(acc)


def dtw64(X, Y):
    """(S, L) at (Tx-1, Ty-1): anti-diagonals in order, ties preferring (i-1,j-1), then (i-1,j), then (i,j-1)."""
    X, Y = np.asarray(X, np.float32), np.asarray(Y, np.float32)
    Tx, Ty = len(X), len(Y)
    S = np.full((Tx, Ty), np.nan)
    Ln = np.zeros((Tx, Ty), np.int64)
    for g in range(Tx + Ty - 1):
        i = np.arange(max(0, g - (Ty - 1)), min(g, Tx - 1) + 1)
        j = g - i
        d = dist_rows(X[i], Y[j])
        best = np.full(len(i), np.inf)
        bl = np.zeros(len(i), np.int64)
        have = np.zeros(len(i), bool)
        for di, dj in ((1, 1), (1, 0), (0, 1)):
            ok = (i >= di) & (j >= dj)
            v = np.where(ok, S[np.maximum(i - di, 0), np.maximum(j - dj, 0)], np.inf)
            take = ok & (~have | (v < best))
            best = np.where(take, v, best)
            bl = np.where(take, Ln[np.maximum(i - di, 0), np.maximum(j - dj, 0)], bl)
            have |= ok
        S[i, j] = np.where(have, d + best, d)
        Ln[i, j] = bl + 1
    return float(S[-1, -1]), int(Ln[-1, -1])


def mcd64(X, Y):
    S, Ln = dtw64(X, Y)
    return MCD_SCALE * S / Ln
