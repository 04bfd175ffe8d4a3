"""float64 restatement of the speaker probes (adaptive_voice_conversion_b200/speaker_probe.py, csrc/probe.cu): frame
rows, standardisation, the MLP's forward and backward passes, the cross-entropy with its rank rule, Adam and the frame
vote."""
import math

import numpy as np


def frames64(x, lengths, row_off, n_rows):
    """out[row_off[b] + t] = x[b, :, t] for t < lengths[b] of a padded [B, C, T] batch."""
    out = np.full((n_rows, x.shape[1]), np.nan, np.float32)
    for b, n in enumerate(lengths):
        out[row_off[b]:row_off[b] + n] = x[b, :, :n].T
    return out


def moments64(x):
    """(mean, std) float64 per column, added in ascending row order; std 0 -> 1."""
    x = np.asarray(x, np.float64)
    n = len(x)
    mean = np.cumsum(x, axis=0)[-1] / n
    var = np.cumsum((x - mean) ** 2, axis=0)[-1] / n
    std = np.sqrt(var)
    return mean, np.where(std == 0.0, 1.0, std)


def standardize64(x, mean, std):
    return ((np.asarray(x, np.float64) - mean) / std).astype(np.float32)


def rank_of(scores, y):
    """#{j : s_j > s_y, or s_j == s_y and j < y}."""
    s = np.asarray(scores)
    return int((s > s[y]).sum() + (s[:y] == s[y]).sum())


def log_softmax64(z):
    z = np.asarray(z, np.float64)
    m = z.max(axis=-1, keepdims=True)
    return z - m - np.log(np.exp(z - m).sum(axis=-1, keepdims=True))


def xent64(z, labels, scale=1.0):
    """(loss [R], dlogits [R, S], rank [R]) in float64."""
    z = np.asarray(z, np.float64)
    ls = log_softmax64(z)
    R = len(z)
    loss = -ls[np.arange(R), labels]
    d = np.exp(ls)
    d[np.arange(R), labels] -= 1.0
    return loss, d * scale, np.array([rank_of(z[r], labels[r]) for r in range(R)], np.int32)


def vote64(z, offsets, labels):
    """(scores [U, S], rank [U]): the sum of each utterance's rows' log-softmax, ascending rows."""
    ls = log_softmax64(z)
    U = len(offsets) - 1
    scores = np.zeros((U, z.shape[1]))
    for u in range(U):
        for r in range(offsets[u], offsets[u + 1]):
            scores[u] += ls[r]
    return scores, np.array([rank_of(scores[u], labels[u]) for u in range(U)], np.int32)


def forward64(P, x):
    """(h1, h2, z) of the MLP with P = [W1, b1, W2, b2, W3, b3] (float64)."""
    W1, b1, W2, b2, W3, b3 = P
    h1 = np.maximum(x @ W1.T + b1, 0.0)
    h2 = np.maximum(h1 @ W2.T + b2, 0.0)
    return h1, h2, h2 @ W3.T + b3


def loss64(P, x, labels):
    """The mean cross-entropy of the MLP on (x, labels)."""
    return float(xent64(forward64(P, x)[2], labels)[0].mean())


def grads64(P, x, labels):
    """The gradients of loss64 with respect to P."""
    W1, b1, W2, b2, W3, b3 = P
    h1, h2, z = forward64(P, x)
    dz = xent64(z, labels, 1.0 / len(x))[1]
    dh2 = (dz @ W3) * (h2 > 0)
    dh1 = (dh2 @ W2) * (h1 > 0)
    return [dh1.T @ x, dh1.sum(0), dh2.T @ h1, dh2.sum(0), dz.T @ h2, dz.sum(0)]


def adam64(P, G, m, v, t, lr=1e-3, b1=0.9, b2=0.999, eps=1e-8):
    """One Adam step (no weight decay, no amsgrad) at step t (1-based); returns (P, m, v)."""
    m = [b1 * mi + (1 - b1) * g for mi, g in zip(m, G)]
    v = [b2 * vi + (1 - b2) * g * g for vi, g in zip(v, G)]
    bc1, bc2 = 1 - b1 ** t, 1 - b2 ** t
    P = [p - (lr / bc1) * mi / (np.sqrt(vi) / math.sqrt(bc2) + eps) for p, mi, vi in zip(P, m, v)]
    return P, m, v


def train64(P, x, labels, order_batches, lr=1e-3):
    """The parameters after one Adam step per batch of row indices in order_batches, from P."""
    P = [np.asarray(p, np.float64) for p in P]
    m = [np.zeros_like(p) for p in P]
    v = [np.zeros_like(p) for p in P]
    for t, rows in enumerate(order_batches, 1):
        G = grads64(P, x[rows], labels[rows])
        P, m, v = adam64(P, G, m, v, t, lr)
    return P
