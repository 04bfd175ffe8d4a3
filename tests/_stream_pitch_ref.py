"""Float64 restatement of the streamed pitch stage's shift rule (streaming.PitchTracker), frame by frame from the
tracker's outputs, with the profile of every prefix recomputed in two passes rather than updated.

Frame t is voiced when aperiodicity < theta, energy > 0 and 10 log10(energy / max(energy[0..t])) >= -silence_db.  Its
l = log2(sr / tau).  (mu_c, sigma_c) = the mean and the (ddof 0) std about that mean of l over the voiced frames 0..t,
each a sequential float64 sum.  A voiced frame's shift is 12 (mu_t - mu_c) for "match", and for "mv" while fewer than
`warmup` voiced frames have been seen or while every voiced l so far is the same (sigma_c = 0); otherwise "mv" gives
12 (mu_t + sigma_t / sigma_c (l - mu_c) - l).  Shifts are clamped to +-limit; an unvoiced frame holds the last voiced
frame's shift, 0 before the first.
"""
import math

import numpy as np


def shifts(tau, ap, en, mode, mu_t, sd_t, warmup, sr, theta, silence_db, limit=24.0):
    """(log2 F0 with NaN where unvoiced, voiced, shifts) float64 / bool / float64 of one stream's frames."""
    T = len(tau)
    out, logs, voiced = np.zeros(T), np.full(T, np.nan), np.zeros(T, bool)
    ls, last = [], 0.0
    for t in range(T):
        emax = max(float(e) for e in en[:t + 1])
        v = ap[t] < theta and en[t] > 0 and emax > 0 and 10.0 * math.log10(en[t] / emax) >= -silence_db
        if v:
            l = math.log2(sr / tau[t])
            ls.append(l)
            logs[t], voiced[t] = l, True
            m = 0.0
            for x in ls:
                m += x
            m /= len(ls)
            q = 0.0
            for x in ls:
                q += (x - m) ** 2
            sd = math.sqrt(q / len(ls))
            if mode == "mv" and len(ls) >= warmup and any(x != ls[0] for x in ls):
                s = 12.0 * (mu_t + sd_t / sd * (l - m) - l)
            else:
                s = 12.0 * (mu_t - m)
            last = min(limit, max(-limit, s))
        out[t] = last
    return logs, voiced, out
