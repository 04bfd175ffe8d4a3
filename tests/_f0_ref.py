"""Float64 numpy restatement of the YIN tracker (csrc/pitch.cu, adaptive_voice_conversion_b200/f0.py), its voicing
rule, the speaker profiles and every per-pair and per-set value of evaluate_f0.  Written from the definitions, loops
where the definition is sequential; it imports nothing from the package."""
import math

import numpy as np

METRICS = ("vuv_agree", "f0_corr", "st_target", "st_source", "f0_success", "st_target_source")


def taus(sr, fmin=50.0, fmax=500.0):
    return int(math.floor(sr / fmax)), int(math.ceil(sr / fmin))


def reflect(i, n):
    i = np.abs(i)
    return np.where(i >= n, 2 * (n - 1) - i, i)


def frames_of(y, hop, win, tau_max, frames=None):
    """x[f][j] = y[reflect(f hop - floor((win + tau_max)/2) + j)], j < win + tau_max, float64 [F, span]."""
    y = np.asarray(y, np.float32).astype(np.float64)
    n = len(y)
    span = win + tau_max
    fs = np.arange(1 + n // hop) if frames is None else np.asarray(frames)
    idx = fs[:, None] * hop - span // 2 + np.arange(span)[None, :]
    assert (idx >= -(n - 1)).all() and (idx <= 2 * (n - 1)).all(), "signal too short for one reflection"
    return y[reflect(idx, n)]


def difference(x, win, tau_max):
    """d[f][tau] for tau = 0..tau_max (d[:, 0] = 0)."""
    d = np.zeros((x.shape[0], tau_max + 1))
    a = x[:, :win]
    for tau in range(1, tau_max + 1):
        e = a - x[:, tau:tau + win]
        d[:, tau] = np.sum(e * e, axis=1)
    return d


def cmnd(d):
    """d'[tau] = d[tau] tau / sum_{k=1..tau} d[k] (1 where that sum is 0), tau >= 1; d'[0] = 1."""
    d = np.asarray(d, np.float64)
    s = np.cumsum(d[..., 1:], axis=-1)
    tau = np.arange(1, d.shape[-1])
    with np.errstate(divide="ignore", invalid="ignore"):
        dp = np.where(s == 0, 1.0, d[..., 1:] * tau / np.where(s == 0, 1.0, s))
    return np.concatenate([np.ones(d.shape[:-1] + (1,)), dp], axis=-1)


def choose(dp, tau_min, tau_max, theta):
    """(tau*, delta) of one d' curve dp[0..tau_max]."""
    ts = None
    for t in range(tau_min, tau_max + 1):
        if dp[t] < theta:
            ts = t
            break
    if ts is not None:
        while ts < tau_max and dp[ts + 1] < dp[ts]:
            ts += 1
    else:
        ts = tau_min
        for t in range(tau_min, tau_max + 1):
            if dp[t] < dp[ts]:
                ts = t
    delta = 0.0
    if ts - 1 >= 1 and ts + 1 <= tau_max:
        a, b, c = dp[ts - 1], dp[ts], dp[ts + 1]
        den = a - 2.0 * b + c
        if den > 0:
            delta = min(0.5, max(-0.5, (a - c) / (2.0 * den)))
    return ts, delta


def yin(y, sr, hop, win=1024, fmin=50.0, fmax=500.0, threshold=0.1, frames=None):
    """{tau, aperiodicity, energy, tau_star} float64 / int arrays of the frames of y (all 1 + len//hop by default)."""
    tau_min, tau_max = taus(sr, fmin, fmax)
    theta = float(np.float32(threshold))
    x = frames_of(y, hop, win, tau_max, frames)
    dp = cmnd(difference(x, win, tau_max))
    out = {"tau": [], "aperiodicity": [], "tau_star": []}
    for row in dp:
        ts, delta = choose(row, tau_min, tau_max, theta)
        out["tau"].append(ts + delta)
        out["aperiodicity"].append(row[ts])
        out["tau_star"].append(ts)
    out = {k: np.asarray(v) for k, v in out.items()}
    out["energy"] = np.sum(x[:, :win] ** 2, axis=1) / win
    return out


def voicing(tau, ap, energy, sr, threshold=0.1, silence_db=40.0):
    """(f0, voiced): voiced when ap < theta (float32), energy > 0 and 10 log10(energy / max energy) >= -silence_db."""
    theta = float(np.float32(threshold))
    tau, ap, energy = (np.asarray(v, np.float64) for v in (tau, ap, energy))
    emax = energy.max()
    voiced = np.zeros(len(tau), bool)
    for i in range(len(tau)):
        voiced[i] = ap[i] < theta and energy[i] > 0 and emax > 0 and 10.0 * math.log10(energy[i] / emax) >= -silence_db
    f0 = np.full(len(tau), np.nan)
    f0[voiced] = sr / tau[voiced]
    return f0, voiced


def seq_sum(v):
    s = 0.0
    for x in v:
        s += float(x)
    return s


def profile(series):
    """(mean, std) of the concatenated log2 F0 series, sequential sums; (None, None) when empty."""
    v = [float(x) for s in series for x in s]
    if not v:
        return None, None
    m = seq_sum(v) / len(v)
    return m, math.sqrt(seq_sum([(x - m) ** 2 for x in v]) / len(v))


def pearson(a, b):
    ma, mb = seq_sum(a) / len(a), seq_sum(b) / len(b)
    da, db = [x - ma for x in a], [x - mb for x in b]
    return seq_sum([x * y for x, y in zip(da, db)]) / math.sqrt(seq_sum([x * x for x in da]) * seq_sum([y * y for y in db]))


def pair(conv, src, target_mean, source_mean):
    """The six values of one pair from (f0, voiced) tracks, or None (n_unvoiced)."""
    (fc, vc), (fs, vs) = conv, src
    both = [i for i in range(len(vc)) if vc[i] and vs[i]]
    if target_mean is None or source_mean is None or len(both) < 2:
        return None
    a = [math.log2(fc[i]) for i in both]
    b = [math.log2(fs[i]) for i in both]
    if len(set(a)) == 1 or len(set(b)) == 1:
        return None
    mc = seq_sum([math.log2(fc[i]) for i in range(len(vc)) if vc[i]]) / sum(bool(x) for x in vc)
    ms = seq_sum([math.log2(fs[i]) for i in range(len(vs)) if vs[i]]) / sum(bool(x) for x in vs)
    st_t, st_s = 12.0 * abs(mc - target_mean), 12.0 * abs(mc - source_mean)
    agree = seq_sum([1.0 if bool(vc[i]) == bool(vs[i]) else 0.0 for i in range(len(vc))]) / len(vc)
    return [agree, pearson(a, b), st_t, st_s, float(st_t < st_s), 12.0 * abs(ms - target_mean)]


def speaker(u):
    return u.split("_")[0]


def measure(pairs, real, conv):
    """evaluate_f0's numbers from the tracks: pairs [(source, [references])], real {utterance: (f0, voiced)} of every
    embedded utterance, conv [(f0, voiced)] per pair.  Returns (rows {pair index: values}, n_unvoiced, set means,
    per-target-speaker means, profiles)."""
    logs = {u: [math.log2(f) for f, v in zip(*real[u]) if v] for u in real}
    by = {}
    for u in sorted(real):
        by.setdefault(speaker(u), []).append(u)
    rows, n_unv = {}, 0
    for i, (u, refs) in enumerate(pairs):
        tm = profile([logs[v] for v in by.get(speaker(refs[0]), []) if v not in refs])[0]
        sm = profile([logs[v] for v in by.get(speaker(u), []) if v != u])[0]
        r = pair(conv[i], real[u], tm, sm)
        if r is None:
            n_unv += 1
        else:
            rows[i] = r

    def means(idx):
        return {k: seq_sum([rows[i][j] for i in idx]) / len(idx) for j, k in enumerate(METRICS)} | {"n": len(idx)}
    total = means(list(rows)) if rows else {"n": 0}
    spk = {}
    for i in rows:
        spk.setdefault(speaker(pairs[i][1][0]), []).append(i)
    profiles = {}
    for s, us in by.items():
        m, sd = profile([logs[u] for u in us])
        profiles[s] = {"log2_mean": m, "log2_std": sd, "voiced": sum(len(logs[u]) for u in us),
                       "frames": sum(len(real[u][1]) for u in us)}
    return rows, n_unv, total, {s: means(ix) for s, ix in spk.items()}, profiles


def harmonic(f0, seconds, sr=24000, n_harm=10, amp=0.5, phase_seed=0):
    """sum_{k=1..n_harm} (amp / k) sin(2 pi k phi(t) + phi_k), phi the integral of f0 (a scalar or a callable of
    t in seconds); harmonics above sr/2 dropped.  float32."""
    t = np.arange(int(round(seconds * sr))) / sr
    if callable(f0):
        inst = f0(t)
        phi = np.concatenate([[0.0], np.cumsum((inst[1:] + inst[:-1]) / 2.0) / sr])
    else:
        inst = np.full_like(t, float(f0))
        phi = float(f0) * t
    rng = np.random.default_rng(phase_seed)
    y = np.zeros_like(t)
    for k in range(1, n_harm + 1):
        ok = k * inst < sr / 2
        y += np.where(ok, amp / k * np.sin(2 * np.pi * k * phi + rng.uniform(0, 2 * np.pi)), 0.0)
    return y.astype(np.float32)
