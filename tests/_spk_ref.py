"""float64 restatement of the speaker measures (adaptive_voice_conversion_b200/speaker_eval.py, include/avc_b200.h):
pooling and scores adding in exactly the kernels' order, the EER from sorted scores, the same EER as the kernel finds
it (three radix searches over order-preserving keys, by counting), a literal brute force over every threshold, and a
literal restatement of the conversion-pair rules."""
import random

import numpy as np


def pool64(x, L):
    """x [C, T] float32, L valid frames -> [2C] float32: means, then stds (ddof 0), float64 sums in ascending t."""
    x = np.asarray(x, np.float32)[:, :L].astype(np.float64)
    s = np.zeros(x.shape[0])
    for t in range(L):
        s = s + x[:, t]
    mean = s / L
    v = np.zeros(x.shape[0])
    for t in range(L):
        e = x[:, t] - mean
        v = v + e * e
    return np.concatenate([mean.astype(np.float32), np.sqrt(v / L).astype(np.float32)])


def rnorms64(V):
    V = np.asarray(V, np.float32).astype(np.float64)
    acc = np.zeros(V.shape[0])
    for k in range(V.shape[1]):
        acc = acc + V[:, k] * V[:, k]
    return np.sqrt(acc)


def cosine64(dot, ra, rb):
    with np.errstate(invalid="ignore", divide="ignore"):
        s = dot / (ra * rb)
    return np.where((ra == 0) | (rb == 0), 0.0, s)


def scores64(V):
    """[N, N] float64: s(i, j) of the rows of V (float32), dots added in ascending d, every operation rounded."""
    V = np.asarray(V, np.float32).astype(np.float64)
    dot = np.zeros((V.shape[0], V.shape[0]))
    for k in range(V.shape[1]):
        dot = dot + np.multiply.outer(V[:, k], V[:, k])
    r = rnorms64(V)
    return cosine64(dot, r[:, None], r[None, :])


def trials(S, labels):
    """(scores, is_target) of the pairs i < j of a score matrix."""
    labels = np.asarray(labels)
    i, j = np.triu_indices(len(labels), 1)
    return S[i, j], labels[i] == labels[j]


def _result(frr_num, nT, far_num, nN, thr):
    frr, far = np.float64(frr_num) / np.float64(nT), np.float64(far_num) / np.float64(nN)
    return {"eer": float(max(frr, far)), "threshold": float(thr), "frr": float(frr), "far": float(far),
            "n_target": int(nT), "n_nontarget": int(nN)}


def _null(nT, nN):
    return {"eer": None, "threshold": None, "frr": None, "far": None, "n_target": int(nT), "n_nontarget": int(nN)}


def eer64(scores, is_target):
    """The EER definition from sorted scores: every distinct score and +inf as candidates, max(FRR, FAR) compared
    exactly as integers over n_target n_nontarget, the first (smallest) minimiser."""
    scores = np.asarray(scores, np.float64) + 0.0        # -0 -> +0
    is_target = np.asarray(is_target, bool)
    nT, nN = int(is_target.sum()), int((~is_target).sum())
    if nT == 0 or nN == 0:
        return _null(nT, nN)
    u, inv = np.unique(scores, return_inverse=True)
    t_at = np.bincount(inv, weights=is_target, minlength=len(u)).astype(np.int64)
    n_at = np.bincount(inv, weights=~is_target, minlength=len(u)).astype(np.int64)
    t_lt = np.concatenate([[0], np.cumsum(t_at)])                  # at u[0..], then +inf
    n_ge = nN - np.concatenate([[0], np.cumsum(n_at)])
    f = np.maximum(t_lt * nN, n_ge * nT)
    k = int(np.argmin(f))
    return _result(t_lt[k], nT, n_ge[k], nN, u[k] if k < len(u) else np.inf)


def eer_brute(scores, is_target):
    """Literal: every candidate threshold in ascending order, FRR and FAR counted one trial at a time."""
    scores = [float(s) for s in scores]
    is_target = [bool(t) for t in is_target]
    nT = sum(is_target)
    nN = len(is_target) - nT
    if nT == 0 or nN == 0:
        return _null(nT, nN)
    best = None
    for th in sorted(set(scores)) + [float("inf")]:
        a = sum(1 for s, t in zip(scores, is_target) if t and s < th)
        b = sum(1 for s, t in zip(scores, is_target) if not t and s >= th)
        f = max(a * nN, b * nT)
        if best is None or f < best[0]:
            best = (f, a, b, th)
    return _result(best[1], nT, best[2], nN, best[3])


# ------------------------------------------------------------------ the kernel's search, on the host
def score_keys(scores):
    b = (np.asarray(scores, np.float64) + 0.0).view(np.uint64)
    return np.where(b >> np.uint64(63) == 1, ~b, b | np.uint64(1 << 63))


def key_scores(keys):
    keys = np.asarray(keys, np.uint64)
    return np.where(keys >> np.uint64(63) == 1, keys & np.uint64((1 << 63) - 1), ~keys).view(np.float64)


PASSES = [(53, 11), (42, 11), (31, 11), (20, 11), (9, 11), (0, 9)]


def _search(keys, is_target, alpha, beta, gamma):
    """Largest key k with alpha #{target < k} + beta #{non-target < k} - gamma < 0, digit by digit over histograms;
    returns (k, #{target < k}, #{non-target < k}, #{target == k}, #{non-target == k})."""
    lo, t_lt, n_lt = 0, 0, 0
    for p, (shift, width) in enumerate(PASSES):
        top = shift + width
        inb = np.ones(len(keys), bool) if top == 64 else (keys >> np.uint64(top)) == (np.uint64(lo) >> np.uint64(top))
        dig = ((keys[inb] >> np.uint64(shift)) & np.uint64((1 << width) - 1)).astype(np.int64)
        th = np.bincount(dig[is_target[inb]], minlength=2048)
        nh = np.bincount(dig[~is_target[inb]], minlength=2048)
        te, ne = np.concatenate([[0], np.cumsum(th)]), np.concatenate([[0], np.cumsum(nh)])
        F = alpha * (t_lt + te) + beta * (n_lt + ne) - gamma           # at the start of bin b, and past the last
        b = int(np.nonzero(F[:2048] < 0)[0].max())
        assert F[b + 1] >= 0
        lo += b << shift
        t_lt, n_lt = t_lt + int(te[b]), n_lt + int(ne[b])
        t_eq, n_eq = int(th[b]), int(nh[b])
    return lo, t_lt, n_lt, t_eq, n_eq


def eer_by_counting(scores, is_target):
    """The EER as avc_spk_eer finds it (csrc/spk.cu): m = the largest key with FRR < FAR, then the threshold by rank
    selections, all from integer counts."""
    keys = score_keys(scores)
    is_target = np.asarray(is_target, bool)
    nT, nN = int(is_target.sum()), int((~is_target).sum())
    if nT == 0 or nN == 0:
        return _null(nT, nN)
    m = _search(keys, is_target, nN, nT, nT * nN)
    _, tl, nl, te, ne = m
    if (tl + te) * nN < (nN - nl) * nT:                   # FRR(m+) < FAR(m): the successor of m
        thr = _search(keys, is_target, 1, 1, tl + nl + te + ne + 1)
    elif nl == 0:                                          # no non-target below m: the smallest score
        thr = _search(keys, is_target, 1, 1, 1)
    else:                                                  # q, the largest non-target below m, then its successor
        q = _search(keys, is_target, 0, 1, nl)
        thr = _search(keys, is_target, 1, 1, q[1] + q[2] + q[3] + q[4] + 1)
    return _result(thr[1], nT, nN - thr[2], nN, key_scores(np.array([thr[0]], np.uint64))[0])


def group_mean64(q, q_label, q_ex, V, labels):
    """Mean of s(q, V[v]) over v with labels[v] == q_label, v != q_ex, added in ascending v; NaN when none."""
    V = np.asarray(V, np.float32)
    rs = rnorms64(V)
    rq = rnorms64(np.asarray(q, np.float32)[None])[0]
    qd = np.asarray(q, np.float32).astype(np.float64)
    tot, n = 0.0, 0
    for v in range(len(V)):
        if labels[v] != q_label or v == q_ex:
            continue
        dot = 0.0
        for k in range(V.shape[1]):
            dot = dot + qd[k] * float(V[v, k])
        tot = tot + float(cosine64(np.float64(dot), rq, rs[v]))
        n += 1
    return tot / n if n else float("nan")


def pairs_literal(utts, lengths, seed, max_pairs, min_src, min_ref, min_set, speaker_of):
    """The conversion-pair rules of speaker_eval written out literally."""
    utts = sorted(utts)
    spk = {u: speaker_of(u) for u in utts}
    qual = [u for u in utts if sum(spk[v] == spk[u] for v in utts) >= 2]
    rng = random.Random(seed)
    out, n_short = [], 0
    for u in qual:
        refs = [r for r in qual if spk[r] != spk[u]]
        if not refs:
            continue
        r = rng.choice(refs)
        others_u = [v for v in utts if spk[v] == spk[u] and v != u and lengths[v] >= min_set]
        others_r = [v for v in utts if spk[v] == spk[r] and v != r and lengths[v] >= min_set]
        if lengths[u] < min_src or lengths[r] < min_ref or not others_u or not others_r:
            n_short += 1
            continue
        out.append((u, r))
    if max_pairs > 0 and len(out) > max_pairs:
        out = [out[i] for i in sorted(rng.sample(range(len(out)), max_pairs))]
    return out, n_short
