"""Float64 restatement of the mean-and-variance log-F0 transform (f0.mv_shifts) and of the banks' target profiles
(SpeakerBank.pitch_profile / morph_pitch_profile), written frame by frame in plain Python floats."""
import math

LIMIT = 24.0


def stats(logs):
    """(mean, ddof-0 std) of a list of log2 F0 values: sequential sums, the std in a second pass about the mean."""
    m = 0.0
    for x in logs:
        m += x
    m /= len(logs)
    v = 0.0
    for x in logs:
        v += (x - m) ** 2
    return m, math.sqrt(v / len(logs))


def at(x, f):
    return x if isinstance(x, float) else float(x[f])


def mv(f0, voiced, target, limit=LIMIT):
    """(shifts, flags) of one conversion: f0 (Hz) and voiced per frame, target (mu_t, sigma_t) of floats or per-frame
    sequences, or None.  flags = {"mean_only", "unmatched", "clamped_frames"}."""
    T = len(voiced)
    vidx = [f for f in range(T) if voiced[f]]
    if not vidx or target is None:
        return [0.0] * T, {"mean_only": False, "unmatched": True, "clamped_frames": 0}
    logs = [math.log2(f0[f]) for f in vidx]
    mc, sc = stats(logs)
    mu, sd = target
    clamp = lambda s: min(limit, max(-limit, s))  # noqa: E731
    if sc == 0.0 or len(vidx) < 2:
        raw = [12.0 * (at(mu, f) - mc) for f in range(T)]
        return [clamp(s) for s in raw], {"mean_only": True, "unmatched": False,
                                         "clamped_frames": sum(abs(s) > limit for s in raw)}
    raw = {f: 12.0 * (at(mu, f) + at(sd, f) / sc * (l - mc) - l) for f, l in zip(vidx, logs)}
    sv = {f: clamp(s) for f, s in raw.items()}
    out = []
    for f in range(T):
        if f in sv:
            out.append(sv[f])
            continue
        before = [p for p in vidx if p < f]
        after = [q for q in vidx if q > f]
        if not before:
            out.append(sv[after[0]])
        elif not after:
            out.append(sv[before[-1]])
        else:
            p, q = before[-1], after[0]
            out.append(sv[p] + (f - p) / (q - p) * (sv[q] - sv[p]))
    return out, {"mean_only": False, "unmatched": False, "clamped_frames": sum(abs(s) > limit for s in raw.values())}


def mix(profiles, weights):
    """(mu, sigma) of a weighted mix of (mu_i, sigma_i) profiles, zero weights skipped; None when a positively
    weighted profile is None."""
    mu = sd = ws = 0.0
    for p, w in zip(profiles, weights):
        if w == 0:
            continue
        if p is None:
            return None
        mu, sd, ws = mu + w * p[0], sd + w * p[1], ws + w
    return mu / ws, sd / ws
