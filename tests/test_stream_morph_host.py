"""Host checks of retargeting live streams (streaming.TargetSchedule, StreamingConverter.retarget, inference.py
-stream_morph): the schedule's weights against a direct float64 restatement, its refusals, its pruning, PitchTracker
with per-frame targets, and the CLI's refusals."""
import math
import os
import subprocess
import sys

import numpy as np
import pytest
import torch

import _stream_pitch_ref as PR
from adaptive_voice_conversion_b200 import streaming as S
from adaptive_voice_conversion_b200.f0 import F0Params

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SR = 24000
P = F0Params()


def code(i, n=8):
    return torch.from_numpy(np.random.default_rng(1000 + i).standard_normal(n).astype(np.float32))


def direct_weights(keyframes, K, n):
    """float64 [n, K] of keyframes [(frame, {anchor: weight})], restated frame by frame: the last keyframe at or
    before t (the later of several), the first held before it and the last after it, linear in between."""
    out = np.zeros((n, K))
    for t in range(n):
        vec = lambda d: np.array([d.get(k, 0.0) for k in range(K)])  # noqa: E731
        at_or_before = [i for i, (f, _) in enumerate(keyframes) if f <= t]
        if not at_or_before:
            out[t] = vec(keyframes[0][1])
            continue
        i = at_or_before[-1]
        if i == len(keyframes) - 1:
            out[t] = vec(keyframes[i][1])
            continue
        (f0, v0), (f1, v1) = keyframes[i], keyframes[i + 1]
        a = (t - f0) / (f1 - f0)
        out[t] = (1 - a) * vec(v0) + a * vec(v1)
    return out


def replay(ops, n):
    """Keyframes of a sequence of retargets [(anchor, at, ramp)] restated on dicts: drop the keyframes after at, add
    (at, mix at at) and (at + ramp, one-hot)."""
    kfs, anchors = [(0, {0: 1.0})], [0]
    for a, at, ramp in ops:
        if a not in anchors:
            anchors.append(a)
        K = len(anchors)
        mix = direct_weights(kfs, K, at + 1)[at]
        kfs = [kf for kf in kfs if kf[0] <= at]
        kfs += [(at, {k: mix[k] for k in range(K)}), (at + ramp, {anchors.index(a): 1.0})]
    return kfs, anchors


@pytest.mark.parametrize("seed", range(12))
def test_weights_match_direct_restatement(seed):
    rng = np.random.default_rng(seed)
    codes = [code(i) for i in range(5)]
    sch = S.TargetSchedule(codes[0])
    ops, at = [], 0
    for _ in range(int(rng.integers(1, 7))):
        at += int(rng.integers(0, 30))
        ramp = int(rng.choice([0, 0, 1, 5, 17, 40]))        # hard cuts, ramps, and ramps interrupted by the next
        a = int(rng.integers(0, 5))
        ops.append((a, at, ramp))
        sch.retarget(codes[a].clone(), at, ramp)          # a clone: de-duplicated by bits, not by object
    kfs, anchors = replay(ops, 0)
    n = at + 60
    ref = direct_weights(kfs, len(anchors), n)
    assert len(sch.codes) == len(anchors)
    assert all(torch.equal(c, codes[a]) for c, a in zip(sch.codes, anchors))
    np.testing.assert_allclose(sch.mix(0, n), ref, rtol=0, atol=1e-15)
    w = sch.weights(0, n)
    assert w.dtype == np.float32 and np.array_equal(w, sch.mix(0, n).T.astype(np.float32))
    # any window of it: the same bits as the whole
    for f0, f1 in ((0, 8), (5, 40), (n - 24, n)):
        assert np.array_equal(sch.weights(f0, f1), w[:, f0:f1])


def test_holds_cut_and_plain_windows():
    a, b = code(0), code(1)
    sch = S.TargetSchedule(a)
    assert sch.window(0, 128) == (0, None)
    sch.retarget(b, 40, 0)                                # a hard cut at frame 40
    w = sch.weights(0, 80)
    assert (w[0, :40] == 1).all() and (w[1, :40] == 0).all() and (w[1, 40:] == 1).all() and (w[0, 40:] == 0).all()
    assert sch.window(0, 40) == (0, None) and sch.window(40, 80) == (1, None)
    ks, ww = sch.window(32, 48)
    assert ks == [0, 1] and np.array_equal(ww, w[:, 32:48])
    sch.retarget(a, 100, 10)
    assert sch.window(110, 200) == (0, None) and sch.window(40, 101) == (1, None)     # frame 100 is still all b
    assert sch.window(100, 110)[0] == [0, 1]


def test_same_code_adds_nothing():
    a = code(0)
    sch = S.TargetSchedule(a)
    sch.retarget(a.clone(), 0, 0)
    sch.retarget(a.clone(), 30, 12)
    assert len(sch.codes) == 1 and np.array_equal(sch.weights(0, 100), np.ones((1, 100), np.float32))
    assert sch.window(0, 100) == (0, None)


def test_interrupted_ramp_starts_from_reached_mix():
    a, b, c = code(0), code(1), code(2)
    sch = S.TargetSchedule(a)
    sch.retarget(b, 10, 20)
    before = sch.mix(15, 16)[0]
    sch.retarget(c, 15, 10)
    m = sch.mix(0, 40)
    np.testing.assert_array_equal(m[15], np.append(before, 0.0))
    np.testing.assert_allclose(m[25], [0, 0, 1], atol=0)
    np.testing.assert_allclose(m[20], 0.5 * np.append(before, 0.0) + 0.5 * np.array([0, 0, 1]), atol=1e-15)


def snapshot(sch):
    return ([c.clone() for c in sch.codes], list(sch.pitch), list(sch.frames), sch.V.copy())


def same(sch, snap):
    codes, pitch, frames, V = snap
    return (len(codes) == len(sch.codes) and all(torch.equal(x, y) for x, y in zip(codes, sch.codes))
            and pitch == sch.pitch and frames == sch.frames and np.array_equal(V, sch.V))


def test_refusals_leave_schedule_unchanged():
    sch = S.TargetSchedule(code(0), 2.0)
    sch.retarget(code(1), 20, 8, 3.0)
    snap = snapshot(sch)
    with pytest.raises(ValueError, match="before the end"):
        sch.retarget(code(2), 9, 0, 1.0, first=10)
    assert same(sch, snap)
    with pytest.raises(ValueError, match="ramp"):
        sch.retarget(code(2), 30, -1, 1.0)
    assert same(sch, snap)
    for bad in (None, ("mv", 7.0, 0.1), "up", True, 30.0):
        with pytest.raises(ValueError, match="kind" if bad != 30.0 else "in \\[-24, 24\\]"):
            sch.pitch_value(bad, 30)
    assert same(sch, snap)
    assert sch.pitch_value(0, 30) == 0.0 and sch.pitch_value(-4, 30) == -4.0
    prof = S.TargetSchedule(code(0), ("mv", 7.5, 0.2))
    for bad in (None, 3.0, ("match", 7.0, 0.1)):
        with pytest.raises(ValueError, match="kind"):
            prof.pitch_value(bad, 0)
    assert prof.pitch_value(("mv", 7, 0.3), 0) == (7.0, 0.3)
    none = S.TargetSchedule(code(0))
    with pytest.raises(ValueError, match="kind"):
        none.pitch_value(2.0, 0)
    assert none.pitch_value(None, 0) is None and none.pitch_value(0.0, 0) is None


def test_anchor_limit():
    """64 anchors of non-zero weight in one window are accepted; the 65th within a window is refused."""
    W = 128
    sch = S.TargetSchedule(code(0))
    for k in range(1, 64):
        sch.retarget(code(k), k, 1, first=0, lo=0, window=W)
    assert len(sch.codes) == 64
    snap = snapshot(sch)
    with pytest.raises(ValueError, match="65 anchors"):
        sch.retarget(code(64), 64, 1, first=0, lo=0, window=W)
    assert same(sch, snap)
    # far enough ahead that no window holds both the first anchor and the new one: accepted
    sch.retarget(code(64), 64 + W + 1, 1, first=0, lo=0, window=W)
    assert len(sch.codes) == 65


def test_pruning_bounded():
    """10 000 retargets, each to a new code, of a stream that moves on by 8 frames (a block) per retarget, each ramp
    done before the next retarget, pruned from 128 frames back: the keyframes and anchors left stay bounded by the
    retargets of the last 128 frames.  (A ramp interrupted by the next retarget keeps its anchors at non-zero weight
    in the mix it reached, so a chain of interrupted ramps keeps them until their weights underflow.)"""
    rng = np.random.default_rng(0)
    sch = S.TargetSchedule(code(0))
    most = (0, 0)
    for i in range(1, 10001):
        lo = max(0, 8 * i - 128)
        sch.retarget(torch.full((8,), float(i)), 8 * i, int(rng.integers(0, 9)), first=8 * i, lo=lo, window=128)
        sch.prune(lo)
        most = (max(most[0], len(sch.frames)), max(most[1], len(sch.codes)))
    # keyframes at or after lo come from the 17 retargets at 8 i - 128 .. 8 i, two each, plus the one before lo
    assert most[0] <= 2 * 17 + 1 and most[1] <= 17 + 1, most


def test_pruning_keeps_values_and_order():
    codes = [code(i) for i in range(4)]
    sch = S.TargetSchedule(codes[0])
    for k, at in ((1, 10), (2, 30), (3, 60)):
        sch.retarget(codes[k], at, 8)
    full = sch.mix(0, 120)
    sch.prune(35)      # frames from 35 on: the ramp from 2 at 30 onwards
    assert [next(i for i, c in enumerate(codes) if torch.equal(c, x)) for x in sch.codes] == [1, 2, 3]
    np.testing.assert_array_equal(sch.mix(35, 120), full[35:, 1:])
    sch.prune(80)
    assert len(sch.codes) == 1 and torch.equal(sch.codes[0], codes[3]) and sch.window(80, 200) == (0, None)


def test_pitch_targets():
    sch = S.TargetSchedule(code(0), 3.0)
    sch.retarget(code(1), 10, 10, -5.0)
    w = sch.weights(0, 30).astype(np.float64)
    np.testing.assert_array_equal(sch.shift(0, 30), w[0] * 3.0 + w[1] * -5.0)
    assert (sch.shift(0, 10) == 3.0).all() and (sch.shift(20, 10) == -5.0).all()
    assert S.KEEP is not None and sch.pitch_value(S.KEEP, 15) == sch.shift(15, 1)[0]
    prof = S.TargetSchedule(code(0), ("mv", 7.0, 0.1))
    prof.retarget(code(1), 4, 8, (8.0, 0.3))
    mu, sd = prof.profile(0, 20)
    w = prof.weights(0, 20).astype(np.float64)
    np.testing.assert_array_equal(mu, (w[0] * 7.0 + w[1] * 8.0) / (w[0] + w[1]))
    np.testing.assert_array_equal(sd, (w[0] * 0.1 + w[1] * 0.3) / (w[0] + w[1]))
    assert (mu[:5] == 7.0).all() and (mu[12:] == 8.0).all()
    # KEEP on a new anchor takes the schedule's target at `at`
    prof.retarget(code(2), 8, 4)
    assert prof.pitch[-1] == (float(mu[8]), float(sd[8]))


def _tracks(T, seed):
    rng = np.random.default_rng(seed)
    tau = rng.uniform(48, 480, T)
    ap = np.where(rng.random(T) < 0.7, rng.uniform(0, 0.09, T), rng.uniform(0.1, 1, T))
    en = rng.uniform(0, 1, T) ** 6 * (rng.random(T) < 0.95)
    return tau, ap, en


def shifts_varying(tau, ap, en, mode, mu, sd, warmup):
    """_stream_pitch_ref.shifts with per-frame targets: a voiced frame t's shift is the constant-target rule at
    (mu[t], sd[t]); an unvoiced frame holds the last voiced frame's, 0 before the first."""
    voiced = PR.shifts(tau, ap, en, mode, 0.0, 0.0, warmup, SR, P.theta(), P.silence_db)[1]
    out, last = [], 0.0
    for t in range(len(tau)):
        if voiced[t]:
            last = PR.shifts(tau[:t + 1], ap[:t + 1], en[:t + 1], mode, mu[t], sd[t], warmup, SR, P.theta(),
                             P.silence_db)[2][-1]
        out.append(last)
    return np.array(out)


@pytest.mark.parametrize("mode", ["mv", "match"])
def test_tracker_per_frame_targets(mode):
    tau, ap, en = _tracks(300, 1)
    a = S.PitchTracker(mode, 7.3, 0.2, 20, SR, P)
    b = S.PitchTracker(mode, 0.0, 0.0, 20, SR, P)
    ra = [a.update(tau[i:i + 37], ap[i:i + 37], en[i:i + 37]) for i in range(0, 300, 37)]
    rb = [b.update(tau[i:i + 37], ap[i:i + 37], en[i:i + 37], np.full(len(tau[i:i + 37]), 7.3),
                   np.full(len(tau[i:i + 37]), 0.2)) for i in range(0, 300, 37)]
    for x, y in zip(ra, rb):
        for u, v in zip(x, y):
            assert np.array_equal(u, v, equal_nan=u.dtype.kind == "f")
    mu = 7.0 + 0.5 * np.sin(np.arange(300) / 17.0)
    sd = 0.1 + 0.05 * np.cos(np.arange(300) / 23.0)
    c = S.PitchTracker(mode, 0.0, 0.0, 20, SR, P)
    got = np.concatenate([c.update(tau[i:i + 50], ap[i:i + 50], en[i:i + 50], mu[i:i + 50], sd[i:i + 50])[2]
                          for i in range(0, 300, 50)])
    assert np.abs(got - shifts_varying(tau, ap, en, mode, mu, sd, 20)).max() <= 1e-9


def _cli(*args):
    return subprocess.run([sys.executable, os.path.join(ROOT, "inference.py"), *args], capture_output=True, text=True,
                          cwd=ROOT)


@pytest.mark.parametrize("extra,msg", [
    (["-bank", "b.pt", "-stream_morph", "p1@0", "p2@1"], "-stream_morph needs -stream"),
    (["-stream", "-stream_morph", "p1@0", "p2@1"], "-stream_morph needs -bank"),
    (["-stream", "-bank", "b.pt", "-t", "t.wav", "-stream_morph", "p1@0"], "excludes -t, -speaker and -pairs"),
    (["-stream", "-bank", "b.pt", "-speaker", "p1", "-stream_morph", "p1@0"], "excludes -t, -speaker and -pairs"),
    (["-stream", "-bank", "b.pt", "-pairs", "x.txt", "-stream_morph", "p1@0"], "excludes -t, -speaker and -pairs"),
    (["-stream", "-bank", "b.pt", "-stream_morph", "p1"], "SPEC@SECONDS"),
    (["-stream", "-bank", "b.pt", "-stream_morph", "p1@-2"], ">= 0"),
    (["-stream", "-bank", "b.pt", "-stream_morph", "p1@2", "p2@1"], "must not decrease"),
    (["-stream", "-bank", "b.pt", "-morph", "p1@0"], "-stream_morph"),
])
def test_cli_stream_morph_refusals(extra, msg):
    r = _cli("-c", "config.yaml", "-s", "s.wav", "-o", "o.wav", *extra)
    assert r.returncode == 2 and msg in r.stderr, r.stderr


def test_cli_stream_morph_needs_profiled_bank(tmp_path):
    bank = tmp_path / "bank.pt"
    torch.save({"speakers": ["p1"], "codes": torch.zeros(1, 128)}, str(bank))
    r = _cli("-c", "config.yaml", "-s", "s.wav", "-o", "o.wav", "-bank", str(bank), "-stream", "-stream_morph",
             "p1@0", "p1@1", "-stream_pitch", "mv")
    assert r.returncode == 2 and "pitch profiles" in r.stderr and "-stream_pitch mv" in r.stderr, r.stderr


def test_keyframe_frames():
    import importlib.util
    spec = importlib.util.spec_from_file_location("inference_cli", os.path.join(ROOT, "inference.py"))
    cli = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(cli)
    assert cli.keyframe_frame(4.0, 24000, 300) == 320 and cli.keyframe_frame(4.3, 24000, 300) == 344
    assert cli.keyframe_frame(0.0, 24000, 300) == 0 and cli.keyframe_frame(0.00625, 24000, 300) == 1   # .5 rounds up
    assert cli.keyframe_frame(0.0062, 24000, 300) == 0 and math.isclose(0.00625 * 24000 / 300, 0.5)
