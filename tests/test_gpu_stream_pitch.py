"""GPU: the streamed pitch stage (streaming.PitchStage) and its tracker kernel (avc_yin_window).

1. avc_yin_window equals avc_yin on the whole signal bit for bit: random origins, frames that reflect at sample 0 and
   at a closed end, 1-sample to random chunkings, several signals in one table; bad arguments get avc_yin's codes and
   messages;
2. a tracked stream's shadow output equals the same stream converted with pitch=None, bit for bit;
3. its tracked (tau, aperiodicity, energy) equal f0.yin of the whole shadow output bit for bit, for three chunkings;
4. its shifts equal the float64 restatement (tests/_stream_pitch_ref.py) from those tracks to 1e-9 semitones;
5. its output equals Rtisi run on pitch_shift(unshifted magnitudes, its shifts) bit for bit; a fixed shift's output
   equals Rtisi(pitch_shift(magnitudes, s)), and s = 0 gives the unshifted bits;
6. bits do not depend on chunking or on the other streams, with tracked, fixed and unshifted streams mixed;
7. every sample n is out once input sample n + tracked_latency_samples has arrived, the worst one exactly then, and
   a stream gives hop (T - 1) samples;
8. on a synthetic harmonic glide pushed as magnitudes through the stage, the output's voiced log2 F0 mean (match, mv)
   and std (mv) after warm-up, tracked offline, are near the target (printed; tolerances from the measured run).
"""
import ctypes as C
import math

import numpy as np
import pytest
import torch

import _stream_pitch_ref as PR
import oracle.ae_oracle as orc
from adaptive_voice_conversion_b200 import _lib as L
from adaptive_voice_conversion_b200 import f0 as F
from adaptive_voice_conversion_b200 import streaming as S
from adaptive_voice_conversion_b200.utils import _stream
from adaptive_voice_conversion_b200.vocoder import _SEG, AudioParams, Vocoder, _ptr, magnitude, pitch_shift
from test_gpu_stream import chunks_of, feed, make_inf, signal

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
SR, HOP = 24000, 300
P = F.F0Params()
TMIN, TMAX = P.tau_min(SR), P.tau_max(SR)
SPAN = P.win + TMAX


# the default span (1504) and two odd ones: W 985 (1465, as W 1024 with fmin 50 Hz at 22 050 Hz) and tau_max 481 (1505)
SPANS = {"default": P, "odd_win": F.F0Params(win=985), "odd_tau": F.F0Params(fmin=49.9)}


def first(o, p=P):
    """avc_yin_window's first sample of an entry with origin o: max(0, o hop - ceil(span / 2) - 1)."""
    span = p.win + p.tau_max(SR)
    return max(0, o * HOP - (span - span // 2) - 1)


def yin_window(entries, p=P):
    """avc_yin_window of entries [(samples (device), origin, n_frames)] in one table: [tau, ap, en] float64 per entry."""
    tab = np.zeros(len(entries), _SEG)
    soff = foff = 0
    for k, (y, o, n) in enumerate(entries):
        tab[k] = (soff, y.numel(), foff, n, o)
        soff += y.numel()
        foff += n
    table = torch.from_numpy(tab.view(np.uint8)).to(DEV)
    y = torch.cat([e[0] for e in entries])
    out = torch.empty(3, foff, dtype=torch.float64, device=DEV)
    d = L.AudioDesc(hop=HOP, n_seg=len(entries), n_frames=foff, n_samples=soff, segs=_ptr(table), y=_ptr(y))
    L.check(L.load().avc_yin_window(C.byref(d), p.win, p.tau_min(SR), p.tau_max(SR), C.c_float(p.threshold), _ptr(out[0]),
                                    _ptr(out[1]), _ptr(out[2]), _stream(DEV)), "avc_yin_window")
    h = out.cpu().numpy()
    res, f = [], 0
    for _, _, n in entries:
        res.append(h[:, f:f + n])
        f += n
    return res


def whole(y, p=P):
    return torch.stack(F.yin([y], SR, HOP, p)[0]).cpu().numpy()


LENS = [3 * SR + 7, HOP * 40, 5000, SR + 150]       # HOP * 40: the last frame's end reflection reaches first(o)


@pytest.mark.parametrize("span", list(SPANS))
def test_yin_window_random_origins(span):
    p = SPANS[span]
    sp = p.win + p.tau_max(SR)
    ys = [signal(n, 20 + i) for i, n in enumerate(LENS)]
    refs = [whole(y, p) for y in ys]
    rng = np.random.default_rng(0)
    entries, want = [], []
    for y, ref in zip(ys, refs):
        T = ref.shape[1]
        origins = {0, 1, 2, T - 1, T - 2} | set(rng.integers(0, T, 12).tolist())
        for o in sorted(origins):
            k = int(rng.integers(1, min(12, T - o) + 1))
            entries.append((y[first(o, p):], o, k))                    # a closed signal: the end reflects
            want.append(ref[:, o:o + k])
            n = int(rng.integers(first(o, p) + 1, y.numel() + 1))      # a signal still arriving: frames inside it
            k2 = min(S.yin_ready(n, HOP, sp), T) - o
            if k2 > 0:
                entries.append((y[first(o, p):n], o, k2))
                want.append(ref[:, o:o + k2])
    got = yin_window(entries, p)
    for i, (g, w) in enumerate(zip(got, want)):
        assert not np.isnan(g).any() and np.array_equal(g, w), (span, i, entries[i][1], np.abs(g - w).max())
    # o = 0 everywhere is avc_yin itself
    got = yin_window([(y, 0, r.shape[1]) for y, r in zip(ys, refs)], p)
    assert all(np.array_equal(g, r) for g, r in zip(got, refs))


@pytest.mark.parametrize("sizes,span", [("one", "default"), (37, "default"), (4800, "default"), ("random", "default"),
                                        ("random", "odd_win"), (37, "odd_tau")])
def test_yin_window_chunkings(sizes, span):
    """Signals arriving in chunks, tracked in lockstep as PitchStage does (one table per update, each entry from the
    first sample its next frame reads), and closed: every frame equals the whole-signal avc_yin."""
    p = SPANS[span]
    sp = p.win + p.tau_max(SR)
    ys = [signal(n, 30 + i) for i, n in enumerate(LENS[:3])]
    refs = [whole(y, p) for y in ys]
    streams = []
    for i, y in enumerate(ys):
        if sizes == "one":   # 1-sample chunks for the first 3 000 samples
            c = [y[k:k + 1] for k in range(3000)] + chunks_of(y[3000:], 4800)
        else:
            c = chunks_of(y, sizes, seed=i)
        streams.append(c)
    got = [[] for _ in ys]
    n_in, done = [0] * len(ys), [0] * len(ys)
    for step in range(max(len(c) for c in streams) + 1):
        entries, who = [], []
        for i, (y, c) in enumerate(zip(ys, streams)):
            closing = step == len(c)
            if step < len(c):
                n_in[i] += c[step].numel()
            elif not closing:
                continue
            T = refs[i].shape[1]
            ready = T if closing else min(T, S.yin_ready(n_in[i], HOP, sp))
            if ready > done[i]:
                entries.append((y[first(done[i], p):n_in[i]], done[i], ready - done[i]))
                who.append(i)
                done[i] = ready
        if entries:
            for i, g in zip(who, yin_window(entries, p)):
                got[i].append(g)
    for i, ref in enumerate(refs):
        g = np.concatenate(got[i], axis=1)
        assert g.shape == ref.shape and np.array_equal(g, ref), (sizes, span, i)


def test_yin_window_argument_errors():
    y = signal(SR, 1)
    tab = np.zeros(1, _SEG)
    tab[0] = (0, y.numel(), 0, 4, 0)
    table = torch.from_numpy(tab.view(np.uint8)).to(DEV)
    out = torch.empty(3, 4, dtype=torch.float64, device=DEV)
    lib = L.load()

    def desc(**kw):
        a = dict(hop=HOP, n_seg=1, n_frames=4, n_samples=y.numel(), segs=_ptr(table), y=_ptr(y))
        a.update(kw)
        return L.AudioDesc(**a)
    o = [_ptr(out[0]), _ptr(out[1]), _ptr(out[2])]
    cases = [
        (lambda: desc(), (P.win, TMIN, TMAX, 0.1), o, False),
        (lambda: desc(n_seg=0), (P.win, TMIN, TMAX, 0.1), o, True),
        (lambda: desc(segs=None), (P.win, TMIN, TMAX, 0.1), o, True),
        (lambda: desc(y=None), (P.win, TMIN, TMAX, 0.1), o, True),
        (lambda: desc(hop=0), (P.win, TMIN, TMAX, 0.1), o, True),
        (lambda: desc(), (P.win, TMIN, TMAX, 0.1), [o[0], None, o[2]], True),
        (lambda: desc(), (P.win, 0, TMAX, 0.1), o, True),
        (lambda: desc(), (P.win, TMAX, TMAX, 0.1), o, True),
        (lambda: desc(), (400, TMIN, TMAX, 0.1), o, True),
        (lambda: desc(), (2800, TMIN, TMAX, 0.1), o, True),
        (lambda: desc(), (P.win, TMIN, TMAX, float("nan")), o, True),
        (lambda: desc(), (P.win, TMIN, TMAX, 0.0), o, True),
        (lambda: desc(), (P.win, TMIN, TMAX, 1.5), o, True),
    ]
    for k, (mk, (win, tmin, tmax, th), outs, bad) in enumerate(cases):
        rcs, msgs = [], []
        for name in ("avc_yin", "avc_yin_window"):
            n0 = L.launch_count()
            rc = getattr(lib, name)(C.byref(mk()), win, tmin, tmax, C.c_float(th), *outs, _stream(DEV))
            rcs.append(rc)
            msgs.append(L.last_error().replace(name, "NAME") if rc else "")
            if rc:
                assert L.launch_count() == n0, (k, name)
        assert rcs[0] == rcs[1] and msgs[0] == msgs[1], (k, rcs, msgs)
        assert (rcs[0] != 0) == bad, (k, rcs)
    assert lib.avc_yin(None, P.win, TMIN, TMAX, C.c_float(0.1), *o, _stream(DEV)) == \
        lib.avc_yin_window(None, P.win, TMIN, TMAX, C.c_float(0.1), *o, _stream(DEV)) == L.ERR_INVALID
    torch.cuda.synchronize()


# ------------------------------------------------------------------ the converter
@pytest.fixture(scope="module")
def small():
    cfg = orc.default_config(80)
    inf = make_inf(cfg)
    voc = Vocoder(n_mels=80, device=DEV)
    return inf, voc


MV = ("mv", math.log2(210.0), 0.12)
MATCH = ("match", math.log2(120.0), 0.2)
FIXED = 5.0


def _run(inf, voc, y, code, size, others, seed):
    """One converter: the same source and code as a mv stream, a match stream, a fixed +5 stream, a pitch=None and a
    pitch=0 stream, plus `others` streams of other signals; returns ({name: output}, {name: id}, converter)."""
    conv = S.StreamingConverter(inf, voc, S.StreamParams(keep_mels=True, pitch_warmup=20))
    ids = {name: conv.open(code, pitch) for name, pitch in
           (("mv", MV), ("match", MATCH), ("fixed", FIXED), ("none", None), ("zero", 0.0))}
    streams = {sid: chunks_of(y, size, seed=seed) for sid in ids.values()}
    for o in range(others):
        sid = conv.open(torch.randn(128, generator=torch.Generator().manual_seed(100 + o)).to(DEV),
                        (MV, None, -3.0)[o % 3])
        streams[sid] = chunks_of(signal(SR + 3000 * o, 60 + o), 700 + 13 * o)
    outs = feed(conv, streams, fn="update")
    return {name: torch.cat(outs[sid]) for name, sid in ids.items()}, ids, conv


def test_tracked_stream_bits(small):
    inf, voc = small
    hp = voc.hp
    y = signal(3 * SR + 777, 42)
    code = torch.randn(128, generator=torch.Generator().manual_seed(5)).to(DEV)
    mean = torch.as_tensor(inf.attr["mean"]).to(DEV)
    std = torch.as_tensor(inf.attr["std"]).to(DEV)
    first_run = None
    for run, (size, others) in enumerate([(480, 0), (37 * 13, 4), ("random", 7)]):
        out, ids, conv = _run(inf, voc, y, code, size, others, run)
        T = 1 + y.numel() // hp.hop_length
        assert all(v.numel() == hp.hop_length * (T - 1) for v in out.values())
        # 5: s = 0 is the unshifted stream's bits
        assert torch.equal(out["zero"], out["none"])
        mags = voc.mel_to_mag([conv.take_mels(ids["none"]) * std + mean])[0]
        for name in ("mv", "match"):
            tm = voc.mel_to_mag([conv.take_mels(ids[name]) * std + mean])[0]
            assert torch.equal(tm, mags)
            d = conv.take_pitch(ids[name])
            # 2: the shadow is the unshifted stream
            assert torch.equal(d["shadow"], out["none"]), name
            # 3: the tracks are f0.yin of the whole shadow output
            ref = whole(d["shadow"])
            got = np.stack([d["tau"], d["aperiodicity"], d["energy"]])
            assert got.shape == ref.shape == (3, T) and np.array_equal(got, ref), name
            # 4: the shifts are the restatement's
            mode, mu, sd = MV if name == "mv" else MATCH
            lf, v, sh = PR.shifts(ref[0], ref[1], ref[2], mode, mu, sd, 20, SR, P.theta(), P.silence_db)
            assert np.array_equal(d["voiced"], v) and np.abs(d["shift"] - sh).max() <= 1e-9, name
            assert np.array_equal(np.isnan(d["log2_f0"]), ~v)
            print(f"run {run} {name}: {int(v.sum())}/{T} voiced, shifts {d['shift'].min():+.3f} .. "
                  f"{d['shift'].max():+.3f} semitones")
            # 5: the output is RTISI-LA of the shifted magnitudes
            rt = S.Rtisi(hp, conv.p.gl_lookahead, conv.p.gl_iters, DEV)
            rt.open(0)
            want = rt.run({0: pitch_shift([mags], [d["shift"]], hp)[0]}, close=(0,))[0]
            assert torch.equal(out[name], want), name
        rt = S.Rtisi(hp, conv.p.gl_lookahead, conv.p.gl_iters, DEV)
        rt.open(0)
        assert torch.equal(out["fixed"], rt.run({0: pitch_shift([mags], FIXED, hp)[0]}, close=(0,))[0])
        # 6: the same bits under every chunking and company
        if first_run is None:
            first_run = out
        for k in out:
            assert torch.equal(out[k], first_run[k]), (run, k)
        with pytest.raises(ValueError):
            conv.take_pitch(ids["fixed"])


def test_tracked_latency(small):
    inf, voc = small
    hp = voc.hp
    conv = S.StreamingConverter(inf, voc)
    lat = conv.tracked_latency_samples
    assert lat == S.tracked_latency_samples(conv.p, hp.win_length, hp.hop_length, conv.m, SPAN)
    n_total = 3 * SR + 123
    y = signal(n_total, 7)
    worst = max(range(0, 60 * hp.hop_length),
                key=lambda n: S.tracked_release_sample(n, conv.p, hp.win_length, hp.hop_length, conv.m, SPAN) - n)
    A = S.tracked_release_sample(worst, conv.p, hp.win_length, hp.hop_length, conv.m, SPAN)
    assert A - worst == lat
    sid = conv.open(torch.randn(128, generator=torch.Generator().manual_seed(1)).to(DEV), MV)
    got = 0
    bounds = sorted({A, A + 1} | set(range(997, n_total, 997)) | {n_total})
    for b0, b1 in zip([0] + bounds[:-1], bounds):
        got += conv.push({sid: y[b0:b1]})[sid].numel()
        assert got >= b1 - lat, (b1, got, lat)
        if b1 == A:
            assert got <= worst, (got, worst)
        if b1 == A + 1:
            assert got > worst, (got, worst)
    got += conv.close(sid).numel()
    T = 1 + n_total // hp.hop_length
    assert got == hp.hop_length * (T - 1)
    print(f"latency {conv.latency_samples} samples, tracked {lat} samples")


# ------------------------------------------------------------------ pitch sanity on a glide
def glide(seconds, f_lo, f_hi, seed):
    """A harmonic signal whose F0 glides geometrically from f_lo to f_hi and back, with a slow vibrato and a little
    noise, and its true log2 F0 per sample."""
    rng = np.random.default_rng(seed)
    n = int(seconds * SR)
    t = np.arange(n) / SR
    u = 0.5 - 0.5 * np.cos(2 * np.pi * t / seconds)
    lf = np.log2(f_lo) + u * (np.log2(f_hi) - np.log2(f_lo)) + 0.02 * np.sin(2 * np.pi * 5.0 * t)
    ph = 2 * np.pi * np.cumsum(2.0 ** lf) / SR
    y = sum((0.5 / k) * np.sin(k * ph + rng.uniform(0, 2 * np.pi)) for k in range(1, 25) if k * 2.0 ** lf.max() < 11000)
    y = 0.3 * y / np.abs(y).max() + 1e-4 * rng.standard_normal(n)
    return y.astype(np.float32)


def glide_errors(target, seed, warmup=50, seconds=8.0):
    """(12 |mean - mu_t|, 12 |std - sigma_t|) of the log2 F0 of the stage's output over its voiced frames after
    warm-up (tracked offline), for a glide pushed as magnitudes in 8-frame blocks."""
    hp = AudioParams()
    y = torch.from_numpy(glide(seconds, 110.0, 170.0, seed)).to(DEV)
    mags = magnitude([y], hp, preemphasis=hp.preemphasis)[0][0]
    st = S.PitchStage(hp, 3, 8, DEV, warmup=warmup, keep=True)
    st.open(0, target)
    blocks = list(torch.split(mags, 8))
    outs = [st.run({0: b}) for b in blocks[:-1]] + [st.run({0: blocks[-1]}, close=(0,))]
    out = torch.cat([o[0] for o in outs if 0 in o])
    assert out.numel() == hp.hop_length * (mags.shape[0] - 1)
    d = st.take(0)
    after = int(np.searchsorted(np.cumsum(d["voiced"]), warmup)) + 1
    f, v = F.track([out], hp.sr, hp.hop_length)[0]
    lv = np.log2(f[after:][v[after:]])
    return 12 * abs(lv.mean() - target[1]), 12 * abs(lv.std() - target[2]), len(lv)


# Measured on an H100 (700 W) over these seeds at GLIDE_TARGET: mv mean errors 1.42 - 1.58 st and std errors 0.04 -
# 0.13 st; match mean errors 1.07 - 1.24 st (its std is the source's, not checked).  tools/bench_stream.py -pitch mv
# reports the same glides (seeds 0 - 4) at the same target.  The running mean lags a glide, so the mean error
# is the larger one.  The tolerances leave a margin over the largest.
MEAN_TOL_ST = 2.0
STD_TOL_ST = 0.3


GLIDE_TARGET = (math.log2(220.0), 0.15)   # (log2 F0 mean, std) of the glide checks here and in tools/bench_stream.py


@pytest.mark.parametrize("mode", ["mv", "match"])
def test_glide_sanity(mode):
    target = (mode, *GLIDE_TARGET)
    errs = [glide_errors(target, seed) for seed in range(3)]
    print(f"{mode}: output voiced log2 F0 after warm-up: mean error (st) {[round(float(e[0]), 3) for e in errs]}, "
          f"std error (st) {[round(float(e[1]), 3) for e in errs]}, voiced frames {[e[2] for e in errs]}")
    assert all(e[2] > 100 for e in errs)
    assert max(e[0] for e in errs) <= MEAN_TOL_ST
    if mode == "mv":
        assert max(e[1] for e in errs) <= STD_TOL_ST
