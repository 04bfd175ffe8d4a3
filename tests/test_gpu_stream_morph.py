"""GPU: retargeting live streams (StreamingConverter.retarget, streaming.TargetSchedule).

1. every emitted block equals a restatement from the offline untrimmed mel, bit for bit: plain windows converted by
   AE.inference_from_embeddings, morph windows by eager AE.inference_morph on the window alone with the schedule's
   anchors and weights as they stood when the window was converted, blended as test_gpu_stream.restate_blocks does;
   hard cuts, ramps, an interrupted ramp, up to 5 anchors, random and fixed chunkings, streams with and without
   retargets in one update, and a close inside a ramp; c80, c512 and sn;
2. a cut from A to B at `at`: blocks whose windows end by `at` are a stream of A's, blocks whose window and previous
   window start at or after `at` a stream of B's, bit for bit;
3. a retarget issued at open and one issued just before the input reaches its frame give the same bits; a retarget to
   the stream's own code changes no bit;
4. a fixed-shift ramp's output is RTISI-LA of pitch_shift at the restated per-frame shifts; a tracked mv stream's
   shifts are PitchTracker's rule on the kernel's YIN outputs with the restated per-frame targets;
5. a stream retargeted every block for 300 blocks keeps its device memory flat and at most the anchors one window can
   read;
6. inference.py -stream -bank -stream_morph (with and without -stream_pitch mv) writes hop (T - 1) samples.
"""
import math
import os
import subprocess
import sys

import numpy as np
import pytest
import torch

import _stream_pitch_ref as PR
import oracle.ae_oracle as orc
from _sn_ref import sn_config
from adaptive_voice_conversion_b200 import streaming as S
from adaptive_voice_conversion_b200.f0 import F0Params
from adaptive_voice_conversion_b200.vocoder import Vocoder, pitch_shift
from test_gpu_stream import chunks_of, make_inf, signal

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
SR, HOP = 24000, 300
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CFGS = {"c80": lambda: orc.default_config(80), "c512": lambda: orc.default_config(512), "sn": lambda: sn_config(80)}


def rcode(i, n=128):
    return torch.randn(n, generator=torch.Generator().manual_seed(500 + i)).to(DEV)


def drive(conv, streams, retargets=None, close=True):
    """Lockstep updates of streams {id: chunks}; retargets {update index: [(id, code, at, ramp, pitch)]} are issued
    before that update, and every stream closed after the last chunk.  Returns ({id: output samples}, {id: [(update
    index, (code, at used, ramp, pitch))]})."""
    retargets = retargets or {}
    outs = {sid: [] for sid in streams}
    log = {sid: [] for sid in streams}
    n = max(len(c) for c in streams.values())
    for u in range(n + (1 if close else 0)):
        for sid, c, at, ramp, pitch in retargets.get(u, []):
            used = conv.retarget(sid, c, at=at, ramp=ramp, pitch=pitch)
            log[sid].append((u, (c, used, ramp, pitch)))
        if u < n:
            res = conv.update({sid: ch[u] for sid, ch in streams.items() if u < len(ch)})
        else:
            res = conv.update({}, close=list(streams))
        for sid, v in res.items():
            outs[sid].append(v)
    return {sid: torch.cat(v) for sid, v in outs.items()}, log


def schedule_at(code0, pitch0, log, u):
    """The stream's TargetSchedule as it stood at update u: its retargets issued before or at u replayed."""
    sch = S.TargetSchedule(code0, S.parse_pitch(pitch0))
    for v, (c, at, ramp, pitch) in log:
        if v <= u:
            sch.retarget(c, at, ramp, pitch if pitch is S.KEEP else sch.pitch_value(pitch, at))
    return sch


def convert_update(hp, n_in_per_update):
    """when(e): the update in which a window ending at frame e is converted, the first whose analysed frames reach e
    (len(n_in_per_update): at close)."""
    frames = [0 if n < hp.win_length // 2 else (n - hp.win_length // 2) // hp.hop_length + 1 for n in n_in_per_update]
    def when(e):
        return next((u for u, f in enumerate(frames) if f >= e), len(frames))
    return when


def restate(inf, conv, mel, T, sched_of_block):
    """restate_blocks with each window converted under sched_of_block(j)'s weights."""
    p, W, m = conv.p, conv.window, conv.m
    mean = torch.as_tensor(inf.attr["mean"]).to(DEV)
    std = torch.as_tensor(inf.attr["std"]).to(DEV)
    x = (mel - mean) / std
    w_new = torch.from_numpy(S.blend_weights(p.hop, p.lookahead)).to(DEV)[:, None]
    w_old = torch.from_numpy(np.float32(1) - S.blend_weights(p.hop, p.lookahead)).to(DEV)[:, None]
    out, prev, j, n_morph = [], None, 0, 0
    while True:
        b0, b1, w0, w1 = S.block_schedule(j, W, p.hop, p.lookahead, m)
        last = w1 > T
        if last:
            if b0 >= T:
                break
            (w0, w1), b1 = S.close_window(T, W), T
        sch = sched_of_block(j, last, w1)
        w = sch.weights(w0, w1)
        nz = np.flatnonzero(w.any(1))
        xw = x[w0:w1].t()[None].contiguous()
        if len(nz) == 1 and (w[nz[0]] == 1).all():
            dec = inf.model.inference_from_embeddings(xw, sch.codes[nz[0]][None])
        else:
            n_morph += 1
            codes = torch.stack([sch.codes[k] for k in nz])[None]
            dec = inf.model.inference_morph(xw, codes, torch.from_numpy(w[nz]).to(DEV)[None])
        dec = dec[0, :, :w1 - w0].t()
        rows = dec[b0 - w0:b1 - w0]
        X = min(w_new.shape[0], rows.shape[0])
        if prev is not None and X:
            rows = torch.cat([rows[:X] * w_new[:X] + prev[:X] * w_old[:X], rows[X:]])
        prev = dec[b1 - w0:b1 - w0 + w_new.shape[0]]
        out.append(rows)
        j += 1
        if last:
            break
    return torch.cat(out), n_morph


def check_stream(inf, conv, voc, y, chunks, code0, log, sid, min_morph=0):
    hp = voc.hp
    n_in = np.cumsum([c.numel() for c in chunks]).tolist()
    when = convert_update(hp, n_in)
    got = conv.take_mels(sid)
    mel = voc.wav_to_mel([y], trim=False)[0][0]
    T = mel.shape[0]
    ref, n_morph = restate(inf, conv, mel, T, lambda j, last, e: schedule_at(
        code0, None, log[sid], 10 ** 9 if last else when(e)))
    assert got.shape == ref.shape == mel.shape, (got.shape, ref.shape)
    assert torch.equal(got, ref), (sid, (got - ref).abs().max())
    assert n_morph >= min_morph, n_morph


@pytest.mark.parametrize("cfg_name", list(CFGS))
def test_blocks_bitwise(cfg_name):
    cfg = CFGS[cfg_name]()
    inf = make_inf(cfg)
    voc = Vocoder(n_mels=cfg["SpeakerEncoder"]["c_in"], device=DEV)
    conv = S.StreamingConverter(inf, voc, S.StreamParams(gl_iters=1, keep_mels=True))
    c_out = conv.c_out
    codes = [rcode(i, c_out) for i in range(6)]
    ys = [signal(n, 70 + i) for i, n in enumerate([3 * SR + 11, 3 * SR + 4000, 2 * SR + 500, 2 * SR])]
    ids = [conv.open(codes[i]) for i in (0, 1, 2, 3)]
    sizes = ["random", 2400, 1000, 1700]
    chunks = {sid: chunks_of(y, s, seed=k) for k, (sid, y, s) in enumerate(zip(ids, ys, sizes))}
    a, b, c, d = ids
    rt = {
        # b: ahead of time, at open: a cut, a ramp interrupted by another, a cut: 5 anchors
        0: [(b, codes[2], 60, 0, S.KEEP), (b, codes[3], 90, 30, S.KEEP), (b, codes[4], 100, 20, S.KEEP),
            (b, codes[5], 150, 0, S.KEEP)],
        # c: while streaming, at the next input frame
        12: [(c, codes[0], None, 40, S.KEEP)],
        30: [(c, codes[4], None, 16, S.KEEP)],
    }
    # d: a ramp the close falls inside
    rt.setdefault(len(chunks[d]) - 20, []).append((d, codes[1], None, 400, S.KEEP))
    _, log = drive(conv, chunks, rt)
    for sid, y, k in zip(ids, ys, (0, 1, 2, 3)):
        check_stream(inf, conv, voc, y, chunks[sid], codes[k], log, sid, min_morph=0 if sid == a else 1)


@pytest.fixture(scope="module")
def small():
    cfg = orc.default_config(80)
    inf = make_inf(cfg)
    voc = Vocoder(n_mels=80, device=DEV)
    return inf, voc


def test_cut_equals_plain_streams(small):
    inf, voc = small
    conv = S.StreamingConverter(inf, voc, S.StreamParams(gl_iters=1, keep_mels=True))
    A, B = rcode(0), rcode(1)
    y = signal(4 * SR, 5)
    at = 96
    x, ya, yb = conv.open(A), conv.open(A), conv.open(B)
    conv.retarget(x, B, at=at)
    drive(conv, {sid: chunks_of(y, 2400) for sid in (x, ya, yb)})
    gx, ga, gb = (conv.take_mels(s) for s in (x, ya, yb))
    T, p, W = gx.shape[0], conv.p, conv.window
    n_a = n_b = 0
    prev_w0 = None
    for j in range(-(-T // p.hop)):
        b0, b1, w0, w1 = S.block_schedule(j, W, p.hop, p.lookahead, conv.m)
        last = w1 > T
        if last:
            (w0, w1), b1 = S.close_window(T, W), T
        if w1 <= at:
            assert torch.equal(gx[b0:b1], ga[b0:b1]), j
            n_a += 1
        if w0 >= at and prev_w0 is not None and prev_w0 >= at:
            assert torch.equal(gx[b0:b1], gb[b0:b1]), j
            n_b += 1
        prev_w0 = w0
        if last:
            break
    assert n_a >= 5 and n_b >= 5, (n_a, n_b)


def test_issue_time_and_self_retarget(small):
    inf, voc = small
    conv = S.StreamingConverter(inf, voc)
    A, B = rcode(0), rcode(1)
    y = signal(3 * SR + 321, 8)
    ch = chunks_of(y, 2400)
    f = 100
    early, late, plain, self_rt = (conv.open(A) for _ in range(4))
    conv.retarget(early, B, at=f, ramp=24)
    u_late = max(u for u in range(len(ch)) if sum(c.numel() for c in ch[:u]) < f * HOP)   # before the input reaches f
    out, _ = drive(conv, {sid: ch for sid in (early, late, plain, self_rt)},
                   {u_late: [(late, B, f, 24, S.KEEP)], 9: [(self_rt, A.clone(), None, 30, S.KEEP)]})
    assert torch.equal(out[early], out[late])
    assert torch.equal(out[self_rt], out[plain])
    assert not torch.equal(out[early], out[plain])


def restated_weights(kfs, K, n):
    """float32 [K, n] of keyframes [(frame, float64 vector)], restated frame by frame."""
    out = np.zeros((n, K))
    fr = [f for f, _ in kfs]
    for t in range(n):
        i = max([k for k, f in enumerate(fr) if f <= t], default=-1)
        if i < 0:
            out[t] = kfs[0][1]
        elif i == len(kfs) - 1:
            out[t] = kfs[i][1]
        else:
            a = (t - fr[i]) / (fr[i + 1] - fr[i])
            out[t] = (1 - a) * kfs[i][1] + a * kfs[i + 1][1]
    return out.T.astype(np.float32)


def test_pitch_follows_schedule(small):
    inf, voc = small
    hp = voc.hp
    conv = S.StreamingConverter(inf, voc, S.StreamParams(keep_mels=True, pitch_warmup=20))
    A, B = rcode(0), rcode(1)
    y = signal(3 * SR + 777, 42)
    T = 1 + y.numel() // HOP
    mv_a, mv_b = ("mv", math.log2(210.0), 0.12), ("mv", math.log2(150.0), 0.2)
    fixed, none, tracked = conv.open(A, 3.0), conv.open(A), conv.open(A, mv_a)
    conv.retarget(fixed, B, at=80, ramp=40, pitch=-4.0)
    conv.retarget(tracked, B, at=60, ramp=50, pitch=mv_b)
    out, _ = drive(conv, {sid: chunks_of(y, "random", seed=3) for sid in (fixed, none, tracked)})
    mean = torch.as_tensor(inf.attr["mean"]).to(DEV)
    std = torch.as_tensor(inf.attr["std"]).to(DEV)
    mags_f = voc.mel_to_mag([conv.take_mels(fixed) * std + mean])[0]
    mags_t = voc.mel_to_mag([conv.take_mels(tracked) * std + mean])[0]
    # the fixed shift: 3 before frame 80, -4 from 120, the weighted sum in between
    w = restated_weights([(0, np.array([1.0, 0])), (80, np.array([1.0, 0])), (120, np.array([0, 1.0]))], 2, T)
    shifts = w[0].astype(np.float64) * 3.0 + w[1].astype(np.float64) * -4.0
    rt = S.Rtisi(hp, conv.p.gl_lookahead, conv.p.gl_iters, DEV)
    rt.open(0)
    assert torch.equal(out[fixed], rt.run({0: pitch_shift([mags_f], [shifts], hp)[0]}, close=(0,))[0])
    # the tracked stream: its targets follow the weights, its shifts are the tracker's rule on its YIN outputs
    d = conv.take_pitch(tracked)
    w = restated_weights([(0, np.array([1.0, 0])), (60, np.array([1.0, 0])), (110, np.array([0, 1.0]))], 2, T)
    w64 = w.astype(np.float64)
    mu = (w64[0] * mv_a[1] + w64[1] * mv_b[1]) / (w64[0] + w64[1])
    sd = (w64[0] * mv_a[2] + w64[1] * mv_b[2]) / (w64[0] + w64[1])
    P = F0Params()
    _, voiced, _ = PR.shifts(d["tau"], d["aperiodicity"], d["energy"], "mv", 0.0, 0.0, 20, SR, P.theta(), P.silence_db)
    want, last = np.zeros(T), 0.0
    for t in range(T):
        if voiced[t]:
            last = PR.shifts(d["tau"][:t + 1], d["aperiodicity"][:t + 1], d["energy"][:t + 1], "mv", mu[t], sd[t], 20,
                             SR, P.theta(), P.silence_db)[2][-1]
        want[t] = last
    assert np.array_equal(d["voiced"], voiced) and np.abs(d["shift"] - want).max() <= 1e-9
    rt = S.Rtisi(hp, conv.p.gl_lookahead, conv.p.gl_iters, DEV)
    rt.open(0)
    assert torch.equal(out[tracked], rt.run({0: pitch_shift([mags_t], [d["shift"]], hp)[0]}, close=(0,))[0])
    print(f"tracked retarget: {int(voiced.sum())}/{T} voiced, shifts {d['shift'].min():+.3f} .. {d['shift'].max():+.3f}")


def test_memory_flat_when_retargeted_every_block(small):
    inf, voc = small
    conv = S.StreamingConverter(inf, voc)
    block = conv.p.hop * HOP
    y = signal(block * 300, 9)
    ids = [conv.open(rcode(0)), conv.open(rcode(1), 2.0)]
    mem, most = [], 0
    for k in range(300):
        for i, sid in enumerate(ids):
            conv.retarget(sid, rcode(10 + k + 1000 * i), ramp=(0, 4, 8)[k % 3], pitch=S.KEEP)
        conv.push({sid: y[k * block:(k + 1) * block] for sid in ids})
        most = max(most, *(len(conv.streams[sid].sched.codes) for sid in ids))
        if k in (149, 299):
            torch.cuda.synchronize()
            mem.append(torch.cuda.memory_allocated(DEV))
    assert mem[1] == mem[0], mem
    # a window reads W frames, one retarget per block of H frames, plus the anchor in force before them and the next
    # block's
    assert most <= conv.window // conv.p.hop + 3, most
    conv.update({}, close=ids)


def test_cli_stream_morph(tmp_path):
    from scipy.io.wavfile import read, write
    from adaptive_voice_conversion_b200.model import AE
    from adaptive_voice_conversion_b200.speaker_bank import SpeakerBank, fingerprint
    from test_gpu_fewshot import _checkpoint
    cfg = orc.default_config(80)
    cfg_path, ckpt = _checkpoint(tmp_path, cfg)
    m = AE(cfg)
    m.load_state_dict(torch.load(ckpt))
    pitch = {"log2_mean": [7.5, 7.9, None], "log2_std": [0.1, 0.2, None], "voiced": [10, 12, 0], "frames": [20, 20, 20],
             "tracker": {}, "griffin_lim": {"n_iter": 100, "momentum": 0.0, "init": "zero"}}
    codes = torch.randn(3, 128, generator=torch.Generator().manual_seed(3))
    SpeakerBank(["p1", "p2", "p3"], codes, [1, 1, 1], [["a"], ["b"], ["c"]], fingerprint(m),
                pitch=pitch).save(str(tmp_path / "bank.pt"))
    n = int(1.7 * SR) + 37
    t = np.arange(n) / SR
    yw = 0.3 * np.sin(2 * np.pi * 140 * t * (1 + 0.2 * t)) + 0.02 * np.random.default_rng(3).standard_normal(n)
    write(str(tmp_path / "s.wav"), SR, (yw * 32767).astype(np.int16))
    env = dict(os.environ, PYTHONPATH=ROOT)
    base = [sys.executable, os.path.join(ROOT, "inference.py"), "-c", cfg_path, "-m", ckpt, "-bank",
            str(tmp_path / "bank.pt"), "-s", str(tmp_path / "s.wav"), "-stream"]
    T = 1 + n // HOP
    for name, extra in (("a.wav", []), ("b.wav", ["-stream_pitch", "mv"]), ("c.wav", ["-stream_pitch", "2.5"])):
        r = subprocess.run(base + ["-o", str(tmp_path / name), "-stream_morph", "p1@0", "p1@0.4", "p2@0.6",
                                   "p1:0.5,p2:0.5@1.2", *extra], env=env, cwd=str(tmp_path), capture_output=True,
                           text=True)
        assert r.returncode == 0, r.stderr
        sr, out = read(str(tmp_path / name))
        assert sr == SR and out.shape[0] == HOP * (T - 1), (name, out.shape)
    # a keyframe without a voiced frame leaves the stream unshifted, and the run says so
    r = subprocess.run(base + ["-o", str(tmp_path / "d.wav"), "-stream_morph", "p1@0", "p3@0.5", "-stream_pitch", "mv"],
                       env=env, cwd=str(tmp_path), capture_output=True, text=True)
    assert r.returncode == 0 and "left unshifted" in r.stdout, (r.stdout, r.stderr)
