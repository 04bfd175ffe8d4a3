"""GPU: streaming conversion (adaptive_voice_conversion_b200/streaming.py) and its RTISI-LA kernel (avc_rtisi_la).

1. the streamed analysis equals the untrimmed offline analysis bit for bit, for any chunking and several streams;
2. every emitted mel block equals the restatement from AE.inference_from_embeddings on the window slices, bit for bit;
3. each RTISI-LA frame step matches the float64 restatement (tests/_rtisi_ref.py) from the kernel's own state;
4. a stream's output bits do not depend on its chunking or on the other streams of its updates;
5. a stream of T frames gives hop (T - 1) samples, and every sample n is out once input sample n + latency_samples
   has arrived, the worst one exactly then;
6. spectral convergence of the streamed synthesis on a harmonic signal, beside offline Griffin-Lim (printed).
"""
import types

import numpy as np
import pytest
import torch

import _rtisi_ref as R
import oracle.ae_oracle as orc
from _sn_ref import sn_config
from adaptive_voice_conversion_b200 import streaming as S
from adaptive_voice_conversion_b200.vocoder import AudioParams, Vocoder, griffin_lim

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
SR = 24000


def signal(n, seed):
    return torch.from_numpy(R.harmonic(n, SR, seed=seed).astype(np.float32)).to(DEV)


def chunks_of(y, sizes, seed=0):
    rng = np.random.default_rng(seed)
    out, k = [], 0
    while k < len(y):
        n = int(rng.integers(1, 3000)) if sizes == "random" else sizes
        out.append(y[k:k + n])
        k += n
    return out


def feed(obj, streams, close=True, fn="push"):
    """Lockstep feeding: streams {id: list of chunks}; returns {id: list of outputs}."""
    outs = {sid: [] for sid in streams}
    for k in range(max(len(c) for c in streams.values())):
        part = {sid: c[k] for sid, c in streams.items() if k < len(c)}
        for sid, v in getattr(obj, fn)(part).items():
            outs[sid].append(v)
    if close:
        for sid, v in getattr(obj, fn)({}, close=list(streams)).items():
            outs[sid].append(v)
    return outs


def test_analysis_bitwise():
    voc = Vocoder(n_mels=80, device=DEV)
    ana = S.StreamAnalyzer(voc)
    lens = [SR + 137, 2 * SR + 5, 30001, 4000, 52000]
    sizes = [1, 37, 300, 4800, "random"]
    ys = [signal(n, i) for i, n in enumerate(lens)]
    for i in range(len(ys)):
        ana.open(i)
    # chunk size 1 over a whole stream is slow: stream 0 gets 1-sample chunks for its first 3000 samples
    streams = {}
    for i, (y, s) in enumerate(zip(ys, sizes)):
        streams[i] = (chunks_of(y[:3000], 1) + chunks_of(y[3000:], 4800)) if s == 1 else chunks_of(y, s, seed=i)
    outs = feed(ana, streams)
    for i, y in enumerate(ys):
        got = torch.cat([o for o in outs[i] if o is not None])
        ref = voc.wav_to_mel([y], trim=False)[0][0]
        assert got.shape == ref.shape, (i, got.shape, ref.shape)
        assert torch.equal(got, ref), (i, (got - ref).abs().max())


def test_analysis_last_frame_alone():
    """hop = win/2 and a length that is a multiple of hop: at close the last frame is an entry of its own, and its end
    reflection reaches back to the entry's first sample that frame reads."""
    voc = Vocoder(n_mels=80, hp=AudioParams(hop_length=600), device=DEV)
    ana = S.StreamAnalyzer(voc)
    y = signal(600 * 40, 77)
    ana.open(0)
    before = ana.push({0: y})[0]
    last = ana.push({}, close=[0])[0]
    assert last.shape[0] == 1
    ref = voc.wav_to_mel([y], trim=False)[0][0]
    assert torch.equal(torch.cat([before, last]), ref)


def make_inf(cfg, attr=True):
    from adaptive_voice_conversion_b200.inference import Inferencer
    torch.manual_seed(0)
    inf = Inferencer(cfg, types.SimpleNamespace())
    inf.model.to(DEV)
    if attr:
        g = np.random.default_rng(3)
        n = cfg["SpeakerEncoder"]["c_in"]
        inf.attr = {"mean": g.uniform(0.2, 0.6, n).astype(np.float32), "std": g.uniform(0.1, 0.3, n).astype(np.float32)}
    return inf


def restate_blocks(inf, conv, mel, code, T):
    """The block schedule restated from the offline mel [T, n_mels]: each window converted alone, eagerly."""
    p, W, m = conv.p, conv.window, conv.m
    mean = torch.as_tensor(inf.attr["mean"]).to(DEV)
    std = torch.as_tensor(inf.attr["std"]).to(DEV)
    x = (mel - mean) / std
    w = torch.from_numpy(S.blend_weights(p.hop, p.lookahead)).to(DEV)[:, None]
    w_old = torch.from_numpy(np.float32(1) - S.blend_weights(p.hop, p.lookahead)).to(DEV)[:, None]
    out, prev, j = [], None, 0
    while True:
        b0, b1, w0, w1 = S.block_schedule(j, W, p.hop, p.lookahead, m)
        last = w1 > T
        if last:
            if b0 >= T:
                break
            (w0, w1), b1 = S.close_window(T, W), T
        dec = inf.model.inference_from_embeddings(x[w0:w1].t()[None].contiguous(), code[None])[0, :, :w1 - w0].t()
        rows = dec[b0 - w0:b1 - w0]
        X = min(w.shape[0], rows.shape[0])
        if prev is not None and X:
            rows = torch.cat([rows[:X] * w[:X] + prev[:X] * w_old[:X], rows[X:]])
        prev = dec[b1 - w0:b1 - w0 + w.shape[0]]
        out.append(rows)
        j += 1
        if last:
            break
    return torch.cat(out)


@pytest.mark.parametrize("cfg_name", ["c80", "c512", "sn"])
def test_blocks_bitwise(cfg_name):
    cfg = {"c80": lambda: orc.default_config(80), "c512": lambda: orc.default_config(512),
           "sn": lambda: sn_config(80)}[cfg_name]()
    inf = make_inf(cfg)
    n_mels = cfg["SpeakerEncoder"]["c_in"]
    voc = Vocoder(n_mels=n_mels, device=DEV)
    conv = S.StreamingConverter(inf, voc, S.StreamParams(gl_iters=1, keep_mels=True))
    lens = [3 * SR + 11, SR + 4000, 2 * SR]
    ys = [signal(n, 10 + i) for i, n in enumerate(lens)]
    codes = [torch.randn(conv.c_out, generator=torch.Generator().manual_seed(i)).to(DEV) for i in range(3)]
    ids = [conv.open(c) for c in codes]
    feed(conv, {sid: chunks_of(y, 2400 if k else "random", seed=k) for k, (sid, y) in enumerate(zip(ids, ys))},
         fn="update")
    for sid, y, code in zip(ids, ys, codes):
        got = conv.take_mels(sid)
        mel = voc.wav_to_mel([y], trim=False)[0][0]
        ref = restate_blocks(inf, conv, mel, code, mel.shape[0])
        assert got.shape == ref.shape == mel.shape, (got.shape, ref.shape, mel.shape)
        assert torch.equal(got, ref), (cfg_name, sid, (got - ref).abs().max())


def _stream_mags(T, seed):
    voc = Vocoder(n_mels=80, device=DEV)
    y = signal(voc.hp.hop_length * (T - 1), seed)
    return voc.mel_to_mag([voc.wav_to_mel([y], trim=False)[0][0]])[0][:T]


# fp32 against float64: a step agrees to a few 1e-4 of the frame's largest value.  The first frame's step is left out
# when K > 1: it enters alone with phase 0, so its spectrum is real, and the sign of each bin near a zero crossing is
# decided by rounding; iterating a lone frame amplifies those flips (K = 1 checks that step)
STEP_TOL = 2e-3


@pytest.mark.parametrize("la", [0, 1, 3, 7])
@pytest.mark.parametrize("K", [1, 8])
def test_rtisi_step_matches_restatement(la, K):
    hp = AudioParams()
    T = 14
    mags = _stream_mags(T, seed=la + 10 * K)
    rt = S.Rtisi(hp, la, K, DEV)
    rt.open(0)
    k, nb = rt.slot[0], la + 1
    win, nbin = hp.win_length, hp.n_bins
    worst = 0.0
    for f in range(T + 1):
        close = f == T
        # the kernel's state before the step, as the restatement's
        st_dev = rt.state[k].double().cpu().numpy()
        c, nbuf = (int(v) for v in rt.count[k].cpu())
        st = R.State(win, hp.hop_length, la)
        st.c, st.nbuf, st.carry = c, nbuf, float(st_dev[nb * win + nb * nbin + win])
        st.num = st_dev[nb * win + nb * nbin:nb * win + nb * nbin + win].copy()
        for F in range(c, c + nbuf):
            st.fr[F] = st_dev[(F % nb) * win:(F % nb + 1) * win].copy()
            st.mag[F] = st_dev[nb * win + (F % nb) * nbin:nb * win + (F % nb + 1) * nbin].copy()
        new = mags[f:f + 1] if not close else mags[:0]
        ref = R.step(st, new.double().cpu().numpy(), close, K, hp.preemphasis)
        got = rt.run({0: new} if not close else {}, close=(0,) if close else ())[0].double().cpu().numpy()
        if f == 0 and K > 1:
            continue
        assert got.shape == ref.shape, (f, got.shape, ref.shape)
        if len(ref):
            e = np.abs(got - ref).max() / (np.abs(ref).max() + 1e-6)
            worst = max(worst, e)
            assert e <= STEP_TOL, (la, K, f, e)
        if not close:
            after = rt.state[k].double().cpu().numpy()
            scale = np.abs(after[:nb * win]).max() + 1e-6
            for F in range(st.c, st.c + st.nbuf):
                e = np.abs(after[(F % nb) * win:(F % nb + 1) * win] - st.fr[F]).max() / scale
                worst = max(worst, e)
                assert e <= STEP_TOL, (la, K, f, F, e)
            assert [int(v) for v in rt.count[k].cpu()] == [st.c, st.nbuf]
    print(f"RTISI-LA step, lookahead {la}, K {K}: largest relative difference {worst:.2e}")


@pytest.fixture(scope="module")
def small():
    cfg = orc.default_config(80)
    inf = make_inf(cfg)
    voc = Vocoder(n_mels=80, device=DEV)
    return inf, voc


def test_invariance(small):
    inf, voc = small
    y = signal(2 * SR + 777, 42)
    code = torch.randn(128, generator=torch.Generator().manual_seed(5)).to(DEV)
    results = []
    for run, (size, others) in enumerate([(480, 0), (37 * 13, 3), ("random", 9)]):
        conv = S.StreamingConverter(inf, voc)
        streams = {}
        for o in range(others):
            sid = conv.open(torch.randn(128, generator=torch.Generator().manual_seed(100 + o)).to(DEV))
            streams[sid] = chunks_of(signal(SR + 1000 * o, 50 + o), 700 + 13 * o)
        sid = conv.open(code)
        streams[sid] = chunks_of(y, size, seed=run)
        results.append(torch.cat(feed(conv, streams, fn="update")[sid]))
    for r in results[1:]:
        assert torch.equal(r, results[0])


def test_memory_bounded_without_kept_mels(small):
    """Without keep_mels a stream keeps nothing that grows: after start-up, updates of the same size leave the same
    device memory allocated, and a closed stream leaves nothing behind."""
    inf, voc = small
    conv = S.StreamingConverter(inf, voc)
    ids = [conv.open(torch.randn(128, generator=torch.Generator().manual_seed(i)).to(DEV)) for i in range(4)]
    block = conv.p.hop * voc.hp.hop_length
    y = signal(block * 60, 9)
    mem = []
    for k in range(60):
        conv.push({sid: y[k * block:(k + 1) * block] for sid in ids})
        if k in (29, 59):
            torch.cuda.synchronize()
            mem.append(torch.cuda.memory_allocated(DEV))
    assert mem[1] == mem[0], mem
    assert all(not conv.streams[sid].mels for sid in ids)
    with pytest.raises(ValueError):
        conv.take_mels(ids[0])
    conv.update({}, close=ids)
    assert not conv.streams and not conv.closed


def test_grid_and_latency(small):
    inf, voc = small
    hp = voc.hp
    conv = S.StreamingConverter(inf, voc)
    lat = conv.latency_samples
    n_total = 3 * SR + 123
    y = signal(n_total, 7)
    # the output sample that waits longest, and the input sample whose arrival releases it
    worst = max(range(0, 40 * hp.hop_length),
                key=lambda n: S.release_sample(n, conv.p, hp.win_length, hp.hop_length, conv.m) - n)
    A = S.release_sample(worst, conv.p, hp.win_length, hp.hop_length, conv.m)
    assert A - worst == lat
    sid = conv.open(torch.randn(128, generator=torch.Generator().manual_seed(1)).to(DEV))
    got = 0
    bounds = sorted({A, A + 1} | set(range(997, n_total, 997)) | {n_total})
    for b0, b1 in zip([0] + bounds[:-1], bounds):
        got += conv.push({sid: y[b0:b1]})[sid].numel()
        # every sample n is out once input sample n + latency has arrived (samples 0 .. b1 - 1 have)
        assert got >= b1 - lat, (b1, got, lat)
        if b1 == A:            # the worst sample waits for input sample A ...
            assert got <= worst, (got, worst)
        if b1 == A + 1:        # ... and is out as soon as it arrives: the bound is reached
            assert got > worst, (got, worst)
    got += conv.close(sid).numel()
    T = 1 + n_total // hp.hop_length
    assert got == hp.hop_length * (T - 1)


def test_harmonic_sanity():
    hp = AudioParams()
    T = 160
    mags = _stream_mags(T, seed=3)
    S_ = mags.double().cpu().numpy()
    sc = {}
    for name, la, K in (("stream K=8", 3, 8), ("stream K=0", 3, 0)):
        rt = S.Rtisi(replace_pre(hp), la, K, DEV)
        rt.open(0)
        y = torch.cat([rt.run({0: mags[:T // 2]})[0], rt.run({0: mags[T // 2:]}, close=(0,))[0]])
        sc[name] = R.spectral_convergence(S_, y.double().cpu().numpy(), hp.win_length, hp.hop_length)
    for it in (8, 100):
        y = griffin_lim([mags], hp, n_iter=it)[0]
        sc[f"offline GL {it}"] = R.spectral_convergence(S_, y.double().cpu().numpy(), hp.win_length, hp.hop_length)
    print("spectral convergence:", {k: round(v, 4) for k, v in sc.items()})
    assert sc["stream K=8"] < sc["stream K=0"], sc


def replace_pre(hp):
    from dataclasses import replace
    return replace(hp, preemphasis=0.0)   # compare the synthesis itself, before de-emphasis
