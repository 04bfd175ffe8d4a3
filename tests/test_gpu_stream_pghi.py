"""GPU: the streamed PGHI start of RTISI-LA.  avc_pghi_stream against the float64 restatement
(tests/_stream_pghi_ref.py) and against avc_pghi, its launch splits and neighbouring streams; avc_rtisi_la_from against
avc_istft and the restatement; Rtisi and StreamingConverter with gl_init "pghi"; the argument checks."""
import ctypes as C

import numpy as np
import pytest
import torch

import _pghi_ref as P
import _rtisi_ref as R
import _stream_pghi_ref as SP
from adaptive_voice_conversion_b200 import _lib as L
from adaptive_voice_conversion_b200 import streaming as S
from adaptive_voice_conversion_b200.vocoder import AudioParams, _ptr
from test_gpu_vocoder_pghi import PHASE_BOUND, V, consistent, dev, mel_inverse, tied  # noqa: F401 (V: fixture)

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
NB = 1025
TOL = 1e-5


class Pool:
    """avc_pghi_stream state slots and one launch over a table of (slot, new rows, close)."""

    def __init__(self, slots, win=1200, hop=300):
        self.win, self.hop = win, hop
        self.state = torch.zeros(slots, int(L.load().avc_pghi_stream_state_floats(2048)), device=DEV)
        self.n = [0] * slots

    def launch(self, entries, parent=True):
        rows, offs, slots, closes, outs = [], [0], [], [], [0]
        for slot, m, close in entries:
            p = 0 if m is None else m.shape[0]
            if p:
                rows.append(torch.as_tensor(m, device=DEV))
            n0, n1 = self.n[slot], self.n[slot] + p
            done = (n1 if close else max(0, n1 - 1)) - max(0, n0 - 1)
            self.n[slot] = n1
            offs.append(offs[-1] + p)
            slots.append(slot)
            closes.append(int(close))
            outs.append(outs[-1] + done)
        n = len(entries)
        mag = torch.cat(rows).float().contiguous() if rows else torch.zeros(1, NB, device=DEV)
        i32 = torch.tensor(offs + slots + closes + outs, dtype=torch.int32, device=DEV)
        mout = torch.full((max(1, outs[-1]), NB), float("nan"), device=DEV)
        X = torch.full((max(1, outs[-1]), NB, 2), float("nan"), device=DEV)
        par = torch.full((max(1, outs[-1]), NB), -1, dtype=torch.int8, device=DEV)
        d = L.PghiStreamDesc(n_fft=2048, hop=self.hop, win=self.win, n_streams=n, mag=_ptr(mag),
                             mag_off=_ptr(i32[:n + 1]), slot=_ptr(i32[n + 1:2 * n + 1]),
                             close=_ptr(i32[2 * n + 1:3 * n + 1]), out_off=_ptr(i32[3 * n + 1:]), mag_out=_ptr(mout),
                             X=_ptr(X), state=_ptr(self.state))
        L.check(L.load().avc_pghi_stream(C.byref(d), C.c_float(TOL), _ptr(par) if parent else None, None),
                "avc_pghi_stream")
        torch.cuda.synchronize()
        return [(mout[a:b].cpu(), torch.view_as_complex(X[a:b]).cpu(), par[a:b].cpu())
                for a, b in zip(outs[:-1], outs[1:])]


def run_stream(s, win=1200, hop=300, split=None):
    """One stream through avc_pghi_stream in the launches split gives (frame counts, the last closing)."""
    pool = Pool(1, win, hop)
    split = split or [len(s)]
    outs, f = [], 0
    for i, p in enumerate(split):
        outs.append(pool.launch([(0, s[f:f + p] if p else None, i == len(split) - 1)])[0])
        f += p
    return tuple(torch.cat(v) for v in zip(*outs))


def cases(V):
    out = []
    for i, T in enumerate([1, 2, 5, 40, 300]):
        c = consistent(T, 10 + i).astype(np.float32)
        ramp = np.linspace(0.2, 1.0, T, dtype=np.float32)[:, None]
        out += [("consistent", c), ("crescendo", c * ramp), ("mel80", mel_inverse(V, T, 80, 20 + i)),
                ("mel512", mel_inverse(V, T, 512, 30 + i) * ramp), ("tied", tied(T, 40 + i)),
                ("silent", np.zeros((T, NB), np.float32))]
    return out


def check(kind, s, got, win=1200, hop=300):
    mout, x, par = got
    phi, want = SP.stream_pghi(s, TOL, hop, win)
    assert np.array_equal(mout.numpy(), s)
    assert np.array_equal(par.numpy(), want), (kind, s.shape, np.argwhere(par.numpy() != want)[:5])
    sig = want != P.NONE
    x = x.numpy()
    if not sig.any():
        assert not x.any()
        return 0.0
    assert np.allclose(np.abs(x), s, rtol=1e-6, atol=0)
    return float(np.abs(P.wrap(np.angle(x[sig]) - phi[sig])).max())


def test_matches_restatement(V):
    worst = 0.0
    for kind, s in cases(V):
        worst = max(worst, check(kind, s, run_stream(s)))
    print(f"worst wrapped phase error {worst:.2e} rad")
    assert worst < PHASE_BOUND, worst


@pytest.mark.parametrize("win,hop", [(4, 1), (64, 1), (600, 150), (1200, 300), (2046, 1023), (2048, 512),
                                     (2048, 1024), (1024, 256)])
def test_every_window(V, win, hop):
    for kind, s in [("consistent", consistent(40, 3).astype(np.float32) * np.linspace(0.2, 1, 40, dtype=np.float32)[:, None]),
                    ("tied", tied(5, 4))]:
        assert check(kind, s, run_stream(s, win, hop), win, hop) < PHASE_BOUND


def test_early_maximum_is_avc_pghi_bitwise(V):
    for T in (1, 2, 5, 40, 300):
        s = consistent(T, 50 + T).astype(np.float32)
        s[min(1, T - 1)] *= 4
        assert s[:2].max() == s.max()
        m, x, par = run_stream(s)
        X, par_o = V.pghi([dev(s)], parent=True)
        assert torch.equal(torch.view_as_real(x), torch.view_as_real(X[0].cpu()))
        assert torch.equal(par, par_o[0].cpu())


def test_launch_splits_bitwise(V):
    s = mel_inverse(V, 40, 512, 7) * np.linspace(0.2, 1, 40, dtype=np.float32)[:, None]
    whole = run_stream(s)
    for split in ([1] * 40 + [0], [0, 3, 0, 0, 17, 1, 19, 0], [1, 1, 38], [39, 1], [40, 0]):
        got = run_stream(s, split=split)
        assert torch.equal(whole[0].view(torch.int32), got[0].view(torch.int32)), split
        assert torch.equal(torch.view_as_real(whole[1]).view(torch.int32), torch.view_as_real(got[1]).view(torch.int32))
        assert torch.equal(whole[2], got[2]), split


def test_many_streams_and_slot_reuse(V):
    rng = np.random.default_rng(1)
    mags = [mel_inverse(V, int(T), 80, 60 + i) for i, T in enumerate(rng.integers(2, 30, 12))]
    alone = [run_stream(s) for s in mags]
    pool = Pool(16)
    pos, got = [0] * 12, [[] for _ in mags]
    slots = list(rng.permutation(16)[:12])
    pool.state[:].normal_()                          # reuse: a stream starts from a zeroed slot
    for k in slots:
        pool.state[int(k)].zero_()
    while any(p < len(s) for p, s in zip(pos, mags)):
        ent, who = [], []
        for i, s in enumerate(mags):
            if pos[i] >= len(s):
                continue
            p = int(rng.integers(0, 4))
            p = min(p, len(s) - pos[i])
            ent.append((int(slots[i]), s[pos[i]:pos[i] + p] if p else None, pos[i] + p == len(s)))
            who.append(i)
            pos[i] += p
        for i, o in zip(who, pool.launch(ent)):
            got[i].append(o)
    for i in range(12):
        g = tuple(torch.cat(v) for v in zip(*got[i]))
        assert torch.equal(torch.view_as_real(g[1]), torch.view_as_real(alone[i][1])) and torch.equal(g[2], alone[i][2])


def _istft_frames_X(X, hop=300, win=1200):
    """avc_istft of X (complex [T, NB]) through Vocoder's own path."""
    from adaptive_voice_conversion_b200.vocoder import _Ragged, _call
    hp = AudioParams(hop_length=hop, win_length=win)
    T = X.shape[0]
    r = _Ragged([hop * (T - 1)], [T], DEV)
    Xd = torch.view_as_real(X.to(DEV)).contiguous()
    y = torch.empty(hop * (T - 1), device=DEV)
    fr = torch.empty(T, win, device=DEV)
    _call("avc_istft", r.desc(hp, X=_ptr(Xd), frames=_ptr(fr), y=_ptr(y)), torch.device(DEV))
    return y


def rtisi_from(hp, X, mags, la, K, split=None):
    rt = S.Rtisi(hp, la, K, DEV)
    rt.open("a")
    T = X.shape[0]
    split = split or [T]
    out, f = [], 0
    for i, p in enumerate(split):
        close = ("a",) if i == len(split) - 1 else ()
        launch = rt.prepare({"a": mags[f:f + p]} if p else {}, close)
        f += p
        if launch is None:                 # an empty update launches nothing
            continue
        p0 = f - p
        Xd = torch.view_as_real(X[p0:f].to(DEV)).contiguous() if p else torch.zeros(1, NB, 2, device=DEV)
        L.check(L.load().avc_rtisi_la_from(C.byref(launch[0]), _ptr(Xd), None), "avc_rtisi_la_from")
        out.append(launch[1]["a"].clone())
    torch.cuda.synchronize()
    return torch.cat(out)


def test_rtisi_from_k0_is_istft(V):
    hp = AudioParams(preemphasis=0.0)
    s = consistent(40, 5).astype(np.float32)
    X = V.pghi([dev(s)])[0]
    y = rtisi_from(hp, X.cpu(), dev(s), 3, 0)
    ref = _istft_frames_X(X.cpu())
    assert y.shape == ref.shape
    print("max |rtisi_from - istft|", float((y - ref).abs().max()), "peak", float(ref.abs().max()))
    assert torch.allclose(y, ref, rtol=0, atol=2e-6 * float(ref.abs().max()))


@pytest.mark.parametrize("la", [0, 1, 3, 7])
def test_rtisi_from_matches_restatement(V, la):
    hp = AudioParams(preemphasis=0.97)
    s = consistent(24, 6).astype(np.float32)
    X = SP.stream_X(s).astype(np.complex64)
    y = rtisi_from(hp, torch.from_numpy(X), dev(s), la, 8).cpu().numpy()
    ref = SP.rtisi_from(X.astype(np.complex128), s, 1200, 300, la, 8, 0.97)
    assert len(y) == len(ref) == 300 * 23
    assert np.abs(y - ref).max() <= 5e-4 * np.abs(ref).max(), np.abs(y - ref).max() / np.abs(ref).max()
    # launch splits bitwise
    y2 = rtisi_from(hp, torch.from_numpy(X), dev(s), la, 8, split=[1, 0, 5, 1, 17]).cpu().numpy()
    assert np.array_equal(y.view(np.int32), y2.view(np.int32))


def test_rtisi_pghi_pool_chunking_and_neighbours(V):
    hp = AudioParams()
    mags = [mel_inverse(V, T, 512, 70 + T) for T in (9, 33, 50)]

    def run(splits, order):
        rt = S.Rtisi(hp, 3, 8, DEV, init="pghi")
        for i in order:
            rt.open(i)
        pos, out = [0, 0, 0], {i: [] for i in order}
        for step in range(max(len(s) for s in splits)):
            ch, close = {}, []
            for i in order:
                if step < len(splits[i]):
                    p = splits[i][step]
                    if p:
                        ch[i] = dev(mags[i][pos[i]:pos[i] + p])
                    pos[i] += p
                    if step == len(splits[i]) - 1:
                        close.append(i)
            for k, v in rt.run(ch, close).items():
                out[k].append(v.clone())
        return {i: torch.cat(v) for i, v in out.items()}

    a = run([[9], [33], [50]], [0, 1, 2])
    b = run([[1] * 9, [5, 0, 7, 21], [2] * 25], [2, 1, 0])
    for i, T in enumerate((9, 33, 50)):
        assert a[i].numel() == 300 * (T - 1)
        assert torch.equal(a[i], b[i])
    # frame by frame: X from the kernel equals the stream's own, through Rtisi
    X = SP.stream_X(mags[1]).astype(np.complex64)
    ref = rtisi_from(hp, torch.from_numpy(X), dev(mags[1]), 3, 8).cpu().numpy()
    assert np.abs(a[1].cpu().numpy() - ref).max() <= 1e-3 * np.abs(ref).max()


def test_argument_checks_launch_nothing():
    lib = L.load()
    n0 = lib.avc_launch_count()
    z = torch.zeros(4, dtype=torch.int32, device=DEV)
    f = torch.zeros(2, NB, device=DEV)
    st = torch.zeros(1, int(lib.avc_pghi_stream_state_floats(2048)), device=DEV)
    assert lib.avc_pghi_stream_state_floats(1024) == 0

    def pd(**kw):
        a = dict(n_fft=2048, hop=300, win=1200, n_streams=1, mag=_ptr(f), mag_off=_ptr(z), slot=_ptr(z),
                 close=_ptr(z), out_off=_ptr(z), mag_out=_ptr(f), X=_ptr(f), state=_ptr(st))
        a.update(kw)
        return L.PghiStreamDesc(**a)
    for kw, tol in [(dict(n_fft=1024), TOL), (dict(win=1201), TOL), (dict(hop=601), TOL), (dict(hop=0), TOL),
                    (dict(n_streams=-1), TOL), ({}, 0.0), ({}, 1.0), ({}, float("nan")), (dict(X=None), TOL),
                    (dict(state=None), TOL), (dict(mag_out=None), TOL)]:
        assert lib.avc_pghi_stream(C.byref(pd(**kw)), C.c_float(tol), None, None) != 0, kw
    assert lib.avc_pghi_stream(None, C.c_float(TOL), None, None) != 0
    rd = L.RtisiDesc(n_fft=2048, hop=300, win=1200, lookahead=3, n_iter=8, n_streams=1, mag=_ptr(f), mag_off=_ptr(z),
                     slot=_ptr(z), close=_ptr(z), out_off=_ptr(z), y=_ptr(f), state=_ptr(f), count=_ptr(z))
    assert lib.avc_rtisi_la_from(C.byref(rd), None, None) != 0
    for k, v in (("n_fft", 1024), ("hop", 601), ("lookahead", 8), ("n_iter", -1), ("win", 1201)):
        bad = L.RtisiDesc.from_buffer_copy(rd)
        setattr(bad, k, v)
        assert lib.avc_rtisi_la_from(C.byref(bad), _ptr(f), None) != 0, k
    bad = L.RtisiDesc.from_buffer_copy(rd)
    bad.deemph = float("inf")
    assert lib.avc_rtisi_la_from(C.byref(bad), _ptr(f), None) != 0
    assert lib.avc_launch_count() == n0


# ------------------------------------------------------------------ the converter with gl_init="pghi"
from test_gpu_stream import chunks_of, feed, signal, small  # noqa: E402,F401 (small: fixture)

SR = 24000
PGHI = S.StreamParams(gl_init="pghi")


def test_converter_invariance(small):
    inf, voc = small
    y = signal(2 * SR + 777, 42)
    code = torch.randn(128, generator=torch.Generator().manual_seed(5)).to(DEV)
    results = []
    for run, (size, others) in enumerate([(480, 0), (37 * 13, 3), ("random", 5)]):
        conv = S.StreamingConverter(inf, voc, PGHI)
        streams = {}
        for o in range(others):
            sid = conv.open(torch.randn(128, generator=torch.Generator().manual_seed(100 + o)).to(DEV))
            streams[sid] = chunks_of(signal(SR + 1000 * o, 50 + o), 700 + 13 * o)
        sid = conv.open(code)
        streams[sid] = chunks_of(y, size, seed=run)
        results.append(torch.cat(feed(conv, streams, fn="update")[sid]))
    T = 1 + y.numel() // voc.hp.hop_length
    assert results[0].numel() == voc.hp.hop_length * (T - 1)
    for r in results[1:]:
        assert torch.equal(r, results[0])


def _worst_case(conv, hp, release):
    worst = max(range(0, 60 * hp.hop_length), key=lambda n: release(n) - n)
    return worst, release(worst)


@pytest.mark.parametrize("pitch", [None, "mv"])
def test_converter_grid_and_latency(small, pitch):
    """The measured wait of the output sample that waits longest equals latency_samples (tracked_latency_samples for
    an mv stream), as test_gpu_stream.test_grid_and_latency measures it."""
    inf, voc = small
    hp = voc.hp
    conv = S.StreamingConverter(inf, voc, PGHI)
    if pitch is None:
        lat = conv.latency_samples
        worst, A = _worst_case(conv, hp, lambda n: S.release_sample(n, conv.p, hp.win_length, hp.hop_length, conv.m))
        assert lat == S.latency_samples(PGHI, hp.win_length, hp.hop_length, conv.m)
    else:
        lat = conv.tracked_latency_samples
        worst, A = _worst_case(conv, hp, lambda n: S.tracked_release_sample(n, conv.p, hp.win_length, hp.hop_length,
                                                                            conv.m, conv.stage.span))
    assert A - worst == lat
    n_total = 3 * SR + 123
    y = signal(n_total, 7)
    sid = conv.open(torch.randn(128, generator=torch.Generator().manual_seed(1)).to(DEV),
                    None if pitch is None else ("mv", 7.5, 0.2))
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
    assert got == hp.hop_length * (n_total // hp.hop_length)


def test_converter_pitch_and_retarget_compose(small):
    inf, voc = small
    y = signal(2 * SR, 11)
    codes = [torch.randn(128, generator=torch.Generator().manual_seed(k)).to(DEV) for k in (1, 2)]
    outs = []
    for size in (480, "random"):
        conv = S.StreamingConverter(inf, voc, S.StreamParams(gl_init="pghi", keep_mels=True))
        a = conv.open(codes[0], 3.0)
        b = conv.open(codes[0], ("mv", 7.5, 0.2))
        conv.retarget(a, codes[1], at=60, ramp=16)
        conv.retarget(b, codes[1], at=80, ramp=0)
        out = feed(conv, {a: chunks_of(y, size, 1), b: chunks_of(y, size, 2)}, fn="update")
        outs.append({k: torch.cat(v) for k, v in out.items()})
        mels = conv.take_mels(a)
        # the mel frames do not depend on the start phase
        ref = S.StreamingConverter(inf, voc, S.StreamParams(keep_mels=True))
        r = ref.open(codes[0], 3.0)
        ref.retarget(r, codes[1], at=60, ramp=16)
        feed(ref, {r: chunks_of(y, size, 1)}, fn="update")
        assert torch.equal(mels, ref.take_mels(r))
    for k in outs[0]:
        assert outs[0][k].numel() == 300 * (y.numel() // 300)
        assert torch.equal(outs[0][k], outs[1][k])


def test_harmonic_sanity():
    """Spectral convergence of the estimate and PGHI starts on the mel pseudo-inverse of a synthetic crescendo."""
    from adaptive_voice_conversion_b200 import vocoder
    T, sc = 160, {}
    y = R.harmonic(300 * (T - 1), SR, seed=3) * np.linspace(0.2, 1.0, 300 * (T - 1))
    A = R.stft_mag(y, 1200, 300)
    import oracle.audio_oracle as ao
    for n_mels in (80, 512):
        voc = vocoder.Vocoder(n_mels=n_mels, device=DEV)
        mel = ao.mel_filterbank(n_mels=n_mels) @ A.T
        norm = np.clip((20 * np.log10(np.maximum(1e-5, mel.T)) - 20 + 100) / 100, 1e-8, 1).astype(np.float32)
        mags = voc.mel_to_mag([dev(norm)])[0]
        S_ = mags.double().cpu().numpy()
        hp = AudioParams(preemphasis=0.0)
        for init in ("estimate", "pghi"):
            for la, K in ((3, 8), (2, 8), (1, 2), (0, 0)):
                rt = S.Rtisi(hp, la, K, DEV, init)
                rt.open(0)
                out = torch.cat([rt.run({0: mags[:T // 2]})[0], rt.run({0: mags[T // 2:]}, close=(0,))[0]])
                sc[(n_mels, init, la, K)] = R.spectral_convergence(S_, out.double().cpu().numpy(), 1200, 300)
    for k, v in sorted(sc.items()):
        print("spectral convergence", k, round(v, 4))
    for n_mels in (80, 512):
        assert sc[(n_mels, "pghi", 0, 0)] < sc[(n_mels, "estimate", 0, 0)], sc
    assert sc[(512, "pghi", 3, 8)] < sc[(512, "estimate", 3, 8)], sc
