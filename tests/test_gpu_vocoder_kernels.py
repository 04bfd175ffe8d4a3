"""GPU: the vocoder kernels (csrc/audio.cu) called through the C ABI, each against a float64 reference computed from
the kernel's own float32 inputs, at every window and hop the ABI accepts, 1 to 512 mels, full ragged batches and the
mel projection's largest row counts.

Every output buffer sits between sentinel guards, and the utterance table leaves NaN-filled gaps between utterances
in the signal: a kernel that reads a signal (STFT, frame power) gives the bits it gives on a packed table, and a
kernel that writes one (overlap-add, de-emphasis) leaves the gaps and guards as they were.  Bounds scale with the
magnitude of the terms (a frame's peak, sum |a_k b_k|, sum |a|^k |x[n-k]|), so quiet parts are held as tightly as
loud ones.  The tolerances are about 3x the worst error measured on the H100 (DESIGN.md section 6); each test prints
its worst per case."""
import ctypes as C

import numpy as np
import pytest
import scipy.signal as ss
import torch

import oracle.audio_oracle as ao
from test_gpu_vocoder import utterance

pytestmark = pytest.mark.gpu

NFFT, NBIN = 2048, 1025
FLT_MIN = float(np.finfo(np.float32).tiny)
GUARD = 64                                         # sentinel floats before and after every output buffer
SENTINEL = np.float32(-1.2345e33)
GAP_NAN = np.array([0x7FC0BEEF], np.uint32).view(np.float32)[0]   # a NaN payload no kernel produces

# every (win, hop) below is legal: even win <= 2048, 0 < hop <= win
PAIRS = [(1200, 300), (2048, 512), (2048, 2048), (600, 150), (300, 150), (2046, 1023), (2, 1)]

# about 3x the worst error measured on 1x H100 80GB HBM3 (700 W power limit); DESIGN.md section 6 lists the worst
TAU_STFT = 2.2e-6       # |X - E| / frame peak |E| (COMPLEX, MAG, X_prev of the projections)
TAU_PROJECT = 2e-6     # |X - S A/|A|| / (S peak|E| / max(1e-8, |A|))
TAU_ISTFT = 6e-7       # |y - ref| / ((P + WIN_ERR |ref| / TAU_ISTFT) sum|w| / sum w^2)
TAU_MEL_TO_MAG = 2.5e-6  # |out - ref| / sum_k |a_k b_k|, a_k the amplitude (its float32 prologue's error included)
TAU_MAG_TO_MEL = 1.2e-6  # the same before the dB epilogue (see check_mel)
EPI_MEL = 5e-7         # the dB epilogue's own float32 rounding (log10f within 2 ulp on |log10 v| <= 5), normalised
WIN_ERR = 2.0 ** -23   # absolute error of the float32 window 0.5 - 0.5 cospif(2q / win) (cancellation near its ends)
TAU_DEEMPH = 2e-6      # |y - lfilter| / lfilter(|x|) with |coef|
TAU_POWER = 3.4e-7      # relative


@pytest.fixture(scope="module")
def L():
    from adaptive_voice_conversion_b200 import _lib
    _lib.load()
    return _lib


def stream():
    return C.c_void_p(torch.cuda.current_stream().cuda_stream)


def ptr(t):
    return None if t is None else C.c_void_p(t.data_ptr())


def bits(t):
    return t.detach().view(torch.int32).cpu().numpy() if t.dtype == torch.float32 else t.cpu().numpy()


class Guarded:
    """A float32 device buffer of n elements between GUARD sentinels; ``check()`` asserts the guards are intact."""

    def __init__(self, n, fill=None):
        self.n = int(n)
        self.buf = torch.full((self.n + 2 * GUARD,), float(SENTINEL), device="cuda")
        self.t = self.buf[GUARD:GUARD + self.n]
        if fill is not None:
            self.t.copy_(torch.as_tensor(np.ascontiguousarray(fill, np.float32).reshape(-1)))

    def check(self, what=""):
        b = self.buf.view(torch.int32)
        b = torch.cat([b[:GUARD], b[GUARD + self.n:]]).cpu().numpy()
        want = np.array([SENTINEL], np.float32).view(np.int32)[0]
        assert (b == want).all(), f"{what}: a guard was overwritten"

    def np(self):
        return self.t.cpu().numpy()


class Table:
    """An avc_audio_seg table: utterance u's signal at sample_offs[u], with ``gap`` NaN floats before every utterance
    and after the last (gap 0: packed, as vocoder._Ragged lays them); frame rows packed."""

    def __init__(self, n_samples, n_frames, gap):
        from adaptive_voice_conversion_b200.vocoder import _SEG
        self.n_samples, self.n_frames, self.gap = [int(n) for n in n_samples], [int(n) for n in n_frames], gap
        self.sample_offs = [gap * (u + 1) + sum(self.n_samples[:u]) for u in range(len(self.n_samples))]
        self.frame_offs = [sum(self.n_frames[:u]) for u in range(len(self.n_frames))]
        self.span = gap * (len(self.n_samples) + 1) + sum(self.n_samples)
        self.rows = sum(self.n_frames)
        tab = np.zeros(len(self.n_samples), _SEG)
        tab["sample_off"], tab["n_samples"] = self.sample_offs, self.n_samples
        tab["frame_off"], tab["n_frames"] = self.frame_offs, self.n_frames
        self.dev = torch.from_numpy(tab.view(np.uint8)).cuda()

    def signal(self, ys):
        """The span as a guarded buffer: the signals at their offsets, GAP_NAN in the gaps."""
        h = np.full(self.span, GAP_NAN, np.float32)
        for o, y in zip(self.sample_offs, ys):
            h[o:o + len(y)] = y
        return Guarded(self.span, h)

    def split(self, y):
        return [y[o:o + n] for o, n in zip(self.sample_offs, self.n_samples)]

    def rows_of(self, x):
        return [x[o:o + n] for o, n in zip(self.frame_offs, self.n_frames)]

    def check_gaps(self, y, what):
        """The gaps of a signal buffer still hold GAP_NAN, bit for bit."""
        b = y.np().view(np.uint32)
        mask = np.ones(self.span, bool)
        for o, n in zip(self.sample_offs, self.n_samples):
            mask[o:o + n] = False
        assert (b[mask] == np.array([GAP_NAN], np.float32).view(np.uint32)[0]).all(), f"{what}: a gap was written"

    def desc(self, L, win, hop, n_fft=NFFT, **kw):
        d = L.AudioDesc(n_fft=n_fft, hop=hop, win=win, n_seg=len(self.n_samples), n_frames=self.rows,
                        n_samples=self.span, max_db=100.0, ref_db=20.0, segs=ptr(self.dev))
        for k, v in kw.items():
            if isinstance(v, Guarded):
                v = v.t
            setattr(d, k, ptr(v) if isinstance(v, torch.Tensor) or v is None else v)
        return d


def call(L, fn, d, *extra):
    L.check(getattr(L.load(), fn)(C.byref(d), *extra, stream()), fn)
    torch.cuda.synchronize()


def stft_lengths(hop):
    """The shortest legal utterance (1025 samples), lengths just over multiples of hop, a 512-frame utterance and one
    of 2000 frames; hop 1 gets short utterances only."""
    if hop == 1:
        return [1025, 1026, 1031, 1100]
    m = -(-1025 // hop)
    return [1025, m * hop + 1, (m + 3) * hop + 1, max(1025, 511 * hop + hop // 2), 2000 * hop + 7]


def signals(lengths, seed):
    """utterance()'s tones and noise, loud and quiet parts (the third utterance at 1e-3), silence in one of them."""
    out = []
    for i, n in enumerate(lengths):
        sil = (min(3000, n // 4), min(2500, n // 4)) if i == 1 else (0, 0)
        y = utterance(n, seed + i, silence=sil)
        if i == 2:
            y = y * np.float32(1e-3)
        out.append(y.astype(np.float32))
    return out


def frame_peak(E):
    return np.abs(E).max(axis=1, keepdims=True)


# ------------------------------------------------------------------ STFT
@pytest.fixture(scope="module", params=PAIRS, ids=[f"win{w}-hop{h}" for w, h in PAIRS])
def stft_case(request, L):
    """One ragged batch per (win, hop): signals, both tables, and the float64 spectra with and without pre-emphasis."""
    win, hop = request.param
    lengths = stft_lengths(hop)
    ys = signals(lengths, 100 + win + hop)
    frames = [1 + n // hop for n in lengths]
    pe = float(np.float32(0.97))
    ref = {pre: [ao.stft(ao.preemphasis(y, pe) if pre else y.astype(np.float64), NFFT, hop, win) for y in ys]
           for pre in (0.0, pe)}
    return dict(win=win, hop=hop, ys=ys, frames=frames, ref=ref, pe=pe,
                gapped=Table(lengths, frames, gap=37), packed=Table(lengths, frames, gap=0))


def run_stft(L, c, tab, mode, preemph, outs, **inputs):
    """avc_stft on the table; outs: {field: initial contents} of guarded outputs, inputs: other fields."""
    y = tab.signal(c["ys"])
    out = {k: Guarded(v.size, fill=v) for k, v in outs.items()}
    call(L, "avc_stft", tab.desc(L, c["win"], c["hop"], mode=mode, preemph=preemph, y=y, **out, **inputs))
    for k, g in out.items():
        g.check(f"avc_stft mode {mode} {k}")
    tab.check_gaps(y, "avc_stft input")
    return out


@pytest.mark.parametrize("pre", [False, True], ids=["plain", "preemph"])
def test_stft_mag_and_complex(L, stft_case, pre):
    c = stft_case
    pe = c["pe"] if pre else 0.0
    refs = c["ref"][pe]
    peaks = [frame_peak(E) for E in refs]
    worst = {"complex": 0.0, "mag": 0.0, "db_epilogue": 0.0}
    results = {}
    for name, tab in (("gapped", c["gapped"]), ("packed", c["packed"])):
        nan = np.full(tab.rows * NBIN, np.nan, np.float32)
        both = run_stft(L, c, tab, L.STFT_MAG, pe, dict(mag_out=nan, mag_db=nan))
        only_mag = run_stft(L, c, tab, L.STFT_MAG, pe, dict(mag_out=nan))
        only_db = run_stft(L, c, tab, L.STFT_MAG, pe, dict(mag_db=nan))
        cplx = run_stft(L, c, tab, L.STFT_COMPLEX, pe, dict(X=np.full(2 * tab.rows * NBIN, np.nan, np.float32)))
        # each output of MAG is the same with or without the other
        assert np.array_equal(bits(both["mag_out"].t), bits(only_mag["mag_out"].t))
        assert np.array_equal(bits(both["mag_db"].t), bits(only_db["mag_db"].t))
        results[name] = [bits(both["mag_out"].t), bits(both["mag_db"].t), bits(cplx["X"].t)]
        mag = tab.rows_of(both["mag_out"].np().reshape(-1, NBIN))
        db = tab.rows_of(both["mag_db"].np().reshape(-1, NBIN))
        X = tab.rows_of(cplx["X"].np().reshape(-1, NBIN, 2))
        for E, pk, m, g, x in zip(refs, peaks, mag, db, X):
            assert x.shape[0] == E.shape[0]
            scale = np.maximum(pk, 1e-300)
            ex = np.abs(x[..., 0] + 1j * x[..., 1].astype(np.float64) - E)
            em = np.abs(m - np.abs(E))
            assert (ex <= TAU_STFT * pk).all() and (em <= TAU_STFT * pk).all(), \
                (c["win"], c["hop"], float((ex / scale).max()), float((em / scale).max()))
            worst["complex"] = max(worst["complex"], float((ex / scale).max()))
            worst["mag"] = max(worst["mag"], float((em / scale).max()))
            # the dB epilogue on the kernel's own |X|
            ed = float(np.abs(g - ao.normalize_db(m.astype(np.float64))).max())
            assert ed < 1e-6, ed
            worst["db_epilogue"] = max(worst["db_epilogue"], ed)
    # a table with gaps reads the same samples as a packed one
    for a, b in zip(results["gapped"], results["packed"]):
        assert np.array_equal(a, b)
    print(f"\nstft win={c['win']} hop={c['hop']} preemph={pe:g} frames={c['frames']}: worst "
          + ", ".join(f"{k} {v:.2e}" for k, v in worst.items()))


@pytest.mark.parametrize("momentum", [0.0, 0.99])
@pytest.mark.parametrize("mode", ["PROJECT_FIRST", "PROJECT"])
def test_stft_projection(L, stft_case, mode, momentum):
    c = stft_case
    tab = c["gapped"]
    refs = c["ref"][0.0]
    E = np.concatenate(refs)
    pk = np.concatenate([frame_peak(e) for e in refs])
    rng = np.random.default_rng(7 + c["win"] + c["hop"])
    S = rng.uniform(0.0, 2.0, E.shape).astype(np.float32)
    P = (pk * (rng.standard_normal(E.shape) + 1j * rng.standard_normal(E.shape))).astype(np.complex64)
    m = np.float32(momentum)
    first = mode == "PROJECT_FIRST"
    p_in = np.full(2 * E.size, np.nan, np.float32) if first else P.view(np.float32).reshape(-1)
    out = run_stft(L, c, tab, getattr(L, "STFT_" + mode), 0.0, dict(X=np.full(2 * E.size, np.nan, np.float32),
                   X_prev=p_in), mag=torch.from_numpy(S.reshape(-1)).cuda(), momentum=float(m))
    # kernel's c: float32 m / (1 + m)
    cm = float(m / (np.float32(1) + m)) if m > 0 and not first else 0.0
    A = E - cm * P.astype(np.complex128)
    ref = S * A / np.maximum(1e-8, np.abs(A))
    got = out["X"].np().reshape(-1, NBIN, 2)
    err = np.abs(got[..., 0] + 1j * got[..., 1].astype(np.float64) - ref)
    bound = S * pk / np.maximum(1e-8, np.abs(A))
    r = err / np.maximum(bound, 1e-300)
    assert (err <= TAU_PROJECT * bound).all(), (mode, momentum, float(r.max()), np.unravel_index(r.argmax(), r.shape))
    msg = f"\nstft {mode} momentum={momentum} win={c['win']} hop={c['hop']}: worst err / bound-scale {r.max():.2e}"
    xp = out["X_prev"].np()
    if m > 0:          # P becomes E
        xp = xp.reshape(-1, NBIN, 2)
        ep = np.abs(xp[..., 0] + 1j * xp[..., 1].astype(np.float64) - E) / np.maximum(pk, 1e-300)
        assert (ep <= TAU_STFT).all(), float(ep.max())
        msg += f", X_prev {ep.max():.2e}"
    else:              # momentum 0 ignores X_prev: the buffer is untouched
        assert np.array_equal(xp.view(np.int32), p_in.view(np.int32))
    print(msg)


# ------------------------------------------------------------------ iSTFT
def cover_sums(n_frames, hop, win):
    """(sum |w|, sum w^2) over the frames covering each output sample (the oracle's grid, n_fft/2 cut at both ends)."""
    w = ao.window(NFFT, win)
    s1 = np.zeros(NFFT + hop * (n_frames - 1))
    s2 = np.zeros_like(s1)
    for f in range(n_frames):
        s1[f * hop:f * hop + NFFT] += np.abs(w)
        s2[f * hop:f * hop + NFFT] += w * w
    return s1[NFFT // 2:len(s1) - NFFT // 2], s2[NFFT // 2:len(s2) - NFFT // 2]


@pytest.mark.parametrize("win,hop", PAIRS, ids=[f"win{w}-hop{h}" for w, h in PAIRS])
def test_istft(L, win, hop):
    min_frames = 1 + -(-(NFFT // 2 + 1) // hop)
    T = [min_frames, min_frames + 1, min_frames + 37] + ([512, 2001] if hop > 1 else [1500])
    # spectra of signals at this window (consistent) and of a quiet one, as complex and as zero-phase magnitude
    specs = []
    for i, t in enumerate(T):
        y = utterance(max(1025, hop * (t - 1)), 300 + i, silence=(0, 0)).astype(np.float64)
        X = ao.stft(y, NFFT, hop, win)[:t] * (1e-3 if i == 1 else 1.0)
        specs.append(X.astype(np.complex64))
    n_samples = [hop * (t - 1) for t in T]
    tab = Table(n_samples, T, gap=53)
    worst = {}
    for kind in ("complex", "zero_phase"):
        if kind == "complex":
            spec = np.concatenate(specs).view(np.float32).reshape(-1)
            ins = [s.astype(np.complex128) for s in specs]
        else:
            spec = np.abs(np.concatenate(specs)).astype(np.float32).reshape(-1)
            ins = [np.abs(s).astype(np.float32).astype(np.float64) for s in specs]
        src = torch.from_numpy(spec).cuda()
        frames = Guarded(tab.rows * win)
        y = tab.signal([np.full(n, np.nan, np.float32) for n in n_samples])
        kw = dict(X=src, mag=None) if kind == "complex" else dict(X=None, mag=src)
        call(L, "avc_istft", tab.desc(L, win, hop, frames=frames, y=y, **kw))
        frames.check("avc_istft frames")
        y.check("avc_istft y")
        tab.check_gaps(y, "avc_istft")
        w = 0.0
        for X, z in zip(ins, tab.split(y.np())):
            ref = ao.istft(X, NFFT, hop, win)
            assert len(z) == len(ref)
            P = np.abs(np.fft.irfft(X, n=NFFT, axis=1)).max()
            s1, s2 = cover_sums(X.shape[0], hop, win)
            dead = s2 <= FLT_MIN
            assert (z[dead] == 0).all(), "where the window sum-square is 0 the output is exactly 0"
            live = ~dead
            # the frames' error (tau P |w| each) and the float32 window's own error, which the division by its
            # sum-square turns into a relative error WIN_ERR / |w| of the output where a single frame covers it
            scale = (TAU_ISTFT * P + WIN_ERR * np.abs(ref[live])) * s1[live] / s2[live] / TAU_ISTFT
            e = np.abs(z[live] - ref[live])
            assert (e <= TAU_ISTFT * scale).all(), (kind, float((e / scale).max()))
            w = max(w, float((e / scale).max()))
        worst[kind] = w
    print(f"\nistft win={win} hop={hop} T={T}: worst error / ((P + WIN_ERR |y| / tau) sum|w| / sum w^2) "
          + ", ".join(f"{k} {v:.2e}" for k, v in worst.items()))


# ------------------------------------------------------------------ mel projections
def mel_call(L, direction, rows, n_mels, n_bins, x, mat, max_db=100.0, ref_db=20.0):
    n_out = n_bins if direction == L.MEL_TO_MAG else n_mels
    out = Guarded(rows * n_out)
    d = L.MelDesc(rows=rows, n_mels=n_mels, n_bins=n_bins, dir=direction, max_db=max_db, ref_db=ref_db,
                  in_=ptr(x), mat=ptr(mat), out=ptr(out.t))
    L.check(L.load().avc_mel_project(C.byref(d), stream()), "avc_mel_project")
    torch.cuda.synchronize()
    out.check("avc_mel_project out")
    return out


def amplitude(v, max_db=100.0, ref_db=20.0):
    return 10.0 ** ((np.clip(np.asarray(v, np.float64), 0, 1) * max_db - max_db + ref_db) / 20.0)


def mel_ref(direction, x, mat, L):
    """(float64 result, sum_k |a_k b_k|) from the kernel's float32 operands; MEL_TO_MAG's a is the amplitude."""
    a = amplitude(x) if direction == L.MEL_TO_MAG else x.astype(np.float64)
    b = mat.astype(np.float64)
    return a @ b, np.abs(a) @ np.abs(b)


def norm_db(v):
    return np.clip((20 * np.log10(np.maximum(1e-5, v)) - 20.0 + 100.0) / 100.0, 1e-8, 1)


def amp_of(n):
    """The amplitude whose normalised dB is n (the epilogue's inverse on (1e-8, 1))."""
    return 10.0 ** ((n * 100.0 + 20.0 - 100.0) / 20.0)


def check_mel(direction, got, ref, mag, L):
    """Asserts the bound and returns the worst err / sum_k |a_k b_k|.  MAG_TO_MEL is compared after the dB
    epilogue, which is monotone: the kernel's value must lie in the epilogue's image of [ref - tau mag, ref + tau mag],
    widened by EPI_MEL.  The returned value is then the least tau that holds: the distance from ref to the amplitudes
    whose images, widened by EPI_MEL, reach the kernel's value (0 where the value is within EPI_MEL of the image)."""
    scale = np.maximum(mag, 1e-300)
    if direction == L.MEL_TO_MAG:
        e = np.abs(got - ref)
        assert (e <= TAU_MEL_TO_MAG * mag).all(), float((e / scale).max())
        return float((e / scale).max())
    lo, hi = norm_db(ref - TAU_MAG_TO_MEL * mag), norm_db(ref + TAU_MAG_TO_MEL * mag)
    assert ((got >= lo - EPI_MEL) & (got <= hi + EPI_MEL)).all(), \
        float(np.maximum(lo - EPI_MEL - got, got - hi - EPI_MEL).max())
    up, down = got - EPI_MEL, got + EPI_MEL          # the image must reach up to `up` and down to `down`
    need_up = np.where(up > 1e-8, amp_of(np.minimum(up, 1.0)) - ref, 0.0)
    need_down = np.where(down < 1.0, ref - amp_of(np.maximum(down, 1e-8)), 0.0)
    need_down = np.where(down <= 1e-8, 0.0, need_down)
    return float((np.maximum(0.0, np.maximum(need_up, need_down)) / scale).max())


def mel_operands(direction, rows, n_mels, n_bins, kind, rng):
    """(input, matrix) float32: the real filterbank / pseudo-inverse or a signed random matrix; MEL_TO_MAG inputs
    reach past both ends of [0, 1]; MAG_TO_MEL magnitudes span 1e-7 .. 1e3 (below the 1e-5 floor and above the clip)
    with a zero row."""
    if kind == "filterbank":
        fb = ao.mel_filterbank(24000, NFFT, n_mels)
        mat = (ao.mel_to_linear_matrix(fb).T if direction == L_MEL_TO_MAG else fb.T)
    else:
        shape = (n_mels, n_bins) if direction == L_MEL_TO_MAG else (n_bins, n_mels)
        mat = rng.standard_normal(shape) * 0.1
    if direction == L_MEL_TO_MAG:
        x = rng.uniform(-0.3, 1.3, (rows, n_mels))
    else:
        x = 10.0 ** rng.uniform(-7, 3, (rows, n_bins))
        x[0] = 0.0
    return np.ascontiguousarray(x, np.float32), np.ascontiguousarray(mat, np.float32)


L_MEL_TO_MAG = 0
MEL_SHAPES = ([(m, NBIN, "filterbank") for m in (1, 17, 80, 100, 512)]
              + [(m, b, "random") for m in (1, 17, 80, 100, 512) for b in (NBIN, 63, 64, 65)])


@pytest.mark.parametrize("direction", [0, 1], ids=["mel_to_mag", "mag_to_mel"])
def test_mel_project(L, direction):
    assert L.MEL_TO_MAG == L_MEL_TO_MAG
    rng = np.random.default_rng(11 + direction)
    worst = {}
    cases = [(r, *s) for s in MEL_SHAPES for r in (1, 63, 64, 65)]
    cases += [(64 * 512, 80, NBIN, "filterbank"), (64 * 512, 512, NBIN, "filterbank"), (64 * 512, 512, NBIN, "random")]
    for rows, n_mels, n_bins, kind in cases:
        x, mat = mel_operands(direction, rows, n_mels, n_bins, kind, rng)
        out = mel_call(L, direction, rows, n_mels, n_bins, torch.from_numpy(x).cuda(), torch.from_numpy(mat).cuda())
        got = out.np().reshape(rows, -1).astype(np.float64)
        ref, mag = mel_ref(direction, x, mat, L)
        key = f"{kind} n_mels={n_mels} n_bins={n_bins}"
        worst[key] = max(worst.get(key, 0.0), check_mel(direction, got, ref, mag, L))
    print(f"\nmel_project dir={direction}: worst error / sum|ab| per shape (rows 1, 63, 64, 65 and 32768):")
    for k, v in worst.items():
        print(f"  {k}: {v:.2e}")


def test_mel_project_beyond_65535_row_tiles(L):
    """4 194 321 rows: 65 537 row tiles of 64, the last one partial.  Tiny n_mels / n_bins keep it under 0.5 GB."""
    rows, n_mels, n_bins = 4194304 + 17, 3, 5
    split = 65535 * 64
    g = torch.Generator(device="cuda").manual_seed(3)
    for direction in (L.MEL_TO_MAG, L.MAG_TO_MEL):
        k_in, n_out = (n_mels, n_bins) if direction == L.MEL_TO_MAG else (n_bins, n_mels)
        x = torch.rand(rows, k_in, device="cuda", generator=g) * 1.4 - 0.2
        if direction == L.MAG_TO_MEL:
            x = x.abs() * 50
        mat = torch.rand(k_in, n_out, device="cuda", generator=g) - 0.25
        big = mel_call(L, direction, rows, n_mels, n_bins, x, mat).t.view(rows, n_out)
        lo = mel_call(L, direction, split, n_mels, n_bins, x[:split], mat).t.view(split, n_out)
        hi = mel_call(L, direction, rows - split, n_mels, n_bins, x[split:], mat).t.view(rows - split, n_out)
        assert torch.equal(big[:split], lo) and torch.equal(big[split:], hi)
        tail = slice(rows - 17 - 64, rows)      # the last full tile and the partial one
        ref, mag = mel_ref(direction, x[tail].cpu().numpy(), mat.cpu().numpy(), L)
        w = check_mel(direction, big[tail].cpu().numpy().astype(np.float64), ref, mag, L)
        print(f"\nmel_project dir={direction} rows={rows}: equal to two smaller calls; last tiles {w:.2e} of sum|ab|")


# ------------------------------------------------------------------ de-emphasis
DEEMPH_LENGTHS = [1, 2, 1023, 1024, 1025, 2049, 3073, 4000, 7777, 10000, 1_000_003]


@pytest.mark.parametrize("coef", [0.0, 0.5, 0.97, 0.999, 1.0, -0.97])
def test_deemphasis(L, coef):
    """1025 and 2049 samples leave trailing threads with empty chunks (per = 2 and 3); 4000 to 10000 give chunks of
    4 to 10 samples, so a carry at coef >= 0.999 crosses many warps before it decays."""
    rng = np.random.default_rng(17)
    xs = []
    for n in DEEMPH_LENGTHS:
        env = 10.0 ** rng.uniform(-3, 0, 1 + n // 500).repeat(500)[:n]
        xs.append((rng.standard_normal(n) * env).astype(np.float32))
    tab = Table(DEEMPH_LENGTHS, [0] * len(xs), gap=29)
    y = tab.signal(xs)
    a = np.float32(coef)
    call(L, "avc_deemphasis", tab.desc(L, 1200, 300, y=y), C.c_float(a))
    y.check("avc_deemphasis")
    tab.check_gaps(y, "avc_deemphasis")
    worst = 0.0
    for x, z in zip(xs, tab.split(y.np())):
        if coef == 0.0:
            assert np.array_equal(z, x)
            continue
        ref = ss.lfilter([1.0], [1.0, -float(a)], x.astype(np.float64))
        scale = ss.lfilter([1.0], [1.0, -abs(float(a))], np.abs(x.astype(np.float64)))
        e = np.abs(z - ref)
        assert (e <= TAU_DEEMPH * scale).all(), (len(x), float((e / scale).max()))
        worst = max(worst, float((e / scale).max()))
    print(f"\ndeemphasis coef={coef}: worst error / lfilter(|x|, |coef|) {worst:.2e}")


# ------------------------------------------------------------------ frame power
@pytest.mark.parametrize("n_fft,hop", [(2048, 512), (2, 1), (4096, 2048)])
def test_frame_power(L, n_fft, hop):
    rng = np.random.default_rng(n_fft + hop)
    lengths = [n_fft // 2 + 1, 5000, 3 * hop + 1, 48013] if hop > 1 else [2, 3, 700, 5001]
    ys = [np.zeros(lengths[0], np.float32),                                        # silent
          (0.5 * rng.standard_normal(lengths[1])).astype(np.float32),              # loud
          utterance(max(lengths[2], 1025), 5, silence=(0, 0))[:lengths[2]],         # tone
          utterance(lengths[3], 6) if lengths[3] > 6000 else                        # mixed: silence, tone, silence
          np.concatenate([np.zeros(2000, np.float32), utterance(1001, 7, silence=(0, 0)),
                          np.zeros(lengths[3] - 3001, np.float32)])]
    frames = [1 + len(y) // hop for y in ys]
    res = []
    worst = 0.0
    for gap in (41, 0):
        tab = Table([len(y) for y in ys], frames, gap)
        y = tab.signal(ys)
        p = Guarded(tab.rows, np.full(tab.rows, np.nan, np.float32))
        call(L, "avc_frame_power", tab.desc(L, n_fft, hop, n_fft=n_fft, y=y), ptr(p.t))
        p.check("avc_frame_power")
        res.append(bits(p.t))
        for yy, got in zip(ys, tab.rows_of(p.np())):
            ref = ao.frame_power(yy, n_fft, hop)
            assert (got[ref == 0] == 0).all()
            nz = ref > 0
            e = np.abs(got[nz] - ref[nz]) / ref[nz]
            assert (e <= TAU_POWER).all(), float(e.max())
            worst = max(worst, float(e.max(initial=0.0)))
    assert np.array_equal(res[0], res[1])
    print(f"\nframe_power n_fft={n_fft} hop={hop}: worst relative error {worst:.2e}")


# ------------------------------------------------------------------ argument checks
def test_argument_checks(L):
    lib = L.load()
    tab = Table([5000], [1 + 5000 // 300], gap=0)
    y = torch.zeros(5000, device="cuda")
    X = torch.zeros(tab.rows * NBIN * 2, device="cuda")
    fr = torch.zeros(tab.rows * 1200, device="cuda")
    pw = torch.zeros(tab.rows, device="cuda")
    s = stream()
    INVALID, UNSUPPORTED = L.ERR_INVALID, L.ERR_UNSUPPORTED
    n0 = L.launch_count()

    def expect(rc, code, text):
        assert rc == code, (rc, code, L.last_error())
        assert text in L.last_error(), (text, L.last_error())

    good = dict(X=X, frames=fr, y=y)
    for change, code, text in [
            (dict(X=None, mag=None), INVALID, "null X/mag, frames or y"),
            (dict(frames=None), INVALID, "null X/mag, frames or y"),
            (dict(y=None), INVALID, "null X/mag, frames or y"),
            (dict(win=1201), UNSUPPORTED, "win must be even"),
            (dict(win=2050), UNSUPPORTED, "win must be even"),
            (dict(hop=1201), UNSUPPORTED, "hop must be in (0, win]"),
            (dict(hop=0), UNSUPPORTED, "hop must be in (0, win]"),
            (dict(n_fft=1024), UNSUPPORTED, "only n_fft = 2048"),
            (dict(segs=None), INVALID, "empty or missing utterance table"),
            (dict(n_seg=0), INVALID, "empty or missing utterance table")]:
        kw = dict(good)
        geo = {k: change.pop(k) for k in list(change) if k in ("win", "hop", "n_fft")}
        kw.update(change)
        d = tab.desc(L, geo.get("win", 1200), geo.get("hop", 300), n_fft=geo.get("n_fft", NFFT), **kw)
        expect(lib.avc_istft(C.byref(d), s), code, text)
    expect(lib.avc_istft(None, s), INVALID, "null descriptor")

    for change, text in [(dict(y=None), "null argument or empty table"), (dict(segs=None), "null argument or empty table"),
                         (dict(n_seg=0), "null argument or empty table")]:
        d = tab.desc(L, 1200, 300, y=y)
        for k, v in change.items():
            setattr(d, k, v)
        expect(lib.avc_deemphasis(C.byref(d), C.c_float(0.97), s), INVALID, text)
    expect(lib.avc_deemphasis(None, C.c_float(0.97), s), INVALID, "null argument or empty table")

    d = tab.desc(L, 2048, 512, y=y)
    expect(lib.avc_frame_power(C.byref(d), None, s), INVALID, "null argument or empty table")
    expect(lib.avc_frame_power(None, ptr(pw), s), INVALID, "null argument or empty table")
    for change, text in [(dict(y=None), "null argument or empty table"), (dict(n_seg=0), "null argument or empty table"),
                         (dict(n_fft=2047), "bad frame length"), (dict(n_fft=0), "bad frame length"),
                         (dict(hop=0), "bad frame length"), (dict(n_frames=-1), "bad frame length")]:
        d = tab.desc(L, 2048, 512, y=y)
        for k, v in change.items():
            setattr(d, k, v)
        expect(lib.avc_frame_power(C.byref(d), ptr(pw), s), INVALID, text)

    a = torch.zeros(64 * 80, device="cuda")
    m = torch.zeros(80 * NBIN, device="cuda")
    o = torch.zeros(64 * NBIN, device="cuda")
    for change, text in [(dict(in_=None), "null argument"), (dict(mat=None), "null argument"),
                         (dict(out=None), "null argument"), (dict(rows=-1), "bad shape"), (dict(n_mels=0), "bad shape"),
                         (dict(n_bins=0), "bad shape"), (dict(max_db=0.0), "bad shape"), (dict(dir=2), "unknown dir"),
                         (dict(dir=-1), "unknown dir")]:
        d = L.MelDesc(rows=64, n_mels=80, n_bins=NBIN, dir=L.MEL_TO_MAG, max_db=100.0, ref_db=20.0, in_=ptr(a),
                      mat=ptr(m), out=ptr(o))
        for k, v in change.items():
            setattr(d, k, v)
        expect(lib.avc_mel_project(C.byref(d), s), INVALID, text)
    expect(lib.avc_mel_project(None, s), INVALID, "null argument")
    assert L.launch_count() == n0
    # the checks left the stream usable, and rows = 0 is a valid empty call
    d = L.MelDesc(rows=0, n_mels=80, n_bins=NBIN, dir=L.MEL_TO_MAG, max_db=100.0, ref_db=20.0, in_=ptr(a), mat=ptr(m),
                  out=ptr(o))
    assert lib.avc_mel_project(C.byref(d), s) == 0
    assert L.launch_count() == n0
    d = tab.desc(L, 1200, 300, y=y)
    L.check(lib.avc_deemphasis(C.byref(d), C.c_float(0.97), s))
    torch.cuda.synchronize()
