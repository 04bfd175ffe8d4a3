"""GPU: the corpus-preparation kernels avc_resample_poly, avc_mel_moments and avc_mel_moments_merge (csrc/prep.cu)
called through the C ABI with tables built here, so that every layout the ABI accepts is reachable, not only those
prepare.Preparer produces, and preprocess.py end to end at 512 mels and targets other than 24 kHz.

1. avc_resample_poly against float64 scipy.signal.resample_poly of the float64 channel mean of the same PCM, at every
   pair of the file rates RATES to the targets TARGETS, int16 and float32, 1, 2, 3 and 6 channels, n_in 1, half_len
   +- 1 and lengths whose n_out ends at a tile edge, in ragged batches at odd offsets; the identity rate; batch
   independence; the tap-table limits; an utterance of n_out = 2^31 - 1;
2. avc_mel_moments and avc_mel_moments_merge against math.fsum two-pass sums at 1 to 1025 mels, utterances of 0, 1
   and 50 000 frames, 5 000 utterances fed in chunks, zero counts, and values far from zero;
3. preprocess.run at --n_mels 512 to 16 and 22.05 kHz from files at 8 to 48 kHz against the float64 oracle.

Every output region lies between sentinel guards with GAP_NAN gaps between utterances, and the input has poison
between utterances (NaN for float32, 32767 for int16): a window that reads a neighbour, or a tile that writes past its
utterance's n_out, fails.  The resampler's bound is TAU_RS of sum_k |x_k t_k| per output, about 3x the worst measured
on the H100 (DESIGN.md section 6); each case prints its worst."""
import ctypes as C
import math
import os
import pickle

import numpy as np
import pytest
import torch
from scipy.io import wavfile
from scipy.signal import firwin, resample_poly

import oracle.audio_oracle as ao
from adaptive_voice_conversion_b200 import _lib as L
from adaptive_voice_conversion_b200 import prepare as P
from adaptive_voice_conversion_b200.vocoder import _SEG
from test_gpu_prepare import to_s16, utterance
from test_gpu_vocoder_kernels import GAP_NAN, Guarded

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
TILE = L.RESAMPLE_TILE
RATES = [8000, 11025, 12000, 16000, 22050, 24000, 32000, 44100, 48000, 88200, 96000, 176400, 192000]
TARGETS = [16000, 22050, 24000, 44100, 48000]
PAIRS = sorted({P.rate_pair(r, t) for r in RATES for t in TARGETS} - {(1, 1)})
CHANNELS = [1, 2, 3, 6]
S16_POISON = 32767
GAP_BITS = np.array([GAP_NAN], np.float32).view(np.uint32)[0]
GAP_I32 = int(np.array([GAP_NAN], np.float32).view(np.int32)[0])
# |kernel - float64| <= TAU_RS * sum_k |x_k| |t_k| per output, |x_k| the mean of the channels' magnitudes (a float32
# channel sum of random-sign values can cancel to far below its terms)
TAU_RS = 2e-6


def stream():
    return C.c_void_p(torch.cuda.current_stream().cuda_stream)


def rates_of(up, down):
    return [f"{r / 1000:g}->{t / 1000:g} kHz" for t in TARGETS for r in RATES if P.rate_pair(r, t) == (up, down)]


# ------------------------------------------------------------------ resampler helpers
class Batch:
    """Utterances of one PCM format in one device buffer, each at an odd element offset with poison in the gaps, and
    their outputs in one Guarded buffer with GAP_NAN gaps; tile0 in the order given."""

    def __init__(self, utts, n_outs, gap=5):
        s16 = utts[0].dtype == np.int16
        self.fmt = L.PCM_S16 if s16 else L.PCM_F32
        self.in_offs, pos = [], gap
        for a in utts:
            pos += 1 - pos % 2
            self.in_offs.append(pos)
            pos += a.size + gap
        pcm = np.full(pos, S16_POISON if s16 else np.nan, np.int16 if s16 else np.float32)
        for o, a in zip(self.in_offs, utts):
            pcm[o:o + a.size] = a.reshape(-1)
        self.pcm = torch.from_numpy(pcm).to(DEV)
        self.n_outs = [int(n) for n in n_outs]
        self.out_offs, pos = [], gap
        for n in self.n_outs:
            self.out_offs.append(pos)
            pos += n + gap
        self.span = pos
        tab = np.zeros(len(utts), P._RSEG)
        tab["in_off"], tab["out_off"] = self.in_offs, self.out_offs
        tab["n_in"] = [a.shape[0] for a in utts]
        tab["n_out"] = self.n_outs
        tab["channels"] = [1 if a.ndim == 1 else a.shape[1] for a in utts]
        tiles = -(-tab["n_out"].astype(np.int64) // TILE)
        tab["tile0"] = np.concatenate([[0], np.cumsum(tiles)[:-1]])
        self.n_tiles = int(tiles.sum())
        self.segs = torch.from_numpy(tab.view(np.uint8)).to(DEV)

    def run(self, up, down):
        """One avc_resample_poly launch; asserts the guards and gaps are intact; the outputs as float32 numpy."""
        out = Guarded(self.span, np.full(self.span, GAP_NAN, np.float32))
        half, n_taps, taps = table(up, down)
        d = L.ResampleDesc(format=self.fmt, up=up, down=down, half_len=half, n_taps=n_taps, n_seg=len(self.n_outs),
                           n_tiles=self.n_tiles, segs=self.segs.data_ptr(), pcm=self.pcm.data_ptr(),
                           taps=None if taps is None else taps.data_ptr(), out=out.t.data_ptr())
        L.check(L.load().avc_resample_poly(C.byref(d), stream()), "avc_resample_poly")
        torch.cuda.synchronize()
        out.check(f"avc_resample_poly {up}/{down}")
        h = out.np()
        mask = np.ones(self.span, bool)
        for o, n in zip(self.out_offs, self.n_outs):
            mask[o:o + n] = False
        assert (h.view(np.uint32)[mask] == GAP_BITS).all(), f"{up}/{down}: a gap between outputs was written"
        return [h[o:o + n].copy() for o, n in zip(self.out_offs, self.n_outs)]


_TABLES = {}


def table(up, down):
    """(half_len, n_taps, float32 device taps) of prepare.resample_taps, or (0, 0, None) at the identity."""
    if (up, down) == (1, 1):
        return 0, 0, None
    if (up, down) not in _TABLES:
        half, tab = P.resample_taps(up, down)
        _TABLES[(up, down)] = (half, tab.shape[1], torch.from_numpy(tab.astype(np.float32)).to(DEV))
    return _TABLES[(up, down)]


def mono64(a, magnitude=False):
    """The float64 channel mean of PCM as the kernel reads it, or with magnitude the mean of the channels' |values|."""
    x = a.astype(np.float64) / (32768.0 if a.dtype == np.int16 else 1.0)
    if magnitude:
        x = np.abs(x)
    return x.mean(axis=1) if x.ndim == 2 else x


def pcm(rng, n, fmt, ch):
    shape = (n, ch) if ch > 1 else (n,)
    if fmt == "s16":
        return rng.integers(-32768, 32768, shape).astype(np.int16)
    return (0.5 * rng.standard_normal(shape)).astype(np.float32)


def lengths(up, down):
    """(n_in, n_out): n_in 1 and half_len +- 1 at their own n_out; and the shortest n_in whose n_out reaches 511, 512,
    513 and 1025, with the table's n_out set to exactly that (the ABI takes any n_out up to ceil(n_in up / down))."""
    half = 10 * max(up, down)
    out = [(n, P.n_resampled(n, up, down)) for n in (1, half - 1, half + 1)]
    return out + [((t - 1) * down // up + 1, t) for t in (511, 512, 513, 1025)]


def errors(a, y, up, down):
    """|y - float64| / sum_k |x_k| |t_k| per output (0 where both are exactly 0; inf where the sum is 0 and y is not)."""
    x = mono64(a)
    h = firwin(20 * max(up, down) + 1, 1.0 / max(up, down), window=("kaiser", 5.0))
    ref = resample_poly(x, up, down, window=h)[:len(y)]
    scale = resample_poly(mono64(a, magnitude=True), up, down, window=np.abs(h))[:len(y)]
    assert len(ref) == len(y), (up, down, len(x), len(y), len(ref))
    assert np.isfinite(y).all(), (up, down, len(x), "non-finite output: a window read poison, or a tile was skipped")
    d = np.abs(y.astype(np.float64) - ref)
    with np.errstate(divide="ignore", invalid="ignore"):
        return np.where(scale > 0, d / np.where(scale > 0, scale, 1), np.where(d == 0, 0.0, np.inf))


def pair_cases(up, down, seed):
    """Per format, the utterances of every channel count and length, in a seeded shuffled order."""
    rng = np.random.default_rng(seed)
    cases = {}
    for fmt in ("s16", "f32"):
        items = [(pcm(rng, n, fmt, ch), n_out) for ch in CHANNELS for n, n_out in lengths(up, down)]
        cases[fmt] = [items[i] for i in rng.permutation(len(items))]
    return cases


# ------------------------------------------------------------------ resampler
@pytest.mark.parametrize("up, down", PAIRS)
def test_resampler_matches_resample_poly_at_every_rate_pair(up, down):
    worst = (0.0, None)
    for fmt, items in pair_cases(up, down, up * 7919 + down).items():
        ys = Batch([a for a, _ in items], [n for _, n in items]).run(up, down)
        for (a, n_out), y in zip(items, ys):
            e = float(errors(a, y, up, down).max())
            if e > worst[0] or worst[1] is None:
                worst = (e, (fmt, a.shape, n_out))
    print(f"resample {up}/{down} ({', '.join(rates_of(up, down))}): worst {worst[0]:.2e} of sum|x t| at {worst[1]}"
          f" (bound {TAU_RS:.0e})")
    assert worst[0] <= TAU_RS, worst


def test_identity_rate_is_exact_for_mono_and_within_one_ulp_for_stereo():
    rng = np.random.default_rng(11)
    for fmt in ("s16", "f32"):
        items = [pcm(rng, n, fmt, ch) for ch in (1, 2) for n in (1, 511, 512, 513, 1025, 4099)]
        ys = Batch(items, [a.shape[0] for a in items]).run(1, 1)
        for a, y in zip(items, ys):
            r32 = mono64(a).astype(np.float32)
            if a.ndim == 1 or a.dtype == np.int16:
                assert np.array_equal(y.view(np.uint32), r32.view(np.uint32)), (fmt, a.shape)
            else:
                assert (np.abs(y - r32) <= np.spacing(np.abs(r32))).all(), (fmt, a.shape)


@pytest.mark.parametrize("up, down", [(1, 2), (80, 147), (640, 147), (147, 1280), (1, 12)])
def test_each_utterance_gets_the_same_bits_alone_shuffled_and_at_another_tile0(up, down):
    items = pair_cases(up, down, 5)["s16"][:12] + pair_cases(up, down, 6)["f32"][:12]
    by_fmt = {}
    for i, (a, n) in enumerate(items):
        by_fmt.setdefault(a.dtype.str, []).append(i)
    for idx in by_fmt.values():
        batch = Batch([items[i][0] for i in idx], [items[i][1] for i in idx]).run(up, down)
        perm = np.random.default_rng(up + down).permutation(len(idx))
        shuffled = Batch([items[idx[j]][0] for j in perm], [items[idx[j]][1] for j in perm]).run(up, down)
        for k, j in enumerate(perm):
            assert np.array_equal(shuffled[k].view(np.uint32), batch[j].view(np.uint32)), (up, down, "shuffled", j)
        for k, i in enumerate(idx):
            a, n = items[i]
            alone = Batch([a], [n]).run(up, down)[0]
            later = Batch([items[idx[0]][0], items[idx[-1]][0], a], [items[idx[0]][1], items[idx[-1]][1], n]).run(up, down)[2]
            assert np.array_equal(alone.view(np.uint32), batch[k].view(np.uint32)), (up, down, "alone", i)
            assert np.array_equal(later.view(np.uint32), batch[k].view(np.uint32)), (up, down, "later tile0", i)


# (up, down) whose table is exactly at a limit, and one past each
AT_LIMIT = [(4, 51), (128, 1633)]        # 256 taps per phase; 256 and 32 768 in all
PAST_LIMIT = [(5, 64), (331, 1638)]      # 257 taps per phase; 99 per phase, 32 769 in all


@pytest.mark.parametrize("up, down", AT_LIMIT)
def test_tables_at_the_limits_are_computed(up, down):
    half, n_taps, taps = table(up, down)
    assert n_taps == L.RESAMPLE_MAX_PHASE_TAPS and up * n_taps in (1024, L.RESAMPLE_MAX_TAPS)
    worst = 0.0
    for fmt, items in pair_cases(up, down, up + 3 * down).items():
        items = [it for it in items if it[0].ndim == 1 or it[0].shape[1] in (2, 3)]
        ys = Batch([a for a, _ in items], [n for _, n in items]).run(up, down)
        worst = max([worst] + [float(errors(a, y, up, down).max()) for (a, _), y in zip(items, ys)])
    print(f"resample {up}/{down} ({n_taps} taps per phase, {up * n_taps} in all): worst {worst:.2e} (bound {TAU_RS:.0e})")
    assert worst <= TAU_RS


@pytest.mark.parametrize("up, down", PAST_LIMIT)
def test_tables_past_the_limits_are_refused_without_a_launch(up, down):
    half, tab = P.resample_taps(up, down)
    assert tab.shape[1] > L.RESAMPLE_MAX_PHASE_TAPS or tab.size > L.RESAMPLE_MAX_TAPS
    taps = torch.from_numpy(tab.astype(np.float32)).to(DEV)
    b = Batch([np.zeros(4000, np.int16)], [P.n_resampled(4000, up, down)])
    out = torch.zeros(b.span, device=DEV)
    d = L.ResampleDesc(format=b.fmt, up=up, down=down, half_len=half, n_taps=tab.shape[1], n_seg=1, n_tiles=b.n_tiles,
                       segs=b.segs.data_ptr(), pcm=b.pcm.data_ptr(), taps=taps.data_ptr(), out=out.data_ptr())
    n0 = L.launch_count()
    assert L.load().avc_resample_poly(C.byref(d), stream()) == L.ERR_UNSUPPORTED
    assert "taps per phase" in L.last_error() and L.launch_count() == n0, L.last_error()
    assert not P.resample_supported(up, down)


def test_an_utterance_of_two_to_the_31_minus_1_outputs_is_written_to_its_end():
    """Up 2 / down 1 from n_in = 2^30 int16 samples with n_out = 2^31 - 1 (about 10 GiB): the last tile's m0 + 512
    passes INT_MAX.  Every output is written, the guard after the last is intact, and the first and last tiles equal
    float64 resample_poly over the input window they read."""
    n_in, n_out, up, down = 2 ** 30, 2 ** 31 - 1, 2, 1
    need = 2 * n_in + 4 * (n_out + 2 * 64) + (1 << 30)
    free = torch.cuda.mem_get_info()[0]
    if free < need:
        pytest.skip(f"needs {need / 2 ** 30:.1f} GiB of free device memory, {free / 2 ** 30:.1f} GiB free")
    g = torch.Generator(device=DEV).manual_seed(31)
    x = torch.randint(-32768, 32768, (n_in,), dtype=torch.int16, device=DEV, generator=g)
    tab = np.zeros(1, P._RSEG)
    tab["n_in"], tab["n_out"], tab["channels"], tab["out_off"] = n_in, n_out, 1, 64
    segs = torch.from_numpy(tab.view(np.uint8)).to(DEV)
    out = torch.full((n_out + 128,), GAP_I32, dtype=torch.int32, device=DEV).view(torch.float32)
    half, n_taps, taps = table(up, down)
    n_tiles = -(-n_out // TILE)
    d = L.ResampleDesc(format=L.PCM_S16, up=up, down=down, half_len=half, n_taps=n_taps, n_seg=1, n_tiles=n_tiles,
                       segs=segs.data_ptr(), pcm=x.data_ptr(), taps=taps.data_ptr(), out=out.data_ptr())
    L.check(L.load().avc_resample_poly(C.byref(d), stream()), "avc_resample_poly")
    torch.cuda.synchronize()
    ob = out.view(torch.int32)
    assert (ob[:64] == GAP_I32).all() and (ob[64 + n_out:] == GAP_I32).all(), "a guard was overwritten"
    step = 1 << 28
    for s in range(64, 64 + n_out, step):
        assert not torch.isnan(out[s:min(64 + n_out, s + step)]).any(), f"outputs from {s - 64} on were not written"
    h = firwin(2 * half + 1, 1.0 / max(up, down), window=("kaiser", 5.0))
    worst = 0.0
    for m0 in (0, (n_tiles - 1) * TILE):
        m1 = min(n_out, m0 + TILE)
        # resample_poly of x[a:] gives y[a up + j] for every j >= 2 half_len: the terms before a fall off the filter
        a = max(0, (m0 - 2 * half) // up)
        k1 = min(n_in, (m1 - 1) * down // up + half + 1)
        xs = x[a:k1].cpu().numpy().astype(np.float64) / 32768.0
        ref = resample_poly(xs, up, down, window=h)[m0 - a * up:m1 - a * up]
        scale = resample_poly(np.abs(xs), up, down, window=np.abs(h))[m0 - a * up:m1 - a * up]
        y = out[64 + m0:64 + m1].double().cpu().numpy()
        assert len(ref) == m1 - m0
        worst = max(worst, float((np.abs(y - ref) / scale).max()))
    print(f"n_out 2^31 - 1: first and last tiles within {worst:.2e} of sum|x t| (bound {TAU_RS:.0e})")
    assert worst <= TAU_RS


# ------------------------------------------------------------------ corpus statistics
def moments(mels, n_mels, mom, first, gap=2):
    """avc_mel_moments of `mels` ([frames, n_mels] float32 each) into mom[first ...]; every utterance has `gap` NaN
    rows before it, and the last one after it."""
    offs, pos = [], 0
    for m in mels:
        pos += gap
        offs.append(pos)
        pos += len(m)
    host = np.full((pos + gap, n_mels), np.nan, np.float32)
    for o, m in zip(offs, mels):
        host[o:o + len(m)] = m
    x = torch.from_numpy(host).to(DEV)
    tab = np.zeros(len(mels), _SEG)
    tab["frame_off"], tab["n_frames"] = offs, [len(m) for m in mels]
    segs = torch.from_numpy(tab.view(np.uint8)).to(DEV)
    d = L.MomentsDesc(n_mels=n_mels, n_seg=len(mels), first=first, segs=segs.data_ptr(), mels=x.data_ptr(),
                      moments=mom.data_ptr())
    L.check(L.load().avc_mel_moments(C.byref(d), stream()), "avc_mel_moments")


def merge(mom, counts, n_mels):
    cnt = torch.tensor(counts, dtype=torch.int32, device=DEV)
    f32 = torch.full((2, n_mels), float("nan"), device=DEV)
    f64 = torch.full((2, n_mels), float("nan"), dtype=torch.float64, device=DEV)
    L.check(L.load().avc_mel_moments_merge(mom.data_ptr(), cnt.data_ptr(), len(counts), n_mels, f32[0].data_ptr(),
                                           f32[1].data_ptr(), f64[0].data_ptr(), f64[1].data_ptr(), stream()),
            "avc_mel_moments_merge")
    return f32.cpu().numpy(), f64.cpu().numpy()


def fsum_moments(cols):
    """Two-pass (mean, M2) of each row of cols [n_mels, frames] float64 with math.fsum."""
    n = cols.shape[1]
    mean = np.array([math.fsum(c) / n for c in cols.tolist()])
    return mean, np.array([math.fsum(v) for v in ((cols - mean[:, None]) ** 2).tolist()])


def check_merge(f32, f64, frames, what):
    """f32 / f64 of avc_mel_moments_merge against the fsum two-pass mean and std (ddof 0) of all frames: float64
    within 1e-12 of max(|mean|, std) per mel (the magnitude of the values: a float64 sum of values near c has an
    absolute error of order eps c, whatever their spread), float32 within one ulp of the rounded reference.  Returns the
    reference (mean, std) and the float64 errors relative to that scale."""
    mean, m2 = fsum_moments(np.concatenate(frames).astype(np.float64).T)
    std = np.sqrt(m2 / sum(len(f) for f in frames))
    scale = np.maximum(np.abs(mean), std)
    errs = []
    for got, ref, name in ((f64[0], mean, "mean"), (f64[1], std, "std")):
        errs.append(float((np.abs(got - ref) / scale).max()))
        assert errs[-1] <= 1e-12, (what, name, errs[-1])
    for got, ref in ((f32[0], mean), (f32[1], std)):
        r32 = ref.astype(np.float32)
        assert (np.abs(got - r32) <= np.spacing(np.abs(r32))).all(), (what, np.abs(got - r32).max())
    return mean, std, errs


@pytest.mark.parametrize("n_mels", [1, 80, 127, 128, 129, 512, 1025])
def test_moments_and_merge_match_fsum(n_mels):
    rng = np.random.default_rng(n_mels)
    frames = [0, 1, 50000, 3, 0, 700, 2]
    mels = [(0.3 + 0.4 * rng.random((t, n_mels))).astype(np.float32) for t in frames]
    mom = torch.full((len(mels) + 3, n_mels, 2), float("nan"), dtype=torch.float64, device=DEV)
    moments(mels, n_mels, mom, 2)
    host = mom.cpu().numpy()
    assert np.isnan(host[:2]).all() and np.isnan(host[2 + len(mels):]).all(), "moments written outside [first, first+n)"
    worst = 0.0
    for u, m in enumerate(mels):
        got = host[2 + u]
        if len(m) == 0:
            assert (got == 0).all(), (n_mels, u)
            continue
        mean, m2 = fsum_moments(m.astype(np.float64).T)
        em = float((np.abs(got[:, 0] - mean) / np.abs(mean)).max())
        eq = float(np.abs(got[:, 1] - m2).max() / max(m2.max(), 1e-300)) if len(m) > 1 else float(np.abs(got[:, 1]).max())
        assert em <= 1e-12 and eq <= 1e-12, (n_mels, len(m), em, eq)
        worst = max(worst, em, eq)
    f32, f64 = merge(mom[2:2 + len(mels)], frames, n_mels)
    _, _, errs = check_merge(f32, f64, mels, n_mels)
    print(f"moments at {n_mels} mels: worst relative {worst:.1e} per utterance, merged mean and std {max(errs):.1e} "
          "(bound 1e-12)")


def test_merge_of_values_far_from_zero_and_zero_counts():
    """Values 1e4 + U(0, 2) in utterances of different means: Chan's update keeps the std within 1e-12 of the values'
    magnitude, where a running sum of squares minus N mean^2 does not.  Zero and negative counts are skipped even
    when their moments are NaN."""
    n_mels = 200
    rng = np.random.default_rng(9)
    mels = [(1e4 + rng.random() + rng.random((int(t), n_mels))).astype(np.float32) for t in rng.integers(1, 3000, 9)]
    mom = torch.full((len(mels), n_mels, 2), float("nan"), dtype=torch.float64, device=DEV)
    moments(mels, n_mels, mom, 0)
    f32, f64 = merge(mom, [len(m) for m in mels], n_mels)
    mean, std, errs = check_merge(f32, f64, mels, "offset")
    cat = np.concatenate(mels).astype(np.float64)
    n = len(cat)
    naive = np.sqrt(np.maximum(0, np.cumsum(cat ** 2, axis=0)[-1] / n - (np.cumsum(cat, axis=0)[-1] / n) ** 2))
    naive_err = float((np.abs(naive - std) / np.maximum(np.abs(mean), std)).max())
    print(f"offset values: merged mean and std within {max(errs):.1e}, a running sum of squares {naive_err:.1e}")
    assert naive_err > 1e-11, "the values are not far enough from zero to tell the two updates apart"
    poisoned = torch.cat([torch.full((2, n_mels, 2), float("nan"), dtype=torch.float64, device=DEV), mom[:4],
                          torch.full((1, n_mels, 2), float("nan"), dtype=torch.float64, device=DEV), mom[4:]])
    counts = [0, -3] + [len(m) for m in mels[:4]] + [0] + [len(m) for m in mels[4:]]
    g32, g64 = merge(poisoned, counts, n_mels)
    assert np.array_equal(g64.view(np.uint64), f64.view(np.uint64)) and np.array_equal(g32.view(np.uint32),
                                                                                       f32.view(np.uint32))


def test_five_thousand_utterances_in_chunks_give_the_bytes_of_one_call():
    n_mels, n_utts = 512, 5000
    rng = np.random.default_rng(5000)
    frames = rng.integers(0, 40, n_utts)
    frames[[0, 17, 4999]] = 0
    mels = [(0.2 + 0.6 * rng.random((int(t), n_mels))).astype(np.float32) for t in frames]
    one = torch.full((n_utts, n_mels, 2), float("nan"), dtype=torch.float64, device=DEV)
    moments(mels, n_mels, one, 0)
    split = torch.full_like(one, float("nan"))
    for a, b in ((0, 1), (1, 700), (700, 701), (701, 2500), (2500, 5000)):
        moments(mels[a:b], n_mels, split, a)
    assert np.array_equal(one.cpu().numpy().view(np.uint64), split.cpu().numpy().view(np.uint64))
    f32, f64 = merge(one, [int(t) for t in frames], n_mels)
    check_merge(f32, f64, mels, "5000 utterances")


# ------------------------------------------------------------------ preprocess.py at 512 mels, 16 and 22.05 kHz
FILE_RATES = [8000, 16000, 22050, 44100, 48000]
E2E_OPTS = dict(n_out_speakers=1, test_prop=0.34, n_utts_attr=10, n_mels=512, segment_size=128, training_samples=50,
                testing_samples=10, seed=3)


@pytest.fixture(scope="module")
def rate_tree(tmp_path_factory):
    root = tmp_path_factory.mktemp("rates")
    rng = np.random.default_rng(1616)
    wav = os.path.join(str(root), "wav")
    speakers = ["225", "226", "227", "228"]
    for s, spk in enumerate(speakers):
        os.makedirs(os.path.join(wav, f"p{spk}"))
        for i in range(3):
            rate = FILE_RATES[(3 * s + i) % len(FILE_RATES)]
            wavfile.write(os.path.join(wav, f"p{spk}", f"p{spk}_{i + 1:03d}.wav"), rate,
                          to_s16(utterance(rng, rate, rng.uniform(3.5, 4.5))))
    info = os.path.join(str(root), "speaker-info.txt")
    with open(info, "w") as f:
        f.write("ID  AGE  GENDER  ACCENTS  REGION\n")
        f.writelines(f"{s}  23  F  English  Somewhere\n" for s in speakers)
    return root, wav, info


@pytest.mark.parametrize("sr", [16000, 22050])
def test_preprocess_at_512_mels_to_other_targets_tracks_the_oracle(rate_tree, sr):
    root, wav, info = rate_tree
    outs = []
    for chunk in (1800.0, 0.001):
        out = os.path.join(str(root), f"out_{sr}_{chunk}")
        P.run(wav, info, out, sample_rate=sr, chunk_seconds=chunk, log=lambda *a: None, **E2E_OPTS)
        outs.append(out)
    names = sorted(os.listdir(outs[0]))
    assert names == sorted(os.listdir(outs[1])) and "attr.pkl" in names
    for f in names:
        assert open(os.path.join(outs[0], f), "rb").read() == open(os.path.join(outs[1], f), "rb").read(), (sr, f)
    with open(os.path.join(outs[0], "attr.pkl"), "rb") as f:
        attr = pickle.load(f)
    mean, std = attr["mean"].astype(np.float64), attr["std"].astype(np.float64)
    paths = {os.path.basename(p): p for lst in P.read_filenames(wav).values() for p in lst}
    worst, worst_ratio, seen = 0.0, 0.0, set()
    for name in P.SETS:
        with open(os.path.join(outs[0], f"{name}.pkl"), "rb") as f:
            data = pickle.load(f)
        for key, v in data.items():
            rate, pcm = wavfile.read(paths[key])
            seen.add(rate)
            x = pcm / 32768.0
            if rate != sr:
                x = resample_poly(x, *P.rate_pair(rate, sr))
            ref, _ = ao.get_spectrograms(x, n_mels=512, sr=sr)
            raw = v.astype(np.float64) * std + mean
            assert raw.shape == ref.shape, (sr, key, raw.shape, ref.shape)
            below = ref.max(axis=1, keepdims=True) - ref          # 1 = 100 dB below the frame's peak
            loud = below <= 0.6
            # 1e-5 within 40 dB of the peak; further down, a fixed float32 amplitude error of the resampled signal and
            # the STFT moves the dB value by 0.087 of its ratio to the entry, so the bound grows as the peak over it
            bound = 1e-5 * np.maximum(1.0, 10.0 ** (5.0 * below - 2.0))
            err = np.abs(raw - ref)
            worst = max(worst, float(err[loud].max()))
            ratio = float((err / bound)[loud].max())
            worst_ratio = max(worst_ratio, ratio)
            assert ratio <= 1.0, (sr, key, rate, ratio)
    assert seen == set(FILE_RATES), seen
    print(f"preprocess to {sr} Hz at 512 mels: within 60 dB of the frame peak, worst {worst:.2e} and at most "
          f"{worst_ratio:.2f} of the bound (1e-5 within 40 dB)")
