"""Streaming conversion: many live streams converted at once in fixed blocks, with a stated latency.

Three stages run once per update, each batched over every stream with pending input:

* analysis: each stream keeps the tail of its samples that later frames still need; frame f is analysed as soon as
  sample f hop + win/2 - 1 has arrived, by ``avc_stft_window`` (the offline STFT kernel with a frame origin) and the
  offline MAG_TO_MEL projection.  The result is bit for bit the offline analysis of the whole stream, untrimmed
  (``Vocoder.wav_to_mel(..., trim=False)``): a stream cannot know its leading silence in advance.  Reflect padding
  applies at the stream's start, and at its end only after ``close``.
* conversion: block j is output frames [jH, (j+1)H); its window [max(0, e_j - W), e_j), e_j = max((j+1)H + LA, m),
  is converted with the stream's speaker code by ``AE.inference_from_embeddings`` as an utterance of its own, and its
  first X = min(LA, H) frames are blended linearly with the previous window's look-ahead rows.  Windows of one length
  run as one batch (a CUDA graph per batch bucket and length), which gives each its stand-alone bits.
* synthesis: the blocks' magnitudes go through RTISI-LA (``avc_rtisi_la``), one CTA per stream, which releases
  samples on ``mel_to_signal``'s grid as their frames are committed.  With ``StreamParams(gl_init="pghi")`` each frame
  enters from a streamed PGHI phase (``avc_pghi_stream``, then ``avc_rtisi_la_from``), a frame later.
* pitch (``PitchStage``, per stream, optional): a fixed shift passes each block's magnitudes through
  ``avc_pitch_shift`` before RTISI-LA.  A target profile (mode, mu_t, sigma_t) synthesises the unshifted magnitudes in
  a second RTISI-LA pool (the shadow), tracks every shadow frame whose span has been released with
  ``avc_yin_window``, turns the new frames into shifts on the host (``PitchTracker``, causal) and shifts the buffered
  magnitudes of those frames before they enter the output RTISI-LA.

A stream's target voice follows its ``TargetSchedule``: anchor codes and keyframes of weights over them at mel frames.
``StreamingConverter.retarget`` cuts or glides to another code from a frame no converted window has reached.  A window
whose weights are one anchor at weight 1 on every frame converts as above; any other (a morph window) converts through
``AE.inference_morph`` with the schedule's per-frame weights, and the pitch targets follow the same weights.

``block_schedule``, ``blend_weights``, ``latency_samples`` and ``tracked_latency_samples`` state the schedule on the
host.
"""
from __future__ import annotations

import ctypes as C
import math
import time
from dataclasses import dataclass

import numpy as np
import torch

from . import _lib as L
from .f0 import F0Params, _yin_launch
from .mcd import min_frames
from .speaker_bank import interpolate_keyframes
from .utils import _stream
from .vocoder import PITCH_SHIFT_MAX, _mel_project, _ptr, _Ragged, _shift_rows


@dataclass(frozen=True)
class StreamParams:
    """The block schedule (mel frames; window, hop and lookahead multiples of 8, so that every window's latent frames
    fall on the stream's 8-frame grid) and RTISI-LA's look-ahead frames and iterations.  None for window:
    the model's segment_size.  These defaults are choices, not searched values."""
    window: int | None = None
    hop: int = 8
    lookahead: int = 8
    gl_lookahead: int = 3
    gl_iters: int = 8
    gl_init: str = "estimate"  # RTISI-LA's start phase of each entering frame: "estimate" (the current estimate's) or
                               # "pghi" (streamed PGHI, Rtisi; one more frame of latency)
    batch_max: int = 1024     # windows per model batch
    keep_mels: bool = False   # keep each stream's emitted mel frames for take_mels, and its pitch diagnostics for
                              # take_pitch (memory grows with the stream)
    pitch_warmup: int = 50    # voiced frames a tracked stream sees before mv scales its range (0.625 s of voicing at
                              # 80 frames/s); not tuned


def check_params(p: StreamParams, window: int):
    for name, v in (("window", window), ("hop", p.hop), ("lookahead", p.lookahead)):
        if v % 8 != 0 or v < (8 if name != "lookahead" else 0):
            raise ValueError(f"StreamParams.{name} must be a {'non-negative' if name == 'lookahead' else 'positive'} "
                             f"multiple of 8 (got {v})")
    if p.hop + p.lookahead > window:
        raise ValueError(f"StreamParams: hop + lookahead ({p.hop + p.lookahead}) must not exceed the window ({window})")
    if not 0 <= p.gl_lookahead <= L.RTISI_MAX_LOOKAHEAD:
        raise ValueError(f"StreamParams.gl_lookahead must be in [0, {L.RTISI_MAX_LOOKAHEAD}] (got {p.gl_lookahead})")
    if p.gl_iters < 0:
        raise ValueError(f"StreamParams.gl_iters must be >= 0 (got {p.gl_iters})")
    if p.gl_init not in RTISI_INITS:
        raise ValueError(f"StreamParams.gl_init must be one of {RTISI_INITS} (got {p.gl_init!r})")
    if p.batch_max < 1:
        raise ValueError("StreamParams.batch_max must be >= 1")
    if p.pitch_warmup < 1:
        raise ValueError(f"StreamParams.pitch_warmup must be >= 1 (got {p.pitch_warmup})")


def min_window(config) -> int:
    """m: the model's minimum source length rounded up to a multiple of 8."""
    return -(-min_frames(config)[0] // 8) * 8


def block_end(j: int, hop: int, lookahead: int, m: int) -> int:
    """e_j: the end (exclusive) of block j's window, in frames."""
    return max((j + 1) * hop + lookahead, m)


def block_schedule(j: int, window: int, hop: int, lookahead: int, m: int):
    """(block start, block end, window start, window end) of block j."""
    e = block_end(j, hop, lookahead, m)
    return j * hop, (j + 1) * hop, max(0, e - window), e


def close_window(T: int, window: int):
    """[start, end) of the last window of a stream of T frames."""
    return max(0, T - window), T


def blend_weights(hop: int, lookahead: int) -> np.ndarray:
    """Weights on the new window of a block's first X = min(lookahead, hop) frames: (i+1)/(X+1) in float32."""
    X = min(lookahead, hop)
    return (np.arange(1, X + 1, dtype=np.float32) / np.float32(X + 1)).astype(np.float32)


def init_delay(p: StreamParams) -> int:
    """Frames a frame waits before it enters RTISI-LA: 1 with the PGHI start (frame f's phase needs frame f+1), else 0."""
    return 1 if p.gl_init == "pghi" else 0


def release_sample(n: int, p: StreamParams, win: int, hop_s: int, m: int) -> int:
    """Index of the input sample whose arrival releases output sample n (before close): n's last covering frame c is
    committed when frame c + gl_lookahead enters RTISI-LA, i.e. (with init_delay) when frame c + gl_lookahead +
    init_delay is emitted in its block j, at the arrival of the sample that completes frame e_j - 1."""
    c = (n + win // 2) // hop_s
    j = (c + p.gl_lookahead + init_delay(p)) // p.hop
    return (block_end(j, p.hop, p.lookahead, m) - 1) * hop_s + win // 2 - 1


def _worst_latency(release, frames: int, win: int, hop_s: int) -> int:
    """max of release(n) - n over the smallest output sample n each frame c < frames is the last covering frame of."""
    worst = 0
    for c in range(frames):
        n = max(0, c * hop_s - win // 2)
        if (n + win // 2) // hop_s == c:
            worst = max(worst, release(n) - n)
    return worst


def latency_samples(p: StreamParams, win: int, hop_s: int, m: int) -> int:
    """max over output samples n >= 0 of release_sample(n) - n.  For a frame c the smallest n it is the last
    frame of is the worst; past the start-up windows the schedule repeats every block, so a few blocks beyond m
    cover every case.  Without start-up effects this is (H + LA + LA_v - 1) hop + win - 1."""
    return _worst_latency(lambda n: release_sample(n, p, win, hop_s, m),
                          m + 4 * p.hop + p.gl_lookahead + init_delay(p) + 2 * (win // hop_s) + 8, win, hop_s)


def yin_last_sample(t: int, hop_s: int, span: int) -> int:
    """The last sample of a signal that YIN frame t (centred at t hop_s, span = W + tau_max samples from
    t hop_s - floor(span / 2)) reads, with the reflection at sample 0."""
    half = span // 2
    return max(t * hop_s + span - half - 1, half - t * hop_s)


def yin_ready(n: int, hop_s: int, span: int) -> int:
    """Frames of a signal still arriving, of which samples 0 .. n - 1 are in, that can be tracked: the t with
    yin_last_sample(t) < n (for t >= 1 that is t hop_s + span - floor(span / 2) - 1)."""
    if n <= yin_last_sample(0, hop_s, span):
        return 0
    return (n - (span - span // 2)) // hop_s + 1


def tracked_release_sample(n: int, p: StreamParams, win: int, hop_s: int, m: int, span: int) -> int:
    """release_sample for a stream with a target profile: n's last covering frame c is committed by the output RTISI-LA
    when frame c + gl_lookahead enters it, which needs frame t = c + gl_lookahead + init_delay shifted, i.e. YIN frame t
    tracked, i.e. the shadow's release of sample yin_last_sample(t); the shadow is synthesised on the output's schedule
    and start, so that is its release_sample."""
    t = (n + win // 2) // hop_s + p.gl_lookahead + init_delay(p)
    return release_sample(yin_last_sample(t, hop_s, span), p, win, hop_s, m)


def tracked_latency_samples(p: StreamParams, win: int, hop_s: int, m: int, span: int) -> int:
    """max over output samples n >= 0 of tracked_release_sample(n) - n, found as latency_samples finds its own.  With
    the defaults the tracking delays each frame by D = gl_lookahead + ceil((span - floor(span / 2) + win / 2) / hop) - 1
    frames (7 at 24 kHz: 3 + 5 - 1)."""
    return _worst_latency(lambda n: tracked_release_sample(n, p, win, hop_s, m, span),
                          m + 4 * p.hop + 2 * (p.gl_lookahead + init_delay(p)) + 2 * (win // hop_s) + span // hop_s + 8,
                          win, hop_s)


class _Tail:
    """The rows of a growing sequence from absolute index ``first`` on: what later work still reads of it."""
    __slots__ = ("x", "first")

    def __init__(self, x):
        self.x, self.first = x, 0

    def append(self, y):
        self.x = torch.cat([self.x, y])

    def view(self, a: int, b: int | None = None):
        """Rows a .. b - 1 (to the end without b), by absolute index."""
        return self.x[a - self.first:None if b is None else b - self.first]

    def trim(self, a: int):
        """Drops the rows before absolute index a."""
        if a > self.first:
            self.x, self.first = self.x[a - self.first:], a


# ------------------------------------------------------------------ analysis
class _AStream:
    __slots__ = ("n_in", "frames", "tail", "closed")

    def __init__(self, dev):
        self.n_in, self.frames, self.closed = 0, 0, False
        self.tail = _Tail(torch.empty(0, device=dev))


class StreamAnalyzer:
    """Streaming mel analysis of many streams: ``push({id: pcm}, close=())`` returns {id: new mel frames
    [n, n_mels]} (normalised dB, as ``Vocoder.wav_to_mel``) for the streams that gained frames, in one avc_stft_window
    launch and one mel projection."""

    def __init__(self, vocoder):
        self.voc = vocoder
        self.hp = vocoder.hp
        self.dev = vocoder.device
        self.streams = {}

    def open(self, sid):
        self.streams[sid] = _AStream(self.dev)

    def drop(self, sid):
        self.streams.pop(sid, None)

    def ready(self, s: _AStream) -> int:
        hp = self.hp
        if s.closed:
            return 1 + s.n_in // hp.hop_length
        return 0 if s.n_in < hp.win_length // 2 else (s.n_in - hp.win_length // 2) // hp.hop_length + 1

    def first_sample(self, f: int) -> int:
        """avc_stft_window's first sample of an entry with frame origin f."""
        return max(0, f * self.hp.hop_length - self.hp.win_length // 2 - 2)

    def push(self, chunks, close=()):
        hp = self.hp
        for sid, x in chunks.items():
            s = self.streams[sid]
            if s.closed:
                raise ValueError(f"stream {sid!r} is closed")
            x = torch.as_tensor(x).to(device=self.dev, dtype=torch.float32).reshape(-1)
            if x.numel():
                s.tail.append(x)
                s.n_in += x.numel()
        for sid in close:
            s = self.streams[sid]
            if s.n_in < hp.min_samples:
                raise ValueError(f"stream {sid!r} has {s.n_in} samples; an STFT with n_fft={hp.n_fft} needs at least "
                                 f"{hp.min_samples}")
            s.closed = True
        ys, ids, counts, origins = [], [], [], []
        for sid in dict.fromkeys(list(chunks) + list(close)):
            s = self.streams[sid]
            n = self.ready(s) - s.frames
            if n <= 0:
                continue
            ys.append(s.tail.view(self.first_sample(s.frames)))
            ids.append(sid)
            counts.append(n)
            origins.append(s.frames)
            s.frames += n
            s.tail.trim(self.first_sample(s.frames))
        if not ids:
            return {}
        r = _Ragged([y.numel() for y in ys], counts, self.dev, origins)
        mag = torch.empty(sum(counts), hp.n_bins, device=self.dev)
        y = torch.cat(ys)
        d = r.desc(hp, mode=L.STFT_MAG, preemph=hp.preemphasis, y=y, mag_out=mag)
        L.check(L.load().avc_stft_window(C.byref(d), _stream(self.dev)), "avc_stft_window")
        mel = _mel_project(mag, self.voc.fb_t, L.MAG_TO_MEL, hp)
        return dict(zip(ids, r.split_frames(mel)))


# ------------------------------------------------------------------ RTISI-LA
RTISI_MAX_FRAMES = 2 ** 31 - 1   # frames of one stream (int32 counts): about 310 days at hop 300 and 24 kHz


RTISI_INITS = ("estimate", "pghi")


class Rtisi:
    """RTISI-LA state of many streams in a pool of slots, and one avc_rtisi_la launch per update.
    ``run({id: mags [n, n_bins]}, close=())`` returns {id: released samples}.

    ``init`` is the start phase of each entering frame: "estimate" (the phase of the current estimate's STFT) or
    "pghi", the stream's own streamed PGHI phase (``avc_pghi_stream``, tolerance ``hp.pghi_tol``), which holds each
    frame until the next one has arrived (or the stream closes): an update is then one avc_pghi_stream launch and one
    avc_rtisi_la_from launch on the same tables, and the PGHI state pool sits beside the slot pool."""
    init = "estimate"

    def __init__(self, hp, lookahead: int = 3, n_iter: int = 8, device=None, init: str = "estimate"):
        if init not in RTISI_INITS:
            raise ValueError(f"Rtisi: init must be one of {RTISI_INITS} (got {init!r})")
        self.hp, self.la, self.n_iter, self.init = hp, int(lookahead), int(n_iter), init
        self.dev = torch.device(device) if device is not None else torch.device("cuda")
        self.stride = int(L.load().avc_rtisi_state_floats(hp.win_length, self.la))
        self.state = torch.zeros(0, self.stride, device=self.dev)
        self.count = torch.zeros(0, 2, dtype=torch.int32, device=self.dev)
        self.pstate = None
        if init == "pghi":
            self.pstride = int(L.load().avc_pghi_stream_state_floats(hp.n_fft))
            self.pstate = torch.zeros(0, self.pstride, device=self.dev)
        self.free, self.slot, self.host, self.held = [], {}, {}, {}

    def open(self, sid):
        if not self.free:
            n = max(16, 2 * self.state.shape[0])
            old = self.state.shape[0]
            state = torch.zeros(n, self.stride, device=self.dev)
            count = torch.zeros(n, 2, dtype=torch.int32, device=self.dev)
            state[:old].copy_(self.state)
            count[:old].copy_(self.count)
            self.state, self.count = state, count
            if self.pstate is not None:
                pstate = torch.zeros(n, self.pstride, device=self.dev)
                pstate[:old].copy_(self.pstate)
                self.pstate = pstate
            self.free = list(range(n - 1, old - 1, -1))
        k = self.free.pop()
        self.state[k].zero_()
        self.count[k].zero_()
        if self.pstate is not None:
            self.pstate[k].zero_()
            self.held[sid] = 0
        self.slot[sid], self.host[sid] = k, [0, 0]

    def drop(self, sid):
        if sid in self.slot:
            self.free.append(self.slot.pop(sid))
            self.host.pop(sid)
            self.held.pop(sid, None)

    def released(self, c: int) -> int:
        return max(0, c * self.hp.hop_length - self.hp.win_length // 2)

    def run(self, mags, close=()):
        launch = self.prepare(mags, close)
        if launch is None:
            return {}
        desc, res = launch[0], launch[1]
        self.launch(desc)
        for sid in close:
            self.drop(sid)
        return res

    def launch(self, desc):
        """The launches of a prepared update (its tables and buffers are kept alive by prepare's result): avc_rtisi_la,
        or with init "pghi" avc_pghi_stream then avc_rtisi_la_from."""
        lib, st = L.load(), _stream(self.dev)
        if self.init == "pghi":
            pd, rd = desc
            L.check(lib.avc_pghi_stream(C.byref(pd), C.c_float(self.hp.pghi_tol), None, st), "avc_pghi_stream")
            L.check(lib.avc_rtisi_la_from(C.byref(rd), pd.X, st), "avc_rtisi_la_from")
        else:
            L.check(lib.avc_rtisi_la(C.byref(desc), st), "avc_rtisi_la")

    def prepare(self, mags, close=()):
        """(descriptor, {id: output view}, buffers) of one update, the host's counts advanced; None when empty.  With
        init "pghi" the descriptor is the pair (avc_pghi_stream's, avc_rtisi_la_from's), and the frames entering
        RTISI-LA are the ones PGHI completes: each but the newest, all of them at close."""
        hp, pghi = self.hp, self.init == "pghi"
        ids = list(dict.fromkeys(list(mags) + list(close)))
        if not ids:
            return None
        for sid in ids:   # avc_rtisi_la's frame counts are int32: refuse before any state changes
            c, nb = self.host[sid]
            m = mags.get(sid)
            # (avc_pghi_stream forms frame f + 2 for its last frame f: one frame fewer)
            if c + nb + (self.held[sid] if pghi else 0) + (0 if m is None else int(m.shape[0])) > RTISI_MAX_FRAMES - pghi:
                raise ValueError(f"stream {sid!r} would pass {RTISI_MAX_FRAMES} frames, the RTISI-LA limit")
        rows, offs, slots, closes, outs, counts, ents = [], [0], [], [], [0], [], [0]
        for sid in ids:
            c, nb = self.host[sid]
            m = mags.get(sid)
            p = 0 if m is None else int(m.shape[0])
            if m is not None and p:
                rows.append(m)
            offs.append(offs[-1] + p)
            if pghi:   # the newest frame waits for the next one, or for close
                h = self.held[sid] + p
                self.held[sid] = 0 if sid in close else min(h, 1)
                p = h - self.held[sid]
                ents.append(ents[-1] + p)
            if sid in close:
                T = c + nb + p
                n_out = max(0, (T - 1) * hp.hop_length) - self.released(c)
                self.host[sid] = [T, 0]
            else:
                nb2 = min(nb + p, self.la)
                c2 = c + nb + p - nb2
                n_out = self.released(c2) - self.released(c)
                self.host[sid] = [c2, nb2]
            slots.append(self.slot[sid])
            closes.append(1 if sid in close else 0)
            counts.append(n_out)
            outs.append(outs[-1] + n_out)
        mag = torch.cat(rows).float().contiguous() if rows else torch.zeros(1, hp.n_bins, device=self.dev)
        n = len(ids)
        i32 = torch.tensor(offs + slots + closes + (ents if pghi else []), dtype=torch.int32).to(self.dev)
        out_off = torch.tensor(outs[:-1], dtype=torch.int64).to(self.dev)
        y = torch.empty(max(1, outs[-1]), device=self.dev)
        keep = (mag, i32, out_off, y)
        rmag, roff = mag, i32[:n + 1]
        if pghi:
            rmag = torch.empty(max(1, ents[-1]), hp.n_bins, device=self.dev)
            X = torch.empty(max(1, ents[-1]), hp.n_bins, 2, device=self.dev)
            roff = i32[3 * n + 1:]
            pd = L.PghiStreamDesc(n_fft=hp.n_fft, hop=hp.hop_length, win=hp.win_length, n_streams=n, mag=_ptr(mag),
                                  mag_off=_ptr(i32[:n + 1]), slot=_ptr(i32[n + 1:2 * n + 1]),
                                  close=_ptr(i32[2 * n + 1:3 * n + 1]), out_off=_ptr(roff), mag_out=_ptr(rmag),
                                  X=_ptr(X), state=_ptr(self.pstate))
            keep += (rmag, X)
        d = L.RtisiDesc(n_fft=hp.n_fft, hop=hp.hop_length, win=hp.win_length, lookahead=self.la, n_iter=self.n_iter,
                        n_streams=n, deemph=hp.preemphasis, mag=_ptr(rmag), mag_off=_ptr(roff),
                        slot=_ptr(i32[n + 1:2 * n + 1]), close=_ptr(i32[2 * n + 1:3 * n + 1]), out_off=_ptr(out_off),
                        y=_ptr(y), state=_ptr(self.state), count=_ptr(self.count))
        return (pd, d) if pghi else d, dict(zip(ids, torch.split(y[:outs[-1]], counts))), keep


# ------------------------------------------------------------------ pitch
PITCH_MODES = ("match", "mv")


def parse_pitch(pitch):
    """None, a fixed shift (float semitones in [-24, 24]; 0 becomes None: nothing to launch) or a target profile
    (mode, mu_t, sigma_t) with mode "match" or "mv" and finite float64 log2 F0 statistics, sigma_t >= 0.
    ValueError otherwise."""
    if pitch is None:
        return None
    if isinstance(pitch, (int, float, np.floating, np.integer)) and not isinstance(pitch, bool):
        v = float(pitch)
        if not np.isfinite(v) or abs(v) > PITCH_SHIFT_MAX:
            raise ValueError(f"pitch: a fixed shift must be finite and in [-{PITCH_SHIFT_MAX:g}, {PITCH_SHIFT_MAX:g}] "
                             f"semitones (got {pitch})")
        return None if v == 0.0 else v
    if isinstance(pitch, (tuple, list)) and len(pitch) == 3 and pitch[0] in PITCH_MODES:
        try:
            mu, sd = float(pitch[1]), float(pitch[2])
        except (TypeError, ValueError):
            mu = sd = float("nan")
        if np.isfinite(mu) and np.isfinite(sd) and sd >= 0.0:
            return (pitch[0], mu, sd)
    raise ValueError(f"pitch: expected None, semitones or (mode in {PITCH_MODES}, log2 mean, log2 std >= 0), "
                     f"got {pitch!r}")


class PitchTracker:
    """The causal shift rule of one tracked stream, in float64, fed its YIN frames in order.

    Frame t is voiced when aperiodicity < theta, energy > 0 and 10 log10(energy / e_max(t)) >= -silence_db, e_max(t) the
    largest energy of frames 0..t (``f0.voicing`` with a running floor); its l = log2(sr / tau).  (mu_c, sigma_c) are
    Welford's running mean and (ddof 0) std of l over the voiced frames 0..t, in frame order.  On a voiced frame the
    shift is 12 (mu_t - mu_c) for "match" and, for "mv", while fewer than `warmup` voiced frames have been seen or while
    sigma_c = 0; after that "mv" gives 12 (mu_t + sigma_t / sigma_c (l - mu_c) - l).  Every shift is clamped to +-24.
    An unvoiced frame holds the last voiced frame's shift, 0 before the first."""

    def __init__(self, mode: str, mu_t: float, sd_t: float, warmup: int, sr: int, params: F0Params = F0Params()):
        self.mode, self.mu_t, self.sd_t, self.warmup, self.sr = mode, float(mu_t), float(sd_t), int(warmup), sr
        self.theta, self.floor = params.theta(), -float(params.silence_db)
        self.emax, self.n, self.mean, self.m2, self.last = 0.0, 0, 0.0, 0.0, 0.0

    def update(self, tau, ap, en, mu_t=None, sd_t=None):
        """(log2 F0 (NaN where unvoiced), voiced, shift) float64 / bool / float64 arrays of the next frames.  mu_t and
        sd_t, when given, are float64 per-frame targets of these frames (TargetSchedule.profile) in place of the
        constant ones; equal targets on every frame give the constant targets' bits."""
        tau, ap, en = (np.asarray(v, np.float64) for v in (tau, ap, en))
        emax = np.maximum.accumulate(np.concatenate([[self.emax], en]))[1:]
        self.emax = float(emax[-1]) if len(emax) else self.emax
        with np.errstate(divide="ignore", invalid="ignore"):
            rel = np.where(emax > 0, 10.0 * np.log10(en / np.where(emax > 0, emax, 1.0)), -np.inf)
            logf = np.where(ap < self.theta, np.log2(self.sr / tau), np.nan)
        voiced = (ap < self.theta) & (en > 0) & (rel >= self.floor)
        logf = np.where(voiced, logf, np.nan)
        shift = np.empty(len(tau))
        for i in range(len(tau)):
            if voiced[i]:
                l = float(logf[i])
                self.n += 1
                d = l - self.mean
                self.mean += d / self.n
                self.m2 += d * (l - self.mean)
                sd = math.sqrt(self.m2 / self.n)
                mu = self.mu_t if mu_t is None else float(mu_t[i])
                sdt = self.sd_t if sd_t is None else float(sd_t[i])
                if self.mode == "mv" and self.n >= self.warmup and sd != 0.0:
                    v = 12.0 * (mu + sdt / sd * (l - self.mean) - l)
                else:
                    v = 12.0 * (mu - self.mean)
                self.last = min(PITCH_SHIFT_MAX, max(-PITCH_SHIFT_MAX, v))
            shift[i] = self.last
        return logf, voiced, shift


# ------------------------------------------------------------------ target schedule
class _Keep:
    def __repr__(self):
        return "KEEP"


KEEP = _Keep()    # retarget's pitch: the new anchor takes the pitch target the schedule has at `at`


def pitch_kind(pitch):
    """The kind of a parsed pitch setting: None, "shift" or the profile's mode."""
    return None if pitch is None else "shift" if isinstance(pitch, float) else pitch[0]


class TargetSchedule:
    """The target voice of one stream over its mel frames: anchor codes in order of first use, each with a pitch
    target of the stream's kind (None; semitones for a fixed shift; (mu, sigma) of log2 F0 for a profile), and
    keyframes (frame, float64 weights over the anchors) at non-decreasing frames.

    The weights of frame t follow speaker_bank.morph_weights' rule (interpolate_keyframes) with times in frames: the
    first keyframe held before it and the last after it, linear in between, the later of two keyframes on one frame
    winning (a hard cut); float64, rounded once to float32 (``weights``).  Pitch targets are the weighted sums of the
    anchors' in float64 with the float32 weights: a shift sum_k w_k s_k, a profile's mu and sigma as
    SpeakerBank.morph_pitch_profile gives them.  Anchors are de-duplicated by bitwise equality of their codes (and
    of the pitch target, when one is given).  ``prune`` drops what no frame from a given one on can read."""

    def __init__(self, code, pitch=None):
        self.kind = pitch_kind(pitch)
        self.codes = [code]
        self.pitch = [None if pitch is None else pitch if isinstance(pitch, float) else (float(pitch[1]),
                                                                                         float(pitch[2]))]
        self.frames = [0]
        self.V = np.ones((1, 1))       # float64 [keyframes, anchors]

    def mix(self, f0: int, f1: int) -> np.ndarray:
        """float64 [f1 - f0, K]: the weights of frames f0 .. f1 - 1 before rounding."""
        return interpolate_keyframes(self.frames, self.V, np.arange(f0, f1))

    def weights(self, f0: int, f1: int) -> np.ndarray:
        """float32 [K, f1 - f0]: the weights of frames f0 .. f1 - 1."""
        if self.V.shape == (1, 1):
            return np.ones((1, f1 - f0), np.float32)
        return self.mix(f0, f1).T.astype(np.float32)

    def window(self, f0: int, f1: int):
        """(k, None) when frames f0 .. f1 - 1 all have anchor k alone at weight 1 (a plain window), otherwise
        (anchors of non-zero weight in schedule order, their float32 weights [K, f1 - f0])."""
        if self.V.shape == (1, 1):
            return 0, None
        w = self.weights(f0, f1)
        nz = np.flatnonzero(w.any(1))
        if len(nz) == 1 and (w[nz[0]] == 1).all():
            return int(nz[0]), None
        return nz.tolist(), w[nz]

    def shift(self, f0: int, n: int) -> np.ndarray:
        """float64 [n]: the fixed-shift target (semitones) of frames f0 .. f0 + n - 1."""
        if len(self.codes) == 1:
            return np.full(n, self.pitch[0])
        w = self.weights(f0, f0 + n).astype(np.float64)
        s = np.zeros(n)
        for wk, sk in zip(w, self.pitch):
            s = s + wk * sk
        return s

    def profile(self, f0: int, n: int):
        """(mu, sigma) float64 [n]: the profile target of frames f0 .. f0 + n - 1."""
        if len(self.codes) == 1:
            return np.full(n, self.pitch[0][0]), np.full(n, self.pitch[0][1])
        w = self.weights(f0, f0 + n).astype(np.float64)
        mu, sd, wsum = np.zeros(n), np.zeros(n), np.zeros(n)
        for wk, (m, s) in zip(w, self.pitch):
            if not wk.any():
                continue
            mu, sd, wsum = mu + wk * m, sd + wk * s, wsum + wk
        return mu / wsum, sd / wsum

    def pitch_value(self, pitch, at: int):
        """retarget's pitch as an anchor's pitch target: KEEP gives the schedule's at frame `at`; otherwise it must be
        of the stream's kind (None; a number of semitones, 0 included; a profile of the stream's mode).  ValueError
        otherwise."""
        if pitch is KEEP:
            if self.kind is None:
                return None
            if self.kind == "shift":
                return float(self.shift(at, 1)[0])
            mu, sd = self.profile(at, 1)
            return float(mu[0]), float(sd[0])
        if self.kind == "shift":
            ok = isinstance(pitch, (int, float, np.floating, np.integer)) and not isinstance(pitch, bool)
            v = parse_pitch(pitch) if ok else "bad"
            if ok and v is None:
                return 0.0
            if isinstance(v, float):
                return v
        else:
            try:
                v = parse_pitch(pitch)
            except ValueError:
                v = "bad"
            if v != "bad" and pitch_kind(v) == self.kind:
                return None if v is None else (v[1], v[2])
        want = {None: "None", "shift": "a number of semitones"}.get(self.kind, f"a ({self.kind!r}, mu, sigma) profile")
        raise ValueError(f"retarget: the stream's pitch setting takes {want} or KEEP (its kind cannot change), got "
                         f"{pitch!r}")

    def retarget(self, code, at: int, ramp: int, pitch=KEEP, first: int = 0, lo: int = 0, window: int = 0,
                 max_k: int = L.MORPH_MAX_K):
        """Moves the schedule from its mix at frame `at` to code (one-hot) over `ramp` frames: drops the keyframes
        after `at`, then adds (at, mix at `at`) and (at + ramp, one-hot).  pitch: the anchor's pitch target
        (pitch_value).  ValueError, the schedule unchanged, for at < first (a frame already converted), a negative
        ramp, or when a window of `window` frames starting at or after frame lo would need more than max_k anchors of
        non-zero weight."""
        if at < first:
            raise ValueError(f"retarget: frame {at} is before the end of the stream's last converted window ({first})")
        if ramp < 0:
            raise ValueError(f"retarget: ramp must be >= 0 frames (got {ramp})")
        v = self.mix(at, at + 1)[0]
        k = next((i for i, c in enumerate(self.codes) if (c is code or torch.equal(c, code))
                  and (pitch is KEEP or self.pitch[i] == pitch)), None)
        if k is None and pitch is KEEP:
            pitch = self.pitch_value(KEEP, at)
        codes, pitches, V = list(self.codes), list(self.pitch), self.V
        if k is None:
            codes.append(code)
            pitches.append(pitch)
            V = np.concatenate([V, np.zeros((V.shape[0], 1))], 1)
            v = np.concatenate([v, [0.0]])
            k = len(codes) - 1
        keep = sum(1 for f in self.frames if f <= at)
        onehot = np.zeros(len(codes))
        onehot[k] = 1.0
        frames = self.frames[:keep] + [at, at + ramp]
        V = np.concatenate([V[:keep], v[None], onehot[None]])
        need = live_anchors(frames, V, lo, window)
        if need > max_k:
            raise ValueError(f"retarget: a window would need {need} anchors of non-zero weight; at most {max_k} are "
                             f"supported")
        self.codes, self.pitch, self.frames, self.V = codes, pitches, frames, V

    def prune(self, lo: int):
        """Drops the keyframes and anchors no frame from lo on reads: every keyframe before the last one at or before
        lo, then every anchor of zero weight in all the keyframes left (the others keep their order)."""
        i = max(0, sum(1 for f in self.frames if f <= lo) - 1)
        if i:
            self.frames, self.V = self.frames[i:], self.V[i:]
        live = np.flatnonzero(self.V.any(0))
        if len(live) < len(self.codes):
            self.codes = [self.codes[k] for k in live]
            self.pitch = [self.pitch[k] for k in live]
            self.V = self.V[:, live]


def live_anchors(frames, V, lo: int, window: int) -> int:
    """The most anchors of non-zero weight any window of `window` frames from frame lo on can need (counting, on each
    span between consecutive keyframes, the anchors of either end)."""
    segs = []   # (first frame, end frame, anchors)
    nz = [set(np.flatnonzero(r).tolist()) for r in V]
    for i in range(len(frames)):
        end = frames[i + 1] if i + 1 < len(frames) else math.inf
        if end > frames[i] or i + 1 == len(frames):
            segs.append((frames[i], end, nz[i] | (nz[i + 1] if i + 1 < len(frames) else set())))
    segs.insert(0, (-math.inf, frames[0], nz[0]))
    worst = 0
    for a in {lo} | {max(lo, s[1] - 1) for s in segs if s[1] != math.inf}:
        used = set()
        for s0, s1, ks in segs:
            if s0 < a + max(1, window) and s1 > a:
                used |= ks
        worst = max(worst, len(used))
    return worst


class _Clock:
    """Wall time per stage, each stage ended by a device synchronise: ``ms`` None is off, a dict accumulates
    milliseconds per stage."""

    def __init__(self, dev):
        self.dev, self.ms, self.t = dev, None, 0.0

    def lap(self, key=None):
        """Ends stage `key` (None: the time since the last lap belongs to no stage) and starts the next."""
        if self.ms is not None:
            torch.cuda.synchronize(self.dev)
            t, self.t = self.t, time.perf_counter()
            if key is not None:
                self.ms[key] = self.ms.get(key, 0.0) + 1e3 * (self.t - t)


class _PStream:
    __slots__ = ("sched", "track", "pend", "frames", "n_rel", "tail", "tracked", "diag")

    def __init__(self, sched, track=None, dev=None, n_bins=0):
        self.sched, self.track = sched, track
        self.pend = torch.empty(0, n_bins, device=dev)          # unshifted magnitudes of frames not yet tracked
        self.frames = self.n_rel = self.tracked = 0
        self.tail = _Tail(torch.empty(0, device=dev))           # shadow samples
        self.diag = {k: [] for k in ("tau", "aperiodicity", "energy", "log2_f0", "voiced", "shift", "shadow")}


class PitchStage:
    """RTISI-LA synthesis of many streams, each with its own pitch setting (``parse_pitch``): ``open(id, pitch)``, then
    ``run({id: linear magnitudes [n, n_bins]}, close=())`` returns {id: released samples}, one batched update.

    * None: the magnitudes enter the output RTISI-LA (``rt``) as they are; an update of such streams only is one
      avc_rtisi_la launch, as before this stage existed.
    * a fixed shift s: they go through avc_pitch_shift with ratio float32(2^(s/12)) first.
    * a target profile: they enter the shadow pool (``shadow``, the same look-ahead and iterations), whose output is
      the unshifted stream's.  Every shadow frame whose span has been released is tracked by one avc_yin_window launch
      over all streams (F0Params defaults), the YIN outputs come to the host in one copy, ``PitchTracker`` turns them
      into shifts, and the buffered magnitudes of the newly tracked frames are shifted before they enter ``rt``.  A
      stream keeps only the shadow samples later frames read.  At close the shadow is closed, its last frames tracked
      with the end reflection, and the output closed, in the same update.
    All shifted rows of an update go through one avc_pitch_shift launch.  Every step is per stream and row, so a
    stream's bits depend neither on how its frames were split into updates nor on the other streams.
    ``keep`` keeps each tracked stream's per-frame diagnostics and shadow samples for ``take``."""

    def __init__(self, hp, lookahead: int = 3, n_iter: int = 8, device=None, warmup: int = 50, keep: bool = False,
                 params: F0Params = F0Params(), init: str = "estimate"):
        self.hp, self.params, self.warmup, self.keep = hp, params, int(warmup), keep
        # the shadow starts its frames as the output does, so that it is the unshifted stream bit for bit
        self.rt = Rtisi(hp, lookahead, n_iter, device, init)
        self.shadow = Rtisi(hp, lookahead, n_iter, device, init)
        self.dev = self.rt.dev
        self.span = int(params.win) + params.tau_max(hp.sr)
        self.streams, self.closed = {}, {}
        self.clock = _Clock(self.dev)

    def open(self, sid, pitch=None, schedule: TargetSchedule = None):
        """schedule, when given, holds the stream's per-frame pitch targets (TargetSchedule.shift / .profile);
        otherwise they are pitch's constant one.  pitch sets the kind."""
        pitch = parse_pitch(pitch)
        self.rt.open(sid)
        if pitch is None:
            return
        if schedule is None:    # the stage never retargets, so the schedule's code is never read
            schedule = TargetSchedule(None, pitch)
        if isinstance(pitch, float):
            self.streams[sid] = _PStream(schedule)
        else:
            self.shadow.open(sid)
            self.streams[sid] = _PStream(schedule, PitchTracker(*pitch, self.warmup, self.hp.sr, self.params),
                                         self.dev, self.hp.n_bins)

    def next_frame(self, sid):
        """The first frame of stream sid whose pitch target the stage has not read yet; None when it reads none."""
        s = self.streams.get(sid)
        if s is None:
            return None
        return s.frames if s.track is None else s.tracked

    def drop(self, sid):
        self.rt.drop(sid)
        self.shadow.drop(sid)
        self.streams.pop(sid, None)

    def tracked(self, sid) -> bool:
        s = self.streams.get(sid)
        return s is not None and s.track is not None

    def first_sample(self, o: int) -> int:
        """avc_yin_window's first sample of an entry with frame origin o."""
        return max(0, o * self.hp.hop_length - (self.span - self.span // 2) - 1)

    def take(self, sid):
        """The diagnostics of tracked stream sid since the last call (a closed stream's once): float64 arrays tau,
        aperiodicity, energy, log2_f0 (NaN where unvoiced), shift, a bool array voiced, and the shadow samples."""
        if not self.keep:
            raise ValueError("take_pitch: the converter keeps no pitch diagnostics; build it with "
                             "StreamParams(keep_mels=True)")
        if sid in self.closed:
            d = self.closed.pop(sid)
        elif self.tracked(sid):
            d = self.streams[sid].diag
        else:
            raise ValueError(f"take_pitch: stream {sid!r} has no target profile")
        out = {k: (np.concatenate(v) if v else np.zeros(0, bool if k == "voiced" else np.float64)) for k, v in d.items()
               if k != "shadow"}
        out["shadow"] = torch.cat(d["shadow"]) if d["shadow"] else torch.empty(0, device=self.dev)
        for v in d.values():
            v.clear()
        return out

    def run(self, mags, close=()):
        hp = self.hp
        close = list(close)
        ids = list(dict.fromkeys(list(mags) + close))
        tracked = [sid for sid in ids if self.tracked(sid)]
        for sid in tracked:
            s = self.streams[sid]
            T = s.frames + (int(mags[sid].shape[0]) if sid in mags else 0)
            if sid in close and hp.hop_length * (T - 1) < self.params.min_samples(hp.sr):
                raise ValueError(f"stream {sid!r}: {T} frames at close; tracking its pitch needs a signal of at least "
                                 f"{self.params.min_samples(hp.sr)} samples")
        self.clock.lap()
        out = {sid: m for sid, m in mags.items() if sid not in self.streams}
        rows, semis, dest = [], [], []           # the rows of this update's avc_pitch_shift launch
        for sid, m in mags.items():
            s = self.streams.get(sid)
            if s is not None and s.track is None and m.shape[0]:
                n = int(m.shape[0])
                rows.append(m)
                semis.append(s.sched.shift(s.frames, n))
                dest.append(sid)
                s.frames += n
        if tracked:
            self._track(tracked, mags, close, rows, semis, dest)
        if rows:
            out.update(zip(dest, _shift_rows(rows, semis, hp)))
        if tracked or rows:
            self.clock.lap("shift")
        res = self.rt.run(out, close)
        self.clock.lap("rtisi")
        for sid in close:
            s = self.streams.pop(sid, None)
            if s is not None and s.track is not None and self.keep:
                self.closed[sid] = s.diag
        return res

    def _track(self, tracked, mags, close, rows, semis, dest):
        """The shadow synthesis and tracking of an update, and the host shifts; the newly tracked frames' rows are
        appended to rows / semis / dest."""
        hop = self.hp.hop_length
        shadow_in = {}
        for sid in tracked:
            s, m = self.streams[sid], mags.get(sid)
            if m is not None and m.shape[0]:
                shadow_in[sid] = m
                s.pend = torch.cat([s.pend, m.float()])
                s.frames += int(m.shape[0])
        res = self.shadow.run(shadow_in, [sid for sid in tracked if sid in close])
        self.clock.lap("shadow")
        ys, entries = [], []
        for sid in tracked:
            s = self.streams[sid]
            y = res.get(sid)
            if y is not None and y.numel():
                s.tail.append(y)
                s.n_rel += int(y.numel())
                if self.keep:
                    s.diag["shadow"].append(y)
            ready = s.frames if sid in close else min(s.frames, yin_ready(s.n_rel, hop, self.span))
            if ready > s.tracked:
                ys.append(s.tail.view(self.first_sample(s.tracked)))
                entries.append((sid, s, ready - s.tracked))
        if not entries:
            return
        r = _Ragged([y.numel() for y in ys], [n for _, _, n in entries], self.dev, [s.tracked for _, s, _ in entries])
        yin = _yin_launch(r, torch.cat(ys), hop, self.hp.sr, self.params, window=True)
        self.clock.lap("tracking")
        host = yin.cpu().numpy()                 # the update's one device-to-host copy
        self.clock.lap("tracking_copy")
        for (sid, s, n), (tau, ap, en) in zip(entries, np.split(host, r.frame_offs[1:-1], axis=1)):
            logf, voiced, shift = s.track.update(tau, ap, en, *s.sched.profile(s.tracked, n))
            rows.append(s.pend[:n])
            semis.append(shift)
            dest.append(sid)
            s.pend = s.pend[n:]
            s.tracked += n
            s.tail.trim(self.first_sample(s.tracked))
            if self.keep:
                for k, v in (("tau", tau), ("aperiodicity", ap), ("energy", en), ("log2_f0", logf),
                             ("voiced", voiced), ("shift", shift)):
                    s.diag[k].append(np.array(v))


# ------------------------------------------------------------------ the converter
class _CStream:
    __slots__ = ("sched", "hist", "block", "prev", "mels", "e_last")

    def __init__(self, sched, dev, n_mels):
        self.sched = sched
        self.hist = _Tail(torch.empty(0, n_mels, device=dev))
        self.block, self.prev, self.mels, self.e_last = 0, None, [], 0


class StreamingConverter:
    """Converts many live streams at once.  ``open(code, pitch=None)`` starts a stream converted to the speaker code
    ``code`` (float32 [c_out] on the device: a row of ``Inferencer.embed_speakers`` or ``SpeakerBank.code``) with a
    pitch setting (``PitchStage``: None, a fixed shift in semitones, or a target profile ("match" | "mv", mu_t,
    sigma_t) of log2 F0) and returns its id; ``push({id: pcm})`` takes float32 PCM chunks at ``hp.sr`` of any length
    and returns {id: new output samples} (device float32), one batched update; ``close(id)`` returns the stream's last
    samples; ``retarget(id, code, at, ramp, pitch)`` moves a live stream to another code (``TargetSchedule``).
    ``take_mels(id)`` hands over the normalised mel frames the stream emitted so far and ``take_pitch(id)`` a
    tracked stream's per-frame pitch diagnostics, when the converter keeps them (``StreamParams(keep_mels=True)``; off
    by default, since they grow with the stream).  ``latency_samples`` is the worst case, over output samples n, of
    (index of the input sample whose arrival releases n) - n; ``tracked_latency_samples`` the same for streams with a
    target profile."""

    def __init__(self, inferencer, vocoder, params: StreamParams = StreamParams()):
        cfg = inferencer.config
        if int(cfg["data_loader"]["frame_size"]) != 1:
            raise ValueError("StreamingConverter: supports data_loader.frame_size 1 only")
        self.n_mels = int(cfg["SpeakerEncoder"]["c_in"])
        if vocoder.hp.n_mels != self.n_mels:
            raise ValueError(f"StreamingConverter: the vocoder has {vocoder.hp.n_mels} mels, the model {self.n_mels}")
        self.window = int(params.window if params.window is not None else cfg["data_loader"]["segment_size"])
        check_params(params, self.window)
        self.m = min_window(cfg)
        if self.m > self.window:
            raise ValueError(f"StreamingConverter: the window ({self.window}) is shorter than the model's minimum "
                             f"source length ({self.m})")
        self.p, self.inf, self.voc, self.hp = params, inferencer, vocoder, vocoder.hp
        self.dev = vocoder.device
        self.c_out = int(cfg["SpeakerEncoder"]["c_out"])
        self.ana = StreamAnalyzer(vocoder)
        self.stage = PitchStage(self.hp, params.gl_lookahead, params.gl_iters, self.dev, params.pitch_warmup,
                                params.keep_mels, init=params.gl_init)
        self.rt = self.stage.rt
        w = blend_weights(params.hop, params.lookahead)
        self.w_new = torch.from_numpy(w).to(self.dev)[:, None]
        self.w_old = torch.from_numpy(np.float32(1) - w).to(self.dev)[:, None]
        self.norm = None
        if inferencer.attr is not None:
            self.norm = tuple(torch.as_tensor(np.asarray(inferencer.attr[k], np.float32)).to(self.dev)
                              for k in ("mean", "std"))
        self.streams, self.closed = {}, {}
        self._next = 0
        self.clock = self.stage.clock
        self.latency_samples = latency_samples(params, self.hp.win_length, self.hp.hop_length, self.m)
        self.tracked_latency_samples = tracked_latency_samples(params, self.hp.win_length, self.hp.hop_length, self.m,
                                                               self.stage.span)

    @property
    def stage_ms(self):
        """None (off, the default) or a dict: each update adds the wall time (synchronised) of analysis, conversion
        and rtisi, and with pitch streams of shadow, tracking, tracking_copy (the YIN outputs' copy to the host) and
        shift."""
        return self.clock.ms

    @stage_ms.setter
    def stage_ms(self, ms):
        self.clock.ms = ms

    def _check_code(self, code, what):
        if (not isinstance(code, torch.Tensor) or code.dtype != torch.float32 or tuple(code.shape) != (self.c_out,)
                or code.device != self.dev):
            raise ValueError(f"StreamingConverter.{what}: code must be float32 [{self.c_out}] on {self.dev}")

    def open(self, code, pitch=None) -> int:
        self._check_code(code, "open")
        pitch = parse_pitch(pitch)
        sid = self._next
        self._next += 1
        sched = TargetSchedule(code.contiguous(), pitch)
        self.streams[sid] = _CStream(sched, self.dev, self.n_mels)
        self.ana.open(sid)
        self.stage.open(sid, pitch, sched)
        return sid

    def retarget(self, sid, code, at=None, ramp: int = 0, pitch=KEEP) -> int:
        """Moves stream sid from its current mix to `code` (float32 [c_out] on the device, one-hot) over `ramp` mel
        frames from frame `at` (TargetSchedule.retarget), and returns the `at` used.  `at` must not precede the end of
        the stream's last converted window, so that no converted frame changes; None: ceil(n_in / hop_length), the
        first frame centred at or after the next input sample.  pitch: the new anchor's pitch target, of the kind the
        stream was opened with (None; semitones; (mode, mu, sigma) of its mode), or KEEP: the target the schedule has
        at `at`.  Retargets issued ahead of time, in order, compose; one issued during a ramp starts from the mix that
        ramp has reached, so its anchors keep a non-zero weight (decaying along a chain of interrupted ramps) and
        count toward MORPH_MAX_K until that weight underflows.  The decoder's windows reach up to H + LA frames past
        the block they emit, so a block's voice starts to move that much before `at`.  KeyError for an unknown or closed stream; ValueError, the
        schedule unchanged, for an earlier `at`, a pitch of another kind, or a window that would need more than
        MORPH_MAX_K anchors."""
        if sid not in self.streams:
            raise KeyError(f"unknown stream {sid!r}")
        self._check_code(code, "retarget")
        s = self.streams[sid]
        nxt = -(-self.ana.streams[sid].n_in // self.hp.hop_length)
        if at is None:
            # a window is converted only once all its frames are analysed, which needs input past its last centre
            assert nxt >= s.e_last, (nxt, s.e_last)
            at = nxt
        at, ramp = int(at), int(ramp)
        value = pitch if pitch is KEEP else s.sched.pitch_value(pitch, at)
        lo = max(0, self.ana.streams[sid].frames - self.window)
        s.sched.retarget(code.contiguous(), at, ramp, value, first=s.e_last, lo=lo, window=self.window)
        s.sched.prune(self._read_from(sid))
        return at

    def _read_from(self, sid) -> int:
        """The first frame of stream sid whose weights a later window or the pitch stage can still read."""
        lo = max(0, self.ana.streams[sid].frames - self.window)
        f = self.stage.next_frame(sid)
        return lo if f is None else min(lo, f)

    def push(self, chunks):
        return self.update(chunks)

    def close(self, sid):
        return self.update({}, close=(sid,))[sid]

    def take_mels(self, sid):
        """The normalised mel frames [n, n_mels] stream sid emitted since the last call (a closed stream's once, then
        they are dropped).  Needs StreamParams(keep_mels=True): otherwise no frame is kept."""
        if not self.p.keep_mels:
            raise ValueError("take_mels: the converter keeps no mels; build it with StreamParams(keep_mels=True)")
        mels = self.streams[sid].mels if sid in self.streams else self.closed.pop(sid)
        out = torch.cat(mels) if mels else torch.empty(0, self.n_mels, device=self.dev)
        mels.clear()
        return out

    def take_pitch(self, sid):
        """A stream with a target profile: its per-frame diagnostics since the last call (a closed stream's once), a
        dict of float64 arrays tau, aperiodicity, energy (the tracker's outputs), log2_f0 (NaN where unvoiced) and
        shift (semitones), a bool array voiced, and "shadow": the unshifted synthesis released since the last call.
        Needs StreamParams(keep_mels=True)."""
        return self.stage.take(sid)

    @torch.no_grad()
    def update(self, chunks, close=()):
        """One batched update: analysis, conversion and synthesis of every stream in chunks or close."""
        for sid in list(chunks) + list(close):
            if sid not in self.streams:
                raise KeyError(f"unknown stream {sid!r}")
        H, LA, W = self.p.hop, self.p.lookahead, self.window
        for sid in close:
            a = self.ana.streams[sid]
            T = 1 + (a.n_in + (torch.as_tensor(chunks[sid]).numel() if sid in chunks else 0)) // self.hp.hop_length
            if T < self.m:
                raise ValueError(f"stream {sid!r} has {T} frames at close; the model needs at least {self.m}")
        self.clock.lap()
        new = self.ana.push(chunks, close)
        for sid, mel in new.items():
            if self.norm is not None:
                mel = (mel - self.norm[0]) / self.norm[1]
            self.streams[sid].hist.append(mel)
        # the windows of every ready block, and of each closing stream's last one
        wins = []     # (sid, block start, block end, window start, window end)
        for sid in dict.fromkeys(list(chunks) + list(close)):
            s, F = self.streams[sid], self.ana.streams[sid].frames
            while block_end(s.block, H, LA, self.m) <= F:
                b0, b1, w0, w1 = block_schedule(s.block, W, H, LA, self.m)
                wins.append((sid, b0, b1, w0, w1))
                s.block += 1
                s.e_last = w1
            if sid in close and s.block * H < F:
                w0, w1 = close_window(F, W)
                wins.append((sid, s.block * H, F, w0, w1))
                s.block = -(-F // H)
        self.clock.lap("analysis")
        outs = self._convert(wins, final=set(close))
        blocks = {}
        for (sid, b0, b1, w0, w1), dec in zip(wins, outs):
            s = self.streams[sid]
            rows = dec[b0 - w0:b1 - w0]
            X = min(self.w_new.shape[0], rows.shape[0])
            if s.prev is not None and X:
                rows = torch.cat([rows[:X] * self.w_new[:X] + s.prev[:X] * self.w_old[:X], rows[X:]])
            # a compact copy: a view would keep the whole batch output alive while the stream waits
            s.prev = dec[b1 - w0:b1 - w0 + self.w_new.shape[0]].clone() if b1 - w0 < dec.shape[0] else None
            blocks.setdefault(sid, []).append(rows)
            if self.p.keep_mels:
                s.mels.append(rows.clone())
        mags = {}
        if blocks:
            ids = list(blocks)
            cat = [torch.cat(blocks[i]) for i in ids]
            mel = torch.cat(cat)
            if self.norm is not None:
                mel = mel * self.norm[1] + self.norm[0]
            mags = dict(zip(ids, torch.split(self.voc.mel_to_mag([mel])[0], [c.shape[0] for c in cat])))
        # history no longer needed: the next window, or the last one at close, starts at or after frame F - W
        for sid in chunks:
            self.streams[sid].hist.trim(max(0, self.ana.streams[sid].frames - W))
        self.clock.lap("conversion")
        res = self.stage.run(mags, close)
        for sid in chunks:
            if sid not in close:
                self.streams[sid].sched.prune(self._read_from(sid))
        for sid in close:
            mels = self.streams.pop(sid).mels
            if self.p.keep_mels:
                self.closed[sid] = mels
            self.ana.drop(sid)
        return {sid: res.get(sid, torch.empty(0, device=self.dev)) for sid in dict.fromkeys(list(chunks) + list(close))}

    def _convert(self, wins, final):
        """Converted mels [window frames, n_mels] of every window, grouped into batches: plain windows by length, morph
        windows by length and anchor count K rounded up to a power of two (the padding anchors have zero weight)."""
        out = [None] * len(wins)
        groups = {}    # (length, close window, K rounded up; None for plain windows): [(window, codes, weights)]
        for k, (sid, _, _, w0, w1) in enumerate(wins):
            sched = self.streams[sid].sched
            a, w = sched.window(w0, w1)
            Kp = None if w is None else 1 << (len(a) - 1).bit_length()
            codes = [sched.codes[a]] if w is None else [sched.codes[i] for i in a]
            groups.setdefault((w1 - w0, sid in final, Kp), []).append((k, codes, w))
        for (Lw, last, Kp), items in sorted(groups.items(), key=lambda g: g[0][2] is not None):   # plain ones first
            for f in range(0, len(items), self.p.batch_max):
                part = items[f:f + self.p.batch_max]
                # a close window has any length: eager, the exact batch; otherwise padded by repeating row 0
                B = len(part) if last else min(self.p.batch_max, 1 << (len(part) - 1).bit_length())
                rows = part + [part[0]] * (B - len(part))
                x = torch.stack([self._slice(wins[k]) for k, _, _ in rows])
                if Kp is None:
                    ins = (x, torch.stack([c[0] for _, c, _ in rows]))
                else:
                    zero = torch.zeros(self.c_out, device=self.dev)
                    cb = torch.stack([c for _, cs, _ in rows for c in cs + [zero] * (Kp - len(cs))])
                    wh = np.zeros((B, Kp, Lw), np.float32)          # the batch's weights, built on the host
                    for j, (_, _, w) in enumerate(rows):
                        wh[j, :w.shape[0]] = w
                    ins = (x, cb.view(B, Kp, self.c_out), torch.from_numpy(wh))
                model = self.inf.model
                if last:
                    dec = (model.inference_from_embeddings if Kp is None else model.inference_morph)(
                        *(t.to(self.dev) for t in ins))
                else:
                    *bufs, run = (self._slot(B, Lw) if Kp is None else
                                  self.inf._morph_slot(B, self.n_mels, Lw, Kp, self.dev))
                    for b, t in zip(bufs, ins):                      # a morph batch's weights: one upload
                        b.copy_(t)
                    if Kp is not None:
                        bufs[3].fill_(Lw)                           # the slot is shared with Inferencer.inference_morph
                    dec = run()
                for j, (k, _, _) in enumerate(part):
                    out[k] = dec[j, :, :Lw].transpose(0, 1)
        if wins:
            self.inf.model.engine(self.dev).check_tc_status()
        return out

    def _slice(self, win):
        sid, _, _, w0, w1 = win
        return self.streams[sid].hist.view(w0, w1).transpose(0, 1)

    def _slot(self, B, T):
        inf = self.inf

        def make():
            xb = torch.zeros(B, self.n_mels, T, device=self.dev)
            eb = torch.zeros(B, self.c_out, device=self.dev)
            return (xb, eb), lambda: inf.model.inference_from_embeddings(xb, eb)
        return inf._graph_slot(("stream", B, self.n_mels, T, str(self.dev), inf._param_version()), make)
