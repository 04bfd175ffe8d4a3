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
  samples on ``mel_to_signal``'s grid as their frames are committed.

``block_schedule``, ``blend_weights`` and ``latency_samples`` state the schedule on the host.
"""
from __future__ import annotations

import ctypes as C
import time
from dataclasses import dataclass

import numpy as np
import torch

from . import _lib as L
from .mcd import min_frames
from .utils import _stream
from .vocoder import _SEG, _mel_project, _ptr


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
    batch_max: int = 1024     # windows per model batch
    keep_mels: bool = False   # keep each stream's emitted mel frames for take_mels (memory grows with the stream)


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
    if p.batch_max < 1:
        raise ValueError("StreamParams.batch_max must be >= 1")


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


def release_sample(n: int, p: StreamParams, win: int, hop_s: int, m: int) -> int:
    """Index of the input sample whose arrival releases output sample n (before close): n's last covering frame c is
    committed when frame c + gl_lookahead enters RTISI-LA, i.e. when its block j is emitted, at the arrival of the
    sample that completes frame e_j - 1."""
    c = (n + win // 2) // hop_s
    j = (c + p.gl_lookahead) // p.hop
    return (block_end(j, p.hop, p.lookahead, m) - 1) * hop_s + win // 2 - 1


def latency_samples(p: StreamParams, win: int, hop_s: int, m: int) -> int:
    """max over output samples n >= 0 of release_sample(n) - n.  For a frame c the smallest n it is the last
    frame of is the worst; past the start-up windows the schedule repeats every block, so a few blocks beyond m
    cover every case.  Without start-up effects this is (H + LA + LA_v - 1) hop + win - 1."""
    worst = 0
    for c in range(m + 4 * p.hop + p.gl_lookahead + 2 * (win // hop_s) + 8):
        n = max(0, c * hop_s - win // 2)
        if (n + win // 2) // hop_s != c:
            continue
        worst = max(worst, release_sample(n, p, win, hop_s, m) - n)
    return worst


# ------------------------------------------------------------------ analysis
class _AStream:
    __slots__ = ("n_in", "frames", "tail", "tail_first", "closed")

    def __init__(self, dev):
        self.n_in, self.frames, self.tail_first, self.closed = 0, 0, 0, False
        self.tail = torch.empty(0, device=dev)


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
                s.tail = torch.cat([s.tail, x])
                s.n_in += x.numel()
        for sid in close:
            s = self.streams[sid]
            if s.n_in < hp.min_samples:
                raise ValueError(f"stream {sid!r} has {s.n_in} samples; an STFT with n_fft={hp.n_fft} needs at least "
                                 f"{hp.min_samples}")
            s.closed = True
        segs, ys, ids, counts = [], [], [], []
        soff = foff = 0
        for sid in dict.fromkeys(list(chunks) + list(close)):
            s = self.streams[sid]
            n = self.ready(s) - s.frames
            if n <= 0:
                continue
            first = self.first_sample(s.frames)
            y = s.tail[first - s.tail_first:]
            segs.append((soff, y.numel(), foff, n, s.frames))
            ys.append(y)
            ids.append(sid)
            counts.append(n)
            soff += y.numel()
            foff += n
            s.frames += n
            keep = self.first_sample(s.frames)
            s.tail, s.tail_first = s.tail[keep - s.tail_first:], keep
        if not ids:
            return {}
        tab = np.zeros(len(segs), _SEG)
        for k, name in enumerate(("sample_off", "n_samples", "frame_off", "n_frames", "reserved")):
            tab[name] = [g[k] for g in segs]
        table = torch.from_numpy(tab.view(np.uint8)).to(self.dev)
        mag = torch.empty(foff, hp.n_bins, device=self.dev)
        y = torch.cat(ys)
        d = L.AudioDesc(n_fft=hp.n_fft, hop=hp.hop_length, win=hp.win_length, n_seg=len(segs), n_frames=foff,
                        n_samples=int(soff), mode=L.STFT_MAG, preemph=hp.preemphasis, max_db=hp.max_db,
                        ref_db=hp.ref_db, segs=_ptr(table), y=_ptr(y), mag_out=_ptr(mag))
        L.check(L.load().avc_stft_window(C.byref(d), _stream(self.dev)), "avc_stft_window")
        mel = _mel_project(mag, self.voc.fb_t, L.MAG_TO_MEL, hp)
        return dict(zip(ids, torch.split(mel, counts)))


# ------------------------------------------------------------------ RTISI-LA
class Rtisi:
    """RTISI-LA state of many streams in a pool of slots, and one avc_rtisi_la launch per update.
    ``run({id: mags [n, n_bins]}, close=())`` returns {id: released samples}."""

    def __init__(self, hp, lookahead: int = 3, n_iter: int = 8, device=None):
        self.hp, self.la, self.n_iter = hp, int(lookahead), int(n_iter)
        self.dev = torch.device(device) if device is not None else torch.device("cuda")
        self.stride = int(L.load().avc_rtisi_state_floats(hp.win_length, self.la))
        self.state = torch.zeros(0, self.stride, device=self.dev)
        self.count = torch.zeros(0, 2, dtype=torch.int32, device=self.dev)
        self.free, self.slot, self.host = [], {}, {}

    def open(self, sid):
        if not self.free:
            n = max(16, 2 * self.state.shape[0])
            old = self.state.shape[0]
            state = torch.zeros(n, self.stride, device=self.dev)
            count = torch.zeros(n, 2, dtype=torch.int32, device=self.dev)
            state[:old].copy_(self.state)
            count[:old].copy_(self.count)
            self.state, self.count = state, count
            self.free = list(range(n - 1, old - 1, -1))
        k = self.free.pop()
        self.state[k].zero_()
        self.count[k].zero_()
        self.slot[sid], self.host[sid] = k, [0, 0]

    def drop(self, sid):
        if sid in self.slot:
            self.free.append(self.slot.pop(sid))
            self.host.pop(sid)

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
        """The avc_rtisi_la launch of a prepared update (its tables and buffers are kept alive by prepare's result)."""
        L.check(L.load().avc_rtisi_la(C.byref(desc), _stream(self.dev)), "avc_rtisi_la")

    def prepare(self, mags, close=()):
        """(descriptor, {id: output view}, buffers) of one update, the host's counts advanced; None when empty."""
        hp = self.hp
        ids = list(dict.fromkeys(list(mags) + list(close)))
        if not ids:
            return None
        rows, offs, slots, closes, outs, counts = [], [0], [], [], [0], []
        for sid in ids:
            c, nb = self.host[sid]
            m = mags.get(sid)
            p = 0 if m is None else int(m.shape[0])
            if m is not None and p:
                rows.append(m)
            if sid in close:
                T = c + nb + p
                n_out = max(0, (T - 1) * hp.hop_length) - self.released(c)
                self.host[sid] = [T, 0]
            else:
                nb2 = min(nb + p, self.la)
                c2 = c + nb + p - nb2
                n_out = self.released(c2) - self.released(c)
                self.host[sid] = [c2, nb2]
            offs.append(offs[-1] + p)
            slots.append(self.slot[sid])
            closes.append(1 if sid in close else 0)
            counts.append(n_out)
            outs.append(outs[-1] + n_out)
        mag = torch.cat(rows).float().contiguous() if rows else torch.zeros(1, hp.n_bins, device=self.dev)
        n = len(ids)
        i32 = torch.tensor(offs + slots + closes, dtype=torch.int32).to(self.dev)
        out_off = torch.tensor(outs[:-1], dtype=torch.int64).to(self.dev)
        y = torch.empty(max(1, outs[-1]), device=self.dev)
        d = L.RtisiDesc(n_fft=hp.n_fft, hop=hp.hop_length, win=hp.win_length, lookahead=self.la, n_iter=self.n_iter,
                        n_streams=n, deemph=hp.preemphasis, mag=_ptr(mag), mag_off=_ptr(i32[:n + 1]),
                        slot=_ptr(i32[n + 1:2 * n + 1]), close=_ptr(i32[2 * n + 1:]), out_off=_ptr(out_off),
                        y=_ptr(y), state=_ptr(self.state), count=_ptr(self.count))
        return d, dict(zip(ids, torch.split(y[:outs[-1]], counts))), (mag, i32, out_off, y)


# ------------------------------------------------------------------ the converter
class _CStream:
    __slots__ = ("code", "hist", "hist_first", "block", "prev", "mels")

    def __init__(self, code, dev, n_mels):
        self.code = code
        self.hist = torch.empty(0, n_mels, device=dev)
        self.hist_first, self.block, self.prev, self.mels = 0, 0, None, []


class StreamingConverter:
    """Converts many live streams at once.  ``open(code)`` starts a stream converted to the speaker code ``code``
    (float32 [c_out] on the device: a row of ``Inferencer.embed_speakers`` or ``SpeakerBank.code``) and returns its
    id; ``push({id: pcm})`` takes float32 PCM chunks at ``hp.sr`` of any length and returns {id: new output samples}
    (device float32), one batched update; ``close(id)`` returns the stream's last samples.  ``take_mels(id)`` hands
    over the normalised mel frames the stream emitted so far, when the converter keeps them
    (``StreamParams(keep_mels=True)``; off by default, since they grow with the stream).  ``latency_samples`` is the worst case, over output
    samples n, of (index of the input sample whose arrival releases n) - n."""

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
        self.rt = Rtisi(self.hp, params.gl_lookahead, params.gl_iters, self.dev)
        w = blend_weights(params.hop, params.lookahead)
        self.w_new = torch.from_numpy(w).to(self.dev)[:, None]
        self.w_old = torch.from_numpy(np.float32(1) - w).to(self.dev)[:, None]
        self.norm = None
        if inferencer.attr is not None:
            self.norm = tuple(torch.as_tensor(np.asarray(inferencer.attr[k], np.float32)).to(self.dev)
                              for k in ("mean", "std"))
        self.streams, self.closed = {}, {}
        self._next = 0
        self.stage_ms = None   # a dict: each update adds its analysis / conversion / rtisi wall time (synchronised)
        self.latency_samples = latency_samples(params, self.hp.win_length, self.hp.hop_length, self.m)

    def open(self, code) -> int:
        if (not isinstance(code, torch.Tensor) or code.dtype != torch.float32 or tuple(code.shape) != (self.c_out,)
                or code.device != self.dev):
            raise ValueError(f"StreamingConverter.open: code must be float32 [{self.c_out}] on {self.dev}")
        sid = self._next
        self._next += 1
        self.streams[sid] = _CStream(code.contiguous(), self.dev, self.n_mels)
        self.ana.open(sid)
        self.rt.open(sid)
        return sid

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
        t0 = self._tick()
        new = self.ana.push(chunks, close)
        for sid, mel in new.items():
            s = self.streams[sid]
            if self.norm is not None:
                mel = (mel - self.norm[0]) / self.norm[1]
            s.hist = torch.cat([s.hist, mel])
        # the windows of every ready block, and of each closing stream's last one
        wins = []     # (sid, block start, block end, window start, window end)
        for sid in dict.fromkeys(list(chunks) + list(close)):
            s, F = self.streams[sid], self.ana.streams[sid].frames
            while block_end(s.block, H, LA, self.m) <= F:
                b0, b1, w0, w1 = block_schedule(s.block, W, H, LA, self.m)
                wins.append((sid, b0, b1, w0, w1))
                s.block += 1
            if sid in close and s.block * H < F:
                w0, w1 = close_window(F, W)
                wins.append((sid, s.block * H, F, w0, w1))
                s.block = -(-F // H)
        t1 = self._tick()
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
            s = self.streams[sid]
            keep = max(0, self.ana.streams[sid].frames - W)
            if keep > s.hist_first:
                s.hist, s.hist_first = s.hist[keep - s.hist_first:], keep
        t2 = self._tick()
        res = self.rt.run(mags, close)
        if self.stage_ms is not None:
            t3 = self._tick()
            for k, a, b in (("analysis", t0, t1), ("conversion", t1, t2), ("rtisi", t2, t3)):
                self.stage_ms[k] = self.stage_ms.get(k, 0.0) + 1e3 * (b - a)
        for sid in close:
            mels = self.streams.pop(sid).mels
            if self.p.keep_mels:
                self.closed[sid] = mels
            self.ana.drop(sid)
        return {sid: res.get(sid, torch.empty(0, device=self.dev)) for sid in dict.fromkeys(list(chunks) + list(close))}

    def _tick(self):
        if self.stage_ms is None:
            return 0.0
        torch.cuda.synchronize(self.dev)
        return time.perf_counter()

    def _convert(self, wins, final):
        """Converted mels [window frames, n_mels] of every window, grouped by length into batches."""
        out = [None] * len(wins)
        groups = {}
        for k, (sid, _, _, w0, w1) in enumerate(wins):
            groups.setdefault((w1 - w0, sid in final), []).append(k)
        for (Lw, last), idx in groups.items():
            for f in range(0, len(idx), self.p.batch_max):
                part = idx[f:f + self.p.batch_max]
                xs = [self._slice(wins[k]) for k in part]
                codes = [self.streams[wins[k][0]].code for k in part]
                if last:   # a close window has any length: eager, the exact batch
                    dec = self.inf.model.inference_from_embeddings(torch.stack(xs), torch.stack(codes))
                else:
                    Bp = min(self.p.batch_max, 1 << (len(part) - 1).bit_length())
                    xb, eb, run = self._slot(Bp, Lw)
                    rows = list(range(len(part))) + [0] * (Bp - len(part))
                    xb.copy_(torch.stack([xs[r] for r in rows]))
                    eb.copy_(torch.stack([codes[r] for r in rows]))
                    dec = run()
                for j, k in enumerate(part):
                    out[k] = dec[j, :, :Lw].transpose(0, 1)
        if wins:
            self.inf.model.engine(self.dev).check_tc_status()
        return out

    def _slice(self, win):
        sid, _, _, w0, w1 = win
        s = self.streams[sid]
        return s.hist[w0 - s.hist_first:w1 - s.hist_first].transpose(0, 1)

    def _slot(self, B, T):
        inf = self.inf

        def make():
            xb = torch.zeros(B, self.n_mels, T, device=self.dev)
            eb = torch.zeros(B, self.c_out, device=self.dev)
            return (xb, eb), lambda: inf.model.inference_from_embeddings(xb, eb)
        return inf._graph_slot(("stream", B, self.n_mels, T, str(self.dev), inf._param_version()), make)
