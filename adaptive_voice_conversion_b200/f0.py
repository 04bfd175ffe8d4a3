"""F0 of synthesised speech: a YIN tracker on the GPU (``avc_yin``, csrc/pitch.cu) and F0 contour and pitch-level
scores of conversions.  Every F0 here is that of a signal this project's Griffin-Lim vocoder synthesised from a mel
(``Vocoder.mel_to_signal``, untrimmed), never of an original recording: the sets keep mels only.

Tracker (de Cheveigne & Kawahara 2002), per signal s of a ragged batch, frame f centred at sample f hop (1 + len // hop
frames: T frames for a signal synthesised from T mel frames, aligned with them), with tau_min = floor(sr / fmax),
tau_max = ceil(sr / fmin) and x[j] = s[reflect(f hop - floor((W + tau_max) / 2) + j)] (one reflection):
  * d(tau) = sum_{j<W} (x[j] - x[j + tau])^2, tau = 1..tau_max;
  * d'(tau) = d(tau) tau / sum_{k=1..tau} d(k), and 1 where that sum is 0 (digital silence);
  * tau* = the smallest tau in [tau_min, tau_max] with d'(tau) < theta, then descend while d'(tau + 1) < d'(tau) and
    tau < tau_max; if no tau is below theta, the argmin of d' there (smallest tau on ties);
  * refinement: with a, b, c = d'(tau* - 1), d'(tau*), d'(tau* + 1) (when tau* - 1 >= 1 and tau* + 1 <= tau_max),
    delta = (a - c) / (2 (a - 2b + c)) if that denominator is > 0, else 0, clamped to [-1/2, 1/2];
  * tau = tau* + delta, aperiodicity = d'(tau*), energy = (1/W) sum_{j<W} x[j]^2, all float64.
theta is used as float32 (the C ABI's type) everywhere, the voicing rule included.  A frame is voiced when
aperiodicity < theta, energy > 0 and 10 log10(energy / the signal's largest frame energy) >= -silence_db; then
f0 = sr / tau.  Defaults: fmin 50 Hz, fmax 500 Hz (48 and 480 lags at 24 kHz), W = 1024, theta = 0.1, silence_db = 40.
None of them is tuned.

Measure (``evaluate_f0``) of one set, the model in eval mode:
  * pairs: ``speaker_eval.conversion_pairs`` with the arguments ``evaluate_speakers`` gives it, so -f0 and -spk score
    the same (source, reference) pairs; with n_refs K > 1 ``fewshot_pairs`` and the pooled codes, as -spk;
  * each conversion is ``mcd.converted`` (the bits of ``Inferencer.inference_ragged``), cropped to the source's T frames;
  * every mel (attr-normalised) is denormalised with attr and synthesised by ``mel_to_signal`` (Griffin-Lim settings
    ``hp``), in chunks of at most ``frame_budget`` frames: the copy-synthesis of every utterance -spk embeds (at least
    max(min_frames) frames) and every conversion;
  * speaker profile: the mean and (ddof 0) std of log2 F0 over the voiced frames of a speaker's copy-synthesised
    utterances, summed sequentially in float64 in sorted utterance order (the std in a second pass about the mean).
    A pair's target profile leaves out its reference(s), its source profile leaves out the source;
  * per pair (u converted with r, both tracks of T frames):
      vuv_agree = the share of the T frames whose voicing agrees between the conversion and u's copy-synthesis;
      f0_corr = the Pearson correlation of log2 F0 over the frames voiced in both (contour preservation);
      st_target = 12 |mean log2 F0 over the conversion's voiced frames - the target profile's mean| (semitones);
      st_source = the same against the source profile's mean; f0_success = [st_target < st_source];
      st_target_source = st_target of u's copy-synthesis itself: the unconverted baseline.
    Means are sequential float64 sums in frame order.  A pair is counted in ``n_unvoiced`` and not scored when fewer
    than 2 frames are voiced in both, when either log2 F0 series is constant over those frames, or when a profile has
    no voiced frame;
  * per set: the means of the six values over the scored pairs (float64, pair order), ``n`` (scored pairs),
    ``n_short``, ``n_unvoiced``, the same means per target speaker, ``profiles`` per speaker (log2_mean, log2_std,
    voiced, frames; the means None without a voiced frame), and the tracker and Griffin-Lim settings.
Both sides of every comparison carry the same vocoder artefacts; the scores compare checkpoints and vocoder settings of
this project, and say how far a conversion moves pitch, not how natural it sounds.
"""
from __future__ import annotations

import ctypes as C
import math
from dataclasses import dataclass, replace
from typing import Dict, List, Mapping, Sequence

import numpy as np
import torch

from . import _lib as L
from .evaluate import speaker_of
from .utils import _stream, eval_mode, upload_mels
from .vocoder import PITCH_SHIFT_MAX, AudioParams, Vocoder, _Ragged, _ptr

METRICS = ("vuv_agree", "f0_corr", "st_target", "st_source", "f0_success", "st_target_source")


@dataclass(frozen=True)
class F0Params:
    """The tracker's parameters (none of them tuned)."""
    fmin: float = 50.0          # Hz: tau_max = ceil(sr / fmin)
    fmax: float = 500.0         # Hz: tau_min = floor(sr / fmax)
    win: int = 1024             # integration window W (samples)
    threshold: float = 0.1      # voicing threshold theta on the aperiodicity d'(tau*), used as float32
    silence_db: float = 40.0    # frames more than this below the signal's loudest frame are unvoiced

    def tau_min(self, sr: int) -> int:
        return int(math.floor(sr / self.fmax))

    def tau_max(self, sr: int) -> int:
        return int(math.ceil(sr / self.fmin))

    def theta(self) -> float:
        return float(np.float32(self.threshold))

    def min_samples(self, sr: int) -> int:
        """Shortest signal every frame of which needs one reflection at most: ceil((W + tau_max) / 2) + 1."""
        return -(-(self.win + self.tau_max(sr)) // 2) + 1

    def settings(self, sr: int, hop: int) -> dict:
        return {"fmin": self.fmin, "fmax": self.fmax, "win": self.win, "tau_min": self.tau_min(sr),
                "tau_max": self.tau_max(sr), "threshold": self.threshold, "silence_db": self.silence_db, "sr": int(sr),
                "hop": int(hop)}


def yin(wavs, sr: int, hop: int, params: F0Params = F0Params()):
    """[(tau, aperiodicity, energy)] float64 device tensors of 1 + len // hop frames per signal of `wavs` (1-D device
    tensors, float32), one avc_yin launch; the module docstring gives the definition.  ValueError for a signal shorter
    than params.min_samples(sr)."""
    ys = [w.reshape(-1).float().contiguous() for w in wavs]
    if not ys:
        raise ValueError("yin: empty batch")
    if hop < 1:
        raise ValueError(f"yin: hop must be positive (got {hop})")
    need = params.min_samples(sr)
    for i, y in enumerate(ys):
        if y.numel() < need:
            raise ValueError(f"yin: signal {i} has {y.numel()} samples; W = {params.win} and tau_max = "
                             f"{params.tau_max(sr)} need at least {need}")
    r = _Ragged([y.numel() for y in ys], [1 + y.numel() // hop for y in ys], ys[0].device)
    out = _yin_launch(r, torch.cat(ys), hop, sr, params)
    return list(zip(*[r.split_frames(o) for o in out]))


def _yin_launch(r: _Ragged, y, hop: int, sr: int, params: F0Params, window: bool = False):
    """float64 [3, frames of r] (tau, aperiodicity, energy) of the entries of r in the signal y, in one avc_yin launch,
    or with window one avc_yin_window launch (each entry from r's frame origin on)."""
    out = torch.empty(3, int(r.frame_offs[-1]), dtype=torch.float64, device=y.device)
    d = L.AudioDesc(hop=int(hop), n_seg=len(r.n_samples), n_frames=out.shape[1], n_samples=int(r.sample_offs[-1]),
                    segs=_ptr(r.table), y=_ptr(y))
    name = "avc_yin_window" if window else "avc_yin"
    L.check(getattr(L.load(), name)(C.byref(d), int(params.win), params.tau_min(sr), params.tau_max(sr),
                                    C.c_float(params.threshold), _ptr(out[0]), _ptr(out[1]), _ptr(out[2]),
                                    _stream(y.device)), name)
    return out


def voicing(tau: np.ndarray, aperiodicity: np.ndarray, energy: np.ndarray, sr: int, params: F0Params = F0Params()):
    """(f0 Hz, voiced) float64 / bool of one signal's tracker outputs (host, float64); f0 is NaN where unvoiced."""
    tau, ap, en = (np.asarray(v, np.float64) for v in (tau, aperiodicity, energy))
    emax = float(en.max()) if en.size else 0.0
    with np.errstate(divide="ignore", invalid="ignore"):
        rel = 10.0 * np.log10(en / emax) if emax > 0 else np.full(en.shape, -np.inf)
    voiced = (ap < params.theta()) & (en > 0) & (rel >= -params.silence_db)
    f0 = np.where(voiced, sr / np.where(voiced, tau, 1.0), np.nan)
    return f0, voiced


def track(wavs, sr: int, hop: int, params: F0Params = F0Params()):
    """[(f0 Hz, voiced)] per signal: ``yin`` on the device, ``voicing`` on the host in float64."""
    outs = yin(wavs, sr, hop, params)
    host = [torch.stack(o).cpu().numpy() for o in outs]
    return [voicing(h[0], h[1], h[2], sr, params) for h in host]


# ------------------------------------------------------------------ the measure
def _seq_sum(v: np.ndarray) -> float:
    return float(np.cumsum(v)[-1]) if len(v) else 0.0


def _mean_std(v: np.ndarray):
    m = _seq_sum(v) / len(v)
    return m, math.sqrt(_seq_sum((v - m) ** 2) / len(v))


def profile(logs: Sequence[np.ndarray]):
    """(log2 mean, log2 std, voiced frames) of the concatenated voiced log2 F0 series `logs` (None, None, 0 without
    one)."""
    v = np.concatenate([np.asarray(x, np.float64) for x in logs]) if logs else np.zeros(0)
    if not len(v):
        return None, None, 0
    m, s = _mean_std(v)
    return m, s, len(v)


def pearson(a: np.ndarray, b: np.ndarray) -> float:
    """sum (a - ma)(b - mb) / sqrt(sum (a - ma)^2 sum (b - mb)^2), every sum sequential in float64."""
    ma, mb = _seq_sum(a) / len(a), _seq_sum(b) / len(b)
    da, db = a - ma, b - mb
    return _seq_sum(da * db) / math.sqrt(_seq_sum(da * da) * _seq_sum(db * db))


def pair_scores(conv, src, target_mean, source_mean):
    """The six per-pair values of a conversion's and its source's copy-synthesis tracks ((f0, voiced) of T frames
    each) against the profile means, or None when the pair goes to n_unvoiced (the module docstring's rules)."""
    (fc, vc), (fs, vs) = conv, src
    both = vc & vs
    if target_mean is None or source_mean is None or int(both.sum()) < 2:
        return None
    a, b = np.log2(fc[both]), np.log2(fs[both])
    if np.all(a == a[0]) or np.all(b == b[0]):
        return None
    mc = _seq_sum(np.log2(fc[vc])) / int(vc.sum())
    ms = _seq_sum(np.log2(fs[vs])) / int(vs.sum())
    st_t, st_s = 12.0 * abs(mc - target_mean), 12.0 * abs(mc - source_mean)
    return [_seq_sum((vc == vs).astype(np.float64)) / len(vc), pearson(a, b),
            st_t, st_s, float(st_t < st_s), 12.0 * abs(ms - target_mean)]


def _means(rows: np.ndarray) -> dict:
    out = {k: _seq_sum(rows[:, i]) / len(rows) for i, k in enumerate(METRICS)}
    out["n"] = len(rows)
    return out


def synthesize(vocoder: Vocoder, mels, hp: AudioParams, frame_budget: int = 32768, semitones=None):
    """mel_to_signal of each (denormalised) mel, in chunks of at most frame_budget frames (one longer mel alone);
    semitones (one per mel) shifts them, default hp.pitch_shift."""
    out, chunk, shifts, frames = [], [], [], 0
    semitones = [hp.pitch_shift] * len(mels) if semitones is None else list(semitones)

    def flush():
        if chunk:
            out.extend(vocoder.mel_to_signal(chunk, hp.n_iter, hp.momentum, hp.gl_init, semitones=list(shifts)))
            chunk.clear()
            shifts.clear()
    for m, st in zip(mels, semitones):
        if chunk and frames + int(m.shape[0]) > frame_budget:
            flush()
            frames = 0
        chunk.append(m)
        shifts.append(st)
        frames += int(m.shape[0])
    flush()
    return out


def track_chunks(signals, sr: int, hop: int, params: F0Params, frame_budget: int = 1 << 20):
    """``track`` over the signals in chunks of at most frame_budget frames."""
    out, chunk, frames = [], [], 0
    for s in signals:
        n = 1 + s.numel() // hop
        if chunk and frames + n > frame_budget:
            out.extend(track(chunk, sr, hop, params))
            chunk, frames = [], 0
        chunk.append(s)
        frames += n
    if chunk:
        out.extend(track(chunk, sr, hop, params))
    return out


# ------------------------------------------------------------------ matching the target's pitch level
def shifts_from_tracks(conv_tracks, ref_track_sets, limit: float = PITCH_SHIFT_MAX):
    """(shifts, info) from tracks ((f0, voiced) per signal): conversion i's shift is 12 (mu_refs - mu_conv), each mu
    the mean log2 F0 over voiced frames (``profile``: the references' voiced frames pooled), clamped to +-limit; 0 and
    unmatched when either side has no voiced frame.  info[i] = {"shift", "voiced_conv", "voiced_refs", "clamped",
    "unmatched"}."""
    shifts, info = [], []
    for (fc, vc), refs in zip(conv_tracks, ref_track_sets):
        mc, _, nc = profile([np.log2(fc[vc])])
        mr, _, nr = profile([np.log2(f[v]) for f, v in refs])
        unmatched = mc is None or mr is None
        st = 0.0 if unmatched else 12.0 * (mr - mc)
        clamped = abs(st) > limit
        st = float(min(limit, max(-limit, st)))
        shifts.append(st)
        info.append({"shift": st, "voiced_conv": int(nc), "voiced_refs": int(nr), "clamped": bool(clamped),
                     "unmatched": bool(unmatched)})
    return shifts, info


def unshifted_tracks(vocoder: Vocoder, conv_mels, ref_sets, hp: AudioParams, params: F0Params = F0Params(),
                     frame_budget: int = 32768):
    """(conversion tracks, reference track sets): conv_mels [T, n_mels] and ref_sets (lists of [T, n_mels])
    denormalised mels on the device, all synthesised unshifted by mel_to_signal at hp's Griffin-Lim settings (in
    synthesize's chunks) and tracked with the same tracker, as evaluate_f0 does, so both carry the same vocoder
    artefacts."""
    flat = [r for rs in ref_sets for r in rs]
    signals = synthesize(vocoder, list(conv_mels) + flat, hp, frame_budget, semitones=[0.0] * (len(conv_mels) + len(flat)))
    tracks = track_chunks(signals, hp.sr, hp.hop_length, params)
    refs, k = [], len(conv_mels)
    for rs in ref_sets:
        refs.append(tracks[k:k + len(rs)])
        k += len(rs)
    return tracks[:len(conv_mels)], refs


def match_shifts(vocoder: Vocoder, conv_mels, ref_sets, hp: AudioParams, params: F0Params = F0Params(),
                 frame_budget: int = 32768):
    """Shifts (semitones) that move each conversion's mean log2 F0 to its reference set's, both tracked unshifted
    (``unshifted_tracks``); ``shifts_from_tracks`` gives (shifts, info)."""
    if len(conv_mels) != len(ref_sets):
        raise ValueError("match_shifts: one reference set per conversion")
    return shifts_from_tracks(*unshifted_tracks(vocoder, conv_mels, ref_sets, hp, params, frame_budget))


# ------------------------------------------------------------------ matching the target's pitch level and range
def track_profile(tracks):
    """(log2 mean, log2 std) of the voiced frames of tracks ((f0, voiced) per signal) pooled, or None without one."""
    m, s, _ = profile([np.log2(f[v]) for f, v in tracks])
    return None if m is None else (m, s)


def mv_shifts(conv_tracks, targets, limit: float = PITCH_SHIFT_MAX):
    """(per-frame shifts, info) of the mean-and-variance log-F0 transform: conversion i's unshifted track (f0, voiced)
    of T frames toward targets[i], a target profile (mu_t, sigma_t) of log2 F0 (floats, or float64 arrays of T values
    for a profile that varies per frame) or None (unmatched).

    With (mu_c, sigma_c) = ``profile`` of the conversion's voiced log2 F0 l, the shift on a voiced frame f is
    12 (mu_t(f) + sigma_t(f) / sigma_c (l - mu_c) - l), clamped to +-limit; an unvoiced frame's is linearly interpolated
    in frame index between the nearest voiced frames' and held before the first and after the last.  With sigma_c = 0
    or fewer than 2 voiced frames every frame gets 12 (mu_t(f) - mu_c), clamped ("mean_only"); with no voiced frame on
    either side every shift is 0 ("unmatched").  All float64.  info[i] = {"mean_shift" (over the T frames),
    "voiced_conv", "clamped_frames" (the frames whose shift was clamped: voiced ones, or any with mean_only),
    "mean_only", "unmatched"}."""
    shifts, info = [], []
    for (fc, vc), tgt in zip(conv_tracks, targets):
        T = len(vc)
        idx = np.flatnonzero(vc)
        l = np.log2(np.asarray(fc, np.float64)[idx])
        mc, sc, nc = profile([l])
        unmatched = mc is None or tgt is None
        mean_only = not unmatched and (sc == 0.0 or nc < 2)
        clamped = 0
        if unmatched:
            s = np.zeros(T)
        else:
            mu_t, sd_t = (np.broadcast_to(np.asarray(x, np.float64), (T,)) for x in tgt)
            if mean_only:
                s = 12.0 * (mu_t - mc)
                clamped = int(np.count_nonzero(np.abs(s) > limit))
                s = np.clip(s, -limit, limit)
            else:
                sv = 12.0 * (mu_t[idx] + sd_t[idx] / sc * (l - mc) - l)
                clamped = int(np.count_nonzero(np.abs(sv) > limit))
                s = np.interp(np.arange(T, dtype=np.float64), idx.astype(np.float64), np.clip(sv, -limit, limit))
        shifts.append(np.ascontiguousarray(s, np.float64))
        info.append({"mean_shift": _seq_sum(s) / T if T else 0.0, "voiced_conv": int(nc),
                     "clamped_frames": clamped, "mean_only": bool(mean_only), "unmatched": bool(unmatched)})
    return shifts, info


def mv_match(vocoder: Vocoder, conv_mels, hp: AudioParams, ref_sets=None, profiles=None,
             params: F0Params = F0Params(), frame_budget: int = 32768):
    """``mv_shifts`` of denormalised conversion mels [T, n_mels] (device tensors), each toward one target: where
    ref_sets[i] is a list of denormalised reference mels, their pooled profile (``track_profile``); where it is None
    (or ref_sets is omitted), profiles[i], a target profile as ``mv_shifts`` takes it (None: unmatched).  The
    conversions and the references are tracked by ``unshifted_tracks``, as ``match_shifts`` tracks them.  Returns
    (shifts, info).  ValueError when a conversion has both a reference set and a profile, or when a list's length is
    not the number of conversions."""
    n = len(conv_mels)
    ref_sets = [None] * n if ref_sets is None else list(ref_sets)
    profiles = [None] * n if profiles is None else list(profiles)
    if len(ref_sets) != n or len(profiles) != n:
        raise ValueError("mv_match: one reference set or profile per conversion")
    for i, (rs, pr) in enumerate(zip(ref_sets, profiles)):
        if rs is not None and (pr is not None or not isinstance(rs, list) or not rs):
            raise ValueError(f"mv_match: conversion {i}: give a non-empty list of reference mels or a profile, not both")
    conv_tracks, ref_tracks = unshifted_tracks(vocoder, conv_mels, [rs or [] for rs in ref_sets], hp, params,
                                               frame_budget)
    return mv_shifts(conv_tracks, [pr if rs is None else track_profile(rt)
                                   for rs, pr, rt in zip(ref_sets, profiles, ref_tracks)])


def select_pairs(cfg, lengths: Mapping[str, int], seed: int = 0, max_pairs: int = 0, n_refs: int = 1):
    """(embedded utterances, [(source, reference)], [[reference, ...]] per pair, {"n", "n_short"[, "n_refs",
    "n_few"]}): the utterances and pairs evaluate_speakers uses for the same arguments (lengths[u] = frames of u)."""
    from .mcd import min_frames
    from .speaker_eval import conversion_pairs, fewshot_pairs
    min_src, min_ref = min_frames(cfg)
    min_set = max(min_src, min_ref)
    utts = [u for u in sorted(lengths) if lengths[u] >= min_set]
    pairs, n_short = conversion_pairs(list(lengths), lengths, seed, max_pairs, min_set, min_ref, min_set)
    res = {"n": 0, "n_short": n_short, "n_unvoiced": 0}
    if n_refs > 1:
        pairs, n_few = fewshot_pairs(pairs, list(lengths), lengths, n_refs, seed, min_ref, min_set)
        res.update(n_refs=int(n_refs), n_few=n_few)
    return utts, pairs, [list(r) if n_refs > 1 else [r] for _, r in pairs], res


def evaluate_f0(model, data: Mapping[str, np.ndarray], attr, seed: int = 0, max_pairs: int = 0, device=None,
                per_pair: bool = False, n_refs: int = 1, hp: AudioParams = AudioParams(),
                params: F0Params = F0Params(), frame_budget: int = 32768, timings: dict = None,
                pitch_shift: str | None = None) -> dict:
    """F0 measures of `model` (an AE) on one set: data = {utterance key: attr-normalised [T, n_mels]} (the set's
    pickle), attr its mel statistics.  hp gives the Griffin-Lim settings (n_iter, momentum, gl_init; n_mels is the
    model's c_in; its pitch_shift is not used).  Returns the module docstring's set entry; per_pair adds "pairs": [[source, reference(s), the six
    values], ...] for the scored pairs.  timings (a dict) receives the wall seconds of conversion, synthesis, tracking
    and host work, each ended by a device synchronise.

    pitch_shift="match" shifts each conversion toward its reference(s) (``shifts_from_tracks`` on the unshifted
    tracks this call computes anyway), re-synthesises and re-tracks it and scores it against the same leave-out
    profiles; the entry then holds the shifted scores, "pitch_shift": {"mode", "mean_semitones",
    "mean_abs_semitones", "n_unmatched", "n_clamped"} over the pairs, and "unshifted": the entry of the call without
    it.  pitch_shift="mv" does the same with ``mv_shifts`` toward the profile of the reference(s)' tracks
    (``track_profile``); a pair's shift is then the mean of its per-frame shifts (mean_abs_semitones: of their absolute
    values), n_clamped counts the pairs with a clamped frame, and "pitch_shift" adds n_mean_only, n_clamped_frames and
    sd_target / sd_target_unshifted: the mean over the scored pairs whose references have a voiced frame of
    12 |sigma_conv - sigma_target|, sigma the log2 std of the (shifted / unshifted) conversion's voiced frames and of
    the target profile (None without such a pair)."""
    import time
    from .mcd import converted
    from .speaker_eval import SPK_MAX_EXCLUDE
    cfg = model.config
    if pitch_shift not in (None, "match", "mv"):
        raise ValueError(f"evaluate_f0: pitch_shift must be None, 'match' or 'mv' (got {pitch_shift!r})")
    if int(cfg["data_loader"]["frame_size"]) != 1:
        raise ValueError(f"F0 evaluation supports data_loader.frame_size 1 only (got {cfg['data_loader']['frame_size']})")
    if not 1 <= int(n_refs) <= SPK_MAX_EXCLUDE:
        raise ValueError(f"n_refs must lie in [1, {SPK_MAX_EXCLUDE}] (got {n_refs})")
    dev = torch.device(device) if device is not None else next(model.parameters()).device
    clock = {"conversion": 0.0, "synthesis": 0.0, "tracking": 0.0, "host": 0.0}
    t0 = time.perf_counter()

    def lap(k):
        nonlocal t0
        torch.cuda.synchronize(dev)
        t1 = time.perf_counter()
        clock[k] += t1 - t0
        t0 = t1

    utts, pairs, refs, res = select_pairs(cfg, {u: len(v) for u, v in data.items()}, seed, max_pairs, n_refs)
    used = sorted(set(utts) | {u for u, _ in pairs} | {v for rs in refs for v in rs})
    mels = upload_mels(data, used, dev)
    n_mels = int(cfg["SpeakerEncoder"]["c_in"])
    hp = replace(hp, n_mels=n_mels, pitch_shift=0.0)
    res["tracker"] = params.settings(hp.sr, hp.hop_length)
    res["griffin_lim"] = {"n_iter": int(hp.n_iter), "momentum": float(hp.momentum), "init": hp.gl_init}
    mean = torch.as_tensor(np.asarray(attr["mean"], np.float32).reshape(-1)).to(dev)
    std = torch.as_tensor(np.asarray(attr["std"], np.float32).reshape(-1)).to(dev)
    if mean.numel() != n_mels or std.numel() != n_mels:
        raise ValueError(f"evaluate_f0: attr mean / std have {mean.numel()} / {std.numel()} entries, the mels {n_mels}")
    convs = [None] * len(pairs)
    with eval_mode(model, dev):
        codes = None
        if n_refs > 1 and pairs:
            from .inference import embed_reference_sets
            codes = embed_reference_sets(model, [[mels[v].t() for v in rs] for rs in refs])
        if pairs:
            for idx, decs in converted(model, [mels[u] for u, _ in pairs], [mels[rs[0]] for rs in refs], codes=codes):
                for i, dec in zip(idx, decs):
                    convs[i] = dec
    lap("conversion")
    vocoder = Vocoder(hp=hp, device=dev)
    conv_mels = [c * std + mean for c in convs]
    signals = synthesize(vocoder, [mels[u] * std + mean for u in utts] + conv_mels, hp, frame_budget)
    lap("synthesis")
    tracks = track_chunks(signals, hp.sr, hp.hop_length, params)
    lap("tracking")
    real = dict(zip(utts, tracks[:len(utts)]))
    conv_tracks = tracks[len(utts):]
    logs = {u: np.log2(f[v]) for u, (f, v) in real.items()}
    by_speaker: Dict[str, List[str]] = {}
    for u in utts:
        by_speaker.setdefault(speaker_of(u), []).append(u)

    def profile_mean(spk, exclude):
        return profile([logs[v] for v in by_speaker.get(spk, []) if v not in exclude])[0]

    kept = []     # the pairs the last score() call scored

    def score(res, conv_tracks):
        rows = []
        kept.clear()
        for i, ((u, _), rs) in enumerate(zip(pairs, refs)):
            v = pair_scores(conv_tracks[i], real[u], profile_mean(speaker_of(rs[0]), set(rs)),
                            profile_mean(speaker_of(u), {u}))
            if v is None:
                res["n_unvoiced"] += 1
            else:
                rows.append(v)
                kept.append(i)
        vals = np.asarray(rows, np.float64).reshape(-1, len(METRICS))
        res["n"] = len(rows)
        if rows:
            res.update({k: v for k, v in _means(vals).items() if k != "n"})
        groups: Dict[str, List[int]] = {}
        for j, i in enumerate(kept):
            groups.setdefault(speaker_of(refs[i][0]), []).append(j)
        res["speakers"] = {s: _means(vals[js]) for s, js in groups.items()}
        res["profiles"] = {}
        for s, us in by_speaker.items():
            m, sd, nv = profile([logs[u] for u in us])
            res["profiles"][s] = {"log2_mean": m, "log2_std": sd, "voiced": nv,
                                  "frames": sum(len(real[u][1]) for u in us)}
        if per_pair:
            res["pairs"] = [[pairs[i][0], refs[i] if n_refs > 1 else refs[i][0]] + [float(x) for x in vals[j]]
                            for j, i in enumerate(kept)]
        return res

    base = dict(res)
    res = score(res, conv_tracks)
    lap("host")
    if pitch_shift is not None:
        # the references' copy-syntheses are the tracks above; a reference too short to be embedded is tracked here
        extra = sorted({v for rs in refs for v in rs} - set(real))
        if extra:
            sig = synthesize(vocoder, [mels[v] * std + mean for v in extra], hp, frame_budget)
            lap("synthesis")
            real.update(zip(extra, track_chunks(sig, hp.sr, hp.hop_length, params)))
            lap("tracking")
        ref_tracks = [[real[v] for v in rs] for rs in refs]
        if pitch_shift == "match":
            shifts, info = shifts_from_tracks(conv_tracks, ref_tracks)
            pair_shift = np.asarray(shifts, np.float64)
            pair_abs = np.abs(pair_shift)
        else:
            targets = [track_profile(t) for t in ref_tracks]
            unshifted_kept = list(kept)
            shifts, info = mv_shifts(conv_tracks, targets)
            pair_shift = np.asarray([d["mean_shift"] for d in info], np.float64)
            pair_abs = np.asarray([_seq_sum(np.abs(s)) / max(len(s), 1) for s in shifts], np.float64)
        sig = synthesize(vocoder, conv_mels, hp, frame_budget, semitones=shifts)
        lap("synthesis")
        shifted = track_chunks(sig, hp.sr, hp.hop_length, params)
        lap("tracking")
        unshifted, res = res, score(base, shifted)
        n = max(len(shifts), 1)
        res["pitch_shift"] = {"mode": pitch_shift, "mean_semitones": _seq_sum(pair_shift) / n,
                              "mean_abs_semitones": _seq_sum(pair_abs) / n,
                              "n_unmatched": sum(d["unmatched"] for d in info)}
        if pitch_shift == "match":
            res["pitch_shift"]["n_clamped"] = sum(d["clamped"] for d in info)
        else:
            def sd_gap(tracks, pairs_kept):
                gaps = [12.0 * abs(track_profile([tracks[i]])[1] - targets[i][1]) for i in pairs_kept
                        if targets[i] is not None]
                return _seq_sum(np.asarray(gaps, np.float64)) / len(gaps) if gaps else None
            res["pitch_shift"].update(n_clamped=sum(d["clamped_frames"] > 0 for d in info),
                                      n_mean_only=sum(d["mean_only"] for d in info),
                                      n_clamped_frames=sum(d["clamped_frames"] for d in info),
                                      sd_target=sd_gap(shifted, kept), sd_target_unshifted=sd_gap(conv_tracks, unshifted_kept))
        res["unshifted"] = unshifted
        lap("host")
    if timings is not None:
        timings.update(clock)
    return res
