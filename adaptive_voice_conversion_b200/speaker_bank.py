"""Speaker code banks: every usable utterance of each speaker pooled into one saved speaker code.

The speaker encoder's only operation across time is its time mean, so a speaker's code pools the last conv layer over
the valid frames of all their utterances together, then runs the dense stack: what get_speaker_embeddings(groups=)
computes for a set of references, without its limit of PADDED_BATCH_MAX references per set.

Building (``build_bank``): the utterances are grouped by speaker, speakers sorted by name and each speaker's
utterances in sorted id order.  That order is the summation order of the pooled sums, so it is fixed.  An utterance
shorter than the reference minimum (``mcd.min_frames(config)[1]``) is skipped and counted.  The kept utterances of
every speaker are packed by length into ``padded_batches``' batches of at most PADDED_BATCH_MAX rows at
``padded_extent``; each batch gives its per-utterance sums and frame counts (``AE.get_speaker_sums``), which land in
their rows of one table, and one ``AE.speaker_codes_from_sums`` call pools every speaker's rows and runs the dense
stack.  A speaker's code is bit for bit what ``get_speaker_embeddings(groups=)`` gives for the same utterances in the
same order in one batch, whatever the packing.

A bank records a fingerprint of the speaker encoder that made it (sha256 over its state_dict entries: names, shapes and
float32 bytes in key order, then its config).  A code only means something to that encoder, so ``load`` refuses a bank
whose fingerprint does not match the model.

A bank whose codes were fitted to the model (``fit.fit_bank``) also carries a ``fitted`` record: the run's steps and
settings and ``model_fingerprint``, a sha256 of the content encoder and the decoder the codes were fitted through.
``load`` refuses such a bank against a model whose record does not match; a bank without the record loads as before.

A bank built with pitch profiles (``build_pitch_profiles``, speaker_bank.py -f0) carries a ``pitch`` record: per
speaker the ``f0.profile`` (log2 mean and std, voiced and total frames) of the voiced log2 F0 of that speaker's pooled
utterances, each copy-synthesised from its denormalised mel by the project's Griffin-Lim vocoder (untrimmed) and
tracked by ``f0.track_chunks``, as ``evaluate_f0`` makes its speaker profiles; and the tracker and Griffin-Lim settings
used.  Profiles describe recordings, not codes, so fitting keeps the record.  ``pitch_profile`` and
``morph_pitch_profile`` give the target profile of a spec or a morph, which ``f0.mv_shifts`` moves conversions toward.
"""
from __future__ import annotations

import hashlib
import json
import math
from typing import Callable, Dict, List, Mapping, Optional, Sequence

import numpy as np
import torch

from .evaluate import speaker_of as _speaker_of
from .inference import padded_batch, padded_batches
from .mcd import min_frames
from .utils import eval_mode

FORMAT = "avc-speaker-bank-1"


def fingerprint(model) -> str:
    """sha256 (hex) of the speaker encoder of `model` (an AE): every state_dict entry of model.speaker_encoder in key
    order (name, shape, float32 bytes), then its config dict as sorted JSON."""
    h = hashlib.sha256()
    for name, t in model.speaker_encoder.state_dict().items():
        h.update(name.encode())
        h.update(json.dumps(list(t.shape)).encode())
        h.update(t.detach().to(device="cpu", dtype=torch.float32).contiguous().numpy().tobytes())
    h.update(json.dumps(model.config["SpeakerEncoder"], sort_keys=True).encode())
    return h.hexdigest()


def parse_spec(spec: str) -> List[tuple]:
    """[(speaker, weight)] of a target spec: ``"p225"`` (weight 1) or ``"p225:0.7,p226:0.3"`` (a missing weight is 1).
    ValueError for an empty or duplicate name, a weight that is not a finite number >= 0, or weights summing to 0."""
    if not isinstance(spec, str) or not spec.strip():
        raise ValueError(f"speaker spec {spec!r}: expected 'NAME' or 'NAME:WEIGHT,NAME:WEIGHT,...'")
    out, seen = [], set()
    for part in spec.split(","):
        name, sep, w = part.strip().partition(":")
        name = name.strip()
        if not name:
            raise ValueError(f"speaker spec {spec!r}: empty speaker name")
        if name in seen:
            raise ValueError(f"speaker spec {spec!r}: {name} is named twice")
        seen.add(name)
        try:
            weight = float(w) if sep else 1.0
        except ValueError:
            raise ValueError(f"speaker spec {spec!r}: weight {w!r} of {name} is not a number") from None
        if not math.isfinite(weight) or weight < 0:
            raise ValueError(f"speaker spec {spec!r}: weight {w!r} of {name} must be a finite number >= 0")
        out.append((name, weight))
    if sum(w for _, w in out) <= 0:
        raise ValueError(f"speaker spec {spec!r}: the weights sum to 0")
    return out


def parse_keyframe(text: str) -> tuple:
    """(spec, seconds) of a morph keyframe ``SPEC@SECONDS``: SPEC in parse_spec's syntax, SECONDS a finite number >= 0.
    ValueError for a missing @, a malformed or negative time, or a bad SPEC."""
    spec, sep, sec = str(text).rpartition("@")
    if not sep:
        raise ValueError(f"keyframe {text!r}: expected SPEC@SECONDS, e.g. p225@0 or p225:0.5,p226:0.5@12")
    parse_spec(spec)
    try:
        t = float(sec)
    except ValueError:
        raise ValueError(f"keyframe {text!r}: time {sec!r} is not a number") from None
    if not math.isfinite(t) or t < 0:
        raise ValueError(f"keyframe {text!r}: time {sec!r} must be a finite number of seconds >= 0")
    return spec, t


def morph_weights(keyframes: Sequence[tuple], n_frames: int, frames_per_second: float):
    """(names, weights float32 [K, n_frames]) of a morph given as keyframes [(SPEC, seconds), ...]: names are the K
    distinct speakers in order of first mention.  A keyframe's weight vector is its spec's weights over the names,
    divided by their sum (the mix SpeakerBank.code makes of it).  Frame t lies at t / frames_per_second seconds; between
    consecutive keyframes the vectors are interpolated linearly, the first keyframe's is held before it and the last
    one's after it, and at two keyframes of the same time the later one takes over there (a hard cut).  Computed in
    float64, rounded once.  ValueError for an empty list, times that are negative or decrease, or a bad spec."""
    if not keyframes:
        raise ValueError("morph: no keyframes")
    if int(n_frames) < 1 or not frames_per_second > 0:
        raise ValueError("morph: n_frames must be >= 1 and frames_per_second > 0")
    names: List[str] = []
    vecs, times = [], []
    for spec, t in keyframes:
        t = float(t)
        if not math.isfinite(t) or t < 0:
            raise ValueError(f"morph: keyframe time {t} must be a finite number of seconds >= 0")
        if times and t < times[-1]:
            raise ValueError(f"morph: keyframe times must not decrease ({spec}@{t} follows a keyframe at {times[-1]})")
        parts = parse_spec(spec)
        for n, _ in parts:
            if n not in names:
                names.append(n)
        vecs.append(parts)
        times.append(t)
    V = np.zeros((len(vecs), len(names)), dtype=np.float64)
    for i, parts in enumerate(vecs):
        total = sum(w for _, w in parts)
        for n, w in parts:
            V[i, names.index(n)] = w / total
    ts = np.arange(int(n_frames), dtype=np.float64) / float(frames_per_second)
    return names, interpolate_keyframes(times, V, ts).T.astype(np.float32)


def interpolate_keyframes(times, vectors, at) -> np.ndarray:
    """float64 [len(at), K]: the keyframe vectors (float64 [n_keyframes, K] at non-decreasing times) at the times `at`,
    interpolated linearly between consecutive keyframes, the first one held before it and the last one after it; at
    two keyframes of the same time the later one takes over there (a hard cut).  The one statement of that rule, shared
    by morph_weights (times in seconds) and streaming.TargetSchedule (times in frames)."""
    V = np.asarray(vectors, dtype=np.float64)
    ts = np.asarray(at, dtype=np.float64)
    tk = np.asarray(times, dtype=np.float64)
    i = np.searchsorted(tk, ts, side="right") - 1                 # last keyframe at or before the frame
    out = np.empty((len(ts), V.shape[1]), dtype=np.float64)
    before, after = i < 0, i >= len(tk) - 1
    out[before] = V[0]
    out[after & ~before] = V[-1]
    mid = ~before & ~after
    if mid.any():
        j = i[mid]
        a = ((ts[mid] - tk[j]) / (tk[j + 1] - tk[j]))[:, None]
        out[mid] = (1 - a) * V[j] + a * V[j + 1]
    return out


def morph_table(bank: "SpeakerBank", keyframes: Sequence[tuple], n_frames: int, frames_per_second: float):
    """(codes float32 [K, c_out] on the bank's device, weights float32 [K, n_frames] on the host) of a morph through
    `bank` (morph_weights; Inferencer.inference_morph takes them).  ValueError for a speaker not in the bank."""
    names, w = morph_weights(keyframes, n_frames, frames_per_second)
    rows = [bank.index(n) for n in names]
    return bank.codes[rows].contiguous(), torch.from_numpy(w)


PITCH_LISTS = ("log2_mean", "log2_std", "voiced", "frames")


def check_pitch(pitch, n_speakers: int) -> dict:
    """A copy of a bank's pitch record after checking it: the PITCH_LISTS of n_speakers entries each, voiced and frames
    integers with 0 <= voiced <= frames, mean and std finite (std >= 0) exactly where voiced > 0 and None elsewhere,
    and the "tracker" and "griffin_lim" settings dicts.  ValueError naming what is wrong."""
    if not isinstance(pitch, dict):
        raise ValueError("SpeakerBank: the pitch record must be a dict")
    for k in PITCH_LISTS:
        if not isinstance(pitch.get(k), (list, tuple)) or len(pitch[k]) != n_speakers:
            raise ValueError(f"SpeakerBank: pitch record: {k} must list the {n_speakers} speakers")
    for k in ("tracker", "griffin_lim"):
        if not isinstance(pitch.get(k), dict):
            raise ValueError(f"SpeakerBank: pitch record: {k} settings missing")
    for i, (m, sd, nv, nf) in enumerate(zip(*(pitch[k] for k in PITCH_LISTS))):
        if not all(isinstance(n, int) and not isinstance(n, bool) for n in (nv, nf)) or not 0 <= nv <= nf:
            raise ValueError(f"SpeakerBank: pitch record of speaker {i}: voiced {nv!r} / frames {nf!r} must be integers "
                             f"with 0 <= voiced <= frames")
        if nv == 0:
            if m is not None or sd is not None:
                raise ValueError(f"SpeakerBank: pitch record of speaker {i}: a mean and std without a voiced frame")
            continue
        if not all(isinstance(x, float) and math.isfinite(x) for x in (m, sd)) or sd < 0:
            raise ValueError(f"SpeakerBank: pitch record of speaker {i}: mean {m!r} and std {sd!r} must be finite "
                             f"floats, the std >= 0")
    out = dict(pitch)
    out.update({k: list(pitch[k]) for k in PITCH_LISTS}, tracker=dict(pitch["tracker"]),
               griffin_lim=dict(pitch["griffin_lim"]))
    return out


class SpeakerBank:
    """Per-speaker codes of one speaker encoder.

    speakers: names in sorted order; codes: float32 [S, c_out] (row s is speakers[s]'s); n_utts[s]: the utterances
    pooled into code s, which are utterances[s] (sorted ids); n_skipped: utterances too short to embed; fingerprint:
    the speaker encoder's (``fingerprint``); fitted: None, or the record of the fitting run that tuned the codes to a
    content encoder and decoder (``fit.fit_bank``; plain values only, with "model_fingerprint"); pitch: None, or the
    speakers' pitch profiles (``build_pitch_profiles``; checked by ``check_pitch``)."""

    def __init__(self, speakers: Sequence[str], codes: torch.Tensor, n_utts: Sequence[int],
                 utterances: Sequence[Sequence[str]], fingerprint: str, n_skipped: int = 0,
                 fitted: Optional[dict] = None, pitch: Optional[dict] = None):
        speakers = [str(s) for s in speakers]
        if len(set(speakers)) != len(speakers) or list(speakers) != sorted(speakers):
            raise ValueError("SpeakerBank: speakers must be unique and sorted")
        if codes.dtype != torch.float32 or codes.dim() != 2 or codes.shape[0] != len(speakers):
            raise ValueError(f"SpeakerBank: codes must be float32 [{len(speakers)}, c_out], got {codes.dtype} "
                             f"{tuple(codes.shape)}")
        if len(n_utts) != len(speakers) or len(utterances) != len(speakers) or any(
                int(n) != len(u) for n, u in zip(n_utts, utterances)):
            raise ValueError("SpeakerBank: n_utts and utterances must list every speaker's pooled utterances")
        self.speakers = speakers
        self.codes = codes
        self.n_utts = [int(n) for n in n_utts]
        self.utterances = [[str(u) for u in us] for us in utterances]
        self.fingerprint = str(fingerprint)
        self.n_skipped = int(n_skipped)
        if fitted is not None and not isinstance(fitted.get("model_fingerprint"), str):
            raise ValueError("SpeakerBank: a fitted record needs its model_fingerprint")
        self.fitted = None if fitted is None else dict(fitted)
        self.pitch = None if pitch is None else check_pitch(pitch, len(speakers))
        self._index = {s: i for i, s in enumerate(speakers)}

    def __len__(self):
        return len(self.speakers)

    def __contains__(self, name):
        return name in self._index

    def index(self, name: str) -> int:
        if name not in self._index:
            raise ValueError(f"speaker {name!r} is not in the bank ({len(self)} speakers)")
        return self._index[name]

    def utterance_ids(self) -> List[str]:
        """Every pooled utterance id, speaker by speaker."""
        return [u for us in self.utterances for u in us]

    def code(self, spec: str) -> torch.Tensor:
        """The float32 [c_out] code of a spec: ``"p225"`` gives p225's stored code bit for bit; ``"p225:0.7,p226:0.3"``
        gives sum_i w_i c_i / sum_i w_i, computed in float64 (terms added in spec order) and rounded once to float32.

        Mixing acts on the final code on purpose: the decoder reads the code only through its AdaIN affine layers, each
        affine in it, so a mix moves every AdaIN scale and shift along the straight line between the speakers' values.
        ValueError for an unknown or duplicate name, a negative weight or weights summing to 0."""
        parts = parse_spec(spec)
        rows = [self.index(n) for n, _ in parts]
        c = self.codes.detach().to(device="cpu", dtype=torch.float64)
        acc, wsum = torch.zeros(c.shape[1], dtype=torch.float64), 0.0
        for r, (_, w) in zip(rows, parts):
            acc = acc + w * c[r]
            wsum += w
        return (acc / wsum).to(dtype=torch.float32, device=self.codes.device)

    def with_pitch(self, pitch: Optional[dict]) -> "SpeakerBank":
        """This bank with the pitch record `pitch` (the codes shared)."""
        return SpeakerBank(self.speakers, self.codes, self.n_utts, self.utterances, self.fingerprint, self.n_skipped,
                           fitted=self.fitted, pitch=pitch)

    def _pitch_rows(self, names):
        if self.pitch is None:
            raise ValueError("the bank has no pitch profiles: rebuild it with speaker_bank.py -f0")
        rows = [self.index(n) for n in names]
        return [(self.pitch["log2_mean"][r], self.pitch["log2_std"][r]) for r in rows]

    def pitch_profile(self, spec: str):
        """(log2 mean, log2 std) of the target a spec names, or None (unmatched) when a speaker of positive weight has
        no voiced frame: p225's own profile, or for ``"p225:0.7,p226:0.3"`` mu = sum_i w_i mu_i / sum_i w_i and the
        same for the std, in float64 with terms in spec order and zero weights skipped (``code``'s straight line).
        ValueError for a bank without a pitch record or a bad spec."""
        parts = parse_spec(spec)
        profs = self._pitch_rows([n for n, _ in parts])
        mu = sd = wsum = 0.0
        for (_, w), (m, s) in zip(parts, profs):
            if w == 0:
                continue
            if m is None:
                return None
            mu, sd, wsum = mu + w * m, sd + w * s, wsum + w
        return mu / wsum, sd / wsum

    def morph_pitch_profile(self, keyframes: Sequence[tuple], n_frames: int, frames_per_second: float):
        """(log2 mean, log2 std) float64 [n_frames] of a morph's target per frame, or None (unmatched) when a speaker
        of positive weight on some frame has no voiced frame: with w_k(f) = ``morph_weights`` (the float32 table the
        decoder gets), mu(f) = sum_k w_k(f) mu_k / sum_k w_k(f) in float64, terms in order of first mention, and the same
        for the std.  A morph held on one speaker gives that speaker's profile on every frame exactly."""
        names, w = morph_weights(keyframes, n_frames, frames_per_second)
        profs = self._pitch_rows(names)
        w = w.astype(np.float64)
        mu, sd, wsum = np.zeros(w.shape[1]), np.zeros(w.shape[1]), np.zeros(w.shape[1])
        for wk, (m, s) in zip(w, profs):
            if not wk.any():
                continue
            if m is None:
                return None
            mu, sd, wsum = mu + wk * m, sd + wk * s, wsum + wk
        return mu / wsum, sd / wsum

    def save(self, path: str):
        """torch.save of plain tensors, lists and strings (loadable with weights_only=True).  The "fitted" and "pitch"
        entries are written only for a fitted bank and one with pitch profiles."""
        d = {"format": FORMAT, "speakers": list(self.speakers), "codes": self.codes.detach().cpu().contiguous(),
             "n_utts": list(self.n_utts), "utterances": [list(u) for u in self.utterances],
             "fingerprint": self.fingerprint, "n_skipped": self.n_skipped}
        if self.fitted is not None:
            d["fitted"] = dict(self.fitted)
        if self.pitch is not None:
            d["pitch"] = self.pitch
        torch.save(d, path)

    @classmethod
    def load(cls, path: str, model) -> "SpeakerBank":
        """The bank saved at `path`, its codes on `model`'s device.  ValueError when it was not made by `model`'s speaker
        encoder (fingerprint mismatch), when its codes were fitted to another content encoder or decoder (the fitted
        record's model_fingerprint), or when it is not a bank file."""
        d = torch.load(path, map_location="cpu", weights_only=True)
        if not isinstance(d, dict) or d.get("format") != FORMAT:
            raise ValueError(f"{path}: not a speaker bank ({FORMAT})")
        fp = fingerprint(model)
        if d["fingerprint"] != fp:
            raise ValueError(f"{path}: the bank was made by a different speaker encoder (fingerprint "
                             f"{d['fingerprint'][:12]}..., the model's {fp[:12]}...); its codes mean nothing to this model")
        fitted = d.get("fitted")
        if fitted is not None:
            from .fit import model_fingerprint
            mf = model_fingerprint(model)
            if fitted.get("model_fingerprint") != mf:
                raise ValueError(f"{path}: the codes were fitted to a different content encoder or decoder (fingerprint "
                                 f"{str(fitted.get('model_fingerprint'))[:12]}..., the model's {mf[:12]}...); they are "
                                 f"tuned to that model")
        dev = next(model.parameters()).device
        pitch = d.get("pitch")
        if pitch is not None:
            try:
                pitch = check_pitch(pitch, len(d["speakers"]))
            except ValueError as e:
                raise ValueError(f"{path}: {e}") from None
        return cls(d["speakers"], d["codes"].to(dev), d["n_utts"], d["utterances"], d["fingerprint"], d["n_skipped"],
                   fitted=fitted, pitch=pitch)


def bank_order(ids: Sequence[str], lengths: Mapping[str, int], min_len: int,
               speaker_of: Callable[[str], str] = _speaker_of):
    """(speakers, utterances per speaker, n_skipped): speakers sorted by name, each speaker's utterances of at least
    min_len frames in sorted id order (the summation order), and the count of shorter ones."""
    by: Dict[str, List[str]] = {}
    skipped = 0
    for u in sorted(ids):
        if lengths[u] < min_len:
            skipped += 1
            continue
        by.setdefault(speaker_of(u), []).append(u)
    speakers = sorted(by)
    return speakers, [by[s] for s in speakers], skipped


def build_bank(model, mels: Mapping[str, object], speaker_of: Callable[[str], str] = _speaker_of,
               device=None) -> SpeakerBank:
    """A SpeakerBank of `model` (an AE, frame_size 1) from mels: utterance id -> attr-normalised [T, n_mels] mel (a
    tensor or an array).  The module docstring gives the order, the packing and the pooling.  ValueError when no
    utterance is long enough."""
    cfg = model.config
    if int(cfg["data_loader"]["frame_size"]) != 1:
        raise ValueError(f"speaker banks support data_loader.frame_size 1 only (got {cfg['data_loader']['frame_size']})")
    dev = torch.device(device) if device is not None else next(model.parameters()).device
    lengths = {u: int(m.shape[0]) for u, m in mels.items()}
    speakers, utts, skipped = bank_order(list(mels), lengths, min_frames(cfg)[1], speaker_of)
    flat = [u for us in utts for u in us]
    if not flat:
        raise ValueError(f"build_bank: no utterance of at least {min_frames(cfg)[1]} frames ({skipped} skipped)")
    c_h = cfg["SpeakerEncoder"]["c_h"]
    sums = torch.empty(len(flat), c_h, device=dev)
    counts = torch.empty(len(flat), dtype=torch.int32, device=dev)
    lens = [lengths[u] for u in flat]
    frames = [(m if isinstance(m, torch.Tensor) else torch.from_numpy(np.ascontiguousarray(m, np.float32))).t()
              for m in (mels[u] for u in flat)]
    with eval_mode(model, dev):
        for idx, T, _, _ in padded_batches(lens, lens):
            x, lx = padded_batch(frames, idx, T, dev)
            s, n = model.get_speaker_sums(x, lengths=lx)
            rows = torch.tensor(idx, device=dev)
            sums.index_copy_(0, rows, s)
            counts.index_copy_(0, rows, n)
        offsets = torch.tensor([0] + [len(us) for us in utts], dtype=torch.int64).cumsum(0)
        codes = model.speaker_codes_from_sums(sums, counts, groups=offsets.to(dev))
    return SpeakerBank(speakers, codes, [len(us) for us in utts], utts, fingerprint(model), skipped)


def build_pitch_profiles(bank: SpeakerBank, mels: Mapping[str, object], attr, hp=None, params=None,
                         frame_budget: int = 32768, device=None, timings: dict = None) -> dict:
    """The pitch record of `bank` (the module docstring) from mels: utterance id -> attr-normalised [T, n_mels] mel
    (a tensor or an array) of at least every pooled utterance.  Each pooled utterance, in the bank's order, is
    denormalised with attr (mel * std + mean), copy-synthesised by ``f0.synthesize`` at hp's Griffin-Lim settings
    (default AudioParams(); unshifted, n_mels the mels') and tracked by ``f0.track_chunks`` with params (default
    F0Params()), in chunks of at most frame_budget frames: only one chunk's mels and signals are on the device at a
    time, and its tracks go to the host before the next (an utterance's bits do not depend on its chunk).  timings (a dict) receives the wall seconds of synthesis, tracking and host work, each ended by a
    device synchronise."""
    import time
    from dataclasses import replace
    from .f0 import F0Params, profile, synthesize, track_chunks
    from .vocoder import AudioParams, Vocoder
    hp = AudioParams() if hp is None else hp
    params = F0Params() if params is None else params
    dev = torch.device(device) if device is not None else bank.codes.device
    flat = bank.utterance_ids()
    missing = [u for u in flat if u not in mels]
    if missing:
        raise ValueError(f"build_pitch_profiles: {len(missing)} pooled utterances have no mel (e.g. {missing[0]})")
    n_mels = int(mels[flat[0]].shape[1])
    hp = replace(hp, n_mels=n_mels, pitch_shift=0.0)
    mean = torch.as_tensor(np.asarray(attr["mean"], np.float32).reshape(-1)).to(dev)
    std = torch.as_tensor(np.asarray(attr["std"], np.float32).reshape(-1)).to(dev)
    if mean.numel() != n_mels or std.numel() != n_mels:
        raise ValueError(f"build_pitch_profiles: attr mean / std have {mean.numel()} / {std.numel()} entries, the mels "
                         f"{n_mels}")
    clock = {"synthesis": 0.0, "tracking": 0.0, "host": 0.0}
    t0 = time.perf_counter()

    def lap(k):
        nonlocal t0
        torch.cuda.synchronize(dev)
        t1 = time.perf_counter()
        clock[k] += t1 - t0
        t0 = t1
    vocoder = Vocoder(hp=hp, device=dev)
    tracks, k = [], 0
    while k < len(flat):      # one chunk of at most frame_budget frames on the device at a time (one longer mel alone)
        j, frames = k + 1, int(mels[flat[k]].shape[0])
        while j < len(flat) and frames + int(mels[flat[j]].shape[0]) <= frame_budget:
            frames += int(mels[flat[j]].shape[0])
            j += 1
        chunk = [(m if isinstance(m, torch.Tensor) else torch.from_numpy(np.ascontiguousarray(m, np.float32))).to(dev)
                 * std + mean for m in (mels[u] for u in flat[k:j])]
        signals = synthesize(vocoder, chunk, hp, frame_budget)
        lap("synthesis")
        tracks.extend(track_chunks(signals, hp.sr, hp.hop_length, params))
        del chunk, signals
        lap("tracking")
        k = j
    rec = {k: [] for k in PITCH_LISTS}
    k = 0
    for us in bank.utterances:
        ts = tracks[k:k + len(us)]
        k += len(us)
        m, sd, nv = profile([np.log2(f[v]) for f, v in ts])
        for key, val in zip(PITCH_LISTS, (m, sd, int(nv), sum(len(v) for _, v in ts))):
            rec[key].append(val)
    rec["tracker"] = params.settings(hp.sr, hp.hop_length)
    rec["griffin_lim"] = {"n_iter": int(hp.n_iter), "momentum": float(hp.momentum), "init": hp.gl_init}
    lap("host")
    if timings is not None:
        timings.update(clock)
    return check_pitch(rec, len(bank))


def check_disjoint(bank: SpeakerBank, utterance_ids) -> None:
    """ValueError naming the count when any pooled utterance of `bank` is among `utterance_ids` (an evaluation against a
    bank built from the evaluated utterances would leak them into the enrolment)."""
    ids = set(utterance_ids)
    n = sum(u in ids for u in bank.utterance_ids())
    if n:
        raise ValueError(f"the bank pooled {n} of the evaluated utterances; build it from a disjoint set (e.g. train)")
