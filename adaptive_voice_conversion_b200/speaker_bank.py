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
    tk = np.asarray(times, dtype=np.float64)
    i = np.searchsorted(tk, ts, side="right") - 1                 # last keyframe at or before the frame
    out = np.empty((int(n_frames), len(names)), dtype=np.float64)
    before, after = i < 0, i >= len(tk) - 1
    out[before] = V[0]
    out[after & ~before] = V[-1]
    mid = ~before & ~after
    if mid.any():
        j = i[mid]
        a = ((ts[mid] - tk[j]) / (tk[j + 1] - tk[j]))[:, None]
        out[mid] = (1 - a) * V[j] + a * V[j + 1]
    return names, out.T.astype(np.float32)


def morph_table(bank: "SpeakerBank", keyframes: Sequence[tuple], n_frames: int, frames_per_second: float):
    """(codes float32 [K, c_out] on the bank's device, weights float32 [K, n_frames] on the host) of a morph through
    `bank` (morph_weights; Inferencer.inference_morph takes them).  ValueError for a speaker not in the bank."""
    names, w = morph_weights(keyframes, n_frames, frames_per_second)
    rows = [bank.index(n) for n in names]
    return bank.codes[rows].contiguous(), torch.from_numpy(w)


class SpeakerBank:
    """Per-speaker codes of one speaker encoder.

    speakers: names in sorted order; codes: float32 [S, c_out] (row s is speakers[s]'s); n_utts[s]: the utterances
    pooled into code s, which are utterances[s] (sorted ids); n_skipped: utterances too short to embed; fingerprint:
    the speaker encoder's (``fingerprint``); fitted: None, or the record of the fitting run that tuned the codes to a
    content encoder and decoder (``fit.fit_bank``; plain values only, with "model_fingerprint")."""

    def __init__(self, speakers: Sequence[str], codes: torch.Tensor, n_utts: Sequence[int],
                 utterances: Sequence[Sequence[str]], fingerprint: str, n_skipped: int = 0,
                 fitted: Optional[dict] = None):
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

    def save(self, path: str):
        """torch.save of plain tensors, lists and strings (loadable with weights_only=True).  The "fitted" entry is
        written only for a fitted bank."""
        d = {"format": FORMAT, "speakers": list(self.speakers), "codes": self.codes.detach().cpu().contiguous(),
             "n_utts": list(self.n_utts), "utterances": [list(u) for u in self.utterances],
             "fingerprint": self.fingerprint, "n_skipped": self.n_skipped}
        if self.fitted is not None:
            d["fitted"] = dict(self.fitted)
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
        return cls(d["speakers"], d["codes"].to(dev), d["n_utts"], d["utterances"], d["fingerprint"], d["n_skipped"],
                   fitted=fitted)


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


def check_disjoint(bank: SpeakerBank, utterance_ids) -> None:
    """ValueError naming the count when any pooled utterance of `bank` is among `utterance_ids` (an evaluation against a
    bank built from the evaluated utterances would leak them into the enrolment)."""
    ids = set(utterance_ids)
    n = sum(u in ids for u in bank.utterance_ids())
    if n:
        raise ValueError(f"the bank pooled {n} of the evaluated utterances; build it from a disjoint set (e.g. train)")
