"""Mel-cepstral distortion after dynamic time warping (MCD-DTW) of one-shot conversions: speaker A's utterance
converted with a different utterance of speaker B as the reference, against B's own recording of the same sentence.

Triplets of a set (whole utterances of ``<set>.pkl``, attr-normalised; ``frame_size`` 1 only):
  * texts come from the transcripts (``read_transcripts``), normalised by ``normalize_text``;
  * a group is a text spoken by at least two distinct speakers (``evaluate.speaker_of``); groups in sorted text order;
    each speaker of a group contributes its first utterance id in sorted order;
  * for each ordered pair (A, B) of distinct speakers of a group, sorted: source = A's utterance, ground truth = B's,
    reference = ``rng.choice`` over B's utterances of the set (sorted ids) whose text is not the group's (utterances
    without a transcript qualify), with ``rng = random.Random(seed)`` drawn in this order; a pair for which B has no
    such utterance is skipped;
  * a triplet whose source or reference is shorter than ``AE.inference`` accepts (``min_frames``) is then dropped and
    counted in ``n_short``; the draws above do not depend on the lengths;
  * with ``max_pairs > 0`` and more triplets than that, ``sorted(rng.sample(range(n), max_pairs))`` of them are kept.

For each triplet ``dec = AE.inference(source, reference)`` in eval mode, cropped to the source's T frames (the bits
``Inferencer.inference_ragged`` gives).  The cepstrum of a frame x is c_k = sqrt(2/N) sum_m l_m cos(pi k (2m+1) / 2N),
k = 1..dims, of the natural-log amplitude l = (a max_db - max_db + ref_db) ln(10)/20 of a = clip(x std + mean, 0, 1)
(what the vocoder synthesises from): an MFCC-style cepstrum of the model's log-mel, without the energy c_0.  Its values
compare between checkpoints and configs of this project, not with WORLD/SPTK mel-cepstrum MCD figures.

    mcd = (10 sqrt(2) / ln 10) S / L

with (S, L) the accumulated distance and the length of the DTW path (``avc_dtw``) between the converted output and the
ground truth; ``mcd_source`` is the same measure between the unconverted source and the ground truth.  A set reports
the means over its triplets (added in triplet order in float64), ``n``, ``n_short``, ``dims`` and the means per target
speaker.  Cepstra and DTW run on the GPU (csrc/mcd.cu); both kernels give a row or a pair the same bits in any batch.

Few-shot (``n_refs`` K > 1): each triplet keeps its reference and gets K - 1 more (``fewshot_triplets``, drawn from
``random.Random(seed + 1)`` after the ``max_pairs`` subsample); ``dec = AE.inference_from_embeddings(source, code)``
with the set's pooled code, in the same batches as K = 1.
"""
from __future__ import annotations

import ctypes as C
import math
import os
import random
import re
from typing import Dict, List, Mapping, Sequence, Tuple

import numpy as np
import torch

from . import _lib as L
from .engine import conv_geometry
from .evaluate import speaker_of
from .utils import _stream, eval_mode, exact_buckets, upload_mels
from .vocoder import AudioParams

MCD_SCALE = 10.0 * math.sqrt(2.0) / math.log(10.0)
_NON_TEXT = re.compile(r"[^a-z0-9']")


# ------------------------------------------------------------------ transcripts and triplets
def normalize_text(text: str) -> str:
    """Lowercase; every character outside [a-z0-9'] becomes a space; runs of whitespace collapse; ends stripped."""
    return " ".join(_NON_TEXT.sub(" ", text.lower()).split())


def read_transcripts(root: str, utt_ids) -> Dict[str, str]:
    """{utterance key: normalised text} for the keys of `utt_ids` (``<id>.wav``) with a transcript under `root`,
    searched recursively: ``<id>.txt`` (VCTK) or ``<id>.normalized.txt`` (LibriTTS).  Other files are ignored; empty
    texts are dropped.  Two files with different texts for one key raise ValueError naming both."""
    if not os.path.isdir(root):
        raise ValueError(f"transcript directory {root} does not exist")
    wanted = set(utt_ids)
    found: Dict[str, Tuple[str, str]] = {}
    for dirpath, dirnames, files in os.walk(root):
        dirnames.sort()
        for name in sorted(files):
            if name.endswith(".normalized.txt"):
                key = name[: -len(".normalized.txt")] + ".wav"
            elif name.endswith(".txt"):
                key = name[: -len(".txt")] + ".wav"
            else:
                continue
            if key not in wanted:
                continue
            path = os.path.join(dirpath, name)
            with open(path, encoding="utf-8", errors="replace") as f:
                text = normalize_text(f.read())
            if key in found and found[key][0] != text:
                raise ValueError(f"different transcripts for {key}: {found[key][1]} and {path}")
            found.setdefault(key, (text, path))
    return {k: t for k, (t, _) in found.items() if t}


def min_frames(config: dict) -> Tuple[int, int]:
    """(source, reference) frames AE.inference accepts at least: every reflect-padded conv on the path must see an
    input longer than its left pad (conv_geometry).  The shipped config gives (17, 9)."""
    def encoder_ok(c, T):
        if any(T <= k // 2 for k in range(c["bank_scale"], c["bank_size"] + 1, c["bank_scale"])):
            return None
        K = c["kernel_size"]
        for s in c["subsample"][: c["n_conv_blocks"]]:
            if T <= K // 2:
                return None
            T = conv_geometry(K, s, T)[2]
        return T

    def source_ok(T):
        T = encoder_ok(config["ContentEncoder"], T)
        if T is None:
            return False
        de = config["Decoder"]
        for up in de["upsample"][: de["n_conv_blocks"]]:
            if T <= de["kernel_size"] // 2:
                return False
            T *= up
        return True

    def first(ok):
        T = 1
        while not ok(T):
            T += 1
        return T
    return first(source_ok), first(lambda T: encoder_ok(config["SpeakerEncoder"], T) is not None)


def parallel_triplets(utts: Sequence[str], texts: Mapping[str, str], lengths: Mapping[str, int], seed: int = 0,
                      max_pairs: int = 0, min_src: int = 1, min_ref: int = 1):
    """([(source, reference, ground truth)], n_short) of the utterance keys `utts` of a set, as the module docstring
    defines; lengths[u] = frames of u."""
    utts = sorted(utts)
    rng = random.Random(seed)
    by_text: Dict[str, Dict[str, str]] = {}
    by_speaker: Dict[str, List[str]] = {}
    for u in utts:
        by_speaker.setdefault(speaker_of(u), []).append(u)
        t = texts.get(u)
        if t:
            by_text.setdefault(t, {}).setdefault(speaker_of(u), u)     # sorted ids: the first one stays
    out, n_short = [], 0
    for text in sorted(by_text):
        spk = by_text[text]
        if len(spk) < 2:
            continue
        for a in sorted(spk):
            for b in sorted(spk):
                if a == b:
                    continue
                refs = [u for u in by_speaker[b] if texts.get(u) != text]
                if not refs:
                    continue
                ref = rng.choice(refs)
                if lengths[spk[a]] < min_src or lengths[ref] < min_ref:
                    n_short += 1
                    continue
                out.append((spk[a], ref, spk[b]))
    if max_pairs > 0 and len(out) > max_pairs:
        out = [out[i] for i in sorted(rng.sample(range(len(out)), max_pairs))]
    return out, n_short


def fewshot_triplets(trip, utts: Sequence[str], texts: Mapping[str, str], lengths: Mapping[str, int], n_refs: int,
                     seed: int = 0, min_ref: int = 1):
    """([(source, [reference, extra, ...], ground truth)], n_few): parallel_triplets' triplets with n_refs - 1 extra
    references each.  rng2 = random.Random(seed + 1) draws, in triplet order, rng2.sample over the target speaker's
    other utterances (sorted) whose text is not the group's and that have at least min_ref frames; a triplet whose
    speaker has fewer than n_refs such utterances (the reference included) is dropped and counted in n_few."""
    by_speaker: Dict[str, List[str]] = {}
    for u in sorted(utts):
        by_speaker.setdefault(speaker_of(u), []).append(u)
    rng2 = random.Random(seed + 1)
    out, n_few = [], 0
    for s, r, g in trip:
        text = texts.get(g)
        others = [u for u in by_speaker[speaker_of(g)] if u != r and texts.get(u) != text and lengths[u] >= min_ref]
        if len(others) + 1 < n_refs:
            n_few += 1
            continue
        out.append((s, [r] + rng2.sample(others, n_refs - 1), g))
    return out, n_few


# ------------------------------------------------------------------ the two kernels
def dct_matrix(n_mels: int, dims: int) -> np.ndarray:
    """[n_mels][dims] float64: sqrt(2/N) cos(pi k (2m+1) / 2N) at [m][k-1], k = 1..dims (orthonormal DCT-II, no c_0)."""
    m = np.arange(n_mels, dtype=np.float64)[:, None]
    k = np.arange(1, dims + 1, dtype=np.float64)[None, :]
    return np.sqrt(2.0 / n_mels) * np.cos(np.pi * k * (2.0 * m + 1.0) / (2.0 * n_mels))


def _check_dims(dims: int):
    if not 1 <= int(dims) <= L.CEPSTRUM_MAX_DIMS:
        raise ValueError(f"cepstrum dims must be in [1, {L.CEPSTRUM_MAX_DIMS}] (got {dims})")


def mel_cepstrum(mels, attr, hp: AudioParams = AudioParams(), dims: int = 24):
    """Cepstra [T_i, dims] float32 (device) of attr-normalised mels [T_i, n_mels] (device tensors), one launch."""
    _check_dims(dims)
    if not mels:
        raise ValueError("mel_cepstrum: empty batch")
    n_mels = int(mels[0].shape[-1])
    for i, m in enumerate(mels):
        if m.dim() != 2 or m.shape[1] != n_mels or m.shape[0] < 1 or not m.is_cuda:
            raise ValueError(f"mel_cepstrum: mel {i} has shape {tuple(m.shape)} on {m.device}; expected [T >= 1, "
                             f"{n_mels}] on a CUDA device")
    dev = mels[0].device
    x = torch.cat([m.float() for m in mels]).contiguous()
    if x.shape[0] >= 2 ** 31:
        raise ValueError("mel_cepstrum: 2^31 frames at most per call")
    mean = torch.as_tensor(np.asarray(attr["mean"], np.float32).reshape(-1)).to(dev)
    std = torch.as_tensor(np.asarray(attr["std"], np.float32).reshape(-1)).to(dev)
    if mean.numel() != n_mels or std.numel() != n_mels:
        raise ValueError(f"mel_cepstrum: attr mean / std have {mean.numel()} / {std.numel()} entries, the mels {n_mels}")
    dct = torch.from_numpy(dct_matrix(n_mels, dims)).to(dev)
    out = torch.empty(x.shape[0], dims, device=dev)
    d = L.CepstrumDesc(rows=x.shape[0], n_mels=n_mels, dims=dims, max_db=hp.max_db, ref_db=hp.ref_db, in_=x.data_ptr(),
                       mean=mean.data_ptr(), std=std.data_ptr(), dct=dct.data_ptr(), out=out.data_ptr())
    L.check(L.load().avc_mel_cepstrum(C.byref(d), _stream(dev)), "avc_mel_cepstrum")
    return list(torch.split(out, [int(m.shape[0]) for m in mels]))


_PAIR = np.dtype([("x_off", "<i8"), ("y_off", "<i8"), ("tx", "<i4"), ("ty", "<i4")])
assert _PAIR.itemsize == C.sizeof(L.DtwPair)


def dtw(xs, ys):
    """(S, L) float64 [n, 2] (device) of the DTW of every pair (xs[i], ys[i]) of cepstra [T, dims], one launch."""
    if len(xs) != len(ys) or not xs:
        raise ValueError(f"dtw: need two equally long non-empty lists (got {len(xs)} and {len(ys)})")
    dims = int(xs[0].shape[-1])
    _check_dims(dims)
    for i, t in enumerate(list(xs) + list(ys)):
        if t.dim() != 2 or t.shape[1] != dims or t.shape[0] < 1 or t.dtype != torch.float32 or not t.is_cuda:
            raise ValueError(f"dtw: sequence {i % len(xs)} is {t.dtype} {tuple(t.shape)} on {t.device}; expected "
                             f"float32 [T >= 1, {dims}] on a CUDA device")
    tx = np.array([int(t.shape[0]) for t in xs], np.int64)
    ty = np.array([int(t.shape[0]) for t in ys], np.int64)
    max_short = int(np.minimum(tx, ty).max())
    if max_short > L.DTW_MAX_SHORT:
        raise ValueError(f"dtw: a pair's shorter side has {max_short} frames; at most {L.DTW_MAX_SHORT} are supported")
    dev = xs[0].device
    tab = np.zeros(len(xs), _PAIR)
    tab["x_off"], tab["y_off"] = np.cumsum(tx) - tx, np.cumsum(ty) - ty
    tab["tx"], tab["ty"] = tx, ty
    pairs = torch.from_numpy(tab.view(np.uint8)).to(dev)
    x, y = torch.cat(list(xs)).contiguous(), torch.cat(list(ys)).contiguous()
    out = torch.empty(len(xs), 2, dtype=torch.float64, device=dev)
    d = L.DtwDesc(n_pairs=len(xs), dims=dims, max_short=max_short, pairs=pairs.data_ptr(), x=x.data_ptr(),
                  y=y.data_ptr(), out=out.data_ptr())
    L.check(L.load().avc_dtw(C.byref(d), _stream(dev)), "avc_dtw")
    return out


# ------------------------------------------------------------------ conversion and the measure
def converted(model, sources, refs, batch_max: int = 64, codes=None):
    """Yields (indices, [dec cropped to T_i, as [T_i, n_mels]]) per batch of the pairs (sources[i], refs[i]) of
    attr-normalised device mels [T, n_mels]: pairs bucketed by their exact (T, T_ref), each bucket in eager
    AE.inference calls of at most batch_max pairs.  codes [P, c_out] (few-shot): the same batches through
    AE.inference_from_embeddings with pair i's speaker code codes[i] instead of refs[i]'s.  The model must be in eval
    mode."""
    with torch.no_grad():
        for (T, _), idx in exact_buckets([int(x.shape[0]) for x in sources], [int(c.shape[0]) for c in refs]):
            for f in range(0, len(idx), batch_max):
                part = idx[f:f + batch_max]
                xb = torch.stack([sources[i].t() for i in part]).contiguous()
                if codes is not None:
                    dec = model.inference_from_embeddings(xb, codes[torch.tensor(part, device=codes.device)])
                    yield part, [dec[j, :, :T].t() for j in range(len(part))]
                    continue
                cb = torch.stack([refs[i].t() for i in part]).contiguous()
                dec = model.inference(xb, cb)
                yield part, [dec[j, :, :T].t() for j in range(len(part))]


def _means(rows: np.ndarray) -> Dict[str, float]:
    """{mcd, mcd_source, n} of a float64 [n][2] array, each column added sequentially in row order."""
    return {"mcd": float(np.cumsum(rows[:, 0])[-1] / len(rows)), "mcd_source": float(np.cumsum(rows[:, 1])[-1] / len(rows)),
            "n": len(rows)}


def evaluate_mcd(model, data: Mapping[str, np.ndarray], attr, texts: Mapping[str, str], dims: int = 24,
                 max_pairs: int = 0, seed: int = 0, hp: AudioParams = AudioParams(), device=None,
                 per_triplet: bool = False, n_refs: int = 1, target_codes=None) -> dict:
    """MCD-DTW of `model` (an AE) on one set: data = {utterance key: attr-normalised [T, n_mels]} (the set's pickle),
    texts = read_transcripts(...) of its keys.  Returns {"n", "n_short", "dims", "speakers": {target speaker: {"mcd",
    "mcd_source", "n"}}} with "mcd" and "mcd_source" when n > 0; per_triplet adds "triplets": [[source, reference,
    target, mcd, mcd_source], ...].  Only the utterances the triplets use are uploaded.

    n_refs > 1 (few-shot): each triplet keeps its reference and gets n_refs - 1 more (fewshot_triplets); the source is
    converted with the set's pooled speaker code in the batches n_refs = 1 uses.  The result then also reports
    "n_refs" and "n_few", and a triplet row lists the references: [source, [reference, ...], target, ...].

    target_codes {speaker: float32 [c_out] code} (an adapted or banked speaker; n_refs 1 only): only the triplets whose
    target speaker has a code are scored, each source converted with its target's code instead of the triplet's
    reference (converted(..., codes=), the same batches).  The result then also reports "n_no_code", the triplets left
    out.  None (the default) changes nothing."""
    cfg = model.config
    if int(cfg["data_loader"]["frame_size"]) != 1:
        raise ValueError(f"MCD evaluation supports data_loader.frame_size 1 only (got {cfg['data_loader']['frame_size']})")
    _check_dims(dims)
    if not 1 <= int(n_refs) <= 64:
        raise ValueError(f"n_refs must lie in [1, 64] (got {n_refs})")
    dev = torch.device(device) if device is not None else next(model.parameters()).device
    min_src, min_ref = min_frames(cfg)
    lengths = {u: len(v) for u, v in data.items()}
    trip, n_short = parallel_triplets(list(data), texts, lengths, seed, max_pairs, min_src, min_ref)
    res = {"n": len(trip), "n_short": n_short, "dims": int(dims)}
    if n_refs > 1:
        trip, n_few = fewshot_triplets(trip, list(data), texts, lengths, n_refs, seed, min_ref)
        res.update(n=len(trip), n_refs=int(n_refs), n_few=n_few)
    if target_codes is not None:
        if n_refs > 1:
            raise ValueError("target_codes replaces the references: n_refs must be 1")
        kept = [t for t in trip if speaker_of(t[2]) in target_codes]
        res.update(n=len(kept), n_no_code=len(trip) - len(kept))
        trip = kept
    if not trip:
        res["speakers"] = {}
        return res
    used = sorted({u for s, r, g in trip for u in [s, g] + (r if n_refs > 1 else [r])})
    mels = upload_mels(data, used, dev)
    plain = sorted({t[0] for t in trip} | {t[2] for t in trip})
    ceps = dict(zip(plain, mel_cepstrum([mels[u] for u in plain], attr, hp, dims)))
    conv = [None] * len(trip)
    with eval_mode(model, dev):
        codes = None
        if target_codes is not None:
            codes = torch.stack([torch.as_tensor(target_codes[speaker_of(g)], dtype=torch.float32).reshape(-1).to(dev)
                                 for _, _, g in trip]).contiguous()
        elif n_refs > 1:
            from .inference import embed_reference_sets
            codes = embed_reference_sets(model, [[mels[u].t() for u in r] for _, r, _ in trip])
        first = [mels[r if n_refs == 1 else r[0]] for _, r, _ in trip]
        for idx, decs in converted(model, [mels[s] for s, _, _ in trip], first, codes=codes):
            for i, c in zip(idx, mel_cepstrum(decs, attr, hp, dims)):
                conv[i] = c
    gts = [ceps[g] for _, _, g in trip]
    sl = dtw(conv + [ceps[s] for s, _, _ in trip], gts + gts).cpu().numpy()
    n = len(trip)
    vals = np.stack([MCD_SCALE * sl[:n, 0] / sl[:n, 1], MCD_SCALE * sl[n:, 0] / sl[n:, 1]], axis=1)
    res.update(_means(vals))
    groups: Dict[str, List[int]] = {}
    for i, (_, _, g) in enumerate(trip):
        groups.setdefault(speaker_of(g), []).append(i)
    res["speakers"] = {s: _means(vals[rows]) for s, rows in groups.items()}
    if per_triplet:
        res["triplets"] = [[s, r, g, float(v[0]), float(v[1])] for (s, r, g), v in zip(trip, vals)]
    return res
