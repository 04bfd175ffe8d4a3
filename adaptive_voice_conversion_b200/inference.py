"""Inferencer with the reference's surface (inference.py:24-93).

The model call (``AE.inference``) is the H100 path.  ``inference_from_path`` uses a
caller-supplied ``vocoder`` object with ``get_spectrograms(path)`` / ``melspectrogram2wav(mel)``
(``vocoder.Vocoder``, the reference's librosa STFT / Griffin-Lim DSP on the GPU) and raises a
clear error without one.  ``inference_batch`` is
the batched entry point BASELINE config 5 measures.
"""
from __future__ import annotations

import bisect
import collections
import os
import pickle
from typing import List, Sequence, Tuple

import torch
import torch.nn.functional as F

from .mcd import min_frames
from .model import AE
from .utils import cc, exact_buckets, local_device

# Inferencer.inference_padded: pairs per padded batch, and the graphs of padded shapes kept (least recently used evicted)
PADDED_BATCH_MAX = 64
PADDED_GRAPHS = 64


def padded_extent(T: int) -> int:
    """The grid extent a padded batch whose longest utterance has T frames gets: the next multiple of 32 up to 256
    frames, of 64 up to 1024, of 128 beyond -- eleven extents (128 ... 640) cover 100 to 600 frames."""
    step = 32 if T <= 256 else 64 if T <= 1024 else 128
    return -(-T // step) * step


def padded_batches(src_lens: Sequence[int], ref_lens: Sequence[int], batch_max: int = PADDED_BATCH_MAX
                   ) -> List[Tuple[List[int], int, int, int]]:
    """[(pair indices, T, T_c, B)]: pairs sorted by (source frames, reference frames, index), cut into runs of
    batch_max, each padded to the padded_extent of its longest source and reference and to a power-of-two B."""
    if len(src_lens) != len(ref_lens):
        raise ValueError("padded_batches: src_lens and ref_lens must have the same length")
    if batch_max < 1:
        raise ValueError("padded_batches: batch_max must be >= 1")
    order = sorted(range(len(src_lens)), key=lambda i: (int(src_lens[i]), int(ref_lens[i]), i))
    out = []
    for f in range(0, len(order), batch_max):
        idx = order[f:f + batch_max]
        B = min(batch_max, 1 << (len(idx) - 1).bit_length())
        out.append((idx, padded_extent(max(int(src_lens[i]) for i in idx)), padded_extent(max(int(ref_lens[i]) for i in idx)), B))
    return out


def pack_sets(set_sizes: Sequence[int], set_lens: Sequence[int], batch_max: int = PADDED_BATCH_MAX
              ) -> List[Tuple[List[int], int]]:
    """[(set indices, T)]: reference sets of set_sizes[g] utterances, the longest set_lens[g] frames, sorted by (longest
    member, index) and packed greedily into padded batches of at most batch_max utterances, each set whole in one
    batch; T = the padded_extent of the batch's longest member."""
    if len(set_sizes) != len(set_lens):
        raise ValueError("pack_sets: set_sizes and set_lens must have the same length")
    for g, n in enumerate(set_sizes):
        if not 1 <= int(n) <= batch_max:
            raise ValueError(f"pack_sets: reference set {g} has {n} utterances; 1 to {batch_max} are supported")
    order = sorted(range(len(set_sizes)), key=lambda g: (int(set_lens[g]), g))
    out, cur, rows = [], [], 0
    for g in order:
        if rows + int(set_sizes[g]) > batch_max:
            out.append(cur)
            cur, rows = [], 0
        cur.append(g)
        rows += int(set_sizes[g])
    if cur:
        out.append(cur)
    return [(idx, padded_extent(max(int(set_lens[g]) for g in idx))) for idx in out]


def fill_rows(dst, frames, rows) -> List[int]:
    """Copies frames[i] ([C, T_i]) into dst[j, :, :T_i] for the j-th entry i of rows and returns those T_i; the frames
    of dst past T_i are left as they are (a graph slot's static buffers are never re-zeroed)."""
    lens = []
    for j, i in enumerate(rows):
        n = int(frames[i].shape[1])
        dst[j, :, :n].copy_(frames[i])
        lens.append(n)
    return lens


def padded_batch(frames, rows, T: int, device):
    """(x, lengths): x a zero-filled [len(rows), C, T] batch that fill_rows fills, lengths its int32 T_i on device."""
    x = torch.zeros(len(rows), int(frames[rows[0]].shape[0]), T, device=device)
    return x, torch.tensor(fill_rows(x, frames, rows), dtype=torch.int32, device=device)


def scatter_crops(out, dec, idx, lens):
    """out[i] = dec[j] cropped to its 8 ceil(lens[j] / 8) output frames, as [frames, n_mels], for the j-th entry i of
    idx."""
    for j, i in enumerate(idx):
        out[i] = dec[j, :, :8 * -(-lens[j] // 8)].transpose(0, 1)


def embed_reference_sets(model, sets) -> torch.Tensor:
    """[G, c_out] (device): the pooled speaker code of each set of sets, lists of [C, T] model inputs (device tensors,
    validated by the caller), through AE.get_speaker_embeddings(groups=) in pack_sets' padded batches."""
    dev = sets[0][0].device
    out = torch.empty(len(sets), model.config["SpeakerEncoder"]["c_out"], device=dev)
    for idx, T in pack_sets([len(s) for s in sets], [max(int(r.shape[1]) for r in s) for s in sets]):
        members = [r for g in idx for r in sets[g]]
        x, lens = padded_batch(members, range(len(members)), T, dev)
        offs = torch.tensor([0] + [len(sets[g]) for g in idx]).cumsum(0).to(torch.int32)
        emb = model.get_speaker_embeddings(x, lengths=lens, groups=offs.to(dev))
        out.index_copy_(0, torch.tensor(idx, device=dev), emb)
    return out


class Inferencer(object):
    def __init__(self, config, args, vocoder=None):
        self.config = config
        self.args = args
        self.vocoder = vocoder
        self.padded_captures = 0     # CUDA graphs inference_padded has captured
        self.build_model()
        if getattr(args, "model", None):
            self.load_model()
        self.attr = None
        if getattr(args, "attr", None):
            with open(args.attr, "rb") as f:
                self.attr = pickle.load(f)

    def load_model(self):
        print(f"Load model from {self.args.model}")
        self.model.load_state_dict(torch.load(f"{self.args.model}", map_location=local_device()))

    def build_model(self):
        self.model = cc(AE(self.config))
        self.model.eval()

    def utt_make_frames(self, x):
        """[T, n_mels] -> [1, n_mels*frame_size, T/frame_size] (inference.py:54-60)."""
        frame_size = self.config["data_loader"]["frame_size"]
        remains = x.size(0) % frame_size
        if remains != 0:
            x = F.pad(x, (0, remains))
        return x.view(1, x.size(0) // frame_size, frame_size * x.size(1)).transpose(1, 2).contiguous()

    def denormalize(self, x):
        return x * self.attr["std"] + self.attr["mean"]

    def normalize(self, x):
        return (x - self.attr["mean"]) / self.attr["std"]

    @torch.no_grad()
    def inference_batch(self, x, x_cond):
        """x [B, n_mels, T], x_cond [B, n_mels, T_c] device tensors -> dec [B, n_mels, 8*ceil(T/8)].

        One conversion is ~150 dependent kernel launches of a few microseconds each -- issued one by one from Python
        the GPU waits for the host.  The call is therefore captured ONCE per (shape, parameter version) into a CUDA
        graph (the speaker / content branches on two streams, model.AE.inference) and replayed on static input
        buffers; at most 8 shapes (serving buckets) are kept.  AVC_INFER_GRAPH=0: plain eager calls."""
        if os.environ.get("AVC_INFER_GRAPH", "1") != "1" or not x.is_cuda:
            return self.model.inference(x, x_cond)
        key = (tuple(x.shape), tuple(x_cond.shape), str(x.device), self._param_version())
        graphs = self.__dict__.setdefault("_graphs", {})
        g = graphs.get(key)
        if g is None:
            if len(graphs) >= 8:
                graphs.clear()
            sx, sc = x.contiguous().clone(), x_cond.contiguous().clone()
            self.model.inference(sx, sc)          # eager once: weight packs, allocator warm-up, argument checks
            torch.cuda.synchronize(x.device)
            graph = torch.cuda.CUDAGraph()
            with torch.cuda.graph(graph, capture_error_mode="thread_local"):
                out = self.model.inference(sx, sc)
            g = graphs[key] = (graph, sx, sc, out)
        graph, sx, sc, out = g
        sx.copy_(x, non_blocking=True)
        sc.copy_(x_cond, non_blocking=True)
        graph.replay()
        return out.clone()

    def _param_version(self):
        # in-place updates (optimizer steps, load_state_dict) bump a tensor's version counter: a captured graph reads
        # the weight packs of the version it was captured with; the spectral norm's u and v are buffers
        return sum(int(p._version) for p in self.model.parameters()) + sum(int(b._version) for b in self.model.buffers())

    @torch.no_grad()
    def inference_ragged(self, xs, x_conds):
        """Batched one-shot conversion of utterance pairs of DIFFERENT lengths (the serving form of the loop around
        inference.py:62-70).  xs[i]: [T_i, n_mels], x_conds[i]: [Tc_i, n_mels] normalised mels on the device.
        Pairs are bucketed by their exact (T_i, Tc_i): every bucket is one batched AE.inference call, so each
        utterance gets bit-for-bit the result of converting it alone (InstanceNorm statistics are per sample and
        no padded frame ever enters them -- no masking needed).  Returns the list of [8*ceil(T_i/8), n_mels] mels
        in the input order (device tensors, normalised domain)."""
        if len(xs) != len(x_conds):
            raise ValueError("inference_ragged: xs and x_conds must have the same length")
        out = [None] * len(xs)
        for _, idx in exact_buckets([int(x.shape[0]) for x in xs], [int(c.shape[0]) for c in x_conds]):
            xb = torch.cat([self.utt_make_frames(xs[i]) for i in idx], dim=0)
            cb = torch.cat([self.utt_make_frames(x_conds[i]) for i in idx], dim=0)
            dec = self.inference_batch(xb, cb)               # [n, n_mels, 8*ceil(T/8)]
            for j, i in enumerate(idx):
                out[i] = dec[j].transpose(0, 1)
        self.model.engine(xs[0].device).check_tc_status()
        return out

    @torch.no_grad()
    def inference_padded(self, xs, x_conds, batch_max: int = PADDED_BATCH_MAX):
        """inference_ragged's lists and results, as padded batches: the pairs run as the few shapes padded_batches
        gives, through AE.inference with per-utterance lengths; each gets its stand-alone conversion within rounding.
        Each shape is one CUDA graph (AVC_INFER_GRAPH=1, default) with the inputs and lengths in its static device
        buffers, so a later call on the same shapes only replays; PADDED_GRAPHS shapes are kept, least recently used
        evicted.  x_conds[i] may instead be a list of references of the target speaker (every entry then a list or
        tuple; a mix raises): the sets are embedded by embed_speakers, one list object shared by several pairs once,
        and the pairs converted with those codes (AE.inference_from_embeddings) in the same grid."""
        if len(xs) != len(x_conds):
            raise ValueError("inference_padded: xs and x_conds must have the same length")
        if not xs:
            return []
        sets = [isinstance(c, (list, tuple)) for c in x_conds]
        if any(sets):
            if not all(sets):
                raise ValueError("inference_padded: x_conds mixes single references (tensors) and reference sets (lists)")
            return self._inference_padded_sets(xs, x_conds, batch_max)
        src = [self.utt_make_frames(x)[0] for x in xs]          # [C, T_i]
        ref = [self.utt_make_frames(c)[0] for c in x_conds]
        min_src, min_ref = min_frames(self.config)
        for i, (s, r) in enumerate(zip(src, ref)):
            if s.shape[1] < min_src or r.shape[1] < min_ref:
                raise ValueError(f"inference_padded: pair {i} has {s.shape[1]} source / {r.shape[1]} reference frames; "
                                 f"the model needs at least {min_src} / {min_ref}")
        dev = src[0].device
        out = [None] * len(xs)
        for idx, T, Tc, Bp in padded_batches([s.shape[1] for s in src], [r.shape[1] for r in ref], batch_max):
            xb, cb, lx, lc, run = self._padded_slot(Bp, src[0].shape[0], T, ref[0].shape[0], Tc, dev)
            rows = idx + [idx[0]] * (Bp - len(idx))                # rows past the batch repeat its first pair
            lens, ref_lens = fill_rows(xb, src, rows), fill_rows(cb, ref, rows)
            lx.copy_(torch.tensor(lens, dtype=torch.int32))
            lc.copy_(torch.tensor(ref_lens, dtype=torch.int32))
            scatter_crops(out, run(), idx, lens)
        self.model.engine(dev).check_tc_status()
        return out

    def _padded_slot(self, B, C, T, Cc, Tc, dev):
        """(x, x_cond, lengths, cond_lengths, convert) of one padded shape: static buffers and a CUDA-graph replay
        (captured on first use) or, with AVC_INFER_GRAPH=0, an eager AE.inference."""
        def make():
            xb, cb = torch.zeros(B, C, T, device=dev), torch.zeros(B, Cc, Tc, device=dev)
            lx, lc = (torch.full((B,), n, dtype=torch.int32, device=dev) for n in (T, Tc))
            return (xb, cb, lx, lc), lambda: self.model.inference(xb, cb, lengths=lx, cond_lengths=lc)
        return self._graph_slot((B, C, T, Cc, Tc, str(dev), self._param_version()), make)

    def _emb_slot(self, B, C, T, dev):
        """(x, emb, lengths, convert) of one padded shape converted with given speaker codes (AE.inference_from_embeddings),
        as _padded_slot."""
        def make():
            xb = torch.zeros(B, C, T, device=dev)
            eb = torch.zeros(B, self.config["SpeakerEncoder"]["c_out"], device=dev)
            lx = torch.full((B,), T, dtype=torch.int32, device=dev)
            return (xb, eb, lx), lambda: self.model.inference_from_embeddings(xb, eb, lengths=lx)
        return self._graph_slot(("emb", B, C, T, str(dev), self._param_version()), make)

    def _graph_slot(self, key, make):
        """(*static buffers, convert) for `key`: make() gives the buffers and the eager call; with AVC_INFER_GRAPH=1 the
        call is captured once into a CUDA graph replayed on those buffers, PADDED_GRAPHS graphs kept (LRU)."""
        graph_on = os.environ.get("AVC_INFER_GRAPH", "1") == "1"
        graphs = self.__dict__.setdefault("_padded_graphs", collections.OrderedDict())
        if graph_on and key in graphs:
            graphs.move_to_end(key)
            return graphs[key]
        bufs, call = make()
        if not graph_on:
            return (*bufs, call)
        call()                             # eager once: weight packs, allocator warm-up, argument checks
        torch.cuda.synchronize(bufs[0].device)
        graph = torch.cuda.CUDAGraph()
        with torch.cuda.graph(graph, capture_error_mode="thread_local"):
            out = call()
        self.padded_captures += 1
        while len(graphs) >= PADDED_GRAPHS:
            graphs.popitem(last=False)
        graphs[key] = (*bufs, lambda: (graph.replay(), out.clone())[1])
        return graphs[key]

    def _ref_frames(self, ref_sets, what):
        """[[C, T] per reference] per set of ref_sets (lists of [T, n_mels] mels); ValueError naming a bad set."""
        _, min_ref = min_frames(self.config)
        out = []
        for g, refs in enumerate(ref_sets):
            if not isinstance(refs, (list, tuple)) or not refs:
                raise ValueError(f"{what}: reference set {g} must be a non-empty list of tensors")
            if len(refs) > PADDED_BATCH_MAX:
                raise ValueError(f"{what}: reference set {g} has {len(refs)} references; at most {PADDED_BATCH_MAX} "
                                 f"are supported")
            frames = [self.utt_make_frames(r)[0] for r in refs]
            for j, r in enumerate(frames):
                if r.shape[1] < min_ref:
                    raise ValueError(f"{what}: reference {j} of set {g} has {r.shape[1]} frames; the model needs at "
                                     f"least {min_ref}")
            out.append(frames)
        return out

    @torch.no_grad()
    def embed_speakers(self, ref_sets):
        """[G, c_out] speaker codes (device) of G reference sets, each a list of [T, n_mels] normalised mels of one
        speaker on the device: AE.get_speaker_embeddings(groups=) over padded batches (pack_sets: at most
        PADDED_BATCH_MAX references, each set whole in one batch).  A set of more than PADDED_BATCH_MAX references or
        a reference shorter than the model accepts raises ValueError naming it."""
        frames = self._ref_frames(ref_sets, "embed_speakers")
        if not frames:
            raise ValueError("embed_speakers: no reference sets")
        out = embed_reference_sets(self.model, frames)
        self.model.engine(out.device).check_tc_status()
        return out

    def _inference_padded_sets(self, xs, ref_sets, batch_max):
        """inference_padded with a reference set per pair: a set object shared by several pairs is embedded once
        (embed_speakers), then the sources run in padded_batches' grid through AE.inference_from_embeddings, one CUDA
        graph per shape with the codes in a static buffer."""
        slot_of, uniq = {}, []
        for refs in ref_sets:
            if id(refs) not in slot_of:
                slot_of[id(refs)] = len(uniq)
                uniq.append(refs)
        src = self._source_frames(xs, "inference_padded")
        emb = self.embed_speakers(uniq)
        which = torch.tensor([slot_of[id(refs)] for refs in ref_sets], device=emb.device)
        return self._convert_with_codes(src, emb.index_select(0, which), batch_max)

    def _source_frames(self, xs, what):
        """[C, T_i] model inputs of the sources xs ([T_i, n_mels]); ValueError naming a source shorter than the model
        accepts."""
        src = [self.utt_make_frames(x)[0] for x in xs]
        min_src, _ = min_frames(self.config)
        for i, s in enumerate(src):
            if s.shape[1] < min_src:
                raise ValueError(f"{what}: pair {i} has {s.shape[1]} source frames; the model needs at least {min_src}")
        return src

    @torch.no_grad()
    def inference_with_codes(self, xs, codes, batch_max: int = PADDED_BATCH_MAX):
        """Convert each source xs[i] ([T_i, n_mels] normalised mel on the device) with the speaker code codes[i]
        (float32 [len(xs), c_out] on the device, or a list of [c_out] codes: rows of embed_speakers, SpeakerBank.code,
        ...) in inference_padded's grid: padded_batches' shapes, one CUDA graph per shape (AVC_INFER_GRAPH=1) with the
        codes in a static buffer, through AE.inference_from_embeddings.  Returns inference_padded's list of mels.
        inference_padded(xs, sets) runs exactly this on embed_speakers' codes of the pairs' sets."""
        if not isinstance(codes, torch.Tensor):
            codes = torch.stack(list(codes)) if len(codes) else None
        c_out = self.config["SpeakerEncoder"]["c_out"]
        if (codes is None or codes.dtype != torch.float32 or tuple(codes.shape) != (len(xs), c_out)
                or (xs and codes.device != xs[0].device)):
            raise ValueError(f"inference_with_codes: codes must be float32 [{len(xs)}, {c_out}] on the sources' device, "
                             f"got {getattr(codes, 'dtype', None)} {tuple(getattr(codes, 'shape', ()))}")
        if not xs:
            return []
        return self._convert_with_codes(self._source_frames(xs, "inference_with_codes"), codes.contiguous(), batch_max)

    def _convert_with_codes(self, src, codes, batch_max):
        """The sources src ([C, T_i] model inputs) converted with codes[i] in padded_batches' grid (_emb_slot)."""
        dev = src[0].device
        out = [None] * len(src)
        for idx, T, _, Bp in padded_batches([s.shape[1] for s in src], [0] * len(src), batch_max):
            xb, eb, lx, run = self._emb_slot(Bp, src[0].shape[0], T, dev)
            rows = idx + [idx[0]] * (Bp - len(idx))                # rows past the batch repeat its first pair
            lens = fill_rows(xb, src, rows)
            eb.copy_(codes.index_select(0, torch.tensor(rows, device=dev)))
            lx.copy_(torch.tensor(lens, dtype=torch.int32))
            scatter_crops(out, run(), idx, lens)
        self.model.engine(dev).check_tc_status()
        return out

    @torch.no_grad()
    def inference_morph(self, xs, codes, weights, batch_max: int = PADDED_BATCH_MAX):
        """Time-varying speaker morphs (AE.inference_morph) of many sources: xs[i] a [T_i, n_mels] normalised mel,
        codes[i] its [K_i, c_out] anchor codes and weights[i] their [K_i, T_i] weights at the source frame rate (device
        tensors).  The sources run in padded_batches' grid; a batch's K is its largest K_i, shorter anchor lists padded
        with zero-weight anchors (which change no bit).  One CUDA graph per (B, T, K) shape (AVC_INFER_GRAPH=1) with the
        sources, anchors and weights in static buffers, bit for bit the eager result.  Returns inference_padded's list
        of mels.  ValueError, before anything runs, naming a source whose shapes or weights are invalid (weights finite,
        >= 0, a positive sum on every frame)."""
        if not len(xs) == len(codes) == len(weights):
            raise ValueError("inference_morph: xs, codes and weights must have the same length")
        if not xs:
            return []
        if int(self.config["data_loader"]["frame_size"]) != 1:
            raise ValueError("inference_morph: supports data_loader.frame_size 1 only")
        from ._lib import MORPH_MAX_K
        c_out = self.config["SpeakerEncoder"]["c_out"]
        dev = xs[0].device
        for i, (x, c, w) in enumerate(zip(xs, codes, weights)):
            K = int(c.shape[0]) if isinstance(c, torch.Tensor) and c.dim() == 2 else 0
            for t in (c, w):
                if not isinstance(t, torch.Tensor) or t.dtype != torch.float32 or t.device != dev:
                    raise ValueError(f"inference_morph: source {i}: codes and weights must be float32 on {dev}")
            if (not 1 <= K <= MORPH_MAX_K or tuple(c.shape) != (K, c_out)
                    or tuple(w.shape) != (K, int(x.shape[0]))):
                raise ValueError(f"inference_morph: source {i}: expected codes [K, {c_out}] with 1 <= K <= {MORPH_MAX_K} "
                                 f"and weights [K, {int(x.shape[0])}], got {tuple(c.shape)} and {tuple(w.shape)}")
        # every source's frames as rows of one table (absent anchors 0): a handful of launches and one synchronise
        offs = [0]
        for w in weights:
            offs.append(offs[-1] + int(w.shape[1]))
        table = torch.zeros(offs[-1], max(int(w.shape[0]) for w in weights), device=dev)
        for i, w in enumerate(weights):
            table[offs[i]:offs[i + 1], :w.shape[0]].copy_(w.t())
        s = table.sum(1)
        bad = (~torch.isfinite(table) | (table < 0)).any(1) | ~(s > 0) | ~torch.isfinite(s)
        if bool(bad.any()):
            i = bisect.bisect_right(offs, int(bad.nonzero()[0])) - 1
            raise ValueError(f"inference_morph: source {i}: weights must be finite and >= 0 with a positive sum on every "
                             f"frame")
        src = self._source_frames(xs, "inference_morph")
        out = [None] * len(src)
        for idx, T, _, Bp in padded_batches([s.shape[1] for s in src], [0] * len(src), batch_max):
            K = max(int(codes[i].shape[0]) for i in idx)
            xb, cb, wb, lx, run = self._morph_slot(Bp, src[0].shape[0], T, K, dev)
            rows = idx + [idx[0]] * (Bp - len(idx))                # rows past the batch repeat its first source
            cb.zero_()
            wb.zero_()
            lens = fill_rows(xb, src, rows)
            for j, i in enumerate(rows):
                k = codes[i].shape[0]
                cb[j, :k].copy_(codes[i])
                wb[j, :k, :lens[j]].copy_(weights[i])
            lx.copy_(torch.tensor(lens, dtype=torch.int32))
            scatter_crops(out, run(), idx, lens)
        self.model.engine(dev).check_tc_status()
        return out

    def _morph_slot(self, B, C, T, K, dev):
        """(x, codes, weights, lengths, convert) of one padded morph shape (AE.inference_morph), as _padded_slot.  The
        weights start at 1 so that the capture's eager call is a valid morph."""
        def make():
            xb = torch.zeros(B, C, T, device=dev)
            cb = torch.zeros(B, K, self.config["SpeakerEncoder"]["c_out"], device=dev)
            wb = torch.ones(B, K, T, device=dev)
            lx = torch.full((B,), T, dtype=torch.int32, device=dev)
            return (xb, cb, wb, lx), lambda: self.model.inference_morph(xb, cb, wb, lengths=lx)
        return self._graph_slot(("morph", B, C, T, K, str(dev), self._param_version()), make)

    @torch.no_grad()
    def inference_one_utterance(self, x, x_cond):
        """x, x_cond: [T, n_mels] normalised mels on the device (inference.py:62-70).  x_cond may also be a list of
        references of the target speaker: their pooled code (embed_speakers) conditions the decoder."""
        if isinstance(x_cond, (list, tuple)):
            dec = self.model.inference_from_embeddings(self.utt_make_frames(x), self.embed_speakers([x_cond]))
        else:
            dec = self.model.inference(self.utt_make_frames(x), self.utt_make_frames(x_cond))
        dec = dec.transpose(1, 2).squeeze(0).detach().cpu().numpy()
        self.model.engine(x.device).check_tc_status()
        if self.attr is not None:
            dec = self.denormalize(dec)
        wav = self.vocoder.melspectrogram2wav(dec) if self.vocoder is not None else None
        return wav, dec

    def write_wav_to_file(self, wav_data, output_path):
        from scipy.io.wavfile import write
        write(output_path, rate=self.args.sample_rate, data=wav_data)

    def inference_from_path(self):
        if self.vocoder is None:
            raise RuntimeError("inference_from_path needs a vocoder with get_spectrograms/melspectrogram2wav "
                               "(e.g. adaptive_voice_conversion_b200.vocoder.Vocoder)")
        src_mel, _ = self.vocoder.get_spectrograms(self.args.source)
        tar_mel, _ = self.vocoder.get_spectrograms(self.args.target)
        dev = local_device()
        src = torch.from_numpy(self.normalize(src_mel)).float().to(dev)
        tar = torch.from_numpy(self.normalize(tar_mel)).float().to(dev)
        wav, _ = self.inference_one_utterance(src, tar)
        self.write_wav_to_file(wav, self.args.output)
