"""Speaker measures of a held-out set: how well the speaker embedding, the content code and the input mel separate
speakers (verification EER), and whether a conversion carries the target speaker's identity (speaker similarity).

Utterances: the whole utterances of ``<set>.pkl`` (attr-normalised [T, n_mels]; ``frame_size`` 1 only) in sorted key
order, the speaker from ``evaluate.speaker_of``.  An utterance shorter than max(min_frames) (``mcd.min_frames``: 17
frames for the shipped config) is dropped from all three representations and counted in ``n_short``, so the three
EERs cover the same trials.

Representations, one vector per utterance, the model in eval mode, in padded batches (``inference.padded_batches``):
  * ``speaker``: ``AE.get_speaker_embeddings(x, lengths=)`` (c_out of the speaker encoder, 128);
  * ``content``: statistics pooling of the content encoder's mean head mu over the utterance's valid latent frames
    (``AE.get_content_means``, the padded path ``AE.inference`` runs): 2 c_out (256);
  * ``mel``: the same pooling of the normalised input mel itself (2 n_mels): the baseline.
InstanceNorm removes each channel's mean and variance, which is why the pooling keeps both.

Pooling (``avc_time_stats_varlen``), per channel over the L valid frames, in float64 adding in ascending t:
mean = (sum x) / L, then var = (sum (x - mean)^2) / L, std = sqrt(var); the vector is [means | stds], each rounded once
to float32.

Score: s(a, b) = dot(a, b) / (sqrt(|a|^2) sqrt(|b|^2)) of the float32 vectors promoted to float64, sums over d in
ascending order, every multiply, add, sqrt and divide rounded on its own; s = 0 when either norm is 0.  So s(a, b) ==
s(b, a) bit for bit and a permuted set gives the same scores.

EER: the trials are all unordered pairs i < j, target trials when both utterances share a speaker.  FRR(t) =
#{target < t} / n_target, FAR(t) = #{non-target >= t} / n_nontarget; over t in {all scores} U {+inf}, ``eer`` = min
max(FRR, FAR) and ``threshold`` the smallest t reaching it, with ``frr`` and ``far`` there (no interpolation).  ``eer``
and the rest are None when either count is 0.  Scores and the threshold search run on the GPU (``avc_spk_eer``, by
counting: radix selection over the scores' order-preserving keys).

Conversion pairs: ``rng = random.Random(seed)``; for every utterance u in sorted order whose speaker has at least two
utterances in the set, the reference r is ``rng.choice`` over the sorted such utterances of the other speakers.  A pair
is then dropped and counted in ``n_short`` when u is not embedded (shorter than max(min_frames)), r is shorter than the
reference minimum, or u's or r's speaker has no other embedded utterance (both means below need one).  The draws do not
depend on the lengths.  With
``max_pairs > 0`` and more pairs than that, ``sorted(rng.sample(range(n), max_pairs))`` of them are kept.

Each pair is converted with ``AE.inference(x, x_cond, lengths=, cond_lengths=)`` in padded batches; ``dec`` cropped to
u's T frames is embedded y by the padded speaker path.  With emb(v) the speaker embedding of utterance v:
  * ``sim_target`` = mean of s(y, emb(v)) over r's speaker's utterances v != r;
  * ``sim_source`` = mean of s(y, emb(v)) over u's speaker's utterances v != u;
  * ``success`` = [sim_target > sim_source];
  * ``sim_target_source`` = sim_target of the unconverted source emb(u): the baseline, as mcd_source is for MCD.
Means over utterances are float64 added in index order (``avc_spk_group_mean``); a set reports the means of the four
values over its pairs (float64, pair order), ``n``, ``n_short`` and the same means per target speaker.

Few-shot (``n_refs`` K > 1): the pairs above (``max_pairs`` already applied) each get K - 1 more references of r's
speaker (``fewshot_pairs``: ``rng2 = random.Random(seed + 1)``, ``rng2.sample`` in pair order over that speaker's other
utterances of at least the reference minimum, sorted); a pair is dropped and counted in ``n_few`` when the speaker has
fewer than K such utterances or no embedded utterance outside the K.  u is converted with the set's pooled code
(``AE.get_speaker_embeddings(groups=)``, then ``AE.inference_from_embeddings`` in padded batches), and ``sim_target``
skips all K references (``avc_spk_group_mean_multi``); ``sim_source`` and ``sim_target_source`` are as with one.

The speaker encoder that embeds y is the model's own: these similarities compare checkpoints of this project, not an
independent verifier's judgement.  The ``speaker`` EER on real recordings, in the same report, shows how far that
encoder can be trusted.
"""
from __future__ import annotations

import ctypes as C
import random
from typing import Dict, List, Mapping, Sequence

import numpy as np
import torch

from . import _lib as L
from .evaluate import speaker_of
from .inference import padded_batch, padded_batches
from .mcd import min_frames
from .utils import _stream, eval_mode, upload_mels

REPRESENTATIONS = ("speaker", "content", "mel")


# ------------------------------------------------------------------ conversion pairs
class _Others:
    """The sorted utterances of `utts` outside [a, b) (one speaker's run), as a sequence for rng.choice."""

    def __init__(self, utts, a, b):
        self.utts, self.a, self.b = utts, a, b

    def __len__(self):
        return len(self.utts) - (self.b - self.a)

    def __getitem__(self, i):
        if not 0 <= i < len(self):
            raise IndexError(i)
        return self.utts[i if i < self.a else i + self.b - self.a]


def conversion_pairs(utts: Sequence[str], lengths: Mapping[str, int], seed: int = 0, max_pairs: int = 0,
                     min_src: int = 1, min_ref: int = 1, min_set: int = 1):
    """([(source, reference)], n_short) of the utterance keys `utts` of a set, as the module docstring defines;
    lengths[u] = frames of u, min_set = the frames an utterance needs to be embedded."""
    utts = sorted(utts)
    count: Dict[str, int] = {}
    for u in utts:
        count[speaker_of(u)] = count.get(speaker_of(u), 0) + 1
    qual = [u for u in utts if count[speaker_of(u)] >= 2]
    run: Dict[str, List[int]] = {}          # a speaker's utterances are one run of the sorted keys
    for i, u in enumerate(qual):
        run.setdefault(speaker_of(u), [i, i])[1] = i + 1
    embedded: Dict[str, int] = {}
    for u in utts:
        if lengths[u] >= min_set:
            embedded[speaker_of(u)] = embedded.get(speaker_of(u), 0) + 1

    def others_embedded(v):
        return embedded.get(speaker_of(v), 0) - (lengths[v] >= min_set) > 0

    rng = random.Random(seed)
    out, n_short = [], 0
    for u in qual:
        a, b = run[speaker_of(u)]
        if b - a == len(qual):
            break                           # a single speaker qualifies: no pair at all
        r = rng.choice(_Others(qual, a, b))
        if lengths[u] < min_src or lengths[r] < min_ref or not others_embedded(u) or not others_embedded(r):
            n_short += 1
            continue
        out.append((u, r))
    if max_pairs > 0 and len(out) > max_pairs:
        out = [out[i] for i in sorted(rng.sample(range(len(out)), max_pairs))]
    return out, n_short


def fewshot_pairs(pairs, utts: Sequence[str], lengths: Mapping[str, int], n_refs: int, seed: int = 0,
                  min_ref: int = 1, min_set: int = 1):
    """([(source, [reference, extra, ...])], n_few): conversion_pairs' pairs with n_refs - 1 extra references each.
    rng2 = random.Random(seed + 1) draws, in pair order, rng2.sample over the reference's speaker's other utterances of
    at least min_ref frames (sorted).  A pair is dropped and counted in n_few when that speaker has fewer than n_refs
    such utterances (the reference included), or no utterance of at least min_set frames outside the drawn set (the
    embedded utterances sim_target averages over)."""
    by_speaker: Dict[str, List[str]] = {}
    for u in sorted(utts):
        by_speaker.setdefault(speaker_of(u), []).append(u)
    rng2 = random.Random(seed + 1)
    out, n_few = [], 0
    for u, r in pairs:
        spk = by_speaker[speaker_of(r)]
        others = [v for v in spk if v != r and lengths[v] >= min_ref]
        if len(others) + 1 < n_refs:
            n_few += 1
            continue
        refs = [r] + rng2.sample(others, n_refs - 1)
        if not any(lengths[v] >= min_set and v not in refs for v in spk):
            n_few += 1
            continue
        out.append((u, refs))
    return out, n_few


# ------------------------------------------------------------------ the three kernels
def _lengths(lengths, B, dev) -> torch.Tensor:
    if isinstance(lengths, torch.Tensor):
        if lengths.dtype == torch.bool or lengths.is_floating_point() or lengths.is_complex():
            raise ValueError(f"lengths must be integers (got {lengths.dtype})")
        lengths = lengths.to(dev)
    else:
        lengths = torch.as_tensor(np.asarray(lengths, np.int64), device=dev)
    if lengths.dim() != 1 or lengths.shape[0] != B:
        raise ValueError(f"lengths has shape {tuple(lengths.shape)}; expected [{B}]")
    return lengths


def time_stats(x: torch.Tensor, lengths) -> torch.Tensor:
    """[B, 2C] float32 (device): per-channel mean then std (ddof 0) of each sample's first lengths[b] frames of a
    padded batch x [B, C, T] (float32 on a CUDA device), one launch.  Frames past a length are never read."""
    if not isinstance(x, torch.Tensor) or x.dim() != 3 or x.dtype != torch.float32 or not x.is_cuda or min(x.shape) < 1:
        raise ValueError(f"time_stats: x is {getattr(x, 'dtype', type(x).__name__)} {tuple(getattr(x, 'shape', ()))}; "
                         f"expected float32 [B, C, T >= 1] on a CUDA device")
    B, Cc, T = x.shape
    lens = _lengths(lengths, B, x.device)
    lo, hi = int(lens.min()), int(lens.max())
    if lo < 1 or hi > T:
        raise ValueError(f"time_stats: lengths must lie in [1, {T}] (got min {lo}, max {hi})")
    x = x.contiguous()
    lens = lens.to(torch.int32)
    out = torch.empty(B, 2 * Cc, device=x.device)
    L.check(L.load().avc_time_stats_varlen(x.data_ptr(), out.data_ptr(), B, Cc, T, lens.data_ptr(), _stream(x.device)),
            "avc_time_stats_varlen")
    return out


def _check_vectors(v, what: str, n_max: int = L.SPK_MAX_N):
    if not isinstance(v, torch.Tensor) or v.dim() != 2 or v.dtype != torch.float32 or not v.is_cuda:
        raise ValueError(f"{what}: expected float32 [N, D] on a CUDA device (got {getattr(v, 'dtype', type(v).__name__)} "
                         f"{tuple(getattr(v, 'shape', ()))})")
    n, d = v.shape
    if not 1 <= n <= n_max:
        raise ValueError(f"{what}: {n} vectors; 1 to {n_max} are supported")
    if not 1 <= d <= L.SPK_MAX_DIMS:
        raise ValueError(f"{what}: {d} dimensions; 1 to {L.SPK_MAX_DIMS} are supported")
    if not bool(torch.isfinite(v).all()):
        raise ValueError(f"{what}: the vectors must be finite")
    return v.contiguous()


def _labels(labels, n, dev, what):
    lab = torch.as_tensor(np.asarray(labels), device=dev) if not isinstance(labels, torch.Tensor) else labels.to(dev)
    if lab.dim() != 1 or lab.shape[0] != n or lab.dtype == torch.bool or lab.is_floating_point() or lab.is_complex():
        raise ValueError(f"{what}: expected {n} integer labels (got {lab.dtype} {tuple(lab.shape)})")
    if lab.numel() and (int(lab.min()) < -2 ** 31 or int(lab.max()) >= 2 ** 31):
        raise ValueError(f"{what}: labels must fit in int32")
    return lab.to(torch.int32).contiguous()


def eer_workspace(n: int, device) -> torch.Tensor:
    """A workspace for avc_spk_eer over n vectors (uint8, 256-byte aligned by the caching allocator)."""
    nbytes = int(L.load().avc_spk_eer_workspace_bytes(int(n)))
    if nbytes < 0:
        raise ValueError(f"eer: {n} vectors; 1 to {L.SPK_MAX_N} are supported")
    return torch.empty(nbytes, dtype=torch.uint8, device=device)


def eer(vecs: torch.Tensor, labels, workspace: torch.Tensor = None) -> dict:
    """{eer, threshold, frr, far, n_target, n_nontarget} of every pair of the rows of vecs [N, D] (float32, CUDA) as
    trials, target when labels (N integers) agree; the module docstring gives the definition.  eer, threshold, frr and
    far are None when either count is 0.  `workspace` (eer_workspace(N)) keeps the scores for trial_scores."""
    vecs = _check_vectors(vecs, "eer")
    n, d = vecs.shape
    dev = vecs.device
    lab = _labels(labels, n, dev, "eer")
    ws = eer_workspace(n, dev) if workspace is None else workspace
    need = int(L.load().avc_spk_eer_workspace_bytes(n))
    if ws.dtype != torch.uint8 or ws.device != dev or ws.numel() < need or ws.data_ptr() % 256:
        raise ValueError(f"eer: the workspace must be a 256-byte aligned uint8 tensor of at least {need} bytes on {dev}")
    res = torch.empty(C.sizeof(L.EerResult), dtype=torch.uint8, device=dev)
    L.check(L.load().avc_spk_eer(vecs.data_ptr(), lab.data_ptr(), n, d, ws.data_ptr(), ws.numel(), res.data_ptr(),
                                 _stream(dev)), "avc_spk_eer")
    r = L.EerResult.from_buffer_copy(bytes(res.cpu().numpy()))
    null = r.n_target == 0 or r.n_nontarget == 0
    out = {k: None if null else float(getattr(r, k)) for k in ("eer", "threshold", "frr", "far")}
    out.update(n_target=int(r.n_target), n_nontarget=int(r.n_nontarget))
    return out


def trial_scores(workspace: torch.Tensor, n: int) -> np.ndarray:
    """float64 [n, n] (host): s(i, j) at [i][j] for i < j, read from the keys avc_spk_eer left in `workspace`; NaN
    elsewhere."""
    nt = -(-n // 64)
    off = L.SPK_STATE_BYTES + -(-8 * n // 256) * 256
    keys = workspace[off:off + nt * (nt + 1) // 2 * 4096 * 8].cpu().numpy().view(np.uint64).reshape(-1, 64, 64)
    neg = keys >> np.uint64(63) == 0
    bits = np.where(neg, ~keys, keys & np.uint64(0x7FFFFFFFFFFFFFFF))
    tiles = bits.view(np.float64)
    full = np.full((nt * 64, nt * 64), np.nan)
    for tj in range(nt):
        for ti in range(tj + 1):
            full[ti * 64:(ti + 1) * 64, tj * 64:(tj + 1) * 64] = tiles[tj * (tj + 1) // 2 + ti]
    full = full[:n, :n]
    full[np.tril_indices(n)] = np.nan
    return full


SPK_MAX_EXCLUDE = 64   # avc_spk_group_mean_multi's n_exclude


def group_means(queries: torch.Tensor, q_labels, q_exclude, vecs: torch.Tensor, labels) -> torch.Tensor:
    """float64 [M] (device): for each query m, the mean of s(queries[m], vecs[v]) over the v with labels[v] ==
    q_labels[m] and v != q_exclude[m] (-1: none), added in ascending v; NaN when there is none.  One launch.
    q_exclude may also be [M, n_exclude] (1 to 64 indices per query, -1 or any index outside the set: none;
    avc_spk_group_mean_multi)."""
    queries = _check_vectors(queries, "group_means(queries)", n_max=2 ** 31 - 1)
    vecs = _check_vectors(vecs, "group_means(vecs)")
    if queries.shape[1] != vecs.shape[1] or queries.device != vecs.device:
        raise ValueError(f"group_means: queries {tuple(queries.shape)} on {queries.device}, vectors {tuple(vecs.shape)} "
                         f"on {vecs.device}; the dimensions and devices must agree")
    (m, d), n, dev = queries.shape, vecs.shape[0], vecs.device
    ql = _labels(q_labels, m, dev, "group_means(q_labels)")
    multi = np.ndim(q_exclude) == 2 if not isinstance(q_exclude, torch.Tensor) else q_exclude.dim() == 2
    if multi:
        qe = torch.as_tensor(np.asarray(q_exclude), device=dev) if not isinstance(q_exclude, torch.Tensor) else q_exclude.to(dev)
        k = qe.shape[1]
        if qe.shape[0] != m or not 1 <= k <= SPK_MAX_EXCLUDE:
            raise ValueError(f"group_means(q_exclude): expected [{m}, 1..{SPK_MAX_EXCLUDE}], got {tuple(qe.shape)}")
        qe = _labels(qe.reshape(-1), m * k, dev, "group_means(q_exclude)")
    else:
        qe = _labels(q_exclude, m, dev, "group_means(q_exclude)")
    lab = _labels(labels, n, dev, "group_means(labels)")
    out = torch.empty(m, dtype=torch.float64, device=dev)
    desc = L.SpkGroupDesc(m=m, n=n, dims=d, queries=queries.data_ptr(), q_labels=ql.data_ptr(), q_exclude=qe.data_ptr(),
                          set=vecs.data_ptr(), labels=lab.data_ptr(), out=out.data_ptr())
    if multi:
        L.check(L.load().avc_spk_group_mean_multi(C.byref(desc), k, _stream(dev)), "avc_spk_group_mean_multi")
    else:
        L.check(L.load().avc_spk_group_mean(C.byref(desc), _stream(dev)), "avc_spk_group_mean")
    return out


def identify(queries: torch.Tensor, bank: torch.Tensor, targets=None) -> Dict[str, np.ndarray]:
    """Closed-set identification of queries [M, D] against bank codes [S, D] (float32, one CUDA device), one launch
    (avc_spk_identify): {"best": int32 [M] (the highest-scoring bank row, the lowest among ties), "best_score": float64,
    "target_score": float64 (NaN without a target), "target_rank": int32 (rows scoring strictly above the target; -1
    without one)} on the host.  targets: M bank rows, -1 = none (None: no targets).  Scores are s(a, b) above."""
    queries = _check_vectors(queries, "identify(queries)", n_max=2 ** 31 - 1)
    bank = _check_vectors(bank, "identify(bank)")
    if queries.shape[1] != bank.shape[1] or queries.device != bank.device:
        raise ValueError(f"identify: queries {tuple(queries.shape)} on {queries.device}, bank {tuple(bank.shape)} on "
                         f"{bank.device}; the dimensions and devices must agree")
    (m, d), s, dev = queries.shape, bank.shape[0], bank.device
    tg = None if targets is None else _labels(targets, m, dev, "identify(targets)")
    best = torch.empty(m, dtype=torch.int32, device=dev)
    rank = torch.empty(m, dtype=torch.int32, device=dev)
    best_score = torch.empty(m, dtype=torch.float64, device=dev)
    target_score = torch.empty(m, dtype=torch.float64, device=dev)
    desc = L.SpkIdentifyDesc(m=m, s=s, dims=d, queries=queries.data_ptr(), bank=bank.data_ptr(),
                             q_target=None if tg is None else tg.data_ptr(), best=best.data_ptr(),
                             best_score=best_score.data_ptr(), target_score=target_score.data_ptr(),
                             target_rank=rank.data_ptr())
    L.check(L.load().avc_spk_identify(C.byref(desc), _stream(dev)), "avc_spk_identify")
    return {"best": best.cpu().numpy(), "best_score": best_score.cpu().numpy(),
            "target_score": target_score.cpu().numpy(), "target_rank": rank.cpu().numpy()}


def bank_identification(bank, y: torch.Tensor, src_speakers, tgt_speakers, real: torch.Tensor, real_speakers) -> dict:
    """The bank fields of a set's conversion entry: id_target / id_source = the shares of the conversions y (rows of
    pairs whose source and target speakers are both banked) whose nearest bank code is the target's / the source's;
    id_real = the share of the real utterance embeddings `real` of banked speakers nearest their own speaker's code;
    n_banked / n_unbanked pairs; bank_speakers.  Shares are None over no rows.  One identify call."""
    pi = [i for i, (s, t) in enumerate(zip(src_speakers, tgt_speakers)) if s in bank and t in bank]
    ri = [i for i, s in enumerate(real_speakers) if s in bank]
    out = {"id_target": None, "id_source": None, "id_real": None, "n_banked": len(pi),
           "n_unbanked": len(src_speakers) - len(pi), "bank_speakers": len(bank)}
    if not pi and not ri:
        return out
    dev = bank.codes.device
    q = torch.cat([v[torch.tensor(rows, dtype=torch.long, device=v.device)].to(dev) for v, rows in ((y, pi), (real, ri))
                   if rows])
    targets = [bank.index(tgt_speakers[i]) for i in pi] + [bank.index(real_speakers[i]) for i in ri]
    best = identify(q, bank.codes, targets)["best"]
    P = len(pi)
    if P:
        out["id_target"] = float(np.mean(best[:P] == np.array(targets[:P])))
        out["id_source"] = float(np.mean(best[:P] == np.array([bank.index(src_speakers[i]) for i in pi])))
    if ri:
        out["id_real"] = float(np.mean(best[P:] == np.array(targets[P:])))
    return out


# ------------------------------------------------------------------ representations and conversions
def representations(model, mels: Sequence[torch.Tensor]) -> Dict[str, torch.Tensor]:
    """{speaker, content, mel}: [N, D] float32 (device) of the attr-normalised mels [T_i, n_mels] (device tensors, each
    at least max(min_frames) long), in padded batches.  The model must be in eval mode."""
    dev = mels[0].device
    lens = [int(m.shape[0]) for m in mels]
    frames = [m.t() for m in mels]
    out = {k: [None] * len(mels) for k in REPRESENTATIONS}
    for idx, T, _, _ in padded_batches(lens, lens):
        x, lx = padded_batch(frames, idx, T, dev)
        emb = model.get_speaker_embeddings(x, lengths=lx)
        mu, lat = model.get_content_means(x, lengths=lx)
        rows = {"speaker": emb, "content": time_stats(mu, lat), "mel": time_stats(x, lx)}
        for k, v in rows.items():
            for j, i in enumerate(idx):
                out[k][i] = v[j]
    return {k: torch.stack(v) for k, v in out.items()}


def converted_embeddings(model, sources: Sequence[torch.Tensor], refs: Sequence[torch.Tensor]) -> torch.Tensor:
    """[P, c_out] float32 (device): the speaker embedding of each conversion of sources[i] (cropped to its T frames)
    with the reference refs[i], in padded batches of AE.inference.  refs[i] may instead be a list of references of
    one speaker: the sources are then converted with the sets' pooled codes (inference.embed_reference_sets) through
    AE.inference_from_embeddings.  The model must be in eval mode."""
    dev = sources[0].device
    src = [s.t() for s in sources]
    out = [None] * len(sources)
    if isinstance(refs[0], (list, tuple)):
        from .inference import embed_reference_sets
        codes = embed_reference_sets(model, [[r.t() for r in s] for s in refs])
        for idx, T, _, _ in padded_batches([int(s.shape[0]) for s in sources], [0] * len(sources)):
            x, lx = padded_batch(src, idx, T, dev)
            dec = model.inference_from_embeddings(x, codes[torch.tensor(idx, device=dev)], lengths=lx)
            emb = model.get_speaker_embeddings(dec, lengths=lx)
            for j, i in enumerate(idx):
                out[i] = emb[j]
        return torch.stack(out)
    ref = [r.t() for r in refs]
    for idx, T, Tc, _ in padded_batches([int(s.shape[0]) for s in sources], [int(r.shape[0]) for r in refs]):
        x, lx = padded_batch(src, idx, T, dev)
        c, lc = padded_batch(ref, idx, Tc, dev)
        dec = model.inference(x, c, lengths=lx, cond_lengths=lc)
        emb = model.get_speaker_embeddings(dec, lengths=lx)
        for j, i in enumerate(idx):
            out[i] = emb[j]
    return torch.stack(out)


def _means(rows: np.ndarray) -> Dict[str, float]:
    """The four columns' means (added sequentially in row order) and n of a float64 [n][4] array."""
    s = np.cumsum(rows, axis=0)[-1] / len(rows)
    return {"sim_target": float(s[0]), "sim_source": float(s[1]), "success": float(s[2]),
            "sim_target_source": float(s[3]), "n": len(rows)}


def evaluate_speakers(model, data: Mapping[str, np.ndarray], seed: int = 0, max_pairs: int = 0, device=None,
                      per_pair: bool = False, n_refs: int = 1, bank=None) -> dict:
    """Speaker measures of `model` (an AE) on one set: data = {utterance key: attr-normalised [T, n_mels]} (the set's
    pickle).  Returns {"eer": {"speaker", "content", "mel": {eer, threshold, frr, far, n_target, n_nontarget}},
    "n_utts", "n_short", "conversion": {"sim_target", "sim_source", "success", "sim_target_source" (when n > 0), "n",
    "n_short", "speakers": {target speaker: the four means and n}}}; per_pair adds conversion["pairs"]: [[source,
    reference, sim_target, sim_source, success, sim_target_source], ...].  The module docstring gives the definitions.

    n_refs > 1 (few-shot): each pair keeps its reference and gets n_refs - 1 more (fewshot_pairs), the source is
    converted with the set's pooled code, and sim_target skips all n_refs references; sim_source and
    sim_target_source are as with one.  conversion then also reports "n_refs" and "n_few" (the pairs fewshot_pairs
    dropped), and a per-pair row lists the references: [source, [reference, ...], ...].

    bank (a speaker_bank.SpeakerBank of this model, built from utterances outside `data`: ValueError naming the
    overlap otherwise): conversion also reports bank_identification's id_target, id_source, id_real, n_banked,
    n_unbanked and bank_speakers, by nearest bank code (avc_spk_identify)."""
    cfg = model.config
    if bank is not None:
        from .speaker_bank import check_disjoint
        check_disjoint(bank, data.keys())
    if int(cfg["data_loader"]["frame_size"]) != 1:
        raise ValueError(f"speaker evaluation supports data_loader.frame_size 1 only (got {cfg['data_loader']['frame_size']})")
    if not 1 <= int(n_refs) <= SPK_MAX_EXCLUDE:
        raise ValueError(f"n_refs must lie in [1, {SPK_MAX_EXCLUDE}] (got {n_refs})")
    dev = torch.device(device) if device is not None else next(model.parameters()).device
    min_src, min_ref = min_frames(cfg)
    min_set = max(min_src, min_ref)
    lengths = {u: len(v) for u, v in data.items()}
    utts = [u for u in sorted(data) if lengths[u] >= min_set]
    pairs, n_short_pairs = conversion_pairs(list(data), lengths, seed, max_pairs, min_set, min_ref, min_set)
    if n_refs > 1:
        pairs, n_few = fewshot_pairs(pairs, list(data), lengths, n_refs, seed, min_ref, min_set)
        used = sorted(set(utts) | {u for u, _ in pairs} | {r for _, refs in pairs for r in refs})
    else:
        used = sorted(set(utts) | {u for p in pairs for u in p})
    mels = upload_mels(data, used, dev)
    speakers = sorted({speaker_of(u) for u in utts})
    label = {s: i for i, s in enumerate(speakers)}
    labels = [label[speaker_of(u)] for u in utts]
    res = {"eer": {}, "n_utts": len(utts), "n_short": len(data) - len(utts)}
    with eval_mode(model, dev):
        if utts:
            reps = representations(model, [mels[u] for u in utts])
            for k in REPRESENTATIONS:
                res["eer"][k] = eer(reps[k], labels)
        else:
            res["eer"] = {k: {"eer": None, "threshold": None, "frr": None, "far": None, "n_target": 0,
                              "n_nontarget": 0} for k in REPRESENTATIONS}
        conv = {"n": len(pairs), "n_short": n_short_pairs}
        if n_refs > 1:
            conv.update(n_refs=int(n_refs), n_few=n_few)
        if pairs:
            index = {u: i for i, u in enumerate(utts)}
            emb = reps["speaker"]
            src = [label[speaker_of(u)] for u, _ in pairs]
            ex_u = [index.get(u, -1) for u, _ in pairs]
            if n_refs > 1:
                y = converted_embeddings(model, [mels[u] for u, _ in pairs], [[mels[r] for r in refs] for _, refs in pairs])
                tgt = [label[speaker_of(refs[0])] for _, refs in pairs]
                ex_r = [index.get(refs[0], -1) for _, refs in pairs]
                # one launch: sim_target skips every reference, the other two rows exactly what n_refs = 1 skips
                pad = [-1] * (n_refs - 1)
                ex = ([[index.get(r, -1) for r in refs] for _, refs in pairs] + [[e] + pad for e in ex_u]
                      + [[e] + pad for e in ex_r])
            else:
                y = converted_embeddings(model, [mels[u] for u, _ in pairs], [mels[r] for _, r in pairs])
                tgt = [label[speaker_of(r)] for _, r in pairs]
                ex_r = [index.get(r, -1) for _, r in pairs]
                ex = ex_r + ex_u + ex_r
            both = group_means(torch.cat([y, y, emb[torch.tensor(ex_u, device=dev)]]), tgt + src + tgt,
                               ex, emb, labels).cpu().numpy()
            P = len(pairs)
            st, ss, sts = both[:P], both[P:2 * P], both[2 * P:]
            vals = np.stack([st, ss, (st > ss).astype(np.float64), sts], axis=1)
            conv.update(_means(vals))
            groups: Dict[str, List[int]] = {}
            for i, (_, r) in enumerate(pairs):
                groups.setdefault(speaker_of(r if n_refs == 1 else r[0]), []).append(i)
            conv["speakers"] = {s: _means(vals[rows]) for s, rows in groups.items()}
            if per_pair:
                conv["pairs"] = [[u, list(r) if n_refs > 1 else r, float(v[0]), float(v[1]), bool(v[2]), float(v[3])]
                                 for (u, r), v in zip(pairs, vals)]
            if bank is not None:
                conv.update(bank_identification(bank, y, [speaker_of(u) for u, _ in pairs],
                                                [speaker_of(r if n_refs == 1 else r[0]) for _, r in pairs], emb,
                                                [speaker_of(u) for u in utts]))
        else:
            conv["speakers"] = {}
            if per_pair:
                conv["pairs"] = []
            if bank is not None:
                conv.update(bank_identification(bank, None, [], [], reps["speaker"] if utts else None,
                                                [speaker_of(u) for u in utts]))
    res["conversion"] = conv
    return res
