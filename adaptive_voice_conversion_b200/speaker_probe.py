"""Speaker-classifier probes: how much speaker identity a trained classifier can read from the content code, the speaker
code and the input mel, scored on held-out utterances of the fit set's speakers.  A low accuracy on the content code
next to a high one on the speaker code and the mel is the evidence for AdaIN-VC's claim that instance normalisation
strips the speaker from the content code; unlike the cosine EER of ``speaker_eval``, a probe can find speaker
information in a few low-variance channels or in single frames.

Sets: the probe is fitted on one set (``-probe_set``, default ``train``) and scored on others.  VCTK's ``in_test`` and
LibriTTS's ``dev`` hold unseen utterances of the training speakers; ``out_test`` and LibriTTS's ``test`` hold unseen
speakers only, whose utterances count in ``n_unseen`` (accuracies None when no utterance is left).  A fit set that
shares an utterance key with a scored set is refused (ValueError naming the overlap), as ``speaker_bank.check_disjoint``
refuses a bank.

Fit utterances (``probe_utterances``): the fit set's utterances of at least max(``mcd.min_frames(cfg)``) frames, in
sorted key order; ``rng = random.Random(seed)``; for each speaker in sorted order, ``rng.sample(its utterances,
min(per_speaker_utts, count))``; the union sorted.  The classes are the sorted speakers with at least one fit utterance.
A scored utterance shorter than that minimum counts in ``n_short``.

Representations (the model in eval mode): ``speaker``, ``content`` and ``mel`` are exactly
``speaker_eval.representations()`` (c_out, 2 c_out and 2 n_mels dims per utterance); ``content_frames`` makes every
valid latent frame of the content mean head mu (``AE.get_content_means``, the padded path ``AE.inference`` runs) one
row of c_out dims (``avc_probe_frames``), labelled with its utterance's speaker.

Probe (``fit_probe``), for each representation:
  1. standardise every input dimension with the fit rows' float64 mean and population std, added in ascending row
     order, a std of 0 replaced by 1 (``avc_probe_moments``; ``avc_probe_standardize`` rounds once to float32);
  2. an MLP D -> H -> H -> S with ReLU (H = ``ProbeParams.hidden``, 256), ``avc_linear_fwd`` / ``avc_linear_bwd``;
  3. nn.Linear's default initialisation, U(-1/sqrt(fan_in), 1/sqrt(fan_in)) for weight then bias of each layer in
     order, drawn from a CPU ``torch.Generator`` seeded with ``seed`` and uploaded;
  4. mean softmax cross-entropy (``avc_probe_xent``) and Adam (lr 1e-3, betas 0.9 / 0.999, eps 1e-8, no weight decay,
     no amsgrad, no clipping: ``avc_sqnorm`` / ``avc_adam_step`` over one flat buffer with max_norm = inf);
  5. a fixed number of epochs, 50 for utterance probes and 10 for frame probes; batches of 256 utterances or 4096
     frames, at most N;
  6. epoch e visits ``torch.randperm(N, generator=torch.Generator().manual_seed(seed * 65536 + e))`` in batches and
     drops the short last one, so every step has one shape.
None of these values is tuned.

Scores (``score_probe``) per set and representation, over the scored utterances of the fit speakers:
  * ``acc`` and ``top5``: the true class's rank is the number of classes with a strictly larger score, ties going to
    the lower class index (rank 0 = the decision); an utterance probe scores its logits, ``content_frames`` the sum of
    its frames' log-softmax (``avc_probe_vote``, float64, ascending frames);
  * ``per_speaker``: ``acc`` per true speaker;  ``frame_acc`` (``content_frames``): the share of frames at rank 0;
  * ``fit_acc``: the share of the fit rows (frames for ``content_frames``) at rank 0: the probe's capacity;
  * ``fit_loss``: the mean cross-entropy of the last epoch.
A set also reports ``n``, ``n_unseen``, ``n_short``, ``speakers`` (S), ``chance`` = 1 / S, ``majority`` (the share of
the scored utterances whose speaker is the most frequent fit class, the lowest index among equals), ``fit_set`` and
``n_fit`` (fit utterances).
"""
from __future__ import annotations

import ctypes as C
import random
from dataclasses import dataclass
from typing import Dict, List, Mapping, Optional, Sequence

import numpy as np
import torch

from . import _lib as L
from .evaluate import speaker_of
from .inference import padded_batch, padded_batches
from .mcd import min_frames
from .speaker_eval import representations
from .utils import _stream, eval_mode, upload_mels

REPRESENTATIONS = ("speaker", "content", "content_frames", "mel")


@dataclass(frozen=True)
class ProbeParams:
    hidden: int = 256
    lr: float = 1e-3
    betas: tuple = (0.9, 0.999)
    eps: float = 1e-8
    utt_epochs: int = 50
    frame_epochs: int = 10
    utt_batch: int = 256
    frame_batch: int = 4096


# ------------------------------------------------------------------ selection
def probe_utterances(lengths: Mapping[str, int], min_set: int, per_speaker_utts: int, seed: int = 0) -> List[str]:
    """The fit utterances of a set with lengths[u] = frames of u, as the module docstring defines."""
    if per_speaker_utts < 1:
        raise ValueError(f"per_speaker_utts must be >= 1 (got {per_speaker_utts})")
    by: Dict[str, List[str]] = {}
    for u in sorted(lengths):
        if lengths[u] >= min_set:
            by.setdefault(speaker_of(u), []).append(u)
    rng = random.Random(seed)
    out: List[str] = []
    for s in sorted(by):
        out += rng.sample(by[s], min(per_speaker_utts, len(by[s])))
    return sorted(out)


def split_set(lengths: Mapping[str, int], classes, min_set: int):
    """(scored utterances in sorted key order, n_unseen, n_short) of a set with lengths[u] = frames of u: the
    utterances of at least min_set frames whose speaker is in `classes`; n_unseen counts the long enough ones of other
    speakers, n_short the shorter ones."""
    long = [u for u in sorted(lengths) if lengths[u] >= min_set]
    seen = [u for u in long if speaker_of(u) in classes]
    return seen, len(long) - len(seen), len(lengths) - len(long)


def check_disjoint(fit_keys, scored_keys, fit_name: str = "the probe set", scored_name: str = "a scored set") -> None:
    """ValueError naming the overlap when an utterance key of the fit set is also one of a scored set."""
    both = sorted(set(fit_keys) & set(scored_keys))
    if both:
        raise ValueError(f"{fit_name} shares {len(both)} utterance(s) with {scored_name} (e.g. {both[0]}); a probe "
                         f"scored on its own fit utterances measures nothing")


# ------------------------------------------------------------------ kernels
def _dev_ptr(t: Optional[torch.Tensor]):
    return None if t is None else t.data_ptr()


def _check_rows(x, what):
    if not isinstance(x, torch.Tensor) or x.dim() != 2 or x.dtype != torch.float32 or not x.is_cuda or min(x.shape) < 1:
        raise ValueError(f"{what}: expected float32 [N >= 1, D >= 1] on a CUDA device (got "
                         f"{getattr(x, 'dtype', type(x).__name__)} {tuple(getattr(x, 'shape', ()))})")
    if not bool(torch.isfinite(x).all()):
        raise ValueError(f"{what}: the rows must be finite")
    return x.contiguous()


def frame_rows(mu: torch.Tensor, lengths: torch.Tensor, row_off: torch.Tensor, out: torch.Tensor) -> None:
    """out[row_off[b] + t] = mu[b, :, t] for t < lengths[b] (avc_probe_frames): mu [B, C, T] float32, lengths int32 [B],
    row_off int64 [B], out [rows, C], all on one CUDA device."""
    B, Cc, T = mu.shape
    L.check(L.load().avc_probe_frames(mu.data_ptr(), B, Cc, T, lengths.data_ptr(), row_off.data_ptr(), out.data_ptr(),
                                      _stream(mu.device)), "avc_probe_frames")


def moments(x: torch.Tensor):
    """(mean, std) float64 [D] (device) of the rows of x [N, D] (avc_probe_moments; std 0 -> 1)."""
    n, d = x.shape
    mean = torch.empty(d, dtype=torch.float64, device=x.device)
    std = torch.empty(d, dtype=torch.float64, device=x.device)
    L.check(L.load().avc_probe_moments(x.data_ptr(), n, d, mean.data_ptr(), std.data_ptr(), _stream(x.device)),
            "avc_probe_moments")
    return mean, std


def standardize(x: torch.Tensor, mean: torch.Tensor, std: torch.Tensor, index: torch.Tensor = None,
                out: torch.Tensor = None) -> torch.Tensor:
    """(x[index] - mean) / std rounded once to float32 (avc_probe_standardize); index int64 [rows] or None = all."""
    rows = x.shape[0] if index is None else index.shape[0]
    out = torch.empty(rows, x.shape[1], device=x.device) if out is None else out
    L.check(L.load().avc_probe_standardize(x.data_ptr(), _dev_ptr(index), rows, x.shape[1], mean.data_ptr(),
                                           std.data_ptr(), out.data_ptr(), _stream(x.device)), "avc_probe_standardize")
    return out


def xent(logits: torch.Tensor, labels: torch.Tensor, scale: float = 1.0, dlogits: torch.Tensor = None,
         loss_sum: torch.Tensor = None, scratch: torch.Tensor = None):
    """(loss float64 [R], rank int32 [R]) of logits [R, S] against int32 labels (avc_probe_xent); dlogits [R, S] and
    loss_sum (a float64 element, with a scratch of L.PROBE_SUM_SCRATCH doubles) are written when given."""
    R, S = logits.shape
    loss = torch.empty(R, dtype=torch.float64, device=logits.device)
    rank = torch.empty(R, dtype=torch.int32, device=logits.device)
    L.check(L.load().avc_probe_xent(logits.data_ptr(), labels.data_ptr(), R, S, scale, loss.data_ptr(), _dev_ptr(dlogits),
                                    rank.data_ptr(), _dev_ptr(scratch), _dev_ptr(loss_sum), _stream(logits.device)),
            "avc_probe_xent")
    return loss, rank


def vote(logits: torch.Tensor, offsets: torch.Tensor, labels: torch.Tensor):
    """(scores float64 [U, S], rank int32 [U]) of the frame logits [R, S] grouped by offsets int64 [U + 1]
    (avc_probe_vote)."""
    S = logits.shape[1]
    U = offsets.shape[0] - 1
    scores = torch.empty(U, S, dtype=torch.float64, device=logits.device)
    rank = torch.empty(U, dtype=torch.int32, device=logits.device)
    L.check(L.load().avc_probe_vote(logits.data_ptr(), S, offsets.data_ptr(), U, labels.data_ptr(), scores.data_ptr(),
                                    rank.data_ptr(), _stream(logits.device)), "avc_probe_vote")
    return scores, rank


# ------------------------------------------------------------------ the MLP
def layer_shapes(D: int, H: int, S: int):
    """[(out, in)] of the three linear layers."""
    return [(H, D), (H, H), (S, H)]


def init_params(D: int, S: int, params: ProbeParams, seed: int) -> torch.Tensor:
    """The flat float32 parameter vector [W1 b1 W2 b2 W3 b3] (host) with nn.Linear's default initialisation drawn from
    a CPU generator seeded with `seed`."""
    g = torch.Generator().manual_seed(int(seed))
    parts = []
    for n, k in layer_shapes(D, params.hidden, S):
        bound = 1.0 / k ** 0.5
        parts.append(torch.empty(n * k).uniform_(-bound, bound, generator=g))
        parts.append(torch.empty(n).uniform_(-bound, bound, generator=g))
    return torch.cat(parts)


def unflatten(flat: torch.Tensor, D: int, H: int, S: int) -> List[torch.Tensor]:
    """Views [W1, b1, W2, b2, W3, b3] of a flat parameter (or gradient) vector."""
    out, o = [], 0
    for n, k in layer_shapes(D, H, S):
        out.append(flat[o:o + n * k].view(n, k))
        o += n * k
        out.append(flat[o:o + n])
        o += n
    return out


class _Mlp:
    """The probe's forward and backward passes for batches of up to `rows` rows, buffers allocated once."""

    def __init__(self, D, H, S, rows, dev):
        self.D, self.H, self.S = D, H, S
        self.h1 = torch.empty(rows, H, device=dev)
        self.h2 = torch.empty(rows, H, device=dev)
        self.z = torch.empty(rows, S, device=dev)
        self.dz = torch.empty(rows, S, device=dev)
        self.dh2 = torch.empty(rows, H, device=dev)
        self.dh1 = torch.empty(rows, H, device=dev)
        self.lib = L.load()

    def forward(self, P, x, n):
        """z[:n] = MLP(x[:n]) with the parameter views P."""
        st = _stream(x.device)
        for (w, b), inp, out, relu in (((P[0], P[1]), x, self.h1, 1), ((P[2], P[3]), self.h1, self.h2, 1),
                                       ((P[4], P[5]), self.h2, self.z, 0)):
            N, K = w.shape
            d = L.LinearDesc(B=n, N=N, K=K, relu=relu, x=inp.data_ptr(), x_bstride=K, w=w.data_ptr(), bias=b.data_ptr(),
                             out=out.data_ptr(), out_bstride=N)
            L.check(self.lib.avc_linear_fwd(C.byref(d), st), "avc_linear_fwd")
        return self.z[:n]

    def backward(self, P, G, x, n):
        """G += the gradients of the parameters P for the upstream gradient in self.dz[:n] (G zeroed by the caller)."""
        st = _stream(x.device)
        for (w, b, dw, db), inp, y_act, dy, dx, relu in (
                ((P[4], P[5], G[4], G[5]), self.h2, None, self.dz, self.dh2, 0),
                ((P[2], P[3], G[2], G[3]), self.h1, self.h2, self.dh2, self.dh1, 1),
                ((P[0], P[1], G[0], G[1]), x, self.h1, self.dh1, None, 1)):
            N, K = w.shape
            d = L.LinearDesc(B=n, N=N, K=K, relu=relu, x=inp.data_ptr(), x_bstride=K, w=w.data_ptr(),
                             y_act=_dev_ptr(y_act), dy=dy.data_ptr(), dy_bstride=N, dx=_dev_ptr(dx), dw=dw.data_ptr(),
                             db=db.data_ptr())
            L.check(self.lib.avc_linear_bwd(C.byref(d), st), "avc_linear_bwd")


@dataclass
class Probe:
    """A fitted probe: flat parameters (device), the standardisation (float64, device), per-epoch mean losses."""
    flat: torch.Tensor
    mean: torch.Tensor
    std: torch.Tensor
    losses: List[float]
    D: int
    H: int
    S: int

    def views(self):
        return unflatten(self.flat, self.D, self.H, self.S)


def epoch_order(n: int, seed: int, epoch: int) -> torch.Tensor:
    """The visiting order of epoch `epoch` (CPU int64)."""
    return torch.randperm(n, generator=torch.Generator().manual_seed(int(seed) * 65536 + int(epoch)))


def fit_probe(x: torch.Tensor, labels, params: ProbeParams = ProbeParams(), seed: int = 0, n_classes: int = None,
              frames: bool = False) -> Probe:
    """Fits the probe of the module docstring to the rows x [N, D] (float32, CUDA) with integer labels in
    [0, n_classes) (default: the largest label + 1); frames selects the frame probe's epochs and batch."""
    x = _check_rows(x, "fit_probe")
    N, D = x.shape
    dev = x.device
    lab = torch.as_tensor(np.asarray(labels, np.int64)) if not isinstance(labels, torch.Tensor) else labels.cpu().long()
    if lab.shape != (N,) or int(lab.min()) < 0:
        raise ValueError(f"fit_probe: expected {N} labels >= 0 (got {tuple(lab.shape)})")
    n_classes = int(lab.max()) + 1 if n_classes is None else int(n_classes)
    if not 1 <= n_classes <= L.PROBE_MAX_CLASSES or int(lab.max()) >= n_classes:
        raise ValueError(f"fit_probe: {n_classes} classes (labels up to {int(lab.max())}); 1 to "
                         f"{L.PROBE_MAX_CLASSES} are supported")
    lab = lab.to(torch.int32).to(dev)
    E = params.frame_epochs if frames else params.utt_epochs
    Bt = min(params.frame_batch if frames else params.utt_batch, N)
    steps = N // Bt
    H, S = params.hidden, n_classes
    lib = L.load()
    st = _stream(dev)
    mean, std = moments(x)
    flat = init_params(D, S, params, seed).to(dev)
    n_par = flat.numel()
    grad = torch.zeros(n_par, device=dev)
    m, v, vmax = (torch.zeros(n_par, device=dev) for _ in range(3))
    # avc_adam_step's layout: [2] grad scale, [3] lr, [4:6] betas, [6] eps, [7] weight decay, [8] max_norm (inf: no
    # clipping), [9] amsgrad
    hp = torch.tensor([0.0, 0.0, 1.0, params.lr, params.betas[0], params.betas[1], params.eps, 0.0, float("inf"), 0.0],
                      dtype=torch.float32, device=dev)
    step = torch.zeros(1, device=dev)
    sq = torch.zeros(1, device=dev)
    sq_scratch = torch.empty(1024, device=dev)
    sums = torch.zeros(E, max(steps, 1), dtype=torch.float64, device=dev)
    scratch = torch.empty(L.PROBE_SUM_SCRATCH, dtype=torch.float64, device=dev)
    P, G = unflatten(flat, D, H, S), unflatten(grad, D, H, S)
    net = _Mlp(D, H, S, Bt, dev)
    xb = torch.empty(N, D, device=dev)
    for e in range(E):
        order = epoch_order(N, seed, e)[:steps * Bt].to(dev)
        standardize(x, mean, std, order, out=xb[:steps * Bt])
        lab_e = lab[order]
        for k in range(steps):
            xk = xb[k * Bt:(k + 1) * Bt]
            z = net.forward(P, xk, Bt)
            xent(z, lab_e[k * Bt:(k + 1) * Bt], 1.0 / Bt, dlogits=net.dz, loss_sum=sums[e, k:k + 1], scratch=scratch)
            L.check(lib.avc_fill_zero(grad.data_ptr(), n_par * 4, st), "avc_fill_zero")
            net.backward(P, G, xk, Bt)
            L.check(lib.avc_sqnorm(grad.data_ptr(), n_par, sq_scratch.data_ptr(), sq.data_ptr(), st), "avc_sqnorm")
            L.check(lib.avc_adam_step(flat.data_ptr(), grad.data_ptr(), m.data_ptr(), v.data_ptr(), vmax.data_ptr(), n_par,
                                      hp.data_ptr(), sq.data_ptr(), step.data_ptr(), st), "avc_adam_step")
    losses = [float(r) for r in (sums.cpu().numpy().sum(axis=1) / (steps * Bt))] if steps else []
    return Probe(flat, mean, std, losses, D, H, S)


def _logit_chunks(probe: Probe, x: torch.Tensor, bounds: Sequence[int]):
    """Yields (first row, logits) of the standardised rows x in the row ranges bounds[i]..bounds[i + 1]."""
    P = probe.views()
    rows = max(b - a for a, b in zip(bounds[:-1], bounds[1:]))
    net = _Mlp(probe.D, probe.H, probe.S, rows, x.device)
    for a, b in zip(bounds[:-1], bounds[1:]):
        if b > a:
            yield a, net.forward(P, x[a:b], b - a)


def _chunk_bounds(offsets: Sequence[int], max_rows: int) -> List[int]:
    """Row boundaries at utterance offsets, each chunk at most max_rows rows unless one utterance is longer."""
    out = [0]
    for a, b in zip(offsets[:-1], offsets[1:]):
        if b - out[-1] > max_rows and a > out[-1]:
            out.append(a)
    if out[-1] != offsets[-1]:
        out.append(offsets[-1])
    return out


def score_probe(probe: Probe, x: torch.Tensor, labels, offsets: Sequence[int] = None, max_rows: int = 65536) -> dict:
    """Ranks of the rows x [N, D] (float32, CUDA) under `probe` against integer labels: {"rank": int32 [N] (host)}; with
    utterance offsets (U + 1 ascending row indices from 0 to N) the frame votes too: {"rank": per-utterance ranks of
    the votes, "frame_rank": per-row ranks}; labels are then per utterance."""
    x = _check_rows(x, "score_probe")
    N, dev = x.shape[0], x.device
    if x.shape[1] != probe.D:
        raise ValueError(f"score_probe: {x.shape[1]} dims; the probe takes {probe.D}")
    xs = standardize(x, probe.mean, probe.std)
    lab = torch.as_tensor(np.asarray(labels, np.int64)).to(torch.int32).to(dev)
    if offsets is None:
        if lab.shape[0] != N:
            raise ValueError(f"score_probe: {lab.shape[0]} labels for {N} rows")
        rank = torch.empty(N, dtype=torch.int32, device=dev)
        bounds = list(range(0, N, max_rows)) + [N]
        for a, z in _logit_chunks(probe, xs, bounds):
            rank[a:a + z.shape[0]] = xent(z, lab[a:a + z.shape[0]])[1]
        return {"rank": rank.cpu().numpy()}
    offsets = [int(o) for o in offsets]
    U = len(offsets) - 1
    if U < 1 or offsets[0] != 0 or offsets[-1] != N or any(b < a for a, b in zip(offsets[:-1], offsets[1:])):
        raise ValueError(f"score_probe: offsets must ascend from 0 to {N}")
    if lab.shape[0] != U:
        raise ValueError(f"score_probe: {lab.shape[0]} labels for {U} utterances")
    row_lab = torch.repeat_interleave(lab, torch.tensor(np.diff(offsets), device=dev))
    frame_rank = torch.empty(N, dtype=torch.int32, device=dev)
    rank = torch.empty(U, dtype=torch.int32, device=dev)
    first = {o: i for i, o in reversed(list(enumerate(offsets)))}    # the first utterance starting at a row
    last = {o: i for i, o in enumerate(offsets)}                     # the last
    for a, z in _logit_chunks(probe, xs, _chunk_bounds(offsets, max_rows)):
        b = a + z.shape[0]
        frame_rank[a:b] = xent(z, row_lab[a:b])[1]
        u0, u1 = first[a], last[b]
        off = torch.tensor([o - a for o in offsets[u0:u1 + 1]], dtype=torch.int64, device=dev)
        rank[u0:u1] = vote(z, off, lab[u0:u1])[1]
    return {"rank": rank.cpu().numpy(), "frame_rank": frame_rank.cpu().numpy()}


# ------------------------------------------------------------------ features of a set
def features(model, mels: Sequence[torch.Tensor]) -> Dict[str, object]:
    """{speaker, content, mel: [N, D] (representations()), content_frames: [sum L_i, c_out] (device), offsets: [N + 1]
    row offsets (host ints)} of the attr-normalised mels [T_i, n_mels] (device, each at least max(min_frames) long).
    The model must be in eval mode."""
    out = dict(representations(model, mels))
    dev = mels[0].device
    lens = [int(m.shape[0]) for m in mels]
    frames = [m.t() for m in mels]
    held, lat = [], [0] * len(mels)
    for idx, T, _, _ in padded_batches(lens, lens):
        x, lx = padded_batch(frames, idx, T, dev)
        mu, ll = model.get_content_means(x, lengths=lx)
        held.append((idx, mu, ll))
        for j, n in zip(idx, ll.cpu().tolist()):
            lat[j] = int(n)
    offsets = [0]
    for n in lat:
        offsets.append(offsets[-1] + n)
    rows = torch.empty(offsets[-1], int(held[0][1].shape[1]), device=dev)
    for idx, mu, ll in held:
        frame_rows(mu.contiguous(), ll, torch.tensor([offsets[i] for i in idx], dtype=torch.int64, device=dev), rows)
    out["content_frames"] = rows
    out["offsets"] = offsets
    return out


# ------------------------------------------------------------------ evaluation
def _accuracy(rank: np.ndarray, k: int = 1) -> Optional[float]:
    return float(np.mean(rank < k)) if len(rank) else None


def evaluate_probe(model, fit_data: Mapping[str, np.ndarray], data: Mapping[str, Mapping[str, np.ndarray]], seed: int = 0,
                   per_speaker_utts: int = 64, device=None, params: ProbeParams = ProbeParams(),
                   fit_name: str = "the probe set") -> Dict[str, dict]:
    """{set: probe entry} of `model` (an AE): the four probes fitted once on fit_data ({utterance key: attr-normalised
    [T, n_mels]}) and scored on every set of data ({set name: such a mapping}); the module docstring gives the
    definitions.  Each entry holds n, n_unseen, n_short, speakers, chance, majority, fit_set, n_fit and, per
    representation, {acc, top5, per_speaker, fit_acc, fit_loss[, frame_acc]} (accuracies None when n = 0)."""
    cfg = model.config
    for name, d in data.items():
        check_disjoint(fit_data.keys(), d.keys(), fit_name, name)
    if int(cfg["data_loader"]["frame_size"]) != 1:
        raise ValueError(f"speaker probes support data_loader.frame_size 1 only (got {cfg['data_loader']['frame_size']})")
    dev = torch.device(device) if device is not None else next(model.parameters()).device
    min_set = max(min_frames(cfg))
    fit_utts = probe_utterances({u: len(v) for u, v in fit_data.items()}, min_set, per_speaker_utts, seed)
    if not fit_utts:
        raise ValueError(f"{fit_name} has no utterance of at least {min_set} frames")
    speakers = sorted({speaker_of(u) for u in fit_utts})
    label = {s: i for i, s in enumerate(speakers)}
    S = len(speakers)
    if S > L.PROBE_MAX_CLASSES:
        raise ValueError(f"{fit_name} has {S} speakers; a probe supports at most {L.PROBE_MAX_CLASSES}")
    fit_lab = np.array([label[speaker_of(u)] for u in fit_utts], np.int64)
    counts = np.bincount(fit_lab, minlength=S)
    major = int(np.argmax(counts))
    res: Dict[str, dict] = {}
    with eval_mode(model, dev):
        fit = features(model, list(upload_mels(fit_data, fit_utts, dev).values()))
        frame_lab = np.repeat(fit_lab, np.diff(fit["offsets"]))
        probes, fit_part = {}, {}
        for k in REPRESENTATIONS:
            fr = k == "content_frames"
            probes[k] = fit_probe(fit[k], frame_lab if fr else fit_lab, params, seed, n_classes=S, frames=fr)
            r = score_probe(probes[k], fit[k], frame_lab if fr else fit_lab)["rank"]
            fit_part[k] = {"fit_acc": _accuracy(r), "fit_loss": probes[k].losses[-1] if probes[k].losses else None}
        del fit
        for name, d in data.items():
            seen, n_unseen, n_short = split_set({u: len(v) for u, v in d.items()}, label, min_set)
            entry = {"n": len(seen), "n_unseen": n_unseen, "n_short": n_short, "speakers": S, "chance": 1.0 / S, "fit_set": fit_name, "n_fit": len(fit_utts)}
            lab = np.array([label[speaker_of(u)] for u in seen], np.int64)
            entry["majority"] = float(np.mean(lab == major)) if len(seen) else None
            if seen:
                mels = upload_mels(d, seen, dev)
                feats = features(model, [mels[u] for u in seen])
            for k in REPRESENTATIONS:
                e = {"acc": None, "top5": None, "per_speaker": {}}
                if k == "content_frames":
                    e["frame_acc"] = None
                if seen:
                    if k == "content_frames":
                        sc = score_probe(probes[k], feats[k], lab, offsets=feats["offsets"])
                        e["frame_acc"] = _accuracy(sc["frame_rank"])
                    else:
                        sc = score_probe(probes[k], feats[k], lab)
                    e["acc"], e["top5"] = _accuracy(sc["rank"]), _accuracy(sc["rank"], 5)
                    e["per_speaker"] = {s: _accuracy(sc["rank"][lab == label[s]]) for s in speakers
                                        if (lab == label[s]).any()}
                e.update(fit_part[k])
                entry[k] = e
            res[name] = entry
    return res
