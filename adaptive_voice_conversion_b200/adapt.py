"""Speaker adaptation: fine-tune the decoder and one speaker code on that speaker's recordings, with both encoders frozen.

What is trained: every decoder parameter (with ``Decoder.sn`` its ``weight_orig`` values, one power iteration per
forward as in training) and one speaker code c (float32 [c_out]), initialised to the speaker's pooled bank code over the
adaptation clips (``build_bank``).  The content encoder stays as it is because every source still goes through it; the
speaker encoder stays so that bank fingerprints remain valid.

One step (``AdaptTrainer``): B crops of segment_size frames of the speaker's clips (``DeviceSegments``), the content
encoder without saving anything (``content_fwd(train=False)``), z = mu + exp(ls/2) eps drawn as the training step draws
it, the decoder with every sample's AdaIN conditioned on c, loss = lambda_rec * L1 (``avc_vae_loss``; the KL term
reaches no trainable value), the decoder's backward without dz, the code gradient sum_b demb[b] (``avc_bias_grad`` at
T = 1), then clip + Adam over the trainable values only.  No speaker encoder, no encoder backward.

Optimizer layout: the decoder's parameters (registration order), then c, are re-homed into ONE flat buffer
(``AdaptParams``) with gradient, m, v and vmax buffers of the same shape, so a step's update is one ``avc_sqnorm`` and
one ``avc_adam_step`` over exactly the trainable values.  Weight decay (the config's, L2 as in training) applies to c as
well.  The encoders and their storage are never written.

The held-out check scores the conversion path (content mean, no noise, ``AE.inference_from_embeddings`` in
``padded_batches``' grid) with the speaker's code: per utterance the mean |dec - x| over its valid frames
(``avc_rec_loss_varlen``), then the mean over utterances.
"""
from __future__ import annotations

import json
from typing import List, Mapping, Sequence

import numpy as np
import torch
import torch.nn as nn

from . import _lib as L
from .data_utils import DeviceSegments
from .engine import A4
from .optim import FusedAdam
from .trainer import FusedTrainer
from .utils import _stream, eval_mode

FORMAT = "avc-adapt-1"
LOG_EVERY = 100


class _Code(nn.Module):
    def __init__(self, code: torch.Tensor):
        super().__init__()
        self.code = nn.Parameter(code.detach().to(torch.float32).reshape(-1).clone())


class AdaptParams(nn.Module):
    """The trainable set of an adaptation: `model`'s decoder (shared, not copied) and one speaker code.
    ``flatten_parameters`` re-homes the decoder's parameters, then the code, into one flat buffer (what FusedAdam steps
    over); the encoders keep their own storage.  (The code sits in a child module registered after the decoder: a
    module lists its own parameters before its children's.)"""

    def __init__(self, model, code: torch.Tensor):
        super().__init__()
        self.decoder = model.decoder
        self.speaker = _Code(code)
        self._flat = None

    @property
    def code(self) -> nn.Parameter:
        return self.speaker.code

    def flatten_parameters(self) -> torch.Tensor:
        params = list(self.parameters())
        flat = torch.empty(sum(p.numel() for p in params), dtype=torch.float32, device=params[0].device)
        off = 0
        for p in params:
            n = p.numel()
            flat[off:off + n].copy_(p.data.reshape(-1))
            p.data = flat[off:off + n].view(p.shape)
            off += n
        self._flat = flat
        return flat


class AdaptAdam(FusedAdam):
    """FusedAdam over an AdaptParams: gradient views exist for the decoder's parameters and the code only."""

    def named_grad_views(self, model):
        return {name: self.grad_views[p] for name, p in model.named_parameters() if p in self.grad_views}


def make_trainer(model, code: torch.Tensor, config: dict, lr=None) -> "AdaptTrainer":
    """An AdaptTrainer of `model` (an AE on the GPU) starting from `code`: re-homes the decoder (before any pointer table
    or graph of the trainer is built) and sets up Adam from config["optimizer"], `lr` overriding its rate.  No
    optimizer state of the base run is loaded."""
    o = config["optimizer"]
    params = AdaptParams(model, code.to(next(model.parameters()).device))
    params.flatten_parameters()
    opt = AdaptAdam(params, lr=o["lr"] if lr is None else float(lr), betas=(o["beta1"], o["beta2"]), amsgrad=o["amsgrad"],
                    weight_decay=o["weight_decay"], max_norm=o["grad_norm"])
    return AdaptTrainer(model, opt, config, params)


class AdaptTrainer(FusedTrainer):
    """FusedTrainer's step machinery (CUDA-graph capture on the third step of a shape and replay, AVC_GRAPH=0 eager,
    the 16-byte report block, losses_async) around the adaptation step of the module docstring.  ``step(x, lambda_kl)``
    as in training; lambda_kl reaches no trainable value.  ``code`` is the trained code (a view of the flat buffer)."""

    def __init__(self, model, opt: AdaptAdam, config: dict, params: AdaptParams):
        self.params = params
        self.code = params.code
        self.code_grad = opt.grad_views[params.code]
        super().__init__(model, opt, config)

    def _fwd_bwd(self, x: torch.Tensor, eps):
        eng, P, G = self.eng, self.P, self.G
        self.opt.zero_grad()
        self._sn_fwd()
        mu4, ls4, _ = eng.content_fwd(P, x, False)
        if eps is None:
            eps = torch.randn((mu4.B, mu4.C, mu4.T), dtype=torch.float32, device=self.dev)
        mu, ls, z4 = eng.reparam_fwd(mu4, ls4, eps)
        B, c_out = x.shape[0], self.code.numel()
        emb = self.code.detach().view(1, c_out).expand(B, c_out)   # every sample's AdaIN reads the one code
        dec4, cd = eng.decoder_fwd(P, z4, emb, True)
        dec = eng.unpack_a4(dec4)
        ddec, dmu, dls = torch.empty_like(dec), torch.empty_like(mu), torch.empty_like(ls)
        self.n_rec, self.n_lat = dec.numel(), mu.numel()
        L.check(self.lib.avc_vae_loss(dec.data_ptr(), x.data_ptr(), dec.numel(), mu.data_ptr(), ls.data_ptr(), mu.numel(),
                                      self.opt.hp.data_ptr(), self.sums.data_ptr(), self.loss_part.data_ptr(), ddec.data_ptr(),
                                      dmu.data_ptr(), dls.data_ptr(), eng.stream), "vae_loss")
        ddec4 = A4.empty(dec4.B, dec4.C, dec4.T, self.dev)
        eng.pack_a4(ddec, ddec4)
        eng.wgrad_stream = self._wgs
        try:
            _, demb = eng.decoder_bwd(P, G, cd, ddec4, need_dz=False)
            # d/dc of sum_b AdaIN_b(c) = sum_b demb[b]: an A4 tensor of T = 1 is planar [B][c_out]
            L.check(self.lib.avc_bias_grad(demb.data_ptr(), c_out, self.code_grad.data_ptr(), B, c_out, 1, eng.stream),
                    "bias_grad[code]")
            eng.join_wgrad()
            eng.flush_wgrad()
        finally:
            eng.wgrad_stream = None
            eng._wg_keep.clear()
        if self.sn:
            eng.spectral_norm_bwd(P, G)
        return mu, ls, emb, dec

    def _update(self):
        self.opt.step()
        if not self.sn:   # with sn the decoder's packs are made from W_bar at the start of the next forward
            self.eng.pack_weights(self.P, need_dgrad=True, prefixes=("decoder.",))


# ----------------------------------------------------------------------------- clips
def crop_index(lengths: Mapping[str, int], segment_size: int):
    """(index, used, skipped): one (clip, t) entry for every start t in [0, T - segment_size] of every clip of at least
    segment_size frames, clips in the mapping's order; the clips used and the shorter ones skipped, in that order."""
    index, used, skipped = [], [], []
    for u, T in lengths.items():
        if int(T) < segment_size:
            skipped.append(u)
            continue
        used.append(u)
        index.extend((u, t) for t in range(int(T) - segment_size + 1))
    return index, used, skipped


def check_disjoint(adapt: Sequence[str], held_out: Sequence[str], what: str = "utterance") -> None:
    """ValueError naming the overlap when a held-out clip is also an adaptation clip (the same path or utterance id)."""
    both = sorted(set(adapt) & set(held_out))
    if both:
        raise ValueError(f"{len(both)} held-out {what}(s) are also adaptation clips (e.g. {both[0]}); a held-out check "
                         f"on adaptation data measures nothing")


def segments(mels: Mapping[str, object], config: dict, batch_size: int, seed: int, device):
    """(DeviceSegments over the crop index, used, skipped) of the clips `mels` ({id: attr-normalised [T, n_mels]}).
    Every batch holds exactly min(batch_size, crops) crops: an epoch's last, short batch is dropped (drop_last), so that
    every step has one shape, replays one CUDA graph and its loss is a mean over the same number of frames.
    ValueError before any launch when no clip is long enough, or frame_size is not 1."""
    dl = config["data_loader"]
    if int(dl["frame_size"]) != 1:
        raise ValueError(f"speaker adaptation supports data_loader.frame_size 1 only (got {dl['frame_size']})")
    seg = int(dl["segment_size"])
    index, used, skipped = crop_index({u: int(m.shape[0]) for u, m in mels.items()}, seg)
    if not used:
        raise ValueError(f"no adaptation clip has segment_size = {seg} frames ({len(skipped)} shorter ones skipped)")
    data = {u: _host(mels[u]) for u in used}
    ds = DeviceSegments(data, index, seg, 1, min(batch_size, len(index)), config["ContentEncoder"]["c_in"], device=device,
                        seed=seed, drop_last=True)
    return ds, used, skipped


def _host(m) -> np.ndarray:
    if isinstance(m, torch.Tensor):
        m = m.detach().cpu().numpy()
    return np.ascontiguousarray(m, np.float32)


# ----------------------------------------------------------------------------- held-out check
def rec_loss_varlen(dec: torch.Tensor, x: torch.Tensor, lengths: torch.Tensor) -> torch.Tensor:
    """float64 [B]: sample b's sum |dec - x| over its first lengths[b] frames of planar padded dec and x [B, C, T]
    (avc_rec_loss_varlen; frames past a length are never read)."""
    if (dec.shape != x.shape or dec.dim() != 3 or dec.dtype != torch.float32 or x.dtype != torch.float32
            or not dec.is_cuda or x.device != dec.device):
        raise ValueError(f"rec_loss_varlen: dec and x must be float32 [B, C, T] on one CUDA device, got "
                         f"{dec.dtype} {tuple(dec.shape)} and {x.dtype} {tuple(x.shape)}")
    B, Cc, T = dec.shape
    lh = lengths.cpu()
    if tuple(lh.shape) != (B,) or int(lh.min()) < 1 or int(lh.max()) > T:
        raise ValueError(f"rec_loss_varlen: lengths must be [{B}] in [1, {T}]")
    dec, x = dec.contiguous(), x.contiguous()
    lt = lengths.to(device=dec.device, dtype=torch.int32)
    out = torch.empty(B, dtype=torch.float64, device=dec.device)
    d = L.RecVarlenDesc(B=B, C=Cc, T=T, dec=dec.data_ptr(), x=x.data_ptr(), lengths=lt.data_ptr(), out=out.data_ptr())
    L.check(L.load().avc_rec_loss_varlen(d, _stream(dec.device)), "avc_rec_loss_varlen")
    return out


def heldout_rec(model, mels: Mapping[str, object], code: torch.Tensor) -> dict:
    """{"rec", "n", "n_skipped", "skipped"} of the held-out clips `mels` ({id: attr-normalised [T, n_mels]}) converted
    with `code`: the conversion path in padded_batches' grid, per utterance the mean |dec - x| over its valid frames,
    then the mean over utterances (float64, in sorted id order).  Clips shorter than the model accepts are skipped."""
    from .inference import padded_batch, padded_batches
    from .mcd import min_frames
    dev = code.device
    min_src = min_frames(model.config)[0]
    ids = sorted(mels)
    keep = [u for u in ids if int(mels[u].shape[0]) >= min_src]
    skipped = [u for u in ids if int(mels[u].shape[0]) < min_src]
    res = {"rec": None, "n": len(keep), "n_skipped": len(skipped), "skipped": skipped}
    if not keep:
        return res
    lens = [int(mels[u].shape[0]) for u in keep]
    frames = [(m if isinstance(m, torch.Tensor) else torch.from_numpy(_host(m))).t() for m in (mels[u] for u in keep)]
    per = np.zeros(len(keep))
    with eval_mode(model, dev):
        for idx, T, _, _ in padded_batches(lens, lens):
            x, lx = padded_batch(frames, idx, T, dev)
            n_mels = x.shape[1]
            emb = code.detach().reshape(1, -1).expand(len(idx), -1).contiguous()
            dec = model.inference_from_embeddings(x, emb, lengths=lx)
            sums = rec_loss_varlen(dec[:, :, :T], x, lx).cpu().numpy()
            for j, i in enumerate(idx):
                per[i] = sums[j] / (n_mels * lens[i])
    res["rec"] = float(np.cumsum(per)[-1] / len(per))
    return res


# ----------------------------------------------------------------------------- the run
def train(trainer: AdaptTrainer, batches, steps: int, log_every: int = LOG_EVERY) -> List[dict]:
    """`steps` adaptation steps on the iterator `batches`; returns [{"step", "loss_rec", "grad_norm"}] of the first step,
    every log_every-th and the last.  Step i's report is read after step i + 1 is enqueued (Solver.run_steps'
    pattern), so the GPU never waits for the host; every read also checks the tensor-core status word."""
    log, pending = [], None

    def finish(p):
        i, get = p
        loss_rec, _, grad_norm = get()
        if i % log_every == 0 or i == steps - 1:
            log.append({"step": i, "loss_rec": loss_rec, "grad_norm": grad_norm})

    for i in range(steps):
        trainer.step(next(batches), 0.0)
        get = trainer.losses_async()
        if pending is not None:
            finish(pending)
        pending = (i, get)
    if pending is not None:
        finish(pending)
    return log


def adapt(model, config: dict, speaker: str, mels: Mapping[str, object], steps: int, lr=None, batch_size=None,
          seed: int = 0, heldout: Mapping[str, object] = None, mcd=None) -> dict:
    """Adapt `model` (an AE on the GPU, modified in place: its decoder) to `speaker` on the clips `mels` ({id:
    attr-normalised [T, n_mels]}).  Returns {"bank", "code", "report"}: a one-speaker SpeakerBank of the adapted code
    (its clips are the ones used), the code, and the run's report (``report``'s schema).  heldout: clips scored before
    and after (``heldout_rec``).  mcd(model, code) -> dict: a second held-out measure, also run before and after."""
    from .speaker_bank import SpeakerBank, build_bank, fingerprint
    dev = next(model.parameters()).device
    B = int(config["data_loader"]["batch_size"] if batch_size is None else batch_size)
    if steps < 1 or B < 1:
        raise ValueError(f"need steps >= 1 and batch_size >= 1 (got {steps}, {B})")
    ds, used, skipped = segments(mels, config, B, seed, dev)   # raises before any launch
    c_out = config["SpeakerEncoder"]["c_out"]
    trainer = make_trainer(model, torch.zeros(c_out, device=dev), config, lr)
    code0 = build_bank(model, {u: mels[u] for u in used}, speaker_of=lambda u: speaker).codes[0]
    with torch.no_grad():
        trainer.code.copy_(code0)
    before = {} if heldout is None else {"rec": heldout_rec(model, heldout, code0)}
    if mcd is not None:
        before["mcd"] = mcd(model, code0)
    torch.manual_seed(seed)
    log = train(trainer, iter(ds), steps)
    code = trainer.code.detach().clone()
    after = {} if heldout is None else {"rec": heldout_rec(model, heldout, code)}
    if mcd is not None:
        after["mcd"] = mcd(model, code)
    bank = SpeakerBank([speaker], code.reshape(1, -1), [len(used)], [sorted(used)], fingerprint(model), len(skipped))
    g = trainer.opt.param_groups[0]
    settings = {"steps": int(steps), "lr": float(g["lr"]), "batch_size": ds.sampler.batch_size, "seed": int(seed),
                "segment_size": int(config["data_loader"]["segment_size"]), "betas": [float(b) for b in g["betas"]],
                "weight_decay": float(g["weight_decay"]), "grad_norm": float(trainer.opt.max_norm),
                "amsgrad": bool(g["amsgrad"]), "lambda_rec": float(config["lambda"]["lambda_rec"]),
                "precision": trainer.eng.precision, "n_trainable": int(trainer.opt.flat_p.numel())}
    report = make_report(speaker, settings, used, skipped, ds.sampler.n, log, before, after)
    return {"bank": bank, "code": code, "report": report}


REPORT_KEYS = ("format", "speaker", "settings", "clips", "losses", "heldout")


def make_report(speaker, settings, used, skipped, n_entries, losses, before, after) -> dict:
    """The JSON document of a run: {"format", "speaker", "settings", "clips": {"used", "skipped", "n_entries"},
    "losses": [{"step", "loss_rec", "grad_norm"}], "heldout": {"before", "after"} or null}.  before / after map a
    measure ("rec": heldout_rec's dict, "mcd": evaluate_mcd's) to its result."""
    return {"format": FORMAT, "speaker": str(speaker), "settings": dict(settings),
            "clips": {"used": list(used), "skipped": list(skipped), "n_entries": int(n_entries)},
            "losses": list(losses), "heldout": {"before": before, "after": after} if (before or after) else None}


def save(result: dict, model, out: str) -> None:
    """<out>.ckpt (the full AE state_dict), <out>.bank.pt and <out>.json."""
    torch.save({k: v.detach().clone() for k, v in model.state_dict().items()}, f"{out}.ckpt")
    result["bank"].save(f"{out}.bank.pt")
    with open(f"{out}.json", "w") as f:
        json.dump(result["report"], f, indent=1)
