"""Reference-shaped model API on top of the sm_90a kernels.

Drop-in for the reference's ``model.py`` classes used by its Solver / Inferencer
(model.py:209-395 of jjery2243542/adaptive_voice_conversion):

  * ``AE(config)`` with ``forward(x) -> (mu, log_sigma, emb, dec)``, ``inference(x, x_cond)``
    and ``get_speaker_embeddings(x)``;
  * identical constructor kwargs (the keys of config.yaml) and an identical ``state_dict``:
    166 fp32 tensors (218 with the decoder's spectral norm, ``Decoder.sn``) named ``speaker_encoder.conv_bank.0.weight`` ... with nn.Conv1d
    ``[Cout, Cin, k]`` / nn.Linear ``[out, in]`` shapes, so reference checkpoints load both
    ways.  nn.Conv1d / nn.Linear modules are kept purely as *parameter containers* (names,
    shapes, default init); their ``forward`` is never called.

The arithmetic runs in ``engine.Engine`` (hand-written CUDA through the C ABI); autograd
sees three custom Functions (speaker encoder, content encoder, reparam+decoder) whose
backward passes are hand-sequenced kernels as well.  There is no CPU path: calling the
model on CPU tensors raises.
"""
from __future__ import annotations

import math
import os
import types

from typing import Dict, List, Optional

import torch
import torch.nn as nn

from . import _lib as L
from .engine import A4, Engine, Lengths, varlen_extent


def _bank_kernel_sizes(bank_size: int, bank_scale: int) -> List[int]:
    return list(range(bank_scale, bank_size + 1, bank_scale))


class _ParamStack(nn.Module):
    """Base: a bag of nn.Conv1d / nn.Linear parameter holders registered under the
    reference's attribute names."""

    def _convs(self, attr: str, specs, f=lambda m: m):
        setattr(self, attr, nn.ModuleList([f(nn.Conv1d(ci, co, kernel_size=k, stride=s)) for (ci, co, k, s) in specs]))

    def _linears(self, attr: str, specs, f=lambda m: m):
        setattr(self, attr, nn.ModuleList([f(nn.Linear(i, o)) for (i, o) in specs]))

    def forward(self, *a, **k):  # pragma: no cover
        raise L.AvcError("sub-stacks are parameter containers; call AE.forward / AE.inference / AE.get_speaker_embeddings")


class SpeakerEncoder(_ParamStack):
    """Parameters of the reference SpeakerEncoder (model.py:209-235)."""

    def __init__(self, c_in, c_h, c_out, kernel_size, bank_size, bank_scale, c_bank, n_conv_blocks,
                 n_dense_blocks, subsample, act, dropout_rate):
        super().__init__()
        ks = _bank_kernel_sizes(bank_size, bank_scale)
        self._convs("conv_bank", [(c_in, c_bank, k, 1) for k in ks])
        self.in_conv_layer = nn.Conv1d(c_bank * len(ks) + c_in, c_h, kernel_size=1)
        self._convs("first_conv_layers", [(c_h, c_h, kernel_size, 1)] * n_conv_blocks)
        self._convs("second_conv_layers", [(c_h, c_h, kernel_size, s) for s, _ in zip(subsample, range(n_conv_blocks))])
        self._linears("first_dense_layers", [(c_h, c_h)] * n_dense_blocks)
        self._linears("second_dense_layers", [(c_h, c_h)] * n_dense_blocks)
        self.output_layer = nn.Linear(c_h, c_out)


class ContentEncoder(_ParamStack):
    """Parameters of the reference ContentEncoder (model.py:279-299)."""

    def __init__(self, c_in, c_h, c_out, kernel_size, bank_size, bank_scale, c_bank, n_conv_blocks, subsample,
                 act, dropout_rate):
        super().__init__()
        ks = _bank_kernel_sizes(bank_size, bank_scale)
        self._convs("conv_bank", [(c_in, c_bank, k, 1) for k in ks])
        self.in_conv_layer = nn.Conv1d(c_bank * len(ks) + c_in, c_h, kernel_size=1)
        self._convs("first_conv_layers", [(c_h, c_h, kernel_size, 1)] * n_conv_blocks)
        self._convs("second_conv_layers", [(c_h, c_h, kernel_size, s) for s, _ in zip(subsample, range(n_conv_blocks))])
        self.mean_layer = nn.Conv1d(c_h, c_out, kernel_size=1)
        self.std_layer = nn.Conv1d(c_h, c_out, kernel_size=1)


class Decoder(_ParamStack):
    """Parameters of the reference Decoder (model.py:325-345).

    sn=True wraps every layer in ``torch.nn.utils.spectral_norm`` as the reference does, in its order: the state_dict
    then holds ``weight_orig`` / ``weight_u`` / ``weight_v`` (with the ``spectral_norm`` metadata), ``parameters()``
    lists ``bias`` before ``weight_orig``, and u and v are drawn from the global generator right after each layer's
    init.  The hook torch installs is never run (the containers' forward is not called): ``Engine.spectral_norm``
    computes W / sigma on the device."""

    def __init__(self, c_in, c_cond, c_h, c_out, kernel_size, n_conv_blocks, upsample, act, sn, dropout_rate):
        super().__init__()
        self.sn = bool(sn)
        f = nn.utils.spectral_norm if sn else (lambda m: m)
        self.in_conv_layer = f(nn.Conv1d(c_in, c_h, kernel_size=1))
        self._convs("first_conv_layers", [(c_h, c_h, kernel_size, 1)] * n_conv_blocks, f)
        self._convs("second_conv_layers", [(c_h, c_h * up, kernel_size, 1) for _, up in zip(range(n_conv_blocks), upsample)], f)
        self._linears("conv_affine_layers", [(c_cond, c_h * 2)] * (2 * n_conv_blocks), f)
        self.out_conv_layer = f(nn.Conv1d(c_h, c_out, kernel_size=1))


def _check_input(x: torch.Tensor, what: str) -> torch.Tensor:
    if not x.is_cuda:
        raise L.AvcError(f"{what}: tensor is on {x.device}; this implementation has no CPU path (move it to an H100)")
    if x.dtype != torch.float32 or x.dim() != 3:
        raise L.AvcError(f"{what}: expected float32 [B, C, T], got {x.dtype} {tuple(x.shape)}")
    return x.contiguous()


def _check_lengths(lengths: Optional[torch.Tensor], x: torch.Tensor, min_len: int, what: str) -> torch.Tensor:
    """lengths of a padded batch x [B, C, T] as int32 [B] on x's device (None: all T); AvcError on a wrong type, shape
    or range.  Device values are not read during a graph capture (inference_padded checks them on the host)."""
    B, _, T = x.shape
    if lengths is None:
        return torch.full((B,), T, dtype=torch.int32, device=x.device)
    if not isinstance(lengths, torch.Tensor) or lengths.dtype == torch.bool or lengths.is_floating_point() or lengths.is_complex():
        raise L.AvcError(f"{what}: expected an integer tensor, got {getattr(lengths, 'dtype', type(lengths).__name__)}")
    if lengths.dim() != 1 or lengths.shape[0] != B:
        raise L.AvcError(f"{what}: expected shape [{B}] (the batch size), got {tuple(lengths.shape)}")
    if lengths.device.type == "cuda" and lengths.device != x.device:
        raise L.AvcError(f"{what}: on {lengths.device}, the batch on {x.device}")
    if not (lengths.is_cuda and torch.cuda.is_current_stream_capturing()):
        v = lengths.cpu()
        lo, hi = int(v.min()), int(v.max())
        if lo < min_len or hi > T:
            raise L.AvcError(f"{what}: lengths must lie in [{min_len}, {T}] (the shortest input the model accepts, the "
                             f"batch's extent); got min {lo}, max {hi}")
    return lengths.to(device=x.device, dtype=torch.int32)


def _check_groups(groups, x: torch.Tensor, what: str, dtype=torch.int32) -> torch.Tensor:
    """Row offsets [G+1] of groups of a batch x [B, C, T] (or of the rows of a table x [B, ...]) as `dtype` on x's
    device: 0 first, strictly increasing, B last (1 <= G <= B); AvcError otherwise.  As in _check_lengths, device
    values are not read during a graph capture."""
    B = x.shape[0]
    if not isinstance(groups, torch.Tensor) or groups.dtype == torch.bool or groups.is_floating_point() or groups.is_complex():
        raise L.AvcError(f"{what}: expected an integer tensor, got {getattr(groups, 'dtype', type(groups).__name__)}")
    if groups.dim() != 1 or not 2 <= groups.shape[0] <= B + 1:
        raise L.AvcError(f"{what}: expected shape [G + 1] with 1 <= G <= {B} (the batch size), got {tuple(groups.shape)}")
    if groups.device.type == "cuda" and groups.device != x.device:
        raise L.AvcError(f"{what}: on {groups.device}, the batch on {x.device}")
    if not (groups.is_cuda and torch.cuda.is_current_stream_capturing()):
        v = groups.cpu().tolist()
        if v[0] != 0 or v[-1] != B or any(b <= a for a, b in zip(v, v[1:])):
            raise L.AvcError(f"{what}: offsets must start at 0, increase strictly and end at {B} (the batch size); got {v}")
    return groups.to(device=x.device, dtype=dtype)


def _pad_time(x: torch.Tensor, Te: int) -> torch.Tensor:
    """x [B, C, T] in the first T frames of a [B, C, Te] buffer (the later frames are never read for a valid output)."""
    xp = x.new_empty(x.shape[0], x.shape[1], Te)
    xp[:, :, :x.shape[2]].copy_(x)
    return xp


class _StackFn(torch.autograd.Function):
    """Common plumbing: params arrive as *args so autograd tracks them; gradients are
    produced into one zeroed flat buffer and returned as views."""

    @staticmethod
    def _begin(ctx, model, prefix, params, train):
        names = model._names_by_prefix[prefix]
        P = dict(zip(names, params))
        eng = model.engine(params[0].device)
        if prefix == "decoder." and model.decoder.sn:
            # torch's spectral_norm: one power iteration per forward in training mode (also under no_grad), none in eval
            P.update((n, b) for n, b in model.named_buffers() if n.startswith(prefix))
            eng.bind_spectral_norm(P)
            eng.spectral_norm(P, iterate=model.training)
        eng.pack_weights(P, need_dgrad=train, prefixes=(prefix,))
        ctx.model, ctx.prefix, ctx.P, ctx.train = model, prefix, P, train
        return eng, P

    @staticmethod
    def _grads(ctx, eng):
        names = ctx.model._names_by_prefix[ctx.prefix]
        sizes = [ctx.P[n].numel() for n in names]
        flat = eng.zeros(sum(sizes))
        G, off = {}, 0
        for n, s in zip(names, sizes):
            G[n] = flat[off:off + s].view(ctx.P[n].shape)
            off += s
        return G, names


class _SpeakerFn(_StackFn):
    @staticmethod
    def forward(ctx, model, x, *params):
        train = any(ctx.needs_input_grad)  # grad mode is off inside Function.forward
        eng, P = _StackFn._begin(ctx, model, "speaker_encoder.", params, train)
        emb, ctx.saved = eng.speaker_fwd(P, x, train)
        return emb

    @staticmethod
    def backward(ctx, demb):
        eng = ctx.model.engine(demb.device)
        G, names = _StackFn._grads(ctx, eng)
        eng.speaker_bwd(ctx.P, G, ctx.saved, demb.contiguous())
        ctx.saved = None
        return (None, None, *[G[n] for n in names])


class _ContentFn(_StackFn):
    @staticmethod
    def forward(ctx, model, x, *params):
        train = any(ctx.needs_input_grad)  # grad mode is off inside Function.forward
        eng, P = _StackFn._begin(ctx, model, "content_encoder.", params, train)
        mu4, ls4, ctx.saved = eng.content_fwd(P, x, train)
        mu, ls, _ = eng.reparam_fwd(mu4, ls4, None)
        ctx.ls4 = ls4 if train else None
        return mu, ls

    @staticmethod
    def backward(ctx, dmu, dls):
        eng = ctx.model.engine(dmu.device)
        G, names = _StackFn._grads(ctx, eng)
        dmu4, dls4 = eng.reparam_bwd(None, ctx.ls4, None, dmu.contiguous(), dls.contiguous())
        eng.content_bwd(ctx.P, G, ctx.saved, dmu4, dls4)
        ctx.saved = None
        return (None, None, *[G[n] for n in names])


class _DecoderFn(_StackFn):
    """z = mu + exp(log_sigma/2)*eps (model.py:383-384; eps None -> z = mu) then Decoder."""

    @staticmethod
    def forward(ctx, model, mu, log_sigma, eps, emb, *params):
        train = any(ctx.needs_input_grad)
        eng, P = _StackFn._begin(ctx, model, "decoder.", params, train)
        B, Cc, T = mu.shape
        mu4, ls4 = A4.empty(B, Cc, T, mu.device), A4.empty(B, Cc, T, mu.device)
        eng.pack_a4(mu.contiguous(), mu4)
        eng.pack_a4(log_sigma.contiguous(), ls4)
        eps = None if eps is None else eps.contiguous()
        _, _, z4 = eng.reparam_fwd(mu4, ls4, eps, want_planar=False)
        dec4, ctx.saved = eng.decoder_fwd(P, z4, emb.contiguous(), train)
        ctx.ls4, ctx.eps = (ls4, eps) if train else (None, None)
        return eng.unpack_a4(dec4)

    @staticmethod
    def backward(ctx, ddec):
        eng = ctx.model.engine(ddec.device)
        G, names = _StackFn._grads(ctx, eng)
        B, Cc, T = ddec.shape
        ddec4 = A4.empty(B, Cc, T, ddec.device)
        eng.pack_a4(ddec.contiguous(), ddec4)
        sn = ctx.model.decoder.sn
        if sn:
            eng.bind_spectral_norm(ctx.P, G)
        dz4, demb = eng.decoder_bwd(ctx.P, G, ctx.saved, ddec4)
        if sn:
            eng.spectral_norm_bwd(ctx.P, G)
        dmu4, dls4 = eng.reparam_bwd(dz4, ctx.ls4, ctx.eps, None, None)
        dmu, dls = eng.unpack_a4(dmu4), eng.unpack_a4(dls4)
        ctx.saved = None
        return (None, dmu, dls, None, demb, *[G[n] for n in names])


class AE(nn.Module):
    """The auto-encoder of the reference (model.py:373-395), H100-native."""

    def __init__(self, config: dict):
        super().__init__()
        self.config = {k: dict(v) if isinstance(v, dict) else v for k, v in config.items()}
        self.speaker_encoder = SpeakerEncoder(**config["SpeakerEncoder"])
        self.content_encoder = ContentEncoder(**config["ContentEncoder"])
        self.decoder = Decoder(**config["Decoder"])
        self._engines: Dict[str, Engine] = {}
        self._names_by_prefix = {}
        self._flat: Optional[torch.Tensor] = None
        self._index_names()

    # ---- parameter bookkeeping
    def _index_names(self):
        names = [n for n, _ in self.named_parameters()]
        for prefix in ("speaker_encoder.", "content_encoder.", "decoder."):
            self._names_by_prefix[prefix] = [n for n in names if n.startswith(prefix)]

    def _params(self, prefix: str):
        d = dict(self.named_parameters())
        return [d[n] for n in self._names_by_prefix[prefix]]

    def engine(self, device) -> Engine:
        key = str(torch.device(device))
        if key not in self._engines:
            self._engines[key] = Engine(self.config, torch.device(device))
        return self._engines[key]

    def flatten_parameters(self) -> torch.Tensor:
        """Re-home every parameter as a view of one flat fp32 buffer (registration order) so
        the optimizer and the gradient all-reduce are single launches over one buffer."""
        params = list(self.parameters())
        dev = params[0].device
        flat = torch.empty(sum(p.numel() for p in params), dtype=torch.float32, device=dev)
        off = 0
        for p in params:
            n = p.numel()
            flat[off:off + n].copy_(p.data.reshape(-1))
            p.data = flat[off:off + n].view(p.shape)
            off += n
        self._flat = flat
        return flat

    # ---- the reference API
    def forward(self, x: torch.Tensor, *, eps: Optional[torch.Tensor] = None, lengths: Optional[torch.Tensor] = None):
        """AE.forward (model.py:380-385).  ``eps`` (keyword-only extension) injects the
        N(0,1) draw for parity tests; by default it is drawn from the device generator.  Training runs on fixed
        segments: ``lengths`` (padded batches) raise."""
        if lengths is not None:
            raise L.AvcError("AE.forward: padded batches (lengths) are inference-only; training runs on fixed segments")
        x = _check_input(x, "AE.forward(x)")
        emb = _SpeakerFn.apply(self, x, *self._params("speaker_encoder."))
        mu, log_sigma = _ContentFn.apply(self, x, *self._params("content_encoder."))
        if eps is None:
            eps = torch.randn_like(log_sigma)
        dec = _DecoderFn.apply(self, mu, log_sigma, eps, emb, *self._params("decoder."))
        return mu, log_sigma, emb, dec

    def inference(self, x: torch.Tensor, x_cond: torch.Tensor, *, lengths: Optional[torch.Tensor] = None,
                  cond_lengths: Optional[torch.Tensor] = None):
        """AE.inference (model.py:387-391): content mean of x, speaker of x_cond.

        lengths / cond_lengths (keyword-only extension): a padded batch.  x [B, C, T] holds lengths[b] valid frames of
        sample b, x_cond [B, C, T_c] cond_lengths[b] (integer [B] tensors on the host or the device; one of them None =
        every sample full length).  Frames past a sample's length are ignored, whatever they hold.  Returns dec
        [B, C, 8 ceil(T/8)] whose dec[b, :, :8 ceil(lengths[b]/8)] is the conversion of the unpadded pair and whose
        later frames are exactly 0.  Lengths below mcd.min_frames or above the extent raise before any launch."""
        x = _check_input(x, "AE.inference(x)")
        x_cond = _check_input(x_cond, "AE.inference(x_cond)")
        if lengths is not None or cond_lengths is not None:
            if x.shape[0] != x_cond.shape[0]:
                raise L.AvcError(f"AE.inference: x has {x.shape[0]} samples, x_cond {x_cond.shape[0]}")
            min_src, min_ref = self._min_frames()
            lx = _check_lengths(lengths, x, min_src, "AE.inference(lengths)")
            lc = _check_lengths(cond_lengths, x_cond, min_ref, "AE.inference(cond_lengths)")
            with torch.no_grad():
                return self._inference_padded(x, x_cond, lx, lc)
        with torch.no_grad():
            side = self._side_stream(x.device)
            if side is None:
                emb = _SpeakerFn.apply(self, x_cond, *self._params("speaker_encoder."))
                mu, log_sigma = _ContentFn.apply(self, x, *self._params("content_encoder."))
                return _DecoderFn.apply(self, mu, log_sigma, None, emb, *self._params("decoder."))
            # the speaker encoder (on x_cond) and the content encoder (on x) are independent until the decoder: the
            # speaker branch runs on a second stream (fork / join), as in the fused train step (trainer.py)
            main = torch.cuda.current_stream(x.device)
            side.wait_stream(main)
            with torch.cuda.stream(side):
                emb = _SpeakerFn.apply(self, x_cond, *self._params("speaker_encoder."))
            mu, log_sigma = _ContentFn.apply(self, x, *self._params("content_encoder."))
            main.wait_stream(side)
            if not torch.cuda.is_current_stream_capturing():
                emb.record_stream(main)   # allocated on the side stream, read by the decoder on this one
            return _DecoderFn.apply(self, mu, log_sigma, None, emb, *self._params("decoder."))

    def _side_stream(self, dev):
        if os.environ.get("AVC_OVERLAP", "1") != "1":
            return None
        st = getattr(self, "_side_streams", None)
        if st is None:
            st = self._side_streams = {}
        if dev not in st:
            st[dev] = torch.cuda.Stream(dev)
        return st[dev]

    def get_speaker_embeddings(self, x: torch.Tensor, *, lengths: Optional[torch.Tensor] = None,
                               groups: Optional[torch.Tensor] = None):
        """AE.get_speaker_embeddings (model.py:393-395).  lengths: a padded batch, as in inference (no gradient).

        groups (keyword-only, no gradient): integer row offsets [G+1] (0, strictly increasing, B) cutting the batch into G
        reference sets of one speaker; returns one code per set, [G, c_out].  The encoder's only operation across time
        is its time mean, so a set's code pools the last conv layer over the valid frames of all its members together
        (what the encoder computes on their concatenation, but for the conv context at the joins) before the dense
        stack.  lengths=None with groups: every row full length.  A one-member set gives the row the call with lengths
        gives, bit for bit."""
        x = _check_input(x, "AE.get_speaker_embeddings(x)")
        if lengths is not None or groups is not None:
            lx = _check_lengths(lengths, x, self._min_frames()[1], "AE.get_speaker_embeddings(lengths)")
            g = None if groups is None else _check_groups(groups, x, "AE.get_speaker_embeddings(groups)")
            with torch.no_grad():
                eng, P = self._eval_stack("speaker_encoder.", x.device)
                return eng.speaker_fwd(P, _pad_time(x, varlen_extent(self.config, x.shape[2], source=False)), False,
                                       lens=Lengths(lx), groups=g)[0]
        return _SpeakerFn.apply(self, x, *self._params("speaker_encoder."))

    def get_speaker_sums(self, x: torch.Tensor, *, lengths: torch.Tensor):
        """(sums [B, c_h] float32, counts [B] int32) of a padded batch x [B, C, T] (lengths as in get_speaker_embeddings;
        no gradient): the speaker encoder up to its time mean, then each sample's float32 sum over its valid frames of
        the last conv layer and the number of those frames.  Rows from any number of calls, gathered into one table,
        pool into speaker codes with speaker_codes_from_sums, bit for bit as get_speaker_embeddings(groups=) pools the
        same members in one batch."""
        x = _check_input(x, "AE.get_speaker_sums(x)")
        lx = _check_lengths(lengths, x, self._min_frames()[1], "AE.get_speaker_sums(lengths)")
        with torch.no_grad():
            eng, P = self._eval_stack("speaker_encoder.", x.device)
            return eng.speaker_sums(P, _pad_time(x, varlen_extent(self.config, x.shape[2], source=False)), Lengths(lx))

    def speaker_codes_from_sums(self, sums: torch.Tensor, counts: torch.Tensor, *, groups: torch.Tensor):
        """Speaker codes [G, c_out] (no gradient) of groups of rows of a get_speaker_sums table: groups holds integer row
        offsets [G+1] (0, strictly increasing, N = the table's rows).  A group's code pools its rows' sums in ascending
        row over their frames together, then runs the dense stack: the same members in the same order give
        get_speaker_embeddings(groups=)'s code bit for bit, however the rows were spread over batches.  Any number of
        rows per group; a group of 2^31 frames or more raises.  Everything is checked before any launch."""
        c = self.config["SpeakerEncoder"]
        if (not isinstance(sums, torch.Tensor) or sums.dtype != torch.float32 or sums.dim() != 2 or not sums.is_cuda
                or sums.shape[1] != c["c_h"] or sums.shape[0] < 1):
            raise L.AvcError(f"AE.speaker_codes_from_sums(sums): expected float32 [N >= 1, {c['c_h']}] on a CUDA device, got "
                             f"{getattr(sums, 'dtype', type(sums).__name__)} {tuple(getattr(sums, 'shape', ()))} on "
                             f"{getattr(sums, 'device', None)}")
        N = sums.shape[0]
        if (not isinstance(counts, torch.Tensor) or counts.dtype != torch.int32 or tuple(counts.shape) != (N,)
                or counts.device != sums.device):
            raise L.AvcError(f"AE.speaker_codes_from_sums(counts): expected int32 [{N}] on {sums.device}, got "
                             f"{getattr(counts, 'dtype', type(counts).__name__)} {tuple(getattr(counts, 'shape', ()))} on "
                             f"{getattr(counts, 'device', None)}")
        offs = _check_groups(groups, sums, "AE.speaker_codes_from_sums(groups)", dtype=torch.int64)
        hc, ho = counts.cpu().to(torch.int64), offs.cpu()
        if int(hc.min()) < 1:
            raise L.AvcError(f"AE.speaker_codes_from_sums(counts): counts must be >= 1 (got min {int(hc.min())})")
        frames = torch.cat([torch.zeros(1, dtype=torch.int64), hc.cumsum(0)])
        per_group = frames[ho[1:]] - frames[ho[:-1]]
        if int(per_group.max()) >= 2 ** 31:
            g = int(per_group.argmax())
            raise L.AvcError(f"AE.speaker_codes_from_sums: group {g} pools {int(per_group[g])} frames; fewer than 2^31 "
                             f"are supported")
        with torch.no_grad():
            eng, P = self._eval_stack("speaker_encoder.", sums.device)
            return eng.speaker_codes_from_sums(P, sums.contiguous(), counts.contiguous(), offs)

    def inference_from_embeddings(self, x: torch.Tensor, emb: torch.Tensor, *, lengths: Optional[torch.Tensor] = None):
        """AE.inference with a given speaker code: content mean of x [B, C, T], decoder conditioned on emb [B, c_out]
        (e.g. get_speaker_embeddings(..., groups=) of several references).  lengths: a padded batch, as in inference.
        inference_from_embeddings(x, get_speaker_embeddings(c)) is inference(x, c) bit for bit, and so with lengths on
        both sides."""
        x = _check_input(x, "AE.inference_from_embeddings(x)")
        c_out = self.config["SpeakerEncoder"]["c_out"]
        if (not isinstance(emb, torch.Tensor) or emb.dtype != torch.float32 or tuple(emb.shape) != (x.shape[0], c_out)
                or emb.device != x.device):
            raise L.AvcError(f"AE.inference_from_embeddings(emb): expected float32 [{x.shape[0]}, {c_out}] on {x.device}, "
                             f"got {getattr(emb, 'dtype', type(emb).__name__)} {tuple(getattr(emb, 'shape', ()))} on "
                             f"{getattr(emb, 'device', None)}")
        emb = emb.contiguous()
        with torch.no_grad():
            if lengths is not None:
                lx = _check_lengths(lengths, x, self._min_frames()[0], "AE.inference_from_embeddings(lengths)")
                return self._decode_padded(x, lx, emb)
            mu, log_sigma = _ContentFn.apply(self, x, *self._params("content_encoder."))
            return _DecoderFn.apply(self, mu, log_sigma, None, emb, *self._params("decoder."))

    def inference_morph(self, x: torch.Tensor, codes: torch.Tensor, weights: torch.Tensor, *,
                        lengths: Optional[torch.Tensor] = None):
        """A time-varying speaker morph (no gradient): content mean of x [B, C, T], decoder conditioned at every frame
        on a mix of K anchor codes codes [B, K, c_out] with weights [B, K, T] at the source frame rate.  lengths: the
        valid frames L_b of each sample (None: every sample full length); frames past L_b of x and of weights are
        ignored, whatever they hold.  Returns dec [B, C, 8 ceil(T/8)], exactly 0 past each sample's 8 ceil(L_b/8) frames.

        Output frame t < 8 ceil(L_b/8) uses the weights of source frame min(t, L_b - 1), normalised to sum 1; a decoder
        AdaIN layer whose frames are f times coarser uses their mean over its f output frames.  Each AdaIN affine layer
        is affine in the code, so a frame's AdaIN scale and shift are the same mix of the anchors' ordinary ones: one-hot
        weights constant over time give inference_from_embeddings(x, codes[:, k], lengths=) bit for bit, and anchors of
        zero weight change no bit.  Every decoder InstanceNorm still pools its statistics over the whole utterance, so a
        switch of speaker at one time also moves the frames before it a little: a morph is not a splice of separate
        conversions.

        Always the padded path, frame_size 1 only.  AvcError before any launch for wrong shapes, dtypes or devices,
        lengths below mcd.min_frames, K outside [1, AVC_MORPH_MAX_K], or weights on a valid frame that are not finite
        and >= 0 with a positive sum (not checked while a CUDA graph is being captured: the caller checks them)."""
        x = _check_input(x, "AE.inference_morph(x)")
        B, _, T = x.shape
        c_out = self.config["SpeakerEncoder"]["c_out"]
        fs = int(self.config.get("data_loader", {}).get("frame_size", 1))
        ups, subs = self.config["Decoder"]["upsample"], self.config["ContentEncoder"]["subsample"]
        if (fs != 1 or math.prod(ups[: self.config["Decoder"]["n_conv_blocks"]]) != 8
                or math.prod(subs[: self.config["ContentEncoder"]["n_conv_blocks"]]) != 8):
            raise L.AvcError("AE.inference_morph: supports frame_size 1 and a content encoder / decoder that subsample / "
                             "upsample by 8")
        for t, what, shape in ((codes, "codes", "[B, K, c_out]"), (weights, "weights", "[B, K, T]")):
            if (not isinstance(t, torch.Tensor) or t.dtype != torch.float32 or t.dim() != 3 or t.device != x.device):
                raise L.AvcError(f"AE.inference_morph({what}): expected float32 {shape} on {x.device}, got "
                                 f"{getattr(t, 'dtype', type(t).__name__)} {tuple(getattr(t, 'shape', ()))} on "
                                 f"{getattr(t, 'device', None)}")
        K = codes.shape[1]
        if not 1 <= K <= L.MORPH_MAX_K:
            raise L.AvcError(f"AE.inference_morph(codes): K={K} anchors; 1 to {L.MORPH_MAX_K} are supported")
        if tuple(codes.shape) != (B, K, c_out) or tuple(weights.shape) != (B, K, T):
            raise L.AvcError(f"AE.inference_morph: expected codes [{B}, K, {c_out}] and weights [{B}, K, {T}] (x is "
                             f"{tuple(x.shape)}), got {tuple(codes.shape)} and {tuple(weights.shape)}")
        lx = _check_lengths(lengths, x, self._min_frames()[0], "AE.inference_morph(lengths)")
        if not torch.cuda.is_current_stream_capturing():
            valid = torch.arange(T, device=x.device)[None, :] < lx[:, None].to(torch.int64)       # [B, T]
            w = torch.where(valid[:, None, :], weights, torch.ones((), device=x.device))
            s = w.sum(1)
            bad = (~torch.isfinite(w) | (w < 0)).any(1) | ~(s > 0) | ~torch.isfinite(s)           # [B, T]
            if bool(bad.any()):
                b, t = (int(v) for v in bad.nonzero()[0])
                raise L.AvcError(f"AE.inference_morph(weights): sample {b}, frame {t}: the weights must be finite and "
                                 f">= 0 with a positive sum on every valid frame, got {weights[b, :, t].tolist()}")
        with torch.no_grad():
            return self._decode_padded(x, lx, None, morph=(codes.contiguous(), weights.contiguous()))

    def get_content_means(self, x: torch.Tensor, *, lengths: torch.Tensor):
        """(mu [B, c_out, T_lat], latent lengths int32 [B]) of a padded batch x [B, C, T]: the content encoder's mean
        head as the padded AE.inference computes it (no gradient); mu[b, :, :latent[b]] is sample b's, later frames are
        padding."""
        x = _check_input(x, "AE.get_content_means(x)")
        lx = _check_lengths(lengths, x, self._min_frames()[0], "AE.get_content_means(lengths)")
        with torch.no_grad():
            eng, P = self._eval_stack("content_encoder.", x.device)
            xp = _pad_time(x, varlen_extent(self.config, x.shape[2], source=True))
            mu4, _, ctx = eng.content_fwd(P, xp, False, lens=Lengths(lx))
            lat = ctx["lens"]
            return eng.unpack_a4(mu4), ((lat.t + (lat.div - 1)) // lat.div * lat.mul).to(torch.int32)

    # ---- padded batches
    def _min_frames(self):
        from .mcd import min_frames
        return min_frames(self.config)

    def _eval_stack(self, prefix, dev):
        """(engine, parameters) of one stack for an inference call outside autograd (the padded path)."""
        return _StackFn._begin(types.SimpleNamespace(), self, prefix, self._params(prefix), False)

    def _inference_padded(self, x, x_cond, lx, lc):
        cp = _pad_time(x_cond, varlen_extent(self.config, x_cond.shape[2], source=False))
        dev = x.device
        side = self._side_stream(dev)
        main = torch.cuda.current_stream(dev)
        if side is not None:   # the speaker branch on a second stream, as in the unpadded call
            side.wait_stream(main)
        with torch.cuda.stream(side if side is not None else main):
            eng, P = self._eval_stack("speaker_encoder.", dev)
            emb, _ = eng.speaker_fwd(P, cp, False, lens=Lengths(lc))

        def join():
            if side is not None:
                main.wait_stream(side)
                if not torch.cuda.is_current_stream_capturing():
                    emb.record_stream(main)
        return self._decode_padded(x, lx, emb, join)

    def _decode_padded(self, x, lx, emb, join=None, morph=None):
        """The content and decoder half of the padded AE.inference: dec [B, C, 8 ceil(T/8)] of x's content mean
        conditioned on emb.  join(), when given, runs between the content encoder and the decoder (the speaker branch's
        stream join).  morph: (codes, weights) of inference_morph instead of emb."""
        B, Cc, T = x.shape
        xp = _pad_time(x, varlen_extent(self.config, T, source=True))
        dev = x.device
        eng, P = self._eval_stack("content_encoder.", dev)
        mu4, ls4, ctx = eng.content_fwd(P, xp, False, lens=Lengths(lx))
        _, _, z4 = eng.reparam_fwd(mu4, ls4, None, want_planar=False)
        if join is not None:
            join()
        eng, P = self._eval_stack("decoder.", dev)
        dec4, _ = eng.decoder_fwd(P, z4, emb, False, lens=ctx["lens"], morph=morph)
        To = 8 * -(-T // 8)
        return eng.unpack_a4(dec4)[:, :, :To].contiguous()
