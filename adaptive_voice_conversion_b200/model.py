"""Reference-shaped model API on top of the sm_90a kernels.

Drop-in for the reference's ``model.py`` classes used by its Solver / Inferencer
(model.py:209-395 of jjery2243542/adaptive_voice_conversion):

  * ``AE(config)`` with ``forward(x) -> (mu, log_sigma, emb, dec)``, ``inference(x, x_cond)``
    and ``get_speaker_embeddings(x)``;
  * identical constructor kwargs (the keys of config.yaml) and an identical ``state_dict``:
    166 fp32 tensors named ``speaker_encoder.conv_bank.0.weight`` ... with nn.Conv1d
    ``[Cout, Cin, k]`` / nn.Linear ``[out, in]`` shapes, so reference checkpoints load both
    ways.  nn.Conv1d / nn.Linear modules are kept purely as *parameter containers* (names,
    shapes, default init); their ``forward`` is never called.

The arithmetic runs in ``engine.Engine`` (hand-written CUDA through the C ABI); autograd
sees three custom Functions (speaker encoder, content encoder, reparam+decoder) whose
backward passes are hand-sequenced kernels as well.  There is no CPU path: calling the
model on CPU tensors raises.
"""
from __future__ import annotations

import os

from typing import Dict, List, Optional

import torch
import torch.nn as nn

from . import _lib as L
from .engine import A4, Engine


def _bank_kernel_sizes(bank_size: int, bank_scale: int) -> List[int]:
    return list(range(bank_scale, bank_size + 1, bank_scale))


class _ParamStack(nn.Module):
    """Base: a bag of nn.Conv1d / nn.Linear parameter holders registered under the
    reference's attribute names."""

    def _convs(self, attr: str, specs):
        setattr(self, attr, nn.ModuleList([nn.Conv1d(ci, co, kernel_size=k, stride=s) for (ci, co, k, s) in specs]))

    def _linears(self, attr: str, specs):
        setattr(self, attr, nn.ModuleList([nn.Linear(i, o) for (i, o) in specs]))

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
    """Parameters of the reference Decoder (model.py:325-345)."""

    def __init__(self, c_in, c_cond, c_h, c_out, kernel_size, n_conv_blocks, upsample, act, sn, dropout_rate):
        super().__init__()
        if sn:
            raise L.AvcError("spectral norm (sn=True) is not implemented; the reference config uses sn: False")
        self.in_conv_layer = nn.Conv1d(c_in, c_h, kernel_size=1)
        self._convs("first_conv_layers", [(c_h, c_h, kernel_size, 1)] * n_conv_blocks)
        self._convs("second_conv_layers", [(c_h, c_h * up, kernel_size, 1) for _, up in zip(range(n_conv_blocks), upsample)])
        self._linears("conv_affine_layers", [(c_cond, c_h * 2)] * (2 * n_conv_blocks))
        self.out_conv_layer = nn.Conv1d(c_h, c_out, kernel_size=1)


def _check_input(x: torch.Tensor, what: str) -> torch.Tensor:
    if not x.is_cuda:
        raise L.AvcError(f"{what}: tensor is on {x.device}; this implementation has no CPU path (move it to an H100)")
    if x.dtype != torch.float32 or x.dim() != 3:
        raise L.AvcError(f"{what}: expected float32 [B, C, T], got {x.dtype} {tuple(x.shape)}")
    return x.contiguous()


class _StackFn(torch.autograd.Function):
    """Common plumbing: params arrive as *args so autograd tracks them; gradients are
    produced into one zeroed flat buffer and returned as views."""

    @staticmethod
    def _begin(ctx, model, prefix, params, train):
        names = model._names_by_prefix[prefix]
        P = dict(zip(names, params))
        eng = model.engine(params[0].device)
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
        dz4, demb = eng.decoder_bwd(ctx.P, G, ctx.saved, ddec4)
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
    def forward(self, x: torch.Tensor, *, eps: Optional[torch.Tensor] = None):
        """AE.forward (model.py:380-385).  ``eps`` (keyword-only extension) injects the
        N(0,1) draw for parity tests; by default it is drawn from the device generator."""
        x = _check_input(x, "AE.forward(x)")
        emb = _SpeakerFn.apply(self, x, *self._params("speaker_encoder."))
        mu, log_sigma = _ContentFn.apply(self, x, *self._params("content_encoder."))
        if eps is None:
            eps = torch.randn_like(log_sigma)
        dec = _DecoderFn.apply(self, mu, log_sigma, eps, emb, *self._params("decoder."))
        return mu, log_sigma, emb, dec

    def inference(self, x: torch.Tensor, x_cond: torch.Tensor):
        """AE.inference (model.py:387-391): content mean of x, speaker of x_cond."""
        x = _check_input(x, "AE.inference(x)")
        x_cond = _check_input(x_cond, "AE.inference(x_cond)")
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

    def get_speaker_embeddings(self, x: torch.Tensor):
        """AE.get_speaker_embeddings (model.py:393-395)."""
        x = _check_input(x, "AE.get_speaker_embeddings(x)")
        return _SpeakerFn.apply(self, x, *self._params("speaker_encoder."))
