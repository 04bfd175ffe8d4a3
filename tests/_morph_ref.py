"""Float64 restatement of the decoder under a time-varying speaker morph (AE.inference_morph), for one sample.

It mixes CODES, not AdaIN rows: at every frame of a layer it forms the code sum_k w_k c_k of that frame's weights and
runs the layer's AdaIN affine layer on it.  The kernel mixes the anchors' rows instead; the two agree because each
affine layer is affine in the code, so a test against this restatement checks that argument as well as the kernels.
Built on _layer_ref's conv / spec / decoder_specs.
"""
import math

import torch
import torch.nn.functional as F

import oracle.ae_oracle as orc
from _layer_ref import affine_names, conv, decoder_specs, res_apply


def layer_weights(w, L, f):
    """w float [K, >= L] source-rate weights of a sample of L frames -> float64 [K, 8 ceil(L/8) / f]: output frame t
    uses the normalised weights of source frame min(t, L - 1); layer frame j the mean over t in [j f, (j + 1) f)."""
    w = w.double()[:, :L]
    wbar = w / w.sum(0, keepdim=True)
    To = 8 * math.ceil(L / 8)
    src = torch.clamp(torch.arange(To, device=w.device), max=L - 1)
    return wbar[:, src].view(w.shape[0], To // f, f).mean(2)


def factors(cfg):
    ups = cfg["Decoder"]["upsample"][: cfg["Decoder"]["n_conv_blocks"]]
    return [math.prod(ups[l + s:]) for l in range(len(ups)) for s in (0, 1)]


def _post_morph(c, s, rows, res):
    """shuffle, InstanceNorm, per-frame AdaIN (rows [T, 2 C]: beta | gamma), ReLU, + residual."""
    y = orc.pixel_shuffle_1d(c, 2) if s["shuffle"] else c
    y = orc.instance_norm(y)
    C = y.shape[1]
    y = y * rows[:, C:].t()[None] + rows[:, :C].t()[None]
    y = F.relu(y)
    if res is not None:
        y = y + res_apply(res, s["res"])
    return y


def decoder_morph(P, cfg, z, codes, w, L, tf32=False):
    """dec [1, c_out, 8 ceil(L/8)] of one sample: z [1, c_lat, ceil(L/8)] its latent (valid frames only), codes [K, c_out]
    the anchors, w [K, >= L] their source-rate weights.  tf32: round the conv operands as the tensor-core kernels do."""
    inc, blocks, outc = decoder_specs(cfg)
    fs = factors(cfg)
    names = affine_names(cfg)
    codes = codes.double()

    def rows_of(i):
        code = layer_weights(w, L, fs[i]).t() @ codes                          # [T_l, c_out]: the mixed code per frame
        return F.linear(code, P[names[i] + ".weight"].double(), P[names[i] + ".bias"].double())

    def c_of(s, x):
        return conv(x, P[s["name"] + ".weight"], P[s["name"] + ".bias"], s["stride"], tf32)

    out = F.relu(orc.instance_norm(c_of(inc, z.double())))
    for s1, s2 in blocks:
        y = _post_morph(c_of(s1, out), s1, rows_of(s1["row"]), None)
        out = _post_morph(c_of(s2, y), s2, rows_of(s2["row"]), out)
    return c_of(outc, out)
