"""float64 restatement of the AdaIN-VC model one layer at a time, forward and VJP, built from the oracle's ops.

A *layer* is one conv of the model with everything the reference applies after it up to the next conv: pixel shuffle,
InstanceNorm, AdaIN (one row of the conv_affine_layers), ReLU and the block's residual (same, ceil-mode average pool or
nearest upsampling).  The chains below (speaker, content, decoder, reparameterisation and loss, the dense stack, the
AdaIN affine layers, spectral norm) compose those layers into the whole model.

Every boundary value passes through ``tap(kind, name, ref, **info)``, which returns the value the chain continues with.
With the default identity tap the chains are the model in float64 (tests/test_layer_ref_host.py checks them against
oracle.ae_forward / ae_inference and autograd of oracle.ae_loss_and_grads).  tests/test_gpu_step_layers.py passes a tap
that compares each reference value with the engine's and continues with the engine's, so each layer is checked on the
engine's own inputs to it and errors do not compound.

``tc(name, op)`` (op "fwd", "dgrad" or "wgrad") says whether that launch of the layer ran on the tensor cores; the
reference then rounds that conv's two operands to TF32 as the kernels do (the conv kernel rounds, tf32_rna; the weight
gradient truncates, tf32_trunc).

Kinds a tap sees: "out" (a layer's output; info pre, relu, redo(mask)), "dc" (the gradient at a layer's raw conv output
and its AdaIN-row gradient; info pre, redo(mask)), "dx" (the gradient at a block's or a layer's input), "dw" (weight
and bias gradient; info x, dc, spec, tf32), "x" (an encoder's input), "emb", "z", "conds", "ddec", "dconds", "demb", "dmu", "dls" and "grad" (a
parameter gradient computed outside the conv layers).
"""
import torch
import torch.nn.functional as F

import oracle.ae_oracle as orc


def tf32_rna(x):
    """cvt.rna.tf32.f32: round to nearest (ties away from zero) at 10 mantissa bits."""
    b = x.contiguous().view(torch.int32)
    return ((b + 0x1000) & -0x2000).view(torch.float32)


def tf32_trunc(x):
    """The top 19 bits of the fp32 pattern: what the tensor cores multiply for an fp32 operand nobody rounded."""
    return (x.contiguous().view(torch.int32) & -0x2000).view(torch.float32)


def tf32_half_ulp(v):
    """Half a TF32 unit in the last place of each element of v (the most cvt.rna can move it)."""
    _, e = torch.frexp(v.double())
    return torch.ldexp(torch.ones_like(v, dtype=torch.float64), e - 12)


def _ident(kind, name, ref, **info):
    return ref


def _no_tc(name, op):
    return False


def _op(t, tf32):
    """A conv operand as the launch multiplies it: TF32-rounded for a tensor-core launch, in float64."""
    if tf32:
        return tf32_rna(t.float()).double()
    return t.double()


# ------------------------------------------------------------------ one layer
def spec(name, K, *, stride=1, shuffle=False, norm=False, relu=False, res=None, row=None):
    """res: None, "same", "pool" or "up" (the residual the layer adds: its block's input); row: the AdaIN affine row."""
    return dict(name=name, K=K, stride=stride, shuffle=shuffle, norm=norm, relu=relu, res=res, row=row)


def res_apply(r, mode):
    if mode == "same":
        return r
    if mode == "pool":
        return F.avg_pool1d(r, kernel_size=2, ceil_mode=True)
    if mode == "up":
        return F.interpolate(r, scale_factor=2, mode="nearest")
    raise ValueError(mode)


def res_adj(g, mode, T_in):
    """Adjoint of res_apply: the gradient at the residual input of T_in frames."""
    r = torch.zeros(g.shape[0], g.shape[1], T_in, dtype=torch.float64, device=g.device, requires_grad=True)
    return torch.autograd.grad(res_apply(r, mode), r, g.double())[0]


def conv(x, w, b, stride, tf32=False):
    """The raw conv output c of a layer (reflect padding as pad_layer)."""
    return orc.reflect_conv1d(_op(x, tf32), _op(w, tf32), None if b is None else b.double(), stride)


def post(c, s, cond=None, res=None, mask=None):
    """-> (out, pre): shuffle, InstanceNorm, AdaIN, ReLU (mask: the branch of every element; default pre > 0), + res."""
    y = orc.pixel_shuffle_1d(c, 2) if s["shuffle"] else c
    if s["norm"]:
        y = orc.instance_norm(y)
    if cond is not None:
        y = orc.adain(y, cond)
    pre = y
    if s["relu"]:
        y = torch.where(pre > 0 if mask is None else mask, pre, torch.zeros_like(pre))
    if res is not None:
        y = y + res_apply(res, s["res"])
    return y, pre


def post_vjp(c, s, cond, g_out, mask=None):
    """-> (dc, dcond): the gradient at the raw conv output and at the AdaIN row (None without one) for the gradient
    g_out at the layer's output (the residual branch excluded)."""
    c = c.detach().requires_grad_(True)
    leaves = [c]
    if cond is not None:
        cond = cond.detach().double().requires_grad_(True)
        leaves.append(cond)
    out, _ = post(c, s, cond, None, mask)
    g = torch.autograd.grad(out, leaves, g_out.double())
    return g[0], (g[1] if cond is not None else None)


def conv_dx(dc, w, T_in, stride, tf32=False):
    """The gradient at a conv's input (the transposed conv, reflect halo folded back)."""
    W = _op(w, tf32)
    x = torch.zeros(dc.shape[0], W.shape[1], T_in, dtype=torch.float64, device=dc.device, requires_grad=True)
    return torch.autograd.grad(orc.reflect_conv1d(x, W, None, stride), x, _op(dc, tf32))[0]


def conv_dw(x, dc, K, stride, tf32=False):
    """-> (dW, db) of a conv with input x and raw-output gradient dc (db from the unrounded dc).  tf32: "trunc" or "rna",
    how the tensor-core weight gradient reduces an operand the engine did not round (True = "trunc")."""
    def op(t):
        if not tf32:
            return t.double()
        return (tf32_rna(t.float()) if tf32 == "rna" else tf32_trunc(t.float())).double()
    X = op(x)
    w = torch.zeros(dc.shape[1], X.shape[1], K, dtype=torch.float64, device=dc.device, requires_grad=True)
    dw = torch.autograd.grad(orc.reflect_conv1d(X, w, None, stride), w, op(dc))[0]
    return dw, dc.double().sum(dim=(0, 2))


def layer_fwd(P, s, x, tap, tc, cond=None, res=None):
    """One layer forward; returns what the tap returns for its output, and the record its backward needs."""
    name = s["name"]
    c = conv(x, P[name + ".weight"], P[name + ".bias"], s["stride"], tc(name, "fwd"))
    out, pre = post(c, s, cond, res)
    out = tap("out", name, out, pre=pre, relu=s["relu"], redo=lambda m: post(c, s, cond, res, m)[0])
    return out, dict(spec=s, x=x, c=c, pre=pre, cond=cond, T_in=x.shape[2])


def layer_bwd(P, a, g_out, tap, tc):
    """One layer backward from the gradient at its output: -> (dc, dcond) as the tap returns them.  The weight and bias
    gradient go to the tap ("dw"); a bias that feeds a non-shuffled InstanceNorm has the gradient 0 exactly."""
    s = a["spec"]
    name = s["name"]
    if s["norm"] or s["relu"]:
        ref = post_vjp(a["c"], s, a["cond"], g_out)
        dc, dcond = tap("dc", name, ref, pre=a["pre"], spec=s,
                        redo=lambda m: post_vjp(a["c"], s, a["cond"], g_out, m))
    else:
        dc, dcond = tap("dc", name, (g_out.double(), None), pre=None, spec=s, redo=None)
    tf = tc(name, "wgrad")
    dw, db = conv_dw(a["x"], dc, s["K"], s["stride"], tf)
    if s["norm"] and not s["shuffle"]:
        db = torch.zeros_like(db)
    tap("dw", name, (dw, db), x=a["x"], dc=dc, spec=s, tf32=tf)
    return dc, dcond


def layer_dx(P, a, dc, tc):
    s = a["spec"]
    return conv_dx(dc, P[s["name"] + ".weight"], a["T_in"], s["stride"], tc(s["name"], "dgrad"))


# ------------------------------------------------------------------ layer lists
def bank_kernels(c):
    return list(range(c["bank_scale"], c["bank_size"] + 1, c["bank_scale"]))


def encoder_specs(cfg, key):
    """(bank specs, in_conv spec, [(first, second)] per block) of the speaker (no norm) or content encoder."""
    c = cfg[key]
    enc = "speaker_encoder" if key == "SpeakerEncoder" else "content_encoder"
    norm = key == "ContentEncoder"
    bank = [spec(f"{enc}.conv_bank.{i}", k, relu=True) for i, k in enumerate(bank_kernels(c))]
    inc = spec(f"{enc}.in_conv_layer", 1, norm=norm, relu=True)
    K = c["kernel_size"]
    blocks = [(spec(f"{enc}.first_conv_layers.{l}", K, norm=norm, relu=True),
               spec(f"{enc}.second_conv_layers.{l}", K, stride=s, norm=norm, relu=True, res="pool" if s > 1 else "same"))
              for l, s in enumerate(c["subsample"][: c["n_conv_blocks"]])]
    return bank, inc, blocks


def decoder_specs(cfg):
    d = cfg["Decoder"]
    K = d["kernel_size"]
    inc = spec("decoder.in_conv_layer", 1, norm=True, relu=True)
    blocks = [(spec(f"decoder.first_conv_layers.{l}", K, norm=True, relu=True, row=2 * l),
               spec(f"decoder.second_conv_layers.{l}", K, shuffle=up > 1, norm=True, relu=True, res="up" if up > 1 else "same",
                    row=2 * l + 1))
              for l, up in enumerate(d["upsample"][: d["n_conv_blocks"]])]
    return inc, blocks, spec("decoder.out_conv_layer", 1)


def dense_names(cfg):
    nd = cfg["SpeakerEncoder"]["n_dense_blocks"]
    return ([f"speaker_encoder.first_dense_layers.{l}" for l in range(nd)]
            + [f"speaker_encoder.second_dense_layers.{l}" for l in range(nd)] + ["speaker_encoder.output_layer"])


def affine_names(cfg):
    return [f"decoder.conv_affine_layers.{i}" for i in range(2 * cfg["Decoder"]["n_conv_blocks"])]


# ------------------------------------------------------------------ stacks, forward
def _encoder_fwd(P, cfg, key, x, tap, tc, acts):
    bank, inc, blocks = encoder_specs(cfg, key)
    x = tap("x", bank[0]["name"].rsplit(".", 2)[0], x.double())    # (the engine packs x into its concat, rounded to TF32)
    outs = []
    for s in bank:
        o, acts[s["name"]] = layer_fwd(P, s, x, tap, tc)
        outs.append(o)
    out, acts[inc["name"]] = layer_fwd(P, inc, torch.cat([o.double() for o in outs] + [x.double()], 1), tap, tc)
    for s1, s2 in blocks:
        y, acts[s1["name"]] = layer_fwd(P, s1, out, tap, tc)
        out, acts[s2["name"]] = layer_fwd(P, s2, y, tap, tc, res=out.double())
    return out


def dense_fwd(P, cfg, h):
    """The speaker encoder after its conv blocks: time mean, the dense blocks and output_layer."""
    return dense_pooled(P, cfg, h.double().mean(dim=2))


def dense_pooled(P, cfg, h):
    """The dense blocks and output_layer on time-pooled rows h [B, c_h]."""
    h = h.double()
    for l in range(cfg["SpeakerEncoder"]["n_dense_blocks"]):
        n1, n2 = f"speaker_encoder.first_dense_layers.{l}", f"speaker_encoder.second_dense_layers.{l}"
        y = F.relu(F.linear(h, P[n1 + ".weight"].double(), P[n1 + ".bias"].double()))
        h = F.relu(F.linear(y, P[n2 + ".weight"].double(), P[n2 + ".bias"].double())) + h
    return F.linear(h, P["speaker_encoder.output_layer.weight"].double(), P["speaker_encoder.output_layer.bias"].double())


def speaker_convs(P, cfg, x, tap=_ident, tc=_no_tc, acts=None):
    """The speaker encoder's conv layers -> the last one's output [B, c_h, T/8], before the time mean."""
    acts = {} if acts is None else acts
    out = _encoder_fwd(P, cfg, "SpeakerEncoder", x, tap, tc, acts)
    acts["speaker_encoder.last"] = out
    return out


def speaker_fwd(P, cfg, x, tap=_ident, tc=_no_tc, acts=None):
    acts = {} if acts is None else acts
    out = speaker_convs(P, cfg, x, tap, tc, acts)
    return tap("emb", "speaker_encoder", dense_fwd(P, cfg, out)), acts


def content_fwd(P, cfg, x, tap=_ident, tc=_no_tc, acts=None):
    acts = {} if acts is None else acts
    out = _encoder_fwd(P, cfg, "ContentEncoder", x, tap, tc, acts)
    mu, acts["content_encoder.mean_layer"] = layer_fwd(P, spec("content_encoder.mean_layer", 1), out, tap, tc)
    ls, acts["content_encoder.std_layer"] = layer_fwd(P, spec("content_encoder.std_layer", 1), out, tap, tc)
    return mu, ls, acts


def affine_fwd(P, cfg, emb, tap=_ident):
    """conds [B, 2n, 2 c_h]: every AdaIN row of the decoder from the speaker embedding."""
    rows = [F.linear(emb.double(), P[n + ".weight"].double(), P[n + ".bias"].double()) for n in affine_names(cfg)]
    return tap("conds", "decoder", torch.stack(rows, 1))


def decoder_fwd(P, cfg, z, emb, tap=_ident, tc=_no_tc, acts=None):
    acts = {} if acts is None else acts
    inc, blocks, outc = decoder_specs(cfg)
    conds = affine_fwd(P, cfg, emb, tap)
    acts["decoder.emb"] = emb
    out, acts[inc["name"]] = layer_fwd(P, inc, z, tap, tc)
    for s1, s2 in blocks:
        y, acts[s1["name"]] = layer_fwd(P, s1, out, tap, tc, cond=conds[:, s1["row"]])
        out, acts[s2["name"]] = layer_fwd(P, s2, y, tap, tc, cond=conds[:, s2["row"]], res=out.double())
    dec, acts[outc["name"]] = layer_fwd(P, outc, out, tap, tc)
    return dec, acts


def reparam(mu, ls, eps):
    return mu.double() + torch.exp(ls.double() / 2) * eps.double()


def ae_forward(P, cfg, x, eps, tap=_ident, tc=_no_tc):
    """-> (mu, ls, emb, dec, acts): AE.forward with the N(0, 1) draw eps."""
    acts = {}
    emb, _ = speaker_fwd(P, cfg, x, tap, tc, acts)
    mu, ls, _ = content_fwd(P, cfg, x, tap, tc, acts)
    z = tap("z", "decoder", reparam(mu, ls, eps))
    dec, _ = decoder_fwd(P, cfg, z, emb, tap, tc, acts)
    return mu, ls, emb, dec, acts


def ae_inference(P, cfg, x, x_cond, tap=_ident, tc=_no_tc):
    acts = {}
    emb, _ = speaker_fwd(P, cfg, x_cond, tap, tc, acts)
    mu, _, _ = content_fwd(P, cfg, x, tap, tc, acts)
    z = tap("z", "decoder", mu.double())
    dec, _ = decoder_fwd(P, cfg, z, emb, tap, tc, acts)
    return dec, acts


# ------------------------------------------------------------------ stacks, backward
def _blocks_bwd(P, acts, blocks, g, tap, tc, dconds=None):
    """The conv blocks backward from the gradient g at the last block's output -> the gradient at the first one's input."""
    for s1, s2 in reversed(blocks):
        a1, a2 = acts[s1["name"]], acts[s2["name"]]
        dc2, dcond2 = layer_bwd(P, a2, g, tap, tc)
        gy = tap("dx", s2["name"], layer_dx(P, a2, dc2, tc))
        dc1, dcond1 = layer_bwd(P, a1, gy, tap, tc)
        if dconds is not None:
            dconds[s2["row"]], dconds[s1["row"]] = dcond2, dcond1
        g = tap("dx", s1["name"], layer_dx(P, a1, dc1, tc) + res_adj(g, s2["res"], a1["T_in"]))
    return g


def _encoder_bwd(P, cfg, key, acts, g, tap, tc):
    bank, inc, blocks = encoder_specs(cfg, key)
    g = _blocks_bwd(P, acts, blocks, g, tap, tc)
    dc_in, _ = layer_bwd(P, acts[inc["name"]], g, tap, tc)
    gcat = layer_dx(P, acts[inc["name"]], dc_in, tc)
    cb = cfg[key]["c_bank"]
    for i, s in enumerate(bank):
        layer_bwd(P, acts[s["name"]], gcat[:, i * cb:(i + 1) * cb], tap, tc)


def dense_bwd(P, cfg, h_last, demb, tap=_ident):
    """Backward of dense_fwd: the dense layers' gradients go to the tap ("grad"); -> the gradient at h_last."""
    names = dense_names(cfg)
    leaves = {n + sfx: P[n + sfx].detach().double().requires_grad_(True) for n in names for sfx in (".weight", ".bias")}
    h = h_last.detach().double().requires_grad_(True)
    grads = torch.autograd.grad(dense_fwd(leaves, cfg, h), [h] + list(leaves.values()), demb.double())
    for k, gk in zip(leaves, grads[1:]):
        tap("grad", k, gk)
    return grads[0]


def affine_bwd(P, cfg, emb, dconds, tap=_ident):
    """The AdaIN affine layers backward from the row gradients dconds [2n] x [B, 2 c_h] -> demb."""
    demb = 0.0
    for i, n in enumerate(affine_names(cfg)):
        g = dconds[i].double()
        tap("grad", n + ".weight", g.t() @ emb.double())
        tap("grad", n + ".bias", g.sum(0))
        demb = demb + g @ P[n + ".weight"].double()
    return tap("demb", "decoder", demb)


def loss_grads(cfg, x, mu, ls, dec, lambda_kl):
    """-> (loss_rec, loss_kl, ddec, dmu, dls) of lambda_rec * mean|dec - x| + lambda_kl * 0.5 * mean(e^ls + mu^2 - 1 - ls)."""
    lrec = float(cfg["lambda"]["lambda_rec"])
    df = dec.double() - x.double()
    m, l = mu.double(), ls.double()
    e = torch.exp(l)
    return (df.abs().mean(), 0.5 * (e + m * m - 1 - l).mean(), torch.sign(df) * (lrec / df.numel()),
            (lambda_kl / m.numel()) * m, (lambda_kl / m.numel()) * 0.5 * (e - 1))


def ae_backward(P, cfg, x, eps, mu, ls, dec, acts, lambda_kl, tap=_ident, tc=_no_tc):
    """The training step's backward, layer by layer, from the forward's outputs and records; every gradient reaches
    the tap ("dw" for the conv layers, "grad" for the dense and affine layers)."""
    _, _, ddec, dmu, dls = loss_grads(cfg, x, mu, ls, dec, lambda_kl)
    ddec = tap("ddec", "decoder", ddec)
    inc, blocks, outc = decoder_specs(cfg)
    dc_out, _ = layer_bwd(P, acts[outc["name"]], ddec, tap, tc)
    g = layer_dx(P, acts[outc["name"]], dc_out, tc)
    dconds = [None] * (2 * len(blocks))
    g = _blocks_bwd(P, acts, blocks, g, tap, tc, dconds)
    dc_in, _ = layer_bwd(P, acts[inc["name"]], g, tap, tc)
    dz = tap("dx", inc["name"], layer_dx(P, acts[inc["name"]], dc_in, tc))
    dconds = tap("dconds", "decoder", torch.stack(dconds, 0))
    demb = affine_bwd(P, cfg, acts["decoder.emb"], dconds, tap)
    # reparameterisation: z = mu + exp(ls / 2) eps
    dmu = tap("dmu", "content_encoder", dz + dmu)
    dls = tap("dls", "content_encoder", dz * eps.double() * 0.5 * torch.exp(ls.double() / 2) + dls)
    am, al = acts["content_encoder.mean_layer"], acts["content_encoder.std_layer"]
    dc_mu, _ = layer_bwd(P, am, dmu, tap, tc)
    dc_ls, _ = layer_bwd(P, al, dls, tap, tc)
    _encoder_bwd(P, cfg, "ContentEncoder", acts, layer_dx(P, am, dc_mu, tc) + layer_dx(P, al, dc_ls, tc), tap, tc)
    last = acts["speaker_encoder.last"]
    dh = dense_bwd(P, cfg, last, demb, tap)
    _encoder_bwd(P, cfg, "SpeakerEncoder", acts, dh, tap, tc)


# ------------------------------------------------------------------ spectral norm
def sn_wbar(w_orig, u, v):
    """W_bar = weight_orig / sigma after one power iteration (u, v held constant under the gradient, as
    torch.nn.utils.spectral_norm computes them without grad) -> (W_bar, u, v, sigma)."""
    from _sn_ref import power_iteration64
    u1, v1, _, _ = power_iteration64(w_orig.detach(), u, v, iterate=True)
    Wm = w_orig.double().reshape(w_orig.shape[0], -1)
    sigma = u1 @ (Wm @ v1)
    return w_orig.double() / sigma, u1, v1, sigma


def sn_bwd(dwbar, wbar, u, v, sigma):
    from _sn_ref import adjoint64
    return adjoint64(dwbar, wbar, u, v, sigma)
