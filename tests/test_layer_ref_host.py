"""CPU: the layer-by-layer float64 restatement of tests/_layer_ref.py composes to the whole model -- its forward chain
reproduces oracle.ae_forward and ae_inference, and its chain of layer VJPs reproduces float64 autograd of the oracle's
training loss for every parameter, with and without the decoder's spectral norm."""
import pytest
import torch

import _layer_ref as LR
import oracle.ae_oracle as orc
from _sn_ref import sn_config

LAMBDA_KL = 0.7


def _config(kind):
    return {"c80": orc.default_config(80), "c512": orc.default_config(512), "sn": sn_config(80)}[kind]


def _state(cfg, seed=0):
    """float64 parameters; with sn also weight_orig, u and v of every wrapped decoder layer."""
    sd = {k: v.double() for k, v in orc.init_state(cfg, seed=seed).items()}
    sn = {}
    if cfg["Decoder"].get("sn", False):
        g = torch.Generator().manual_seed(seed + 7)
        for k in list(sd):
            if k.startswith("decoder.") and k.endswith(".weight"):
                n = k[: -len(".weight")]
                w = sd.pop(k)
                sn[n] = (w, torch.randn(w.shape[0], generator=g, dtype=torch.float64),
                         torch.randn(w[0].numel(), generator=g, dtype=torch.float64))
    return sd, sn


def _bind(sd, sn, leaves=None):
    """P with W_bar as the weight of every spectral-normed layer (a function of weight_orig in leaves, if given)."""
    P = dict(sd if leaves is None else {k: v for k, v in leaves.items() if not k.endswith(".weight_orig")})
    stats = {}
    for n, (w, u, v) in sn.items():
        w = w if leaves is None else leaves[n + ".weight_orig"]
        wbar, u1, v1, sigma = LR.sn_wbar(w, u, v)
        P[n + ".weight"] = wbar
        stats[n] = (u1, v1, sigma)
    return P, stats


def _data(cfg, B, T, seed=1):
    g = torch.Generator().manual_seed(seed)
    x = torch.randn((B, cfg["SpeakerEncoder"]["c_in"], T), generator=g, dtype=torch.float64)
    eps = torch.randn((B, cfg["ContentEncoder"]["c_out"], -(-T // 8)), generator=g, dtype=torch.float64)
    return x, eps


def _close(a, b, tol=1e-12):
    a, b = a.detach().double(), b.detach().double()
    return float((a - b).abs().max()) <= tol * max(float(b.abs().max()), 1e-30)


@pytest.mark.parametrize("kind", ["c80", "c512", "sn"])
def test_forward_chain_is_ae_forward(kind):
    cfg = _config(kind)
    sd, sn = _state(cfg)
    P, _ = _bind(sd, sn)
    x, eps = _data(cfg, 2, 32)
    ref = orc.ae_forward(P, cfg, x, eps)
    got = LR.ae_forward(P, cfg, x, eps)[:4]
    for name, a, b in zip(("mu", "log_sigma", "emb", "dec"), got, ref):
        assert a.shape == b.shape and _close(a, b), name


@pytest.mark.parametrize("kind", ["c80", "c512", "sn"])
@pytest.mark.parametrize("T,T_c", [(32, 32), (17, 9), (45, 23)])
def test_forward_chain_is_ae_inference(kind, T, T_c):
    cfg = _config(kind)
    sd, sn = _state(cfg)
    P, _ = _bind(sd, sn)
    x, _ = _data(cfg, 2, T, seed=3)
    xc, _ = _data(cfg, 2, T_c, seed=4)
    ref = orc.ae_inference(P, cfg, x, xc)
    got, _ = LR.ae_inference(P, cfg, x, xc)
    assert got.shape == ref.shape and _close(got, ref)


@pytest.mark.parametrize("kind,B,T", [("c80", 2, 32), ("c512", 2, 32), ("sn", 2, 32), ("c80", 3, 24)])
def test_layer_vjps_chain_to_autograd(kind, B, T):
    cfg = _config(kind)
    sd, sn = _state(cfg)
    x, eps = _data(cfg, B, T)
    # float64 autograd of the oracle's loss, through W_bar = weight_orig / sigma for the spectral-normed layers
    leaves = {k: v.clone().requires_grad_(True) for k, v in sd.items()}
    leaves.update({n + ".weight_orig": w.clone().requires_grad_(True) for n, (w, _, _) in sn.items()})
    P, _ = _bind(sd, sn, leaves)
    mu, ls, emb, dec = orc.ae_forward(P, cfg, x, eps)
    loss_rec, loss_kl = orc.ae_losses(x, mu, ls, dec)
    loss = cfg["lambda"]["lambda_rec"] * loss_rec + LAMBDA_KL * loss_kl
    ref = dict(zip(leaves, torch.autograd.grad(loss, list(leaves.values()))))

    # the chain of layer VJPs
    P, stats = _bind(sd, sn)
    got = {}

    def tap(kind_, name, val, **info):
        if kind_ == "dw":
            for k, g in zip((".weight", ".bias"), val):
                assert name + k not in got, name + k
                got[name + k] = g
        elif kind_ == "grad":
            assert name not in got, name
            got[name] = val
        return val
    rmu, rls, remb, rdec, acts = LR.ae_forward(P, cfg, x, eps, tap)
    lr, lk, _, _, _ = LR.loss_grads(cfg, x, rmu, rls, rdec, LAMBDA_KL)
    assert _close(lr, loss_rec) and _close(lk, loss_kl)
    LR.ae_backward(P, cfg, x, eps, rmu, rls, rdec, acts, LAMBDA_KL, tap)
    for n, (u1, v1, sigma) in stats.items():
        got[n + ".weight_orig"] = LR.sn_bwd(got.pop(n + ".weight"), P[n + ".weight"], u1, v1, sigma)
    assert set(got) == set(ref)
    for k in ref:
        # measured against the layer's largest gradient: autograd leaves ~1e-17 rounding noise on the biases whose
        # gradient is exactly 0
        scale = max(float(ref[j].abs().max()) for j in ref if j.rsplit(".", 1)[0] == k.rsplit(".", 1)[0])
        err = float((got[k] - ref[k]).abs().max())
        assert err <= 1e-10 * scale, (k, err, scale)
    # the zero-gradient rule: biases that feed a non-shuffled InstanceNorm
    for k in ("content_encoder.in_conv_layer.bias", "decoder.first_conv_layers.0.bias"):
        w = ref.get(k.replace(".bias", ".weight"), ref.get(k.replace(".bias", ".weight_orig")))
        assert float(ref[k].abs().max()) < 1e-10 * float(w.abs().max()) and not got[k].any()


def test_tf32_rounding_helpers():
    x = torch.tensor([1.0, 1.0 + 2 ** -11, 1.0 + 2 ** -10 + 2 ** -11, -(1.0 + 2 ** -11), 3.0e-3], dtype=torch.float32)
    r = LR.tf32_rna(x)
    assert r.tolist()[:4] == [1.0, 1.0 + 2 ** -10, 1.0 + 2 ** -9, -(1.0 + 2 ** -10)]   # ties away from zero
    assert ((r.view(torch.int32) & 0x1FFF) == 0).all()
    assert ((r.double() - x.double()).abs() <= LR.tf32_half_ulp(x)).all()
