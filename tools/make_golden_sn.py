"""Generate the spectral-norm fixtures tests/golden/train_sn_c80_b4.pt and infer_sn_c80.pt by running the UNMODIFIED
reference model.py with ``Decoder.sn = True`` (a checkout of the original project, given by $AVC_REFERENCE_DIR).

    AVC_REFERENCE_DIR=<checkout> python tools/make_golden_sn.py

The model is the reference's own initialisation after ``torch.manual_seed(0)``: the spectral norm's u and v are
drawn there, in module order, so the fixture pins the construction order too.  The fixture keeps the state_dict's
names, shapes and metadata, the parameter order (what a ``.opt`` file indexes) and float64 checksums of the initial
state; ``AE(cfg)`` after the same seed must reproduce them.  The helpers and the file conventions (seeded inputs,
sampled large tensors) are those of oracle/make_golden.py.
"""
from __future__ import annotations

import os
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from oracle.make_golden import SMALL_GRADS, import_reference, randn, reference_eps, sampled, shrink_train_fixture  # noqa: E402

INIT_SEED = 0
# the layers whose u, v and sigma are recorded after every forward (every decoder layer kind, both ends)
SN_LAYERS = ["decoder.in_conv_layer", "decoder.first_conv_layers.0", "decoder.second_conv_layers.0",
             "decoder.second_conv_layers.5", "decoder.conv_affine_layers.0", "decoder.conv_affine_layers.11",
             "decoder.out_conv_layer"]


def sn_config(c_in):
    import oracle.ae_oracle as orc
    cfg = orc.default_config(c_in)
    cfg["Decoder"]["sn"] = True
    return cfg


def sn_grad_name(k):
    """SMALL_GRADS names a few decoder weights; with sn their parameter is weight_orig."""
    mod = k.rsplit(".", 1)[0]
    return mod + ".weight_orig" if k.endswith(".weight") and mod in SN_LAYERS else k


def state_record(sd):
    return {"state_keys": [(k, tuple(v.shape)) for k, v in sd.items()],
            "state_metadata": {k: dict(v) for k, v in sd._metadata.items() if "spectral_norm" in v},
            "state_checksum": torch.tensor([float(sum(v.double().sum() for v in sd.values())),
                                            float(sum(v.double().abs().sum() for v in sd.values()))])}


def sn_snapshot(ae):
    """u, v (the stored buffers) and sigma = u . (W v) of SN_LAYERS, as torch's hook computes it."""
    mods = dict(ae.named_modules())
    out = {}
    with torch.no_grad():
        for n in SN_LAYERS:
            m = mods[n]
            w = m.weight_orig.reshape(m.weight_orig.shape[0], -1)
            out[n] = {"u": m.weight_u.clone(), "v": m.weight_v.clone(), "sigma": torch.dot(m.weight_u, torch.mv(w, m.weight_v))}
    return out


def make_train_fixture(ref_model, c_in, batch, T, n_steps, name):
    config = sn_config(c_in)
    torch.manual_seed(INIT_SEED)
    ae = ref_model.AE(config)
    fx = {"c_in": c_in, "init_seed": INIT_SEED, "x": randn((batch, c_in, T), seed=1), "lambda_kl": 0.37, "steps": []}
    fx.update(state_record(ae.state_dict()))
    fx["param_names"] = [k for k, _ in ae.named_parameters()]
    fx["sn_layers"] = SN_LAYERS
    fx["sn_init"] = sn_snapshot(ae)
    x = fx["x"]
    o = config["optimizer"]
    opt = torch.optim.Adam(ae.parameters(), lr=o["lr"], betas=(o["beta1"], o["beta2"]),
                           amsgrad=o["amsgrad"], weight_decay=o["weight_decay"])
    small = [sn_grad_name(k) for k in SMALL_GRADS]
    for step in range(n_steps):
        eps_seed = 100 + step
        torch.manual_seed(eps_seed)
        mu, ls, emb, dec = ae(x)            # training mode: one power iteration per wrapped layer
        sn = sn_snapshot(ae)
        loss_rec = torch.nn.L1Loss()(dec, x)
        loss_kl = 0.5 * torch.mean(torch.exp(ls) + mu ** 2 - 1 - ls)
        loss = config["lambda"]["lambda_rec"] * loss_rec + fx["lambda_kl"] * loss_kl
        opt.zero_grad()
        loss.backward()
        grads = {k: (p.grad.detach().clone() if p.grad is not None else torch.zeros_like(p))
                 for k, p in ae.named_parameters()}
        gnorm = torch.nn.utils.clip_grad_norm_(ae.parameters(), max_norm=o["grad_norm"])
        opt.step()
        fx["steps"].append({
            "eps": reference_eps(ls.shape, eps_seed),
            "mu": mu.detach().clone(), "log_sigma": ls.detach().clone(),
            "emb": emb.detach().clone(), "dec": dec.detach().clone(),
            "loss_rec": loss_rec.detach().clone(), "loss_kl": loss_kl.detach().clone(),
            "grad_norm": torch.as_tensor(float(gnorm)),
            "grad_l2": torch.stack([grads[k].norm() for k in grads]),
            "grad_small": {k: grads[k] for k in small},
            "param_l2_after": torch.stack([p.detach().norm() for p in ae.parameters()]),
            "param_small_after": {k: dict(ae.named_parameters())[k].detach().clone() for k in small},
            "sn": sn,
        })
    fx["names"] = fx["param_names"]
    torch.save(shrink_train_fixture(fx), os.path.join(ROOT, "tests", "golden", name))
    print(name, "loss_rec", float(fx["steps"][0]["loss_rec"]), "sigma(in_conv)", float(fx["steps"][0]["sn"][SN_LAYERS[0]]["sigma"]))


def make_infer_fixture(ref_model, c_in, batch, T, T_cond, name):
    """Eval-mode AE.inference (sigma from the stored u, v; they do not move), then the same call in training mode
    (one power iteration)."""
    config = sn_config(c_in)
    torch.manual_seed(INIT_SEED)
    ae = ref_model.AE(config)
    x = randn((batch, c_in, T), seed=3)
    xc = randn((batch, c_in, T_cond), seed=4)
    fx = {"c_in": c_in, "init_seed": INIT_SEED, "x": x, "x_cond": xc, "sn_layers": SN_LAYERS}
    fx.update(state_record(ae.state_dict()))
    fx["sn_init"] = sn_snapshot(ae)
    with torch.no_grad():
        ae.eval()
        fx["dec"] = sampled(ae.inference(x, xc), 7)
        fx["sn_eval"] = sn_snapshot(ae)
        ae.train()
        fx["dec_train"] = sampled(ae.inference(x, xc), 8)
        fx["sn_train"] = sn_snapshot(ae)
    torch.save(fx, os.path.join(ROOT, "tests", "golden", name))
    print(name)


def main():
    ref_model = import_reference()
    torch.set_num_threads(os.cpu_count() or 1)
    make_train_fixture(ref_model, 80, 4, 128, 3, "train_sn_c80_b4.pt")
    make_infer_fixture(ref_model, 80, 2, 301, 173, "infer_sn_c80.pt")


if __name__ == "__main__":
    main()
