"""Float64 restatements of the code-fitting kernels (csrc/fit.cu) and of one fitting step (tests/test_gpu_fit.py).

group_l1_ref follows avc_group_l1's summation order exactly, so its float64 sums are the kernel's bit for bit, and its
gradient is the kernel's float32 value.  code_adam_ref restates avc_code_adam in float64 (per-code clip_grad_norm_ +
Adam(amsgrad, L2 decay)), to be compared within float32 rounding."""
import math

import numpy as np
import torch

THREADS = 512


def rna_tf32(a: np.ndarray) -> np.ndarray:
    """cvt.rna.tf32.f32 of float32 values: round to 10 mantissa bits, ties away from zero."""
    u = np.ascontiguousarray(a, np.float32).view(np.uint32).astype(np.uint64)
    r = ((u + 0x1000) & 0xFFFFE000).astype(np.uint32)
    return r.view(np.float32)


def a4_of(planar: np.ndarray) -> np.ndarray:
    """planar [B, C, T] -> the engine's A4 [B, C/4, T, 4]."""
    B, C, T = planar.shape
    return np.ascontiguousarray(planar.reshape(B, C // 4, 4, T).transpose(0, 1, 3, 2))


def sample_sum(dec: np.ndarray, x: np.ndarray) -> float:
    """One sample's sum of |dec - x| ([C, T] each) in group_l1_kernel's order: unit u = (chunk q, step t) in A4 order,
    thread u % 512 adds the unit's four channels in order; then the warp butterflies and the 16 warp sums, padded to 32
    with zeros, butterflied again."""
    C, T = dec.shape
    terms = np.abs(a4_of(dec[None].astype(np.float64))[0] - a4_of(x[None].astype(np.float64))[0]).reshape(-1, 4)
    acc = np.zeros(THREADS)
    for k in range(0, len(terms), THREADS):
        part = terms[k:k + THREADS]
        for c in range(4):
            acc[:len(part)] = acc[:len(part)] + part[:, c]
    lane = np.arange(32)
    p = acc.reshape(THREADS // 32, 32)
    for o in (16, 8, 4, 2, 1):
        p = p + p[:, lane ^ o]
    w = np.zeros(32)
    w[:THREADS // 32] = p[:, 0]
    for o in (16, 8, 4, 2, 1):
        w = w + w[lane ^ o]
    return float(w[0])


def group_l1_ref(dec: np.ndarray, x: np.ndarray, m: int, lam: float, round_tf32: bool):
    """(ddec planar float32 [B, C, T], part float64 [B], sums float64 [G], total float32) of avc_group_l1 on planar
    dec and x."""
    B, C, T = dec.shape
    grec = np.float32(lam) / np.float32(m * C * T)
    df = dec.astype(np.float32) - x.astype(np.float32)
    g = np.where(df > 0, grec, np.where(df < 0, -grec, np.float32(0))).astype(np.float32)
    if round_tf32:
        g = rna_tf32(g)
    part = np.array([sample_sum(dec[b], x[b]) for b in range(B)])
    sums = []
    for s in range(B // m):
        a = 0.0
        for j in range(m):
            a += part[s * m + j]
        sums.append(a)
    tot = 0.0
    for v in sums:
        tot += v
    return g, part, np.array(sums), np.float32(tot)


class CodeAdamState:
    def __init__(self, S, C):
        self.m = np.zeros((S, C))
        self.v = np.zeros((S, C))
        self.vmax = np.zeros((S, C))
        self.step = np.zeros(S)


def code_adam_ref(codes: np.ndarray, demb: np.ndarray, m: int, st: CodeAdamState, opt: dict, lr=None):
    """One avc_code_adam step in float64: per code s, g_s = the sum of its m rows of demb [S m, C], then
    clip_grad_norm_(max_norm) + Adam(amsgrad, L2 decay) on that code alone.  Updates codes and st in place; returns
    (g [S, C], pre-clip norms [S])."""
    S, C = codes.shape
    lr = opt["lr"] if lr is None else lr
    b1, b2, wd, max_norm, eps = opt["beta1"], opt["beta2"], opt["weight_decay"], opt["grad_norm"], 1e-8
    g = demb.astype(np.float64).reshape(S, m, C).sum(1)
    norms = np.sqrt((g ** 2).sum(1))
    for s in range(S):
        coef = min(1.0, max_norm / (norms[s] + 1e-6))
        st.step[s] += 1
        t = st.step[s]
        gi = g[s] * coef + wd * codes[s]
        st.m[s] = b1 * st.m[s] + (1 - b1) * gi
        st.v[s] = b2 * st.v[s] + (1 - b2) * gi * gi
        second = st.v[s]
        if opt.get("amsgrad", True):
            st.vmax[s] = np.maximum(st.vmax[s], st.v[s])
            second = st.vmax[s]
        denom = np.sqrt(second) / math.sqrt(1 - b2 ** t) + eps
        codes[s] = codes[s] - lr / (1 - b1 ** t) * st.m[s] / denom
    return g, norms


def oracle_codes_step(model, cfg, x: torch.Tensor, codes: torch.Tensor, m: int, lr=None):
    """One fitting step in float64 on the oracle (oracle/ae_oracle.py): the conversion path (z = mu, eval-mode W_bar
    from the stored u and v with Decoder.sn), per speaker s lambda_rec x mean |dec - x| over its m crops, autograd
    with respect to the codes only, then code_adam_ref.  -> (g [S, C], norms [S], updated codes [S, C], losses [S])"""
    import oracle.ae_oracle as orc
    from _sn_ref import power_iteration64
    sd = {k: v.detach().double().cpu() for k, v in model.state_dict().items()}
    st = dict(sd)
    for n in [n for n in sd if n.endswith(".weight_orig")]:
        base = n[: -len(".weight_orig")]
        st[base + ".weight"] = power_iteration64(sd[n], sd[base + ".weight_u"], sd[base + ".weight_v"], iterate=False)[3]
    c = codes.detach().double().cpu().clone().requires_grad_(True)
    xd = x.double().cpu()
    with torch.no_grad():
        mu, _ = orc.content_encoder(st, xd, cfg["ContentEncoder"]["subsample"])
    dec = orc.decoder(st, mu, c.repeat_interleave(m, dim=0), cfg["Decoder"]["upsample"])
    S = c.shape[0]
    lam = cfg["lambda"]["lambda_rec"]
    losses = torch.stack([lam * (dec[s * m:(s + 1) * m] - xd[s * m:(s + 1) * m]).abs().mean() for s in range(S)])
    (gc,) = torch.autograd.grad(losses.sum(), [c])
    # the autograd gradient is the exact sum over the speaker's slots; restate it through code_adam_ref's row sum
    demb = np.repeat(gc.numpy() / m, m, axis=0)
    vals = codes.detach().double().cpu().numpy().copy()
    g, norms = code_adam_ref(vals, demb, m, CodeAdamState(S, c.shape[1]), cfg["optimizer"], lr)
    return g, norms, vals, losses.detach().numpy()
