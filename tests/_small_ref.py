"""float64 restatement of the small kernels of csrc/small_ops.cu and csrc/dense_fused.cu: the dense layers (per layer,
fused stack, L layers per launch), the time mean, the VAE reparameterisation, the L1 + KL loss, the gradient norm and
the clip + Adam(amsgrad) update.  Each function takes the fp32 operands the kernel reads, computes in float64 and
returns float64 tensors, following the contracts of include/avc_b200.h.  Shared by tests/test_small_ref_host.py
(against float64 autograd and torch.optim.Adam) and tests/test_gpu_small_ops_exact.py (against the kernels)."""
import math

import torch

from test_gpu_wgrad_exact import tf32_rna  # noqa: F401  (re-exported: cvt.rna.tf32.f32 on the bit pattern)


def _d(t):
    return None if t is None else t.double()


def rows_at(buf, off, bstride, B, W):
    """The [B][W] rows of a flat buffer starting at float `off`, rows `bstride` floats apart (the *_off / *_bstride
    addressing of the descriptors)."""
    return torch.as_strided(buf.reshape(-1), (B, W), (bstride, 1), off)


def relu(y):
    """max(y, 0) with the mask y > 0 (an exact zero passes no gradient, as torch's relu backward)."""
    return torch.where(y > 0, y, torch.zeros_like(y))


# ------------------------------------------------------------------ avc_linear_fwd / avc_linear_bwd
def linear_fwd(x, w, bias=None, *, relu_=False, res=None):
    """-> (out, y_act): y_act = act(x W^T + b), out = y_act + res."""
    y = _d(x) @ _d(w).T
    if bias is not None:
        y = y + _d(bias)
    if relu_:
        y = relu(y)
    return (y + _d(res) if res is not None else y), y


def linear_bwd(x, w, dy, *, y_act=None, dx_add=None, dw0=None, db0=None):
    """-> (dx, dw, db).  With y_act (the relu layers) the gradient is masked by y_act > 0; dx = g W (+ dx_add);
    dw = dw0 + g^T x and db = db0 + sum_b g accumulate onto what is passed in (db None when db0 is None)."""
    g = _d(dy)
    if y_act is not None:
        g = torch.where(_d(y_act) > 0, g, torch.zeros_like(g))
    dx = g @ _d(w)
    if dx_add is not None:
        dx = dx + _d(dx_add)
    dw = g.T @ _d(x) + (_d(dw0) if dw0 is not None else 0.0)
    db = g.sum(0) + _d(db0) if db0 is not None else None
    return dx, dw, db


# ------------------------------------------------------------------ avc_dense_stack_fwd / _bwd
def dense_stack_fwd(x, params, n_blocks):
    """params = [W1_l, b1_l]* [W2_l, b2_l]* Wo bo.  -> (out, save) with save [3n+1][B][C] = h_0..h_n | y_0.. | a_0..:
    y_l = relu(W1 h_l + b1), a_l = relu(W2 y_l + b2), h_{l+1} = h_l + a_l, out = Wo h_n + bo."""
    P = [_d(p) for p in params]
    nb = n_blocks
    h, ys, as_, hs = _d(x), [], [], [_d(x)]
    for l in range(nb):
        y = relu(h @ P[2 * l].T + P[2 * l + 1])
        a = relu(y @ P[2 * nb + 2 * l].T + P[2 * nb + 2 * l + 1])
        h = h + a
        ys.append(y)
        as_.append(a)
        hs.append(h)
    out = h @ P[4 * nb].T + P[4 * nb + 1]
    return out, torch.stack(hs + ys + as_)


def dense_stack_bwd(params, n_blocks, save, dout):
    """-> (dx, gsave) with gsave [2n+1][B][C] = g1_0.. | g2_0.. | dout: the upstream gradient of every layer after its
    ReLU mask, the masks taken from the given save planes (a_l > 0, y_l > 0)."""
    P = [_d(p) for p in params]
    nb = n_blocks
    S = _d(save)
    dh = _d(dout) @ P[4 * nb]
    g1, g2 = [None] * nb, [None] * nb
    for l in reversed(range(nb)):
        g2[l] = torch.where(S[2 * nb + 1 + l] > 0, dh, torch.zeros_like(dh))
        dy = g2[l] @ P[2 * nb + 2 * l]
        g1[l] = torch.where(S[nb + 1 + l] > 0, dy, torch.zeros_like(dy))
        dh = dh + g1[l] @ P[2 * l]
    return dh, torch.stack(g1 + g2 + [_d(dout)])


# ------------------------------------------------------------------ avc_linear_batch_fwd / _dx / _dw
def linear_batch_fwd(x, x_off, x_bstride, params, B, N, K):
    """-> [L] outputs [B][N]: layer l reads x rows at x_off[l]; params = [W_l, b_l]*, b_l may be None."""
    L = len(params) // 2
    return [linear_fwd(rows_at(x, x_off[l], x_bstride, B, K), params[2 * l], params[2 * l + 1])[0] for l in range(L)]


def linear_batch_dx(y, y_off, y_bstride, params, B, N, K, dx_add=None):
    """-> dx [B][K] = sum_l y_l W_l (+ dx_add), y_l the rows of y at y_off[l]."""
    L = len(params) // 2
    dx = sum(_d(rows_at(y, y_off[l], y_bstride, B, N)) @ _d(params[2 * l]) for l in range(L))
    return dx + _d(dx_add) if dx_add is not None else dx


def linear_batch_dw(x, x_off, x_bstride, y, y_off, y_bstride, grads0, B, N, K):
    """-> [dW_l, db_l]*: grads0 (the preloaded [dW_l, db_l]*, db_l may be None) plus sum_b y_l^T x_l and sum_b y_l."""
    L = len(grads0) // 2
    out = []
    for l in range(L):
        _, dw, db = linear_bwd(rows_at(x, x_off[l], x_bstride, B, K), torch.zeros(N, K), rows_at(y, y_off[l], y_bstride, B, N),
                               dw0=grads0[2 * l], db0=grads0[2 * l + 1])
        out += [dw, db]
    return out


# ------------------------------------------------------------------ avc_time_mean_fwd / _bwd
def time_mean_fwd(x):
    """planar [B][C][T] -> [B][C]: AdaptiveAvgPool1d(1)."""
    return _d(x).mean(dim=2)


def time_mean_bwd(dout, T):
    """[B][C] -> [B][C][T]: every step receives dout / T."""
    return (_d(dout) / T)[:, :, None].expand(-1, -1, T)


# ------------------------------------------------------------------ avc_reparam_fwd / _bwd
def reparam_fwd(mu, ls, eps=None):
    """z = mu + exp(ls / 2) eps; z = mu without eps (inference)."""
    if eps is None:
        return _d(mu)
    return _d(mu) + torch.exp(_d(ls) / 2) * _d(eps)


def reparam_bwd(dz, ls, eps=None, dmu_ext=None, dls_ext=None):
    """-> (dmu, dls): dmu = dz + dmu_ext, dls = dz eps exp(ls / 2) / 2 + dls_ext; a null dz counts as 0."""
    ref = _d(ls) if ls is not None else _d(dmu_ext if dmu_ext is not None else dls_ext)
    dz = _d(dz) if dz is not None else torch.zeros_like(ref)
    dmu = dz + (_d(dmu_ext) if dmu_ext is not None else 0.0)
    dls = dz * _d(eps) * 0.5 * torch.exp(_d(ls) / 2) if eps is not None else torch.zeros_like(dz)
    return dmu, dls + (_d(dls_ext) if dls_ext is not None else 0.0)


# ------------------------------------------------------------------ avc_vae_loss
def vae_loss(dec, x, mu, ls, hp):
    """-> (sum |dec - x|, sum (e^ls + mu^2 - 1 - ls), ddec, dmu, dls), the gradients of lambda_rec * mean|dec - x| +
    lambda_kl * 0.5 * mean(e^ls + mu^2 - 1 - ls); hp is the fp32 device vector ([0] lambda_rec, [1] lambda_kl)."""
    lrec, lkl = float(hp[0]), float(hp[1])
    df = _d(dec) - _d(x)
    m, l = _d(mu), _d(ls)
    e = torch.exp(l)
    return (df.abs().sum(), (e + m * m - 1 - l).sum(), torch.sign(df) * (lrec / df.numel()),
            (lkl / m.numel()) * m, (lkl / m.numel()) * 0.5 * (e - 1))


# ------------------------------------------------------------------ avc_sqnorm / avc_adam_step
HP_GSCALE, HP_LR, HP_B1, HP_B2, HP_EPS, HP_WD, HP_MAXNORM, HP_AMSGRAD = range(2, 10)
CLIP_EPS = 1e-6        # clip_grad_norm_'s max_norm / (norm + 1e-6)


def sqnorm(g):
    return float((_d(g) ** 2).sum())


def clip_coef(hp, sq):
    """min(1, max_norm / (grad_scale sqrt(sqnorm) + 1e-6)) * grad_scale: what multiplies the summed gradient."""
    gs, mx = float(hp[HP_GSCALE]), float(hp[HP_MAXNORM])
    return min(1.0, mx / (gs * math.sqrt(sq) + CLIP_EPS)) * gs


def adam_step(p, g, m, v, vmax, step, hp, sq):
    """One avc_adam_step: clip by the given sum of squares `sq`, L2 weight decay folded into the gradient, Adam with
    bias corrections at step + 1, amsgrad from hp.  hp is the fp32 device vector, read as the kernel reads it.
    -> (p, m, v, vmax, step + 1); vmax is returned unchanged without amsgrad."""
    lr, b1, b2 = float(hp[HP_LR]), float(hp[HP_B1]), float(hp[HP_B2])
    eps, wd, ams = float(hp[HP_EPS]), float(hp[HP_WD]), float(hp[HP_AMSGRAD]) != 0.0
    t = float(step) + 1
    p, m, v, vmax = _d(p), _d(m), _d(v), _d(vmax)
    gi = _d(g) * clip_coef(hp, sq) + wd * p
    m = m + (1 - b1) * (gi - m)
    v = b2 * v + (1 - b2) * gi * gi
    second = torch.maximum(vmax, v) if ams else v
    denom = second.sqrt() / math.sqrt(1 - b2 ** t) + eps
    p = p - lr / (1 - b1 ** t) * m / denom
    return p, m, v, (second if ams else vmax), t
