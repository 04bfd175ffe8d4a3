"""float64 restatement of the InstanceNorm / AdaIN / ReLU / residual epilogue of a conv block, of its backward, of the
reflect-padding + residual adjoint and of the bias gradient, on planar [B][C][T] tensors.  Each function takes exactly
the operands the corresponding kernel of csrc/norm.cu reads.  Shared by tests/test_norm_ref_host.py (against autograd
of the oracle's primitives) and tests/test_gpu_norm_exact.py (against the kernels)."""
import torch

from test_gpu_tc2_exact import from_a4, relerr, tf32, to_a4  # noqa: F401  (re-exported for the GPU module)

RES_NONE, RES_SAME, RES_POOL, RES_UP = 0, 1, 2, 3


def shuffle1d(c):
    """pixel shuffle by 2: conv row 2ch+s at time t -> channel ch at time 2t+s."""
    B, C2, T = c.shape
    return c.reshape(B, C2 // 2, 2, T).transpose(2, 3).reshape(B, C2 // 2, 2 * T)


def unshuffle1d(y):
    """inverse of shuffle1d."""
    B, Cn, T2 = y.shape
    return y.reshape(B, Cn, T2 // 2, 2).transpose(2, 3).reshape(B, 2 * Cn, T2 // 2)


def residual(res, mode, Tn):
    """the residual branch at the block output's length Tn: same, avg-pool 2 (ceil_mode: a lone last sample counts
    alone), nearest-upsample 2."""
    r = res.double()
    if mode == RES_SAME:
        return r
    if mode == RES_UP:
        return r.repeat_interleave(2, dim=2)
    assert mode == RES_POOL
    T = r.shape[2]
    out = torch.zeros(r.shape[0], r.shape[1], (T + 1) // 2, dtype=torch.float64)
    out += r[:, :, 0::2]
    out[:, :, : T // 2] = 0.5 * (out[:, :, : T // 2] + r[:, :, 1::2])
    assert out.shape[2] == Tn
    return out


def norm_apply(c, *, shuffle=False, norm=False, eps=1e-5, cond=None, relu=False, res=None, res_mode=RES_NONE, mask=None):
    """-> (out, mean, rstd) in float64; mean / rstd [B][Cn] (None without norm).  c: raw conv output [B][Cout][Tout];
    cond: AdaIN rows [B][2 Cn] (beta | gamma); res at the length its mode needs; mask like out."""
    y = c.double()
    if shuffle:
        y = shuffle1d(y)
    Cn, Tn = y.shape[1], y.shape[2]
    mean = rstd = None
    if norm:
        mean = y.sum(dim=2) / Tn
        var = ((y - mean[:, :, None]) ** 2).sum(dim=2) / Tn
        rstd = 1.0 / torch.sqrt(var + eps)
        y = (y - mean[:, :, None]) * rstd[:, :, None]
    if cond is not None:
        cd = cond.double()
        y = y * cd[:, Cn:, None] + cd[:, :Cn, None]
    if relu:
        y = torch.where(y > 0, y, torch.zeros_like(y))
    if res is not None:
        y = y + residual(res, res_mode, Tn)
    if mask is not None:
        y = torch.where(mask > 0, y, torch.zeros_like(y))
    return y, mean, rstd


def norm_bwd(c, mean, rstd, cond, dy, *, shuffle=False, norm=False, relu=False):
    """Adjoint of norm_apply's normalisation / AdaIN / ReLU at the GIVEN statistics (the fp32 ones the kernel reads)
    -> (dc [B][Cout][Tout], dcond [B][2 Cn] = (sum g | sum g xhat) or None without norm, dbias [Cout] = sum of dc).

    The part with mean and rstd held constant is float64 autograd; their dependence on c (d mean / dy_t = 1/Tn,
    d rstd / dy_t = -rstd^3 (y_t - mean) / Tn) is added analytically:  dc = rstd gamma (g - s0/Tn - xhat s1/Tn)."""
    c64 = c.double().clone().requires_grad_(True)
    y = shuffle1d(c64) if shuffle else c64
    B, Cn, Tn = y.shape
    dy = dy.double()
    if not norm:
        assert cond is None, "AdaIN without InstanceNorm"
        pre = y
        (torch.relu(pre) if relu else pre).mul(dy).sum().backward()
        dc = c64.grad
        return dc, None, dc.sum(dim=(0, 2))
    m, r = mean.double()[:, :, None], rstd.double()[:, :, None]
    cd = cond.double() if cond is not None else torch.cat([torch.zeros(B, Cn), torch.ones(B, Cn)], 1).double()
    beta = cd[:, :Cn].clone().requires_grad_(True)
    gamma = cd[:, Cn:].clone().requires_grad_(True)
    xh = (y - m) * r
    pre = xh * gamma[:, :, None] + beta[:, :, None]
    (torch.relu(pre) if relu else pre).mul(dy).sum().backward()
    s0, s1 = beta.grad, gamma.grad                      # sum g, sum g * xhat (g: dy behind the ReLU mask)
    corr = -(r * gamma.detach()[:, :, None]) * (s0[:, :, None] + xh.detach() * s1[:, :, None]) / Tn
    dc = c64.grad + (unshuffle1d(corr) if shuffle else corr)
    return dc, torch.cat([s0, s1], 1), dc.sum(dim=(0, 2))


def fold_add(dxp, pl, pr, dres=None, res_mode=RES_NONE):
    """Adjoint of F.pad(x, (pl, pr), mode="reflect") applied to dxp [B][C][T + pl + pr], plus the adjoint of the
    block's residual branch applied to dres -> dx [B][C][T]."""
    g = dxp.double()
    T = g.shape[2] - pl - pr
    dx = g[:, :, pl:pl + T].clone()
    for j in range(pl):                 # padded column j mirrors input pl - j
        dx[:, :, pl - j] += g[:, :, j]
    for j in range(pr):                 # padded column pl + T + j mirrors input T - 2 - j
        dx[:, :, T - 2 - j] += g[:, :, pl + T + j]
    if dres is not None:
        r = dres.double()
        if res_mode == RES_SAME:
            dx += r
        elif res_mode == RES_POOL:      # x[t] fed pooled column t // 2, with weight 1/2 unless it is a lone tail
            w = torch.full((T,), 0.5, dtype=torch.float64)
            if T % 2:
                w[-1] = 1.0
            dx += r.repeat_interleave(2, dim=2)[:, :, :T] * w
        else:
            assert res_mode == RES_UP
            dx += r[:, :, 0::2] + r[:, :, 1::2]
    return dx


def bias_sums(dc, group_c=None):
    """sum over (b, t) of dc [B][C][T] -> [C], or [C / group_c][group_c] for layers side by side."""
    s = dc.double().sum(dim=(0, 2))
    return s if group_c is None else s.reshape(-1, group_c)
