"""CPU: the float64 restatement in tests/_norm_ref.py (what tests/test_gpu_norm_exact.py measures the kernels of
csrc/norm.cu against) equals float64 autograd of the oracle's own primitives, and the entry points of those kernels
reject the descriptors their host checks forbid before anything is launched."""
import itertools

import pytest
import torch
import torch.nn.functional as F

import oracle.ae_oracle as orc
from _norm_ref import RES_NONE, RES_POOL, RES_SAME, RES_UP, bias_sums, fold_add, norm_apply, norm_bwd

EPS = orc.IN_EPS


def oracle_chain(c, *, shuffle, norm, cond, relu, res=None, res_mode=RES_NONE, mask=None):
    """The block epilogue as the oracle writes it (model.py's ConvBlock order)."""
    y = orc.pixel_shuffle_1d(c, 2) if shuffle else c
    if norm:
        y = orc.instance_norm(y)
    if cond is not None:
        y = orc.adain(y, cond)
    if relu:
        y = F.relu(y)
    if res is not None:
        y = y + {RES_SAME: lambda: res, RES_POOL: lambda: F.avg_pool1d(res, 2, ceil_mode=True),
                 RES_UP: lambda: F.interpolate(res, scale_factor=2, mode="nearest")}[res_mode]()
    if mask is not None:
        y = y * (mask > 0)
    return y


def inputs(B, Cout, Tout, seed, edge=True):
    """c with, per sample, a channel constant over time and one with a DC offset 100x its spread."""
    g = torch.Generator().manual_seed(seed)
    c = torch.randn((B, Cout, Tout), generator=g, dtype=torch.float64) + torch.randn((1, Cout, 1), generator=g, dtype=torch.float64)
    if edge:
        c[:, 0:2] = 0.37                                            # rows 0 and 1: normalised channel 0 also under shuffle
        c[:, 4:6] = 100.0 + torch.randn((B, 2, Tout), generator=g, dtype=torch.float64)
    return c, g


def close(a, b, rel=1e-12):
    return float((a - b).abs().max()) <= rel * max(float(b.abs().max()), 1e-300)


FWD = [(s, n, cd, r, m, mk) for s, n, cd, r, m, mk in itertools.product((0, 1), (0, 1), (0, 1), (0, 1), (0, 1, 2, 3), (0, 1))]


@pytest.mark.parametrize("Tout", [1, 7, 16])
@pytest.mark.parametrize("shuffle,norm,cond,relu,mode,mask", FWD)
def test_norm_apply_equals_oracle(shuffle, norm, cond, relu, mode, mask, Tout):
    """Every flag combination, every residual mode (avg-pool with an even and an odd input length), odd lengths."""
    B, Cout = 3, 16
    c, g = inputs(B, Cout, Tout, 1000 * Tout + 7)
    Cn, Tn = (Cout // 2, 2 * Tout) if shuffle else (Cout, Tout)
    if mode == RES_UP and Tn % 2:
        pytest.skip("nearest-upsampling gives even lengths only")
    cd = torch.randn((B, 2 * Cn), generator=g, dtype=torch.float64) * 0.5 + 0.7 if cond else None
    mk = (torch.randn((B, Cn, Tn), generator=g, dtype=torch.float64) > -0.5).double() if mask else None
    res_lens = {RES_NONE: [None], RES_SAME: [Tn], RES_POOL: [2 * Tn, 2 * Tn - 1], RES_UP: [Tn // 2]}[mode]
    for rT in res_lens:
        res = torch.randn((B, Cn, rT), generator=g, dtype=torch.float64) if rT else None
        out, mean, rstd = norm_apply(c, shuffle=bool(shuffle), norm=bool(norm), eps=EPS, cond=cd, relu=bool(relu), res=res,
                                     res_mode=mode, mask=mk)
        ref = oracle_chain(c, shuffle=shuffle, norm=norm, cond=cd, relu=relu, res=res, res_mode=mode, mask=mk)
        assert out.shape == ref.shape and close(out, ref), (rT, float((out - ref).abs().max()))
        if norm:
            y = orc.pixel_shuffle_1d(c, 2) if shuffle else c
            assert close(mean, y.mean(dim=2))
            assert close(rstd, 1 / torch.sqrt(y.var(dim=2, unbiased=False) + EPS))


BWD = [(s, n, cd, r) for s, n, cd, r in itertools.product((0, 1), (0, 1), (0, 1), (0, 1)) if n or not cd]


@pytest.mark.parametrize("Tout", [1, 7, 37])
@pytest.mark.parametrize("shuffle,norm,cond,relu", BWD)
def test_norm_bwd_equals_full_autograd(shuffle, norm, cond, relu, Tout):
    """With the true statistics, the adjoint at fixed statistics plus its analytic correction is the full adjoint of
    the oracle's pixel shuffle -> instance norm -> AdaIN -> ReLU, for dc, the AdaIN-row gradient and the bias
    gradient; a constant channel (rstd = eps^-1/2) and a DC-offset channel included."""
    B, Cout = 3, 16
    c, g = inputs(B, Cout, Tout, 2000 * Tout + 11)
    Cn, Tn = (Cout // 2, 2 * Tout) if shuffle else (Cout, Tout)
    cd = torch.randn((B, 2 * Cn), generator=g, dtype=torch.float64) * 0.5 + 0.7 if cond else None
    dy = torch.randn((B, Cn, Tn), generator=g, dtype=torch.float64)
    x = c.clone().requires_grad_(True)
    cd_ = cd.clone().requires_grad_(True) if cd is not None else None
    (oracle_chain(x, shuffle=shuffle, norm=norm, cond=cd_, relu=relu) * dy).sum().backward()
    _, mean, rstd = norm_apply(c, shuffle=bool(shuffle), norm=bool(norm), eps=EPS)
    dc, dcond, dbias = norm_bwd(c, mean, rstd, cd, dy, shuffle=bool(shuffle), norm=bool(norm), relu=bool(relu))
    # dc's scale is rstd |gamma| |dy| (at Tout = 1 the true dc is exactly 0)
    scale = float(dy.abs().max()) * (float(rstd.max()) if norm else 1.0) * (float(cd[:, Cn:].abs().max()) if cond else 1.0)
    assert float((dc - x.grad).abs().max()) <= 1e-12 * scale
    # (a conv row that feeds an InstanceNorm alone has a bias gradient of 0)
    assert float((dbias - x.grad.sum(dim=(0, 2))).abs().max()) <= 1e-12 * scale * B * Tout
    if cond:
        assert close(dcond, cd_.grad, 1e-12)
    if norm and not cond:   # the AdaIN-row gradient of gamma = 1, beta = 0
        xg = c.clone().requires_grad_(True)
        bg = torch.zeros((B, Cn), dtype=torch.float64, requires_grad=True)
        gg = torch.ones((B, Cn), dtype=torch.float64, requires_grad=True)
        y = orc.instance_norm(orc.pixel_shuffle_1d(xg, 2) if shuffle else xg) * gg[:, :, None] + bg[:, :, None]
        ((F.relu(y) if relu else y) * dy).sum().backward()
        assert close(dcond, torch.cat([bg.grad, gg.grad], 1), 1e-12)
    if not norm:
        assert dcond is None


def test_norm_bwd_holds_the_given_statistics():
    """With statistics off the true ones (as fp32 rounding leaves them) the restatement follows the given values: it
    is the adjoint of the normalisation written with those constants, plus the correction at those constants."""
    B, Cout, Tout = 2, 8, 9
    c, g = inputs(B, Cout, Tout, 5, edge=False)
    _, mean, rstd = norm_apply(c, norm=True, eps=EPS)
    mean_f, rstd_f = mean * (1 + 1e-3), rstd * (1 - 1e-3)
    dy = torch.randn((B, Cout, Tout), generator=g, dtype=torch.float64)
    dc, dcond, _ = norm_bwd(c, mean_f, rstd_f, None, dy, norm=True)
    xh = (c - mean_f[:, :, None]) * rstd_f[:, :, None]
    s0, s1 = dy.sum(2), (dy * xh).sum(2)
    assert close(dcond, torch.cat([s0, s1], 1))
    assert close(dc, rstd_f[:, :, None] * (dy - s0[:, :, None] / Tout - xh * s1[:, :, None] / Tout))
    exact, _, _ = norm_bwd(c, mean, rstd, None, dy, norm=True)
    assert not close(dc, exact, 1e-6)


def pads(K):
    return K // 2, K // 2 - (1 if K % 2 == 0 else 0)


FOLD = [(K, T, m) for K in range(1, 9) for T in sorted({pads(K)[0] + 1, pads(K)[0] + 2, 5, 8})
        for m in (RES_NONE, RES_SAME, RES_POOL, RES_UP)]


@pytest.mark.parametrize("K,Tin,mode", FOLD)
def test_fold_add_equals_pad_adjoint(K, Tin, mode):
    """Every (pl, pr) of K = 1..8, the smallest legal input (Tin = pl + 1: with K = 8 the left and right reflect
    regions overlap), odd lengths under the avg-pool residual, every residual mode."""
    pl, pr = pads(K)
    g =torch.Generator().manual_seed(97 * K + 13 * Tin + mode)
    B, Cc = 2, 8
    dxp = torch.randn((B, Cc, Tin + pl + pr), generator=g, dtype=torch.float64)
    rT = {RES_NONE: 0, RES_SAME: Tin, RES_POOL: (Tin + 1) // 2, RES_UP: 2 * Tin}[mode]
    dres = torch.randn((B, Cc, rT), generator=g, dtype=torch.float64) if rT else None
    xi = torch.zeros((B, Cc, Tin), dtype=torch.float64, requires_grad=True)
    obj = (F.pad(xi, (pl, pr), mode="reflect") * dxp).sum()
    if rT:
        br = {RES_SAME: lambda: xi, RES_POOL: lambda: F.avg_pool1d(xi, 2, ceil_mode=True),
              RES_UP: lambda: F.interpolate(xi, scale_factor=2, mode="nearest")}[mode]()
        obj = obj + (br * dres).sum()
    obj.backward()
    assert close(fold_add(dxp, pl, pr, dres, mode), xi.grad)


def test_bias_sums():
    g = torch.Generator().manual_seed(3)
    dc = torch.randn((3, 16, 5), generator=g, dtype=torch.float64)
    assert close(bias_sums(dc), torch.stack([dc[:, c].sum() for c in range(16)]))
    assert close(bias_sums(dc, 4)[2], torch.stack([dc[:, 8 + c].sum() for c in range(4)]))


def test_host_checks_reject_before_any_launch():
    """Descriptors the host checks forbid return their error code; these calls run on a machine without a GPU too,
    so nothing was launched.  Pointers are placeholders that a rejected call never reads."""
    from adaptive_voice_conversion_b200 import _lib as L
    import ctypes as C
    lib = L.load()
    fake = 1 << 20
    d = L.ConvDesc()
    d.B, d.Cin, d.Cout, d.K, d.stride, d.in_ups, d.Tin, d.Tout = 2, 4, 128, 1, 1, 1, 16, 16
    d.save_c, d.dy, d.dc, d.dy_bstride, d.eps = fake, fake, fake, 128 * 16, EPS
    d.norm, d.stats = 1, None
    assert lib.avc_norm_bwd(C.byref(d), None) == L.ERR_INVALID and "stats" in L.last_error()
    d.norm, d.stats, d.cond, d.cond_bstride = 0, fake, fake, 256
    assert lib.avc_norm_bwd(C.byref(d), None) == L.ERR_UNSUPPORTED and "AdaIN" in L.last_error()
    assert lib.avc_bias_grad(fake, 128 * 1025, fake, 2, 128, 1025, None) == L.ERR_UNSUPPORTED and "1025" in L.last_error()
    assert lib.avc_bias_grad_groups(fake, 1024 * 1025, fake, 128, 2, 1024, 1025, None) == L.ERR_UNSUPPORTED
    assert "1025" in L.last_error()
