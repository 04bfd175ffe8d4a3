"""CPU: the float64 restatement in tests/_small_ref.py (what tests/test_gpu_small_ops_exact.py measures the kernels of
csrc/small_ops.cu and csrc/dense_fused.cu against) equals float64 autograd of the oracle's op sequence -- the dense
blocks and output layer of the speaker encoder (model.py:252-263, :273-276), the AdaIN affine layers (:342-343), the
reparameterisation (:383-384) and the losses (solver.py:84-88) -- and clip_grad_norm_ + torch.optim.Adam; tf32_rna is
checked on hand-made bit patterns."""
import pytest
import torch
import torch.nn.functional as F

import oracle.ae_oracle as orc
import _small_ref as R


def close(a, b, rel=1e-12):
    a, b = a.detach().double(), b.detach().double()
    return float((a - b).abs().max()) <= rel * max(float(b.abs().max()), 1e-300)


def rnd(g, *shape):
    return torch.randn(shape, generator=g)


def leaf(t):
    return t.double().clone().requires_grad_(True)


@pytest.mark.parametrize("B,K,N", [(1, 1, 1), (5, 7, 9), (33, 31, 80)])
@pytest.mark.parametrize("relu", [False, True])
@pytest.mark.parametrize("bias,res,dx_add", [(True, True, True), (False, False, False), (True, False, True)])
def test_linear_equals_autograd(B, K, N, relu, bias, res, dx_add):
    """relu(x W^T + b) + res, its input / weight / bias gradients accumulated onto preloaded values; weight row 0 and
    bias 0 zero, so y_act[:, 0] is an exact 0 whose gradient torch's relu blocks, as the restatement's mask must."""
    g = torch.Generator().manual_seed(B * 1000 + K * 10 + N + 7 * relu + 3 * bias)
    x, w, dy = rnd(g, B, K), rnd(g, N, K), rnd(g, B, N)
    b = rnd(g, N) if bias else None
    r = rnd(g, B, N) if res else None
    xa = rnd(g, B, K) if dx_add else None
    dw0, db0 = rnd(g, N, K), rnd(g, N)
    w[0] = 0.0
    if bias:
        b[0] = 0.0
    xl, wl, bl = leaf(x), leaf(w), (leaf(b) if bias else None)
    y = F.linear(xl, wl, bl)
    y = F.relu(y) if relu else y
    out_t = y + r.double() if res else y
    (out_t * dy.double()).sum().backward()
    out, y_act = R.linear_fwd(x, w, b, relu_=relu, res=r)
    assert close(out, out_t) and close(y_act, y)
    dx, dw, db = R.linear_bwd(x, w, dy, y_act=y_act if relu else None, dx_add=xa, dw0=dw0, db0=db0 if bias else None)
    assert close(dx, xl.grad + (xa.double() if dx_add else 0))
    assert close(dw, wl.grad + dw0.double())
    if bias:
        assert close(db, bl.grad + db0.double())
    else:
        assert db is None
    if relu:
        assert bool((y_act[:, 0] == 0).all()) and float(dw[0].sub(dw0[0].double()).abs().max()) == 0.0


def stack_state(nb, C, g):
    P = []
    for _ in range(2 * nb + 1):
        P += [rnd(g, C, C) / C ** 0.5, 0.1 * rnd(g, C)]
    if nb:
        P[0][0], P[1][0] = 0.0, 0.0          # W1_0 row 0, b1_0[0]: y_0[:, 0] is an exact 0
    return P


@pytest.mark.parametrize("nb", [0, 1, 3])
@pytest.mark.parametrize("B", [1, 5])
def test_dense_stack_equals_autograd(nb, B):
    """The oracle's dense blocks and output layer: out, the save planes (h_l, y_l, a_l), dx, and the gsave planes as
    the left operands of the weight gradients (dW = g^T input, db = sum g)."""
    C = 12
    g = torch.Generator().manual_seed(100 * nb + B)
    P = stack_state(nb, C, g)
    x, dout = rnd(g, B, C), rnd(g, B, C)
    L = [leaf(p) for p in P]
    xl = leaf(x)
    h, hs, ys, as_ = xl, [xl], [], []
    for l in range(nb):                              # oracle/ae_oracle.py speaker_encoder, dense part
        y = F.relu(F.linear(h, L[2 * l], L[2 * l + 1]))
        a = F.relu(F.linear(y, L[2 * nb + 2 * l], L[2 * nb + 2 * l + 1]))
        h = a + h
        hs.append(h)
        ys.append(y)
        as_.append(a)
    out_t = F.linear(h, L[4 * nb], L[4 * nb + 1])
    (out_t * dout.double()).sum().backward()
    out, save = R.dense_stack_fwd(x, P, nb)
    assert save.shape == (3 * nb + 1, B, C)
    assert close(out, out_t) and close(save, torch.stack(hs + ys + as_))
    dx, gsave = R.dense_stack_bwd(P, nb, save, dout)
    assert gsave.shape == (2 * nb + 1, B, C)
    assert close(dx, xl.grad)
    for l in range(nb):
        for gi, inp, wi in ((gsave[l], save[l], 2 * l), (gsave[nb + l], save[nb + 1 + l], 2 * nb + 2 * l)):
            assert close(gi.T @ inp, L[wi].grad) and close(gi.sum(0), L[wi + 1].grad)
    assert close(gsave[2 * nb].T @ save[nb], L[4 * nb].grad)
    if nb:
        assert bool((save[nb + 1][:, 0] == 0).all()) and bool((gsave[0][:, 0] == 0).all())


@pytest.mark.parametrize("layout", ["affine", "planes"])
def test_linear_batch_equals_autograd(layout):
    """L = 4 layers, one of them without bias: the affine layout (shared x, rows L N + 2 apart) and per-layer planes."""
    Ln, B, N, K = 4, 3, 6, 5
    g = torch.Generator().manual_seed(len(layout))
    W = [rnd(g, N, K) for _ in range(Ln)]
    bs = [None if l == 1 else rnd(g, N) for l in range(Ln)]
    dW0 = [rnd(g, N, K) for _ in range(Ln)]
    db0 = [None if l == 1 else rnd(g, N) for l in range(Ln)]
    if layout == "affine":
        xbuf, x_off, x_bs = rnd(g, B * K), [0] * Ln, K
        y_bs, y_off = Ln * N + 2, [l * N for l in range(Ln)]
        ybuf = rnd(g, B * y_bs)
    else:
        xbuf, x_off, x_bs = rnd(g, (Ln + 1) * B * K), [(l + 1) % (Ln + 1) * B * K for l in range(Ln)], K
        ybuf, y_off, y_bs = rnd(g, Ln * B * N), [(Ln - 1 - l) * B * N for l in range(Ln)], N
    dx_add = rnd(g, B, K)
    xl = leaf(xbuf)
    Wl, bl = [leaf(w) for w in W], [leaf(b) if b is not None else None for b in bs]
    outs = [F.linear(R.rows_at(xl, x_off[l], x_bs, B, K), Wl[l], bl[l]) for l in range(Ln)]
    sum((o * R.rows_at(ybuf, y_off[l], y_bs, B, N).double()).sum() for l, o in enumerate(outs)).backward()
    params = [t for l in range(Ln) for t in (W[l], bs[l])]
    got = R.linear_batch_fwd(xbuf, x_off, x_bs, params, B, N, K)
    assert all(close(a, b) for a, b in zip(got, outs))
    dx = R.linear_batch_dx(ybuf, y_off, y_bs, params, B, N, K, dx_add)
    if layout == "affine":                # every layer reads the same x: its gradient is the sum over layers
        assert close(dx, R.rows_at(xl.grad, 0, K, B, K) + dx_add.double())
    else:                                 # layer l's plane receives y_l W_l alone
        for l in range(Ln):
            one = R.linear_batch_dx(ybuf, [y_off[l]], y_bs, params[2 * l:2 * l + 2], B, N, K)
            assert close(one, R.rows_at(xl.grad, x_off[l], x_bs, B, K))
    gr = R.linear_batch_dw(xbuf, x_off, x_bs, ybuf, y_off, y_bs, [t for l in range(Ln) for t in (dW0[l], db0[l])], B, N, K)
    for l in range(Ln):
        assert close(gr[2 * l], Wl[l].grad + dW0[l].double())
        if bs[l] is None:
            assert gr[2 * l + 1] is None
        else:
            assert close(gr[2 * l + 1], bl[l].grad + db0[l].double())


@pytest.mark.parametrize("T", [1, 7, 125])
def test_time_mean_equals_autograd(T):
    g = torch.Generator().manual_seed(T)
    x, dout = rnd(g, 3, 8, T), rnd(g, 3, 8)
    xl = leaf(x)
    m = xl.mean(dim=2)                              # AdaptiveAvgPool1d(1).squeeze(2)
    (m * dout.double()).sum().backward()
    assert close(R.time_mean_fwd(x), m) and close(R.time_mean_bwd(dout, T), xl.grad)


@pytest.mark.parametrize("eps,dz,dmu_ext,dls_ext", [(1, 1, 1, 1), (1, 1, 0, 0), (0, 1, 1, 1), (1, 0, 1, 0), (0, 0, 0, 1)])
def test_reparam_equals_autograd(eps, dz, dmu_ext, dls_ext):
    """z = mu + exp(ls / 2) eps (oracle ae_forward), z = mu without eps; the external gradients add."""
    g = torch.Generator().manual_seed(16 * eps + 8 * dz + 4 * dmu_ext + 2 * dls_ext)
    mu, ls, e, gz = rnd(g, 2, 8, 5), rnd(g, 2, 8, 5), rnd(g, 2, 8, 5), rnd(g, 2, 8, 5)
    em, el = rnd(g, 2, 8, 5), rnd(g, 2, 8, 5)
    ml, ll = leaf(mu), leaf(ls)
    z = ml + torch.exp(ll / 2) * e.double() if eps else ml + 0 * ll
    if dz:
        (z * gz.double()).sum().backward()
    zr = R.reparam_fwd(mu, ls, e if eps else None)
    assert close(zr, z)
    dmu, dls = R.reparam_bwd(gz if dz else None, ls, e if eps else None, em if dmu_ext else None, el if dls_ext else None)
    zero = torch.zeros_like(mu, dtype=torch.float64)
    assert close(dmu, (ml.grad if dz else zero) + (em.double() if dmu_ext else 0))
    assert close(dls, (ll.grad if dz else zero) + (el.double() if dls_ext else 0))


@pytest.mark.parametrize("n_rec,n_lat", [(1, 3), (97, 40), (40, 97)])
def test_vae_loss_equals_autograd(n_rec, n_lat):
    """sums and the gradients of lambda_rec * L1 + lambda_kl * KL (oracle ae_losses), with exact ties dec = x (the
    gradient of |0| is 0 in torch too) and log-sigmas at and near 0."""
    g = torch.Generator().manual_seed(n_rec * 7 + n_lat)
    dec, x = rnd(g, n_rec), rnd(g, n_rec)
    dec[: (n_rec + 2) // 3] = x[: (n_rec + 2) // 3]
    mu, ls = rnd(g, n_lat), rnd(g, n_lat)
    ls[0], ls[1:4] = 0.0, 1e-6
    hp = torch.zeros(16)
    hp[0], hp[1] = 10.0, 0.7
    dl, ml, ll = leaf(dec), leaf(mu), leaf(ls)
    rec, kl = orc.ae_losses(x.double(), ml, ll, dl)
    (float(hp[0]) * rec + float(hp[1]) * kl).backward()
    s_rec, s_kl, ddec, dmu, dls = R.vae_loss(dec, x, mu, ls, hp)
    assert close(s_rec / n_rec, rec) and close(0.5 * s_kl / n_lat, kl)
    assert close(ddec, dl.grad) and close(dmu, ml.grad)
    # autograd forms e^l - 1 from two terms, which cancel near l = 0: compare on the scale of those terms
    assert float((dls - ll.grad).abs().max()) <= 1e-14 * float(hp[1]) / n_lat * float((torch.exp(ls.double()) + 1).max())
    assert bool((ddec[: (n_rec + 2) // 3] == 0).all())


def f32(v):
    return float(torch.tensor(v, dtype=torch.float32))


@pytest.mark.parametrize("step0", [0, 199999])
@pytest.mark.parametrize("gscale", [1.0, 0.5])
@pytest.mark.parametrize("wd", [0.0, 1e-4])
@pytest.mark.parametrize("ams", [0, 1])
def test_adam_step_equals_torch_adam(ams, wd, gscale, step0):
    """adam_step iterated against clip_grad_norm_ + torch.optim.Adam(amsgrad, weight_decay) in float64, the
    hyper-parameters fp32-exact so that both read the same values; clipping on every other step; grad_scale 0.5 with
    twice the gradient is the world-size-2 form (summed gradients); a resumed step counter (bias corrections ~ 1)."""
    n = 50
    g = torch.Generator().manual_seed(ams * 8 + int(wd > 0) * 4 + int(gscale * 2) + step0)
    lr, b1, b2, eps, wdf, mx = f32(5e-4), f32(0.9), f32(0.999), f32(1e-8), f32(wd), 5.0
    hp = torch.tensor([10, 1, gscale, lr, b1, b2, eps, wdf, mx, float(ams)] + [0] * 6, dtype=torch.float32)
    p = rnd(g, n).double()
    pt = p.clone().requires_grad_(True)
    opt = torch.optim.Adam([pt], lr=lr, betas=(b1, b2), eps=eps, weight_decay=wdf, amsgrad=bool(ams))
    m, v, vmax = torch.zeros(n, dtype=torch.float64), torch.zeros(n, dtype=torch.float64), torch.zeros(n, dtype=torch.float64)
    if step0:
        m, v = 1e-3 * rnd(g, n).double(), 1e-6 * rnd(g, n).double() ** 2
        vmax = 1.5 * v
        opt.state[pt] = {"step": torch.tensor(float(step0)), "exp_avg": m.clone(), "exp_avg_sq": v.clone()}
        if ams:
            opt.state[pt]["max_exp_avg_sq"] = vmax.clone()
    step = float(step0)
    vmax0 = vmax.clone()
    clipped = set()
    for s in range(6):
        gr = rnd(g, n).double() * (3.0 if s % 2 == 0 else 0.01)
        gr[0] = 0.0
        pt.grad = gr.clone()
        norm = float(torch.nn.utils.clip_grad_norm_([pt], max_norm=mx))
        clipped.add(norm > mx)
        opt.step()
        gsum = gr / gscale
        p, m, v, vmax, step = R.adam_step(p, gsum, m, v, vmax, step, hp, R.sqnorm(gsum))
        st = opt.state[pt]
        assert close(p, pt.detach()) and close(m, st["exp_avg"]) and close(v, st["exp_avg_sq"]), s
        if ams:
            assert close(vmax, st["max_exp_avg_sq"])
        else:
            assert torch.equal(vmax, vmax0)
        assert step == float(st["step"])
    assert clipped == {True, False}


def test_adam_step_amsgrad_off_leaves_vmax():
    hp = torch.tensor([10, 1, 1.0, 5e-4, 0.9, 0.999, 1e-8, 0, 5, 0] + [0] * 6, dtype=torch.float32)
    vm = torch.full((4,), -7.0)
    _, _, _, vmax, _ = R.adam_step(torch.ones(4), torch.ones(4), torch.zeros(4), torch.zeros(4), vm, 0, hp, 4.0)
    assert torch.equal(vmax, vm.double())


def bitpat(*ints):
    return torch.tensor(ints, dtype=torch.int64).to(torch.int32).view(torch.float32)


def test_tf32_rna_on_bit_patterns():
    """cvt.rna.tf32.f32: low 13 bits cleared, ties (low bits = 0x1000) away from zero for both signs, a carry out of
    the mantissa into the exponent, TF32-exact values unchanged."""
    src = bitpat(0x3F801000, 0xBF801000, 0x3F800FFF, 0xBF800FFF, 0x3F801001, 0x3FFFF000, 0xBFFFF000, 0x3F803000,
                 0x3F802000, 0x00000000, 0x80000000, 0x40490000, 0x7F7FE000)
    want = bitpat(0x3F802000, 0xBF802000, 0x3F800000, 0xBF800000, 0x3F802000, 0x40000000, 0xC0000000, 0x3F804000,
                  0x3F802000, 0x00000000, 0x80000000, 0x40490000, 0x7F7FE000)
    got = R.tf32_rna(src)
    assert torch.equal(got.view(torch.int32), want.view(torch.int32))
    assert float(R.tf32_rna(bitpat(0x3FFFF000))[0]) == 2.0
