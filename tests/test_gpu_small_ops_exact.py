"""GPU: the small kernels of csrc/small_ops.cu and csrc/dense_fused.cu -- avc_linear_fwd/bwd, avc_dense_stack_fwd/bwd,
avc_linear_batch_fwd/_dx/_dw, avc_time_mean_fwd/bwd, avc_pack_a4/avc_unpack_a4, avc_reparam_fwd/bwd, avc_vae_loss,
avc_sqnorm and avc_adam_step -- against the float64 restatement in tests/_small_ref.py, which reads the same fp32
operands.  The entry points are called with hand-built descriptors at the model's shapes and strides (the AdaIN rows
conds[:, i] are 3072 floats apart, A4 tensors can be channel views of a wider one) and at the kernels' tile edges.
Every strided or partial output sits inside a buffer filled with a sentinel that must survive outside it, and every
case launches its kernels twice on the same inputs: the two results must be bit-identical (none of them uses atomics).
The last test asserts that the cases reached every entry of FEATURES and prints the worst error per group.

Error measures, each relative to the scale of the terms rather than to the result, so cancellation cannot inflate it:
  * dot products (linear, stack, batched forward, dx, dw, db): |err| / (sum |a||b| over the element's reduction + |bias|
    + |res| + |dx_add| + the |dw0| / |db0| it accumulates onto).  In the backward the ReLU mask is the kernel's own
    y_act (or save plane), as the contract says;
  * dense stack, layer by layer: each save plane against the float64 layer applied to the kernel's own input plane;
    h_{l+1} = fp32(h_l + a_l) bit for bit; the gsave planes the same way going backwards (the running dh from the
    kernel's planes); end to end (out from x, dx from the kernel's masks) relative to max |reference|;
  * time mean: |err| / (sum |x| / T); its backward is fp32(dout * fp32(1/T)) bit for bit;
  * pack / unpack: bit for bit; with round_tf32 the bits of cvt.rna (ties away from zero, inputs include exact ties);
  * reparameterisation: z in units of |mu| + e^{ls/2}|eps|, dls of |dz eps| e^{ls/2}/2 + |dls_ext|, dmu of |dz| +
    |dmu_ext|; the planar mu / ls outputs are bit copies;
  * vae_loss: the sums over sum |dec - x| and sum (e^l + m^2 + 1 + |l|); ddec = +-fp32(lambda_rec / n_rec) or 0 and
    dmu = fp32(fp32(lambda_kl / n_lat) m) bit for bit; dls over g_kl (e^l + 1) / 2 (the kernel's expf(l) - 1 cancels
    near l = 0 as torch's autograd of the reference does; the measure does not count that as an error);
  * sqnorm: relative to the float64 sum of squares;
  * adam, one step at a time from the kernel's own state read back: m and v in units of 2^-24 of their terms'
    magnitude, vmax = max(vmax_in, v_out) bit for bit (untouched without amsgrad), step exact, and p as |p - p_ref|
    minus half an ulp of p_ref, over the magnitude of the update's terms lr / bc1 * (|m_in| + (1 - b1)(|g_i| + |m_in|))
    / denom (m itself may cancel).  A 20-step run is also compared with float64 torch.optim.Adam at double
    hyper-parameters: the kernel reads beta2 as fp32 0.999 = 0.99900001287, 1 - beta2 is 1.29e-5 smaller in relative
    terms.  Computed on the host (float64 torch.optim.Adam at the fp32-rounded against the double hyper-parameters, same
    schedule), that alone moves a first-step update by up to 3.3e-6 of itself and the 20-step result by 3.8e-7 of the
    summed update magnitudes; the fp32 storage of p (half an ulp per step) is subtracted before the division.

Worst measured on 1x NVIDIA H100 80GB HBM3 (132 SMs, 700 W power limit): linear 3.0e-7, stack (save / gsave / out /
dx) 3.2e-7, stack end to end 9.1e-7, batched 3.4e-7, time mean 1.8e-7, reparam 1.9e-7, vae_loss 6.6e-7 (the sum over
8 388 608 elements), sqnorm 1.3e-7, adam m 4.2 and v 7.7 units of 2^-24, adam p 3.4e-6, adam against torch 8.9e-7.
TOL is about 3x those.  The 83 cases take about 12 s on that GPU.  Deliberately broken kernels (arithmetic and index
mutations on a scratch copy, never committed) each fail cases: linear forward skipping the last k of the reduction, out
1.3e-2 .. 1.0 (13 cases); linear dw skipping the last batch row, dw 0.12 .. 0.97 (11); time mean 1/(T - 1), 2.4e-4 ..
inf (9); batched dx dropping the last layer of the sum, 2.0e-2 .. 0.56 (8); dense-stack backward masking g2 with y
instead of a, gsave inf (8); reparam expf(l) for expf(l / 2), z 2.1 .. 13 (5); vae dls without the 1/2, 0.97 .. 1.0
(6); sqnorm stage 2 skipping the last partial, 2.8e-6 .. 1.0 (8); adam m's lerp weights swapped, 1.3e8 units (8);
vmax not written, the vmax bit check and 9.6e-4 against torch (6); beta1 in the second bias correction, p 7.5 .. 9.0
and 8.0 against torch (6).
"""
import ctypes as C
import math
import time
import zlib
from dataclasses import dataclass

import pytest
import torch

import _small_ref as R
from test_gpu_tc2_exact import from_a4, to_a4

pytestmark = pytest.mark.gpu

SENT = -7777.0
GUARD = 64            # floats of sentinel after a dense output
ULP = 2.0 ** -24
TOL = {"linear": 1e-6, "stack": 1e-6, "stack e2e": 3e-6, "batch": 1e-6, "time mean": 5e-7, "reparam": 6e-7,
       "vae_loss": 2e-6, "sqnorm": 4e-7, "adam m": 12.0, "adam v": 24.0, "adam p": 1e-5, "adam torch": 3e-6}

FEATURES = (
    [("linear B", b) for b in (1, 7, 8, 9, 33, 257)] + [("linear K", k) for k in (1, 31, 32, 33, 128)]
    + [("linear N", n) for n in (1, 80, 128, 256, 300)]
    + ["linear: relu", "linear: res", "linear: null bias", "linear: null dx", "linear: dx_add", "linear: null db",
       "linear: out / dy rows 3072 apart", "linear: x rows wider than K", "linear: dw over B > 32",
       "linear: exact-zero activation masked"]
    + [("stack n_blocks", n) for n in (0, 1, 6)] + [("stack B", b) for b in (1, 3, 4, 5, 128, 257)]
    + ["stack: inference form", "stack: ragged last CTA"]
    + [("batch L", n) for n in (1, 12, 16)]
    + ["batch: affine layout", "batch: dense-dw planes", "batch: null-bias layers", "batch: dx with dx_add",
       "batch: dx without dx_add", "batch: row gap"]
    + [("time mean T", t) for t in (1, 16, 31, 33, 125, 1000, 4097)]
    + ["time mean: warps not a multiple of 8", "time mean: channel view"]
    + [("pack T", t) for t in (1, 37, 128)] + ["pack: channel view", "pack: round_tf32 0", "pack: round_tf32 1"]
    + [f"reparam fwd: ls4 {a} eps {b} mu {c} ls {d}" for a in (0, 1) for b in (0, 1) for c in (0, 1) for d in (0, 1)
       if a or not (b or d)]
    + [f"reparam bwd: dz {a} eps {b} dmu_ext {c} dls_ext {d}" for a in (0, 1) for b in (0, 1) for c in (0, 1) for d in (0, 1)]
    + [("vae n_rec", n) for n in (1, 40960, 2621440, 8388608)]
    + ["vae: n_lat < n_rec", "vae: n_lat > n_rec", "vae: exact ties", "vae: all partials used"]
    + [("sqnorm n", n) for n in (1, 255, 262144, 262145, 4892880, 9040512)] + ["sqnorm: all of scratch used"]
    + [("adam n", n) for n in (1, 300, 4892880)]
    + ["adam: amsgrad 0", "adam: amsgrad 1", "adam: wd 0", "adam: wd 1e-4", "adam: step preloaded 199999",
       "adam: clipped", "adam: not clipped", "adam: v below vmax", "adam: zero-gradient elements"])

RESULTS = {}      # case id -> (group, features, {measure: error})
_T0 = []


# ------------------------------------------------------------------ helpers
def lib():
    from adaptive_voice_conversion_b200 import _lib as L
    return L.load()


def stream():
    return torch.cuda.current_stream().cuda_stream


def ck(rc, what):
    from adaptive_voice_conversion_b200 import _lib as L
    assert rc == 0, f"{what}: rc={rc}: {L.last_error()}"


def ptr(t):
    return None if t is None else t.data_ptr()


def gen_of(cid):
    return torch.Generator().manual_seed(zlib.crc32(cid.encode()))


def randn(g, *shape):
    return torch.randn(shape, generator=g)


def boxed(shape, index):
    """(buffer full of SENT on the device, the view buffer[index])."""
    buf = torch.full(shape, SENT, device="cuda")
    return buf, buf[index]


def intact(buf, index):
    """everything of buf outside buf[index] still holds SENT."""
    m = torch.ones(buf.shape, dtype=torch.bool, device=buf.device)
    m[index] = False
    return bool((buf[m] == SENT).all())


def dense(n):
    """(buffer of n + GUARD floats, the first n): a dense output with a sentinel tail."""
    return boxed((n + GUARD,), slice(0, n))


def bits(t):
    return t.detach().contiguous().view(torch.int32)


def same_bits(a, b):
    return torch.equal(bits(a), bits(b.to(a.device)))


def err(k, ref, scale):
    """max |k - ref| / scale over elements; 0 where they agree exactly, inf where the scale is 0 but they differ."""
    ref = ref.to(k.device).double()
    e = (k.double() - ref).abs()
    s = scale.to(k.device).double() if torch.is_tensor(scale) else torch.full_like(e, float(scale))
    r = torch.where(e == 0, torch.zeros_like(e), e / s)
    return float(r.max()) if r.numel() else 0.0


def twice(launch):
    """launch() resets its outputs, runs the kernels and returns its output buffers: run it twice, demand the same
    bits, return the first run's buffers."""
    a = [t.clone() for t in launch()]
    b = launch()
    for i, (x, y) in enumerate(zip(a, b)):
        assert same_bits(x, y), f"output {i} differs between two launches on the same inputs"
    return a


def a4_view(B, Cc, T, view):
    """(wide A4 buffer full of SENT, index of the [B][C/4][T][4] region, address, bstride): view = channels
    [4, 4 + C) of a tensor 8 channels wider."""
    Cw, q0 = (Cc + 8, 1) if view else (Cc, 0)
    buf = torch.full((B, Cw // 4, T, 4), SENT, device="cuda")
    idx = (slice(None), slice(q0, q0 + Cc // 4))
    return buf, idx, buf.data_ptr() + q0 * T * 16, Cw * T


def record(cid, group, feats, errs):
    if not _T0:
        _T0.append(time.time())
    feats.discard("")
    RESULTS[cid] = (group, feats, errs)
    for k, e in errs.items():
        tol = TOL[k] if k in TOL else TOL[group]
        assert e < tol, f"{k}: error {e:.3e} (tolerance {tol:.0e})"


# ------------------------------------------------------------------ avc_linear_fwd / avc_linear_bwd
@dataclass(frozen=True)
class Lin:
    B: int
    K: int
    N: int
    relu: bool = False
    res: bool = False
    bias: bool = True
    dx: str = "plain"          # "plain" / "add" (dx_add) / "none" (null dx)
    db: bool = True
    strided: bool = False      # out / dy rows of a [B][12][N] tensor, x rows K + 5 wide
    zero_row: bool = False     # weight row 0 and bias 0 zero: y_act[:, 0] is exactly 0

    @property
    def id(self):
        return (f"linear-B{self.B}-K{self.K}-N{self.N}" + ("-relu" if self.relu else "") + ("-res" if self.res else "")
                + ("" if self.bias else "-nobias") + ("" if self.dx == "plain" else f"-dx{self.dx}")
                + ("" if self.db else "-nodb") + ("-strided" if self.strided else "") + ("-zero" if self.zero_row else ""))


LIN_CASES = [
    Lin(1, 128, 256, relu=True, strided=True, zero_row=True),
    Lin(7, 31, 80, res=True, dx="add"),
    Lin(8, 32, 128, relu=True, res=True, db=False),
    Lin(9, 33, 300, bias=False, dx="none"),
    Lin(33, 128, 256, strided=True, dx="add"),
    Lin(257, 128, 128, relu=True, res=True, zero_row=True),
    Lin(257, 1, 1, relu=True),
    Lin(33, 31, 300, relu=True, bias=False, db=False, zero_row=True),
    Lin(1, 33, 80, dx="none", db=False),
    Lin(9, 128, 256, relu=True, res=True, strided=True, dx="none"),
    Lin(7, 1, 128, bias=False, dx="add"),
    Lin(8, 32, 1, relu=True, res=True),
]


@pytest.mark.parametrize("case", LIN_CASES, ids=lambda c: c.id)
def test_linear(case):
    from adaptive_voice_conversion_b200 import _lib as L
    g = gen_of(case.id)
    B, K, N = case.B, case.K, case.N
    x, w = randn(g, B, K), randn(g, N, K) / math.sqrt(K)
    b = 0.3 * randn(g, N) if case.bias else None
    res = randn(g, B, N) if case.res else None
    dx_add = randn(g, B, K) if case.dx == "add" else None
    dw0, db0 = randn(g, N, K), randn(g, N)
    if case.zero_row:
        w[0] = 0.0
        if b is not None:
            b[0] = 0.0
    xw = torch.full((B, K + 5 if case.strided else K), SENT)
    xw[:, :K] = x
    xd = xw.cuda()[:, :K]
    rows = (B + 1, 12, N) if case.strided else (B + 1, N)
    ridx = (slice(0, B), 5) if case.strided else (slice(0, B),)
    dyb, dy = boxed(rows, ridx)
    dy.copy_(randn(g, B, N))
    outb, out = boxed(rows, ridx)
    yab, ya = boxed((B + 1, N), (slice(0, B),))
    dxb, dx = boxed((B + 1, K), (slice(0, B),))
    dwb, dw = boxed((N + 1, K), (slice(0, N),))
    dbb, db = boxed((N + 1,), (slice(0, N),))
    wd = w.cuda()
    bdev = b.cuda() if b is not None else None
    resd = res.cuda() if res is not None else None
    dxad = dx_add.cuda() if dx_add is not None else None

    d = L.LinearDesc()
    d.B, d.N, d.K, d.relu = B, N, K, int(case.relu)
    d.x, d.x_bstride, d.w, d.bias, d.res = xd.data_ptr(), xd.stride(0), wd.data_ptr(), ptr(bdev), ptr(resd)
    d.y_act, d.out, d.out_bstride = ya.data_ptr(), out.data_ptr(), out.stride(0)
    d.dy, d.dy_bstride = dy.data_ptr(), dy.stride(0)
    d.dx_add, d.dx = ptr(dxad), (dx.data_ptr() if case.dx != "none" else None)
    d.dw, d.db = dw.data_ptr(), (db.data_ptr() if case.db else None)

    def launch():
        for t in (outb, yab, dxb, dwb, dbb):
            t.fill_(SENT)
        dw.copy_(dw0)
        db.copy_(db0)
        ck(lib().avc_linear_fwd(C.byref(d), stream()), "linear_fwd")
        ck(lib().avc_linear_bwd(C.byref(d), stream()), "linear_bwd")
        return [outb, yab, dxb, dwb, dbb]

    outb, yab, dxb, dwb, dbb = twice(launch)
    for buf, idx, name in ((outb, ridx, "out"), (yab, (slice(0, B),), "y_act"), (dxb, (slice(0, B),), "dx"),
                           (dwb, (slice(0, N),), "dw"), (dbb, (slice(0, N),), "db")):
        assert intact(buf, idx), f"{name}: write outside the output"
    out_k, ya_k, dx_k, dw_k, db_k = outb[ridx], yab[:B], dxb[:B], dwb[:N], dbb[:N]
    ab = b.abs() if b is not None else None
    out_r, y_r = R.linear_fwd(x, w, b, relu_=case.relu, res=res)
    s_out, s_y = R.linear_fwd(x.abs(), w.abs(), ab, res=res.abs() if res is not None else None)
    errs = {"out": err(out_k, out_r, s_out), "y_act": err(ya_k, y_r, s_y)}
    yk = ya_k.cpu() if case.relu else None
    dx_r, dw_r, db_r = R.linear_bwd(x, w, dy.cpu(), y_act=yk, dx_add=dx_add, dw0=dw0, db0=db0)
    gm = dy.cpu().abs() * ((yk > 0) if yk is not None else 1.0)
    s_dx, s_dw, s_db = R.linear_bwd(x.abs(), w.abs(), gm, dx_add=dx_add.abs() if dx_add is not None else None,
                                    dw0=dw0.abs(), db0=db0.abs())
    if case.dx != "none":
        errs["dx"] = err(dx_k, dx_r, s_dx)
    else:
        assert bool((dxb == SENT).all())
    errs["dw"] = err(dw_k, dw_r, s_dw)
    if case.db:
        errs["db"] = err(db_k, db_r, s_db)
    else:
        assert same_bits(db_k, db0), "db is null: nothing may be written"
    feats = {("linear B", B), ("linear K", K), ("linear N", N)}
    feats |= {"linear: relu" if case.relu else "", "linear: res" if case.res else "", "" if case.bias else "linear: null bias",
              {"plain": "", "add": "linear: dx_add", "none": "linear: null dx"}[case.dx], "" if case.db else "linear: null db"}
    if case.strided:
        feats.add("linear: x rows wider than K")
        if out.stride(0) == 3072:
            feats.add("linear: out / dy rows 3072 apart")
    if B > 32:
        feats.add("linear: dw over B > 32")
    if case.zero_row and case.relu:
        assert bool((ya_k[:, 0] == 0).all())
        assert same_bits(dw_k[0], dw0[0]) and (not case.db or same_bits(db_k[0], db0[0])), "the ReLU mask let y_act = 0 through"
        feats.add("linear: exact-zero activation masked")
    record(case.id, "linear", feats, errs)


# ------------------------------------------------------------------ avc_dense_stack_fwd / _bwd
STACK_CASES = [(6, 1), (6, 3), (6, 4), (6, 5), (6, 128), (6, 257), (0, 5), (0, 1), (1, 257), (1, 4)]
DS_C = 128


def stack_params(g, nb):
    ps = []
    for _ in range(2 * nb + 1):
        ps += [randn(g, DS_C, DS_C) / math.sqrt(DS_C), 0.1 * randn(g, DS_C)]
    # table order [W1_l, b1_l]* [W2_l, b2_l]* Wo bo: the draw above is already in that order
    return ps


@pytest.mark.parametrize("nb,B", STACK_CASES, ids=[f"stack-n{n}-B{b}" for n, b in STACK_CASES])
def test_dense_stack(nb, B):
    from adaptive_voice_conversion_b200 import _lib as L
    cid = f"stack-n{nb}-B{B}"
    g = gen_of(cid)
    P = stack_params(g, nb)
    x, dout = randn(g, B, DS_C), randn(g, B, DS_C)
    Pd = [p.cuda() for p in P]
    tab = torch.tensor([p.data_ptr() for p in Pd], dtype=torch.int64).cuda()
    xd, doutd = x.cuda(), dout.cuda()
    plane = B * DS_C
    ridx = (slice(0, B),)
    outb, out = boxed((B + 4, DS_C), ridx)
    out2b, out2 = boxed((B + 4, DS_C), ridx)
    saveb, save = dense((3 * nb + 1) * plane)
    gsaveb, gsave = dense((2 * nb + 1) * plane)
    dxb, dx = boxed((B + 4, DS_C), ridx)
    d = L.DenseStackDesc()
    d.B, d.C, d.c_out, d.n_blocks = B, DS_C, DS_C, nb
    d.params, d.x, d.save, d.out = tab.data_ptr(), xd.data_ptr(), save.data_ptr(), out.data_ptr()
    d.dout, d.gsave, d.dx = doutd.data_ptr(), gsave.data_ptr(), dx.data_ptr()
    di = L.DenseStackDesc()
    di.B, di.C, di.c_out, di.n_blocks = B, DS_C, DS_C, nb
    di.params, di.x, di.save, di.out = tab.data_ptr(), xd.data_ptr(), None, out2.data_ptr()

    def launch():
        for t in (outb, out2b, saveb, gsaveb, dxb):
            t.fill_(SENT)
        ck(lib().avc_dense_stack_fwd(C.byref(d), stream()), "dense_stack_fwd")
        ck(lib().avc_dense_stack_bwd(C.byref(d), stream()), "dense_stack_bwd")
        ck(lib().avc_dense_stack_fwd(C.byref(di), stream()), "dense_stack_fwd (inference)")
        return [outb, out2b, saveb, gsaveb, dxb]

    outb, out2b, saveb, gsaveb, dxb = twice(launch)
    for buf, idx, name in ((outb, ridx, "out"), (out2b, ridx, "out (inference)"), (dxb, ridx, "dx"),
                           (saveb, slice(0, (3 * nb + 1) * plane), "save"), (gsaveb, slice(0, (2 * nb + 1) * plane), "gsave")):
        assert intact(buf, idx), f"{name}: write outside the output (rows >= B or past the last plane)"
    assert same_bits(out2b[:B], outb[:B]), "the inference form (save = null) differs from the training form"
    S = saveb[:(3 * nb + 1) * plane].view(3 * nb + 1, B, DS_C)
    Gs = gsaveb[:(2 * nb + 1) * plane].view(2 * nb + 1, B, DS_C)
    Pg = [p.double() for p in Pd]
    Pa = [p.abs() for p in Pg]
    h = lambda l: S[l]                   # noqa: E731
    y = lambda l: S[nb + 1 + l]          # noqa: E731
    a = lambda l: S[2 * nb + 1 + l]      # noqa: E731
    assert same_bits(S[0], xd), "h_0 is not x"
    e_save = 0.0
    for l in range(nb):
        W1, b1, W2, b2 = Pg[2 * l], Pg[2 * l + 1], Pg[2 * nb + 2 * l], Pg[2 * nb + 2 * l + 1]
        e_save = max(e_save, err(y(l), R.relu(h(l).double() @ W1.T + b1), h(l).double().abs() @ W1.abs().T + b1.abs()))
        e_save = max(e_save, err(a(l), R.relu(y(l).double() @ W2.T + b2), y(l).double().abs() @ W2.abs().T + b2.abs()))
        assert same_bits(h(l + 1), h(l) + a(l)), f"h_{l + 1} != fp32(h_{l} + a_{l})"
    hn = h(nb).double()
    errs = {"save": e_save, "out": err(out, hn @ Pg[4 * nb].T + Pg[4 * nb + 1], hn.abs() @ Pa[4 * nb].T + Pa[4 * nb + 1])}
    # backward, layer by layer from the kernel's gsave planes
    assert same_bits(Gs[2 * nb], doutd), "the last gsave plane is not dout"
    dh = doutd.double() @ Pg[4 * nb]
    sh = doutd.double().abs() @ Pa[4 * nb]
    e_g = 0.0
    for l in reversed(range(nb)):
        ma, my = a(l) > 0, y(l) > 0
        zero = torch.zeros_like(dh)
        e_g = max(e_g, err(Gs[nb + l], torch.where(ma, dh, zero), torch.where(ma, sh, zero)))
        g2 = Gs[nb + l].double()
        e_g = max(e_g, err(Gs[l], torch.where(my, g2 @ Pg[2 * nb + 2 * l], zero), torch.where(my, g2.abs() @ Pa[2 * nb + 2 * l], zero)))
        g1 = Gs[l].double()
        dh, sh = dh + g1 @ Pg[2 * l], sh + g1.abs() @ Pa[2 * l]
    errs["gsave"] = e_g
    errs["dx"] = err(dxb[:B], dh, sh)
    # end to end: out from x alone; dx from dout through the kernel's own masks
    out_e, _ = R.dense_stack_fwd(xd, Pd, nb)
    dx_e, _ = R.dense_stack_bwd(Pd, nb, S, doutd)
    errs["stack e2e"] = max(err(out, out_e, out_e.abs().max()), err(dxb[:B], dx_e, dx_e.abs().max()))
    feats = {("stack n_blocks", nb), ("stack B", B), "stack: inference form", "stack: ragged last CTA" if B % 4 else ""}
    record(cid, "stack", feats, errs)


# ------------------------------------------------------------------ avc_linear_batch_fwd / _dx / _dw
@dataclass(frozen=True)
class Batch:
    L: int
    B: int
    N: int
    K: int
    layout: str                       # "affine": shared x, row = L * N (+ pad); "planes": one [B][K] / [B][N] plane per layer
    nullbias: tuple = ()
    dx_add: bool = False
    pad: int = 0

    @property
    def id(self):
        return (f"batch-L{self.L}-B{self.B}-N{self.N}-K{self.K}-{self.layout}" + (f"-pad{self.pad}" if self.pad else "")
                + ("-nb" + "_".join(map(str, self.nullbias)) if self.nullbias else "") + ("-dxadd" if self.dx_add else ""))


BATCH_CASES = [
    Batch(12, 3, 256, 128, "affine"),
    Batch(12, 256, 256, 128, "affine", nullbias=(3, 7), dx_add=True),
    Batch(12, 9, 256, 128, "affine", pad=8),
    Batch(13, 5, 128, 128, "planes"),
    Batch(13, 257, 128, 128, "planes", nullbias=(12,), dx_add=True),
    Batch(1, 9, 80, 33, "planes", dx_add=True),
    Batch(16, 33, 300, 31, "affine", nullbias=(0, 15), pad=3),
    Batch(16, 1, 1, 1, "planes"),
]


@pytest.mark.parametrize("case", BATCH_CASES, ids=lambda c: c.id)
def test_linear_batch(case):
    from adaptive_voice_conversion_b200 import _lib as L
    g = gen_of(case.id)
    Ln, B, N, K = case.L, case.B, case.N, case.K
    W = [randn(g, N, K) / math.sqrt(K) for _ in range(Ln)]
    bs = [None if l in case.nullbias else 0.3 * randn(g, N) for l in range(Ln)]
    dW0 = [randn(g, N, K) for _ in range(Ln)]
    db0 = [None if l in case.nullbias else randn(g, N) for l in range(Ln)]
    if case.layout == "affine":
        x = randn(g, B * K)
        x_off, x_bs = [0] * Ln, K
        y_bs = Ln * N + case.pad
        y_off = [l * N for l in range(Ln)]
        ny = B * y_bs
    else:                                    # L + 1 planes, layer l at plane perm[l]: one plane no layer uses
        perm = torch.randperm(Ln + 1, generator=g)[:Ln].tolist()
        x = randn(g, (Ln + 1) * B * K)
        x_off, x_bs = [p * B * K for p in perm], K
        y_off, y_bs = [p * B * N for p in reversed(perm)], N
        ny = (Ln + 1) * B * N
    used = torch.zeros(ny, dtype=torch.bool)
    for l in range(Ln):
        R.rows_at(used, y_off[l], y_bs, B, N).fill_(True)
    yin = torch.where(used, randn(g, ny), torch.full((ny,), SENT))
    dx_add = randn(g, B, K) if case.dx_add else None
    Wd = [w.cuda() for w in W]
    bd = [b.cuda() if b is not None else None for b in bs]
    gW = [torch.empty(N, K, device="cuda") for _ in range(Ln)]
    gb = [torch.empty(N, device="cuda") if b is not None else None for b in db0]
    tab = torch.tensor([ptr(t) or 0 for l in range(Ln) for t in (Wd[l], bd[l])], dtype=torch.int64).cuda()
    gtab = torch.tensor([ptr(t) or 0 for l in range(Ln) for t in (gW[l], gb[l])], dtype=torch.int64).cuda()
    xd, yd = x.cuda(), yin.cuda()
    dxad = dx_add.cuda() if dx_add is not None else None
    outb, out = dense(ny)
    partb, part = dense(Ln * B * K)
    dxb, dx = dense(B * K)
    d = L.LinearBatchDesc()
    d.L, d.B, d.N, d.K = Ln, B, N, K
    d.params, d.grads, d.x, d.x_bstride = tab.data_ptr(), gtab.data_ptr(), xd.data_ptr(), x_bs
    d.y, d.out, d.y_bstride = yd.data_ptr(), out.data_ptr(), y_bs
    for l in range(Ln):
        d.x_off[l], d.y_off[l] = x_off[l], y_off[l]
    d.part, d.dx_add, d.dx = part.data_ptr(), ptr(dxad), dx.data_ptr()

    def launch():
        for t in (outb, partb, dxb):
            t.fill_(SENT)
        for l in range(Ln):
            gW[l].copy_(dW0[l])
            if gb[l] is not None:
                gb[l].copy_(db0[l])
        ck(lib().avc_linear_batch_fwd(C.byref(d), stream()), "linear_batch_fwd")
        ck(lib().avc_linear_batch_dx(C.byref(d), stream()), "linear_batch_dx")
        ck(lib().avc_linear_batch_dw(C.byref(d), stream()), "linear_batch_dw")
        return [outb, partb, dxb] + gW + [t for t in gb if t is not None]

    res = twice(launch)
    outb, dxb = res[0], res[2]
    gWk, gbk = res[3:3 + Ln], res[3 + Ln:]
    assert intact(dxb, slice(0, B * K)) and intact(res[1], slice(0, Ln * B * K))
    # every float of out that no layer owns (row gaps, the unused plane, the guard) keeps its SENT
    assert bool((outb[:ny][~used.cuda()] == SENT).all()) and bool((outb[ny:] == SENT).all()), "write outside the layer rows"
    out_r = R.linear_batch_fwd(x, x_off, x_bs, list(sum(zip(W, bs), ())), B, N, K)
    out_s = R.linear_batch_fwd(x.abs(), x_off, x_bs, list(sum(zip([w.abs() for w in W], [b.abs() if b is not None else None for b in bs]), ())), B, N, K)
    e_f = max(err(R.rows_at(outb, y_off[l], y_bs, B, N), out_r[l], out_s[l]) for l in range(Ln))
    dx_r = R.linear_batch_dx(yin, y_off, y_bs, list(sum(zip(W, bs), ())), B, N, K, dx_add)
    dx_s = R.linear_batch_dx(yin.abs(), y_off, y_bs, list(sum(zip([w.abs() for w in W], bs), ())), B, N, K,
                             dx_add.abs() if dx_add is not None else None)
    gr = R.linear_batch_dw(x, x_off, x_bs, yin, y_off, y_bs, list(sum(zip(dW0, db0), ())), B, N, K)
    gs = R.linear_batch_dw(x.abs(), x_off, x_bs, yin.abs(), y_off, y_bs,
                           list(sum(zip([t.abs() for t in dW0], [t.abs() if t is not None else None for t in db0]), ())), B, N, K)
    e_dw = max(err(gWk[l], gr[2 * l], gs[2 * l]) for l in range(Ln))
    e_db, j = 0.0, 0
    for l in range(Ln):
        if db0[l] is not None:
            e_db = max(e_db, err(gbk[j], gr[2 * l + 1], gs[2 * l + 1]))
            j += 1
    errs = {"out": e_f, "dx": err(dxb[:B * K].view(B, K), dx_r, dx_s), "dw": e_dw, "db": e_db}
    feats = {("batch L", Ln), "batch: affine layout" if case.layout == "affine" else "batch: dense-dw planes",
             "batch: null-bias layers" if case.nullbias else "", "batch: dx with dx_add" if case.dx_add else "batch: dx without dx_add",
             "batch: row gap" if case.pad else ""}
    record(case.id, "batch", feats, errs)


# ------------------------------------------------------------------ avc_time_mean_fwd / _bwd
TM_CASES = [(5, 128, 16, False), (3, 128, 1, True), (2, 128, 31, False), (4, 128, 33, True), (7, 128, 125, False),
            (2, 128, 1000, True), (1, 12, 4097, False), (3, 12, 37, True), (256, 128, 16, True)]


@pytest.mark.parametrize("B,Cc,T,view", TM_CASES, ids=[f"tmean-B{b}-C{c}-T{t}" + ("-view" if v else "") for b, c, t, v in TM_CASES])
def test_time_mean(B, Cc, T, view):
    cid = f"tmean-B{B}-C{Cc}-T{T}" + ("-view" if view else "")
    g = gen_of(cid)
    x = randn(g, B, Cc, T) + 2.0 * randn(g, 1, Cc, 1)
    dout = randn(g, B, Cc)
    src, sidx, sptr, sbs = a4_view(B, Cc, T, view)
    src[sidx] = to_a4(x)
    outb, out = dense(B * Cc)
    dab, didx, dptr, dbs = a4_view(B, Cc, T, view)
    doutd = dout.cuda()

    def launch():
        outb.fill_(SENT)
        dab.fill_(SENT)
        ck(lib().avc_time_mean_fwd(sptr, sbs, out.data_ptr(), B, Cc, T, stream()), "time_mean_fwd")
        ck(lib().avc_time_mean_bwd(doutd.data_ptr(), dptr, dbs, B, Cc, T, stream()), "time_mean_bwd")
        return [outb, dab]

    outb, dab = twice(launch)
    assert intact(outb, slice(0, B * Cc)) and intact(dab, didx), "write outside the output"
    xd = x.cuda()
    errs = {"fwd": err(outb[:B * Cc].view(B, Cc), R.time_mean_fwd(xd), xd.abs().sum(2) / T)}
    inv = torch.tensor(1.0, device="cuda") / torch.tensor(float(T), device="cuda")
    assert same_bits(from_a4(dab[didx]), (doutd * inv)[:, :, None].expand(B, Cc, T)), "backward is not fp32(dout * fp32(1/T))"
    feats = {("time mean T", T), "time mean: channel view" if view else "",
             "time mean: warps not a multiple of 8" if (B * Cc // 4) % 8 else ""}
    record(cid, "time mean", feats, errs)


# ------------------------------------------------------------------ avc_pack_a4 / avc_unpack_a4
PACK_CASES = [(3, 80, 1, False, 0), (2, 80, 37, True, 1), (5, 128, 128, True, 0), (4, 80, 128, False, 1),
              (1, 12, 37, True, 1), (2, 128, 1, True, 1)]


@pytest.mark.parametrize("B,Cc,T,view,rnd", PACK_CASES, ids=[f"pack-B{b}-C{c}-T{t}" + ("-view" if v else "") + f"-r{r}"
                                                               for b, c, t, v, r in PACK_CASES])
def test_pack_unpack(B, Cc, T, view, rnd):
    from _small_ref import tf32_rna
    cid = f"pack-B{B}-C{Cc}-T{T}" + ("-view" if view else "") + f"-r{rnd}"
    g = gen_of(cid)
    x = randn(g, B, Cc, T)
    xb = x.view(torch.int32)
    tie = torch.rand((B, Cc, T), generator=g) < 0.25           # exact ties: low 13 bits = 0x1000
    xb[tie] = (xb[tie] & -0x2000) | 0x1000
    xd = x.cuda()
    dstb, didx, dptr, dbs = a4_view(B, Cc, T, view)
    pb, pl = dense(B * Cc * T)

    def launch():
        dstb.fill_(SENT)
        pb.fill_(SENT)
        ck(lib().avc_pack_a4(xd.data_ptr(), dptr, dbs, B, Cc, T, rnd, stream()), "pack_a4")
        ck(lib().avc_unpack_a4(dptr, dbs, pl.data_ptr(), B, Cc, T, stream()), "unpack_a4")
        return [dstb, pb]

    dstb, pb = twice(launch)
    assert intact(dstb, didx) and intact(pb, slice(0, B * Cc * T)), "write outside the output"
    want = tf32_rna(x) if rnd else x
    assert same_bits(dstb[didx], to_a4(want)), "packed bits"
    if rnd:
        assert bool(((bits(dstb[didx]) & 0x1FFF) == 0).all())
        assert not torch.equal(tf32_rna(x), x)
    assert same_bits(pb[:B * Cc * T].view(B, Cc, T), want), "unpacked bits"
    feats = {("pack T", T), "pack: channel view" if view else "", f"pack: round_tf32 {rnd}"}
    record(cid, "pack", feats, {})


# ------------------------------------------------------------------ avc_reparam_fwd / _bwd
FWD_COMBOS = [(a, b, c, d) for a in (0, 1) for b in (0, 1) for c in (0, 1) for d in (0, 1) if a or not (b or d)]
REPARAM_CASES = [(i, 3, 8, 37) for i in range(16)] + [(15, 256, 128, 16)]


@pytest.mark.parametrize("i,B,Cc,T", REPARAM_CASES, ids=[f"reparam-{i}-B{b}-C{c}-T{t}" for i, b, c, t in REPARAM_CASES])
def test_reparam(i, B, Cc, T):
    cid = f"reparam-{i}-B{B}-C{Cc}-T{T}"
    g = gen_of(cid)
    f_ls4, f_eps, f_mu, f_ls = FWD_COMBOS[i % len(FWD_COMBOS)] if B < 256 else (1, 1, 1, 1)
    b_dz, b_eps, b_dmu, b_dls = i & 1, (i >> 1) & 1, (i >> 2) & 1, (i >> 3) & 1
    mu, ls = randn(g, B, Cc, T), 1.5 * randn(g, B, Cc, T) - 1.0
    eps, dz = randn(g, B, Cc, T), randn(g, B, Cc, T)
    dmu_ext, dls_ext = randn(g, B, Cc, T), randn(g, B, Cc, T)
    mu4, ls4, dz4 = to_a4(mu), to_a4(ls), to_a4(dz)
    epsd, dmud, dlsd = eps.cuda(), dmu_ext.cuda(), dls_ext.cuda()
    n = B * Cc * T
    zb, z = dense(n)
    mb, mo = dense(n)
    lb, lo = dense(n)
    dmb, dm = dense(n)
    dlb, dl = dense(n)

    def launch():
        for t in (zb, mb, lb, dmb, dlb):
            t.fill_(SENT)
        ck(lib().avc_reparam_fwd(mu4.data_ptr(), ptr(ls4) if f_ls4 else None, ptr(epsd) if f_eps else None,
                                 ptr(mo) if f_mu else None, ptr(lo) if f_ls else None, z.data_ptr(), B, Cc, T, stream()), "reparam_fwd")
        ck(lib().avc_reparam_bwd(ptr(dz4) if b_dz else None, ptr(ls4) if b_eps else None, ptr(epsd) if b_eps else None,
                                 ptr(dmud) if b_dmu else None, ptr(dlsd) if b_dls else None, dm.data_ptr(), dl.data_ptr(),
                                 B, Cc, T, stream()), "reparam_bwd")
        return [zb, mb, lb, dmb, dlb]

    zb, mb, lb, dmb, dlb = twice(launch)
    for buf in (zb, dmb, dlb):
        assert intact(buf, slice(0, n)), "write past the output"
    P = lambda t: from_a4(t[:n].view(B, Cc // 4, T, 4))   # noqa: E731
    md, lsd = mu.cuda(), ls.cuda()
    errs = {}
    if f_eps:
        errs["z"] = err(P(zb), R.reparam_fwd(md, lsd, epsd), md.abs() + torch.exp(lsd.double() / 2) * epsd.abs())
    else:
        assert same_bits(P(zb), md), "z = mu without eps"
    assert same_bits(mb[:n], md.reshape(-1)) if f_mu else bool((mb == SENT).all())
    assert same_bits(lb[:n], lsd.reshape(-1)) if f_ls else bool((lb == SENT).all())
    dmu_r, dls_r = R.reparam_bwd(dz.cuda() if b_dz else None, lsd, epsd if b_eps else None,
                                 dmud if b_dmu else None, dlsd if b_dls else None)
    zero = torch.zeros_like(md)
    s_dmu = (dz.cuda().abs() if b_dz else zero) + (dmud.abs() if b_dmu else zero)
    s_dls = ((dz.cuda() * epsd).abs() * 0.5 * torch.exp(lsd.double() / 2) if b_dz and b_eps else zero) + (dlsd.abs() if b_dls else zero)
    errs["dmu"] = err(P(dmb), dmu_r, s_dmu)
    errs["dls"] = err(P(dlb), dls_r, s_dls)
    feats = {f"reparam fwd: ls4 {f_ls4} eps {f_eps} mu {f_mu} ls {f_ls}", f"reparam bwd: dz {b_dz} eps {b_eps} dmu_ext {b_dmu} dls_ext {b_dls}"}
    record(cid, "reparam", feats, errs)


# ------------------------------------------------------------------ avc_vae_loss
VAE_CASES = [(1, 7), (1, 300), (40960, 8192), (1000, 5000), (2621440, 524288), (8388608, 262144)]


@pytest.mark.parametrize("n_rec,n_lat", VAE_CASES, ids=[f"vae-{a}-{b}" for a, b in VAE_CASES])
def test_vae_loss(n_rec, n_lat):
    from adaptive_voice_conversion_b200 import _lib as L
    cid = f"vae-{n_rec}-{n_lat}"
    g = torch.Generator(device="cuda").manual_seed(zlib.crc32(cid.encode()))
    dec = torch.randn(n_rec, generator=g, device="cuda")
    x = torch.randn(n_rec, generator=g, device="cuda")
    tie = torch.rand(n_rec, generator=g, device="cuda") < 0.01
    tie[0] = n_rec > 1
    x[tie] = dec[tie]
    mu = torch.randn(n_lat, generator=g, device="cuda")
    ls = 2.0 * torch.randn(n_lat, generator=g, device="cuda") - 1.0
    ls[: n_lat // 4] *= 1e-4                       # near l = 0, where e^l - 1 cancels
    ls[0] = 0.0
    hp = torch.zeros(16)
    hp[0], hp[1] = 10.0, 0.7
    hpd = hp.cuda()
    partb, part = dense(L.VAE_PARTIALS)
    sb, sums = dense(2)
    ddb, ddec = dense(n_rec)
    dmb, dmu = dense(n_lat)
    dlb, dls = dense(n_lat)

    def launch():
        for t in (partb, sb, ddb, dmb, dlb):
            t.fill_(SENT)
        ck(lib().avc_vae_loss(dec.data_ptr(), x.data_ptr(), n_rec, mu.data_ptr(), ls.data_ptr(), n_lat, hpd.data_ptr(),
                              sums.data_ptr(), part.data_ptr(), ddec.data_ptr(), dmu.data_ptr(), dls.data_ptr(), stream()), "vae_loss")
        return [partb, sb, ddb, dmb, dlb]

    partb, sb, ddb, dmb, dlb = twice(launch)
    for buf, n in ((partb, L.VAE_PARTIALS), (sb, 2), (ddb, n_rec), (dmb, n_lat), (dlb, n_lat)):
        assert intact(buf, slice(0, n)), "write past the output"
    s_rec, s_kl, ddec_r, dmu_r, dls_r = R.vae_loss(dec, x, mu, ls, hp)
    l64, m64 = ls.double(), mu.double()
    e_l = torch.exp(l64)
    errs = {"sum rec": abs(float(sb[0]) - float(s_rec)) / float((dec.double() - x.double()).abs().sum()),
            "sum kl": abs(float(sb[1]) - float(s_kl)) / float((e_l + m64 * m64 + 1 + l64.abs()).sum())}
    f32 = lambda v: torch.tensor(v, dtype=torch.float32, device="cuda")   # noqa: E731
    grec = f32(10.0) / f32(float(n_rec))
    gkl = f32(0.7) / f32(float(n_lat))
    df = dec - x
    want = torch.where(df > 0, grec, torch.where(df < 0, -grec, torch.zeros_like(df)))
    assert same_bits(ddb[:n_rec], want), "ddec is not +-fp32(lambda_rec / n_rec) or 0"
    assert same_bits(dmb[:n_lat], gkl * mu), "dmu is not fp32(fp32(lambda_kl / n_lat) * mu)"
    errs["dls"] = err(dlb[:n_lat], dls_r, float(gkl) * 0.5 * (e_l + 1))
    nb = min(max(-(-n_rec // 256), 1), 132 * 8)
    feats = {("vae n_rec", n_rec), "vae: n_lat < n_rec" if n_lat < n_rec else "vae: n_lat > n_rec",
             "vae: exact ties" if bool(tie.any()) else "", "vae: all partials used" if 2 * nb == L.VAE_PARTIALS else ""}
    record(cid, "vae_loss", feats, errs)


# ------------------------------------------------------------------ avc_sqnorm
SQ_CASES = [1, 255, 262144, 262145, 4892880, 9040512]


@pytest.mark.parametrize("n", SQ_CASES, ids=[f"sqnorm-{n}" for n in SQ_CASES])
def test_sqnorm(n):
    cid = f"sqnorm-{n}"
    gg = torch.Generator(device="cuda").manual_seed(zlib.crc32(cid.encode()))
    gv = 1e-3 * torch.randn(n, generator=gg, device="cuda")
    gv[n // 3] = 10.0                                    # one dominant element
    scb, scratch = dense(1024)
    ob, out = dense(1)

    def launch():
        scb.fill_(SENT)
        ob.fill_(SENT)
        ck(lib().avc_sqnorm(gv.data_ptr(), n, scratch.data_ptr(), out.data_ptr(), stream()), "sqnorm")
        return [scb, ob]

    scb, ob = twice(launch)
    assert intact(scb, slice(0, 1024)) and intact(ob, slice(0, 1)), "write past scratch / out"
    ref = R.sqnorm(gv)
    nb = min(max(-(-n // 256), 1), 1024)
    feats = {("sqnorm n", n), "sqnorm: all of scratch used" if nb == 1024 else ""}
    record(cid, "sqnorm", feats, {"sqnorm": abs(float(ob[0]) - ref) / ref})


# ------------------------------------------------------------------ avc_adam_step
MAX_NORM = 5.0


def hp_vec(wd, ams, lr=5e-4, b1=0.9, b2=0.999, eps=1e-8, gscale=0.5):
    hp = torch.zeros(16)
    hp[0], hp[1] = 10.0, 1.0
    hp[R.HP_GSCALE], hp[R.HP_LR], hp[R.HP_B1], hp[R.HP_B2] = gscale, lr, b1, b2
    hp[R.HP_EPS], hp[R.HP_WD], hp[R.HP_MAXNORM], hp[R.HP_AMSGRAD] = eps, wd, MAX_NORM, float(ams)
    return hp


def grad_schedule(n, steps, seed, device="cuda"):
    """Per-step gradients: a fixed per-element magnitude spanning 1e-8 .. 1e2, a fresh direction each step, 5 % of the
    elements always 0; every third step scaled to 4x max_norm (clipped), the others to 0.2 x 0.8^s of it (not clipped,
    and shrinking, so v falls below vmax)."""
    g = torch.Generator(device=device).manual_seed(seed)
    mag = 10.0 ** (torch.rand(n, generator=g, device=device) * 10 - 8)
    live = torch.rand(n, generator=g, device=device) >= 0.05
    live[0] = n == 1                      # a zero-gradient element, unless it is the only one
    for s in range(steps):
        d = torch.randn(n, generator=g, device=device) * mag * live
        c = 4.0 if s % 3 == 0 else 0.2 * 0.8 ** s
        yield (d * (c * MAX_NORM / float(d.norm()))).float(), c > 1


ADAM_CASES = [(1, 1, 1e-4, 0), (300, 0, 0.0, 0), (300, 1, 0.0, 199999), (300, 1, 1e-4, 0), (4892880, 1, 1e-4, 0),
              (4892880, 0, 1e-4, 199999)]


def half_ulp(r):
    f = r.float()
    return torch.ldexp(torch.ones_like(r), torch.frexp(f)[1].to(torch.int64) - 25)


@pytest.mark.parametrize("n,ams,wd,step0", ADAM_CASES, ids=[f"adam-{n}-a{a}-wd{w:g}-s{s}" for n, a, w, s in ADAM_CASES])
def test_adam_step(n, ams, wd, step0):
    cid = f"adam-{n}-a{ams}-wd{wd:g}-s{step0}"
    gg = torch.Generator(device="cuda").manual_seed(zlib.crc32(cid.encode()))
    hp = hp_vec(wd, ams)
    hpd = hp.cuda()
    p = 0.1 * torch.randn(n, generator=gg, device="cuda")
    m = torch.zeros(n, device="cuda")
    v = torch.zeros(n, device="cuda")
    if step0:
        m = 1e-3 * torch.randn(n, generator=gg, device="cuda")
        v = 1e-6 * torch.randn(n, generator=gg, device="cuda") ** 2
    vmb, vmax = dense(n)
    if ams:
        vmax.copy_(1.5 * v)
    step = torch.full((1,), float(step0), device="cuda")
    sq = torch.zeros(1, device="cuda")
    scratch = torch.zeros(1024, device="cuda")
    b1, b2, lr = float(hp[R.HP_B1]), float(hp[R.HP_B2]), float(hp[R.HP_LR])
    worst = {"adam m": 0.0, "adam v": 0.0, "adam p": 0.0}
    feats = {("adam n", n), f"adam: amsgrad {ams}", "adam: wd 0" if wd == 0 else "adam: wd 1e-4",
             "adam: step preloaded 199999" if step0 == 199999 else ""}
    for gsum, clipped in ((2 * gs, cl) for gs, cl in grad_schedule(n, 30, zlib.crc32(cid.encode()) + 1)):
        st0 = [t.clone() for t in (p, m, v, vmb, step)]

        def launch():
            for t, s in zip((p, m, v, vmb, step), st0):
                t.copy_(s)
            ck(lib().avc_sqnorm(gsum.data_ptr(), n, scratch.data_ptr(), sq.data_ptr(), stream()), "sqnorm")
            ck(lib().avc_adam_step(p.data_ptr(), gsum.data_ptr(), m.data_ptr(), v.data_ptr(), vmax.data_ptr(), n, hpd.data_ptr(),
                                   sq.data_ptr(), step.data_ptr(), stream()), "adam_step")
            return [p, m, v, vmb, step, sq]

        twice(launch)
        p0, m0, v0, vm0, s0 = st0
        sqv = float(sq)
        pr, mr, vr, vmr, tr = R.adam_step(p0, gsum, m0, v0, vm0[:n], float(s0), hp, sqv)
        assert float(step) == tr, "step"
        coef = R.clip_coef(hp, sqv)
        gmag = gsum.double().abs() * coef + wd * p0.double().abs()
        mmag = m0.double().abs() + (1 - b1) * (gmag + m0.double().abs())
        vmag = b2 * v0.double() + (1 - b2) * gmag * gmag
        worst["adam m"] = max(worst["adam m"], err(m, mr, ULP * mmag))
        worst["adam v"] = max(worst["adam v"], err(v, vr, ULP * vmag))
        if ams:
            assert same_bits(vmax, torch.maximum(vm0[:n], v)), "vmax != max(vmax_in, v_out)"
            if bool((v < vm0[:n]).any()):
                feats.add("adam: v below vmax")
            second = torch.maximum(vm0[:n].double(), vr)
        else:
            assert bool((vmb == SENT).all()), "vmax written without amsgrad"
            second = vr
        assert intact(vmb, slice(0, n))
        t = tr
        denom = second.sqrt() / math.sqrt(1 - b2 ** t) + float(hp[R.HP_EPS])
        umag = lr / (1 - b1 ** t) * mmag / denom
        worst["adam p"] = max(worst["adam p"], err(((p.double() - pr).abs() - half_ulp(pr)).clamp_min(0), torch.zeros_like(pr), umag))
        feats.add("adam: clipped" if clipped else "adam: not clipped")
    if n > 1:
        feats.add("adam: zero-gradient elements")
    record(cid, "adam", feats, worst)


def test_adam_matches_torch_adam():
    """20 steps of avc_sqnorm + avc_adam_step (world-size-2 form: summed gradient, grad_scale 0.5) against float64
    clip_grad_norm_ + torch.optim.Adam(amsgrad, weight_decay) at double hyper-parameters; error per element, less the
    fp32 storage rounding of p (half an ulp per step), over the sum of the magnitudes of torch's 20 updates."""
    n, steps = 4096, 20
    hp = hp_vec(1e-4, 1)
    hpd = hp.cuda()
    p0 = 0.1 * torch.randn(n, generator=torch.Generator().manual_seed(11))
    p, m, v, vm = p0.cuda(), torch.zeros(n, device="cuda"), torch.zeros(n, device="cuda"), torch.zeros(n, device="cuda")
    step, sq, scratch = torch.zeros(1, device="cuda"), torch.zeros(1, device="cuda"), torch.zeros(1024, device="cuda")
    pt = p0.double().clone().requires_grad_(True)
    opt = torch.optim.Adam([pt], lr=5e-4, betas=(0.9, 0.999), eps=1e-8, weight_decay=1e-4, amsgrad=True)
    moved = torch.zeros(n, dtype=torch.float64)
    for gs, _ in grad_schedule(n, steps, 12, device="cpu"):
        before = pt.detach().clone()
        pt.grad = gs.double()
        torch.nn.utils.clip_grad_norm_([pt], max_norm=MAX_NORM)
        opt.step()
        moved += (pt.detach() - before).abs()
        g2 = (2 * gs).cuda()
        ck(lib().avc_sqnorm(g2.data_ptr(), n, scratch.data_ptr(), sq.data_ptr(), stream()), "sqnorm")
        ck(lib().avc_adam_step(p.data_ptr(), g2.data_ptr(), m.data_ptr(), v.data_ptr(), vm.data_ptr(), n, hpd.data_ptr(),
                               sq.data_ptr(), step.data_ptr(), stream()), "adam_step")
    assert float(step) == steps
    # p is stored in fp32 after every step: up to half an ulp per step is storage, not arithmetic
    e = err((p.cpu().double() - pt.detach()).abs().sub(steps * half_ulp(pt.detach())).clamp_min(0), torch.zeros(n), moved)
    record("adam-vs-torch", "adam torch", {""}, {"adam torch": e})


# ------------------------------------------------------------------ argument rejection
def test_invalid_arguments_are_rejected_before_any_launch():
    """Each call returns its error code and message, and nothing is launched.  Pointers are placeholders that a
    rejected call never reads."""
    from adaptive_voice_conversion_b200 import _lib as L
    lb = lib()
    f = 1 << 20
    n0 = L.launch_count()
    d = L.LinearDesc()
    d.B, d.N, d.K, d.relu, d.x, d.w, d.dy, d.dw, d.out = 2, 8, 8, 1, f, f, f, f, f
    calls = [(lambda: lb.avc_linear_bwd(C.byref(d), None), L.ERR_INVALID, "relu needs y_act")]
    for Ln in (0, 17):
        bd = L.LinearBatchDesc()
        bd.L, bd.B, bd.N, bd.K, bd.params, bd.grads, bd.x, bd.y, bd.out, bd.part, bd.dx = Ln, 2, 8, 8, f, f, f, f, f, f, f
        calls += [(lambda bd=bd, fn=fn: getattr(lb, fn)(C.byref(bd), None), L.ERR_INVALID, "bad argument")
                  for fn in ("avc_linear_batch_fwd", "avc_linear_batch_dx", "avc_linear_batch_dw")]
    sd = L.DenseStackDesc()
    sd.B, sd.C, sd.c_out, sd.n_blocks, sd.params, sd.x, sd.out = 2, 64, 64, 1, f, f, f
    sd.save, sd.dout, sd.gsave, sd.dx = f, f, f, f
    calls += [(lambda: lb.avc_dense_stack_fwd(C.byref(sd), None), L.ERR_UNSUPPORTED, "C = c_out = 128"),
              (lambda: lb.avc_dense_stack_bwd(C.byref(sd), None), L.ERR_UNSUPPORTED, "C = c_out = 128")]
    calls += [
        (lambda: lb.avc_reparam_fwd(f, None, f, None, None, f, 2, 8, 4, None), L.ERR_INVALID, "eps needs log_sigma"),
        (lambda: lb.avc_reparam_bwd(f, None, f, None, None, f, f, 2, 8, 4, None), L.ERR_INVALID, "eps needs log_sigma"),
        (lambda: lb.avc_reparam_fwd(f, f, None, None, None, f, 2, 6, 4, None), L.ERR_INVALID, "bad argument"),
        (lambda: lb.avc_reparam_bwd(f, f, None, None, None, f, f, 2, 6, 4, None), L.ERR_INVALID, "bad argument"),
        (lambda: lb.avc_pack_a4(f, f, 48, 1, 6, 8, 0, None), L.ERR_INVALID, "C % 4"),
        (lambda: lb.avc_unpack_a4(f, 48, f, 1, 6, 8, None), L.ERR_INVALID, "C % 4"),
        (lambda: lb.avc_time_mean_fwd(f, 48, f, 1, 6, 8, None), L.ERR_INVALID, "bad argument"),
        (lambda: lb.avc_time_mean_bwd(f, f, 48, 1, 6, 8, None), L.ERR_INVALID, "bad argument"),
        (lambda: lb.avc_vae_loss(f, f, 10, f, f, 10, f, f, None, f, f, f, None), L.ERR_INVALID, "bad argument"),
        (lambda: lb.avc_vae_loss(f, f, 0, f, f, 10, f, f, f, f, f, f, None), L.ERR_INVALID, "bad argument"),
        (lambda: lb.avc_vae_loss(f, f, 10, f, f, 0, f, f, f, f, f, f, None), L.ERR_INVALID, "bad argument"),
        (lambda: lb.avc_sqnorm(f, 10, None, f, None), L.ERR_INVALID, "bad argument"),
        (lambda: lb.avc_sqnorm(f, 0, f, f, None), L.ERR_INVALID, "bad argument"),
        (lambda: lb.avc_adam_step(f, f, f, f, f, 10, f, None, f, None), L.ERR_INVALID, "bad argument"),
        (lambda: lb.avc_adam_step(f, f, f, f, f, 0, f, f, f, None), L.ERR_INVALID, "bad argument"),
    ]
    for i, (call, code, msg) in enumerate(calls):
        assert call() == code, i
        assert msg in L.last_error(), (i, L.last_error())
    assert L.launch_count() == n0


# ------------------------------------------------------------------ tie-ins through the engine and the optimizer
def test_engine_linear_into_conds_rows():
    """Engine.linear / linear_bwd on one AdaIN affine layer writing conds[:, 7] of a [B][12][256] tensor."""
    import oracle.ae_oracle as orc
    from adaptive_voice_conversion_b200.engine import Engine
    eng = Engine(orc.default_config(80), torch.device("cuda", 0))
    g = gen_of("engine-linear")
    B, N, K = 9, 256, 128
    w, b, x = randn(g, N, K) / math.sqrt(K), 0.3 * randn(g, N), randn(g, B, K)
    dw0, db0, dx_add = randn(g, N, K), randn(g, N), randn(g, B, K)
    name = "decoder.conv_affine_layers.7"
    P = {name + ".weight": w.cuda(), name + ".bias": b.cuda()}
    G = {name + ".weight": dw0.cuda(), name + ".bias": db0.cuda()}
    conds = torch.full((B, 12, N), SENT, device="cuda")
    dconds = torch.full((B, 12, N), SENT, device="cuda")
    dconds[:, 7] = randn(g, B, N).cuda()
    out, rec = eng.linear(P, name, x.cuda(), out=conds[:, 7], train=True)
    dx = eng.linear_bwd(P, G, rec, dconds[:, 7], dx_add=dx_add.cuda())
    assert out.stride(0) == 3072 and intact(conds, (slice(None), 7))
    out_r, _ = R.linear_fwd(x, w, b)
    dy = dconds[:, 7].cpu()
    dx_r, dw_r, db_r = R.linear_bwd(x, w, dy, dx_add=dx_add, dw0=dw0, db0=db0)
    s_dx, s_dw, s_db = R.linear_bwd(x.abs(), w.abs(), dy.abs(), dx_add=dx_add.abs(), dw0=dw0.abs(), db0=db0.abs())
    errs = {"out": err(conds[:, 7], out_r, R.linear_fwd(x.abs(), w.abs(), b.abs())[0]), "dx": err(dx, dx_r, s_dx),
            "dw": err(G[name + ".weight"], dw_r, s_dw), "db": err(G[name + ".bias"], db_r, s_db)}
    record("engine-linear", "linear", {""}, errs)


def test_fused_adam_on_model_flat_buffers():
    """FusedAdam.step on the 80-mel model's flat parameter buffer (4 892 880 floats): one step from a preloaded state
    against the restatement."""
    import oracle.ae_oracle as orc
    from adaptive_voice_conversion_b200.model import AE
    from adaptive_voice_conversion_b200.optim import FusedAdam
    cfg = orc.default_config(80)
    model = AE(cfg)
    model.load_state_dict(orc.init_state(cfg, seed=0))
    model = model.cuda()
    model.flatten_parameters()
    opt = FusedAdam(model, lr=5e-4, weight_decay=1e-4, max_norm=MAX_NORM)
    n = opt.flat_p.numel()
    assert n == 4892880
    gg = torch.Generator(device="cuda").manual_seed(21)
    opt.flat_g.copy_(1e-2 * torch.randn(n, generator=gg, device="cuda"))
    opt.flat_m.copy_(1e-3 * torch.randn(n, generator=gg, device="cuda"))
    opt.flat_v.copy_(1e-6 * torch.randn(n, generator=gg, device="cuda") ** 2)
    opt.flat_vmax.copy_(opt.flat_v * 1.2)
    opt.step_dev.fill_(7.0)
    st0 = [t.clone() for t in (opt.flat_p, opt.flat_m, opt.flat_v, opt.flat_vmax)]
    opt.step()
    hp = opt.hp.cpu()
    sqv = float(opt.sqnorm)
    assert abs(sqv - R.sqnorm(opt.flat_g)) / R.sqnorm(opt.flat_g) < TOL["sqnorm"]
    pr, mr, vr, vmr, t = R.adam_step(*st0[:1], opt.flat_g, *st0[1:], 7.0, hp, sqv)
    assert float(opt.step_dev) == t == 8.0
    b1, b2 = float(hp[R.HP_B1]), float(hp[R.HP_B2])
    gmag = opt.flat_g.double().abs() * R.clip_coef(hp, sqv) + float(hp[R.HP_WD]) * st0[0].double().abs()
    mmag = st0[1].double().abs() + (1 - b1) * (gmag + st0[1].double().abs())
    vmag = b2 * st0[2].double() + (1 - b2) * gmag * gmag
    assert same_bits(opt.flat_vmax, torch.maximum(st0[3], opt.flat_v))
    denom = vmr.sqrt() / math.sqrt(1 - b2 ** t) + float(hp[R.HP_EPS])
    umag = float(hp[R.HP_LR]) / (1 - b1 ** t) * mmag / denom
    errs = {"adam m": err(opt.flat_m, mr, ULP * mmag), "adam v": err(opt.flat_v, vr, ULP * vmag),
            "adam p": err(((opt.flat_p.double() - pr).abs() - half_ulp(pr)).clamp_min(0), torch.zeros_like(pr), umag)}
    record("fused-adam-model", "adam", {""}, errs)


# ------------------------------------------------------------------ coverage
def _all_ids():
    return ([c.id for c in LIN_CASES] + [f"stack-n{n}-B{b}" for n, b in STACK_CASES] + [c.id for c in BATCH_CASES]
            + [f"tmean-B{b}-C{c}-T{t}" + ("-view" if v else "") for b, c, t, v in TM_CASES]
            + [f"pack-B{b}-C{c}-T{t}" + ("-view" if v else "") + f"-r{r}" for b, c, t, v, r in PACK_CASES]
            + [f"reparam-{i}-B{b}-C{c}-T{t}" for i, b, c, t in REPARAM_CASES] + [f"vae-{a}-{b}" for a, b in VAE_CASES]
            + [f"sqnorm-{n}" for n in SQ_CASES] + [f"adam-{n}-a{a}-wd{w:g}-s{s}" for n, a, w, s in ADAM_CASES]
            + ["adam-vs-torch", "engine-linear", "fused-adam-model"])


def test_small_ops_coverage():
    """The cases reached every entry of FEATURES; reports the worst error per group and measure."""
    ids = _all_ids()
    if any(i not in RESULTS for i in ids):
        pytest.skip("only part of the module ran")
    worst, covered = {}, set()
    for grp, feats, errs in RESULTS.values():
        covered |= feats
        for k, e in errs.items():
            key = k if k in TOL else grp
            worst[key] = max(worst.get(key, 0.0), e)
    print(f"\nsmall ops exact: {len(ids)} cases in {time.time() - _T0[0]:.1f} s on {torch.cuda.get_device_name(0)}; worst "
          "error (tolerance): " + ", ".join(f"{k} {e:.2e} ({TOL[k]:.0e})" for k, e in sorted(worst.items())))
    for cid in ids:
        print(f"  {cid}: " + ", ".join(f"{k} {e:.2e}" for k, e in RESULTS[cid][2].items()))
    missing = [f for f in FEATURES if f not in covered]
    assert not missing, missing
