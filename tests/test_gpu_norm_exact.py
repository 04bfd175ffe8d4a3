"""GPU: the HBM-bound epilogue kernels of csrc/norm.cu -- avc_norm_bwd (norm_bwd_cached_kernel, norm_bwd_kernel<false>,
norm_bwd_kernel<true>, partial_sum_kernel), avc_norm_apply_fwd (both instances), avc_fold_add_fwd, avc_bias_grad(_groups)
-- and the AVC_F_NORMBWD epilogue of the persistent conv kernel, against the float64 restatement in tests/_norm_ref.py.

The kernels read fp32 operands: c, dy, cond, res, mask and the fp32 (mean, rstd) statistics.  The reference reads the
same values, so what is left of the difference is the kernels' fp32 arithmetic.  Tensors are put into the A4 layout on
the host by a permute (bit-exact, no pack kernel), descriptors are built by hand, and the cases use the model's
strides: the decoder's AdaIN rows are views conds[:, i] of a [B][12][2 Cn] tensor (cond_bstride 3072 at Cn = 128), and
the bank's dc and bias gradient are channel sub-ranges of a wider tensor.  Every strided output sits inside a tensor
filled with a sentinel that must survive outside the view.  The last test asserts that the cases reached every entry
of FEATURES and prints the worst error per group.

Error: max |kernel - reference| / max |reference| per output tensor.  Exceptions:
  * outputs rounded to TF32 (AVC_F_ROUND_OUT): every value must have its low 13 bits clear, and the error is what
    exceeds one TF32 ulp of the reference value, over max |reference|;
  * mean: |delta mean| * rstd (the error in units of the channel's spread); rstd: relative per channel;
  * bias gradients, which are added to a nonzero dbias: |dbias - (dbias0 + sums)| / max |sums|;
  * behind a ReLU that follows InstanceNorm the kernel decides pre > 0 in fp32: rows whose reference pre-activation
    comes within 1e-6 of the row's largest |pre| are left out (and must be under 1 % of the rows).

Worst observed on 1x NVIDIA H100 80GB HBM3 (132 SMs, 700 W power limit), per group of cases:
    bwd cached 1.5e-7, bwd plain 3.8e-7, bwd shuffle 3.4e-7, apply plain 4.6e-7, apply shuffle 1.6e-6, fold 7.2e-8,
    bias 2.3e-7;  mean (in units of the spread) 5.7e-6, at Tn = 2;  nbw 1.5e-6 and the engine tie-in 2.1e-6, whose
    operands pass through a TF32 conv (the same level as tests/test_gpu_tc2_exact.py).
TOL, TOL_MEAN and TOL_TC are about 3x those.  For scale, deliberately broken kernels land at: the lone avg-pool tail of
the fold weighted 1/2, 0.30 .. 0.33; 1 / Tout for 1 / Tn under pixel shuffle, 0.05 .. 0.43 on dc and 1.3 .. 2.3 on the
bias gradient (backward), 0.22 .. 6e3 (forward); AdaIN rows indexed 2 Cn apart instead of cond_bstride, 21 .. 3.9e3.
Before the two-pass forward corrected its mean with the sum of the deviations, the constant channel at Tout = 2000 was
off by 7.0e-5 (out) and 5.3e-4 (mean); now 4.6e-7 and 3.3e-6.
The module takes about 20 s on that GPU (the float64 reference on the CPU included).
"""
import ctypes as C
import math
import time
import zlib
from dataclasses import dataclass

import pytest
import torch
import torch.nn.functional as F

from _norm_ref import RES_POOL, RES_UP, bias_sums, fold_add, from_a4, norm_apply, norm_bwd, relerr, tf32, to_a4

pytestmark = pytest.mark.gpu

TOL = 5e-6            # kernels of csrc/norm.cu
TOL_MEAN = 2e-5       # their mean statistic, in units of the channel's spread
TOL_TC = 6e-6         # results computed from the output of a TF32 conv (nbw, the engine tie-in)
EPS = 1e-5
NEAR = 1e-6           # ReLU exclusion threshold, relative to the row's largest |pre|
SENTINEL = -7777.0
PAD_C = 4             # a strided view starts 4 channels into a tensor 8 channels wider

FEATURES = (
    [("bwd kernel", k) for k in ("cached", "plain", "shuffle")]
    + ["bwd: cached at Tout = 128", "bwd: plain at Tout = 129", "bwd: ReLU only", "bwd: norm without ReLU",
       "bwd: AdaIN", "bwd: norm without AdaIN", "bwd: ROUND_OUT", "bwd: fp32 dc", "bwd: dbias null",
       "bwd: dbias partials", "bwd: dbias atomics", "bwd: cached, dead warps with dbias", "bwd: Tout < 32",
       "bwd: Tout % 32 != 0", "bwd: strided cond / dcond", "bwd: non-dense dy", "bwd: constant and DC-offset channels"]
    + [f"bwd: B = {b} with dbias" for b in (1, 5, 9, 257)]
    + [("apply kernel", k) for k in ("plain", "shuffle")]
    + [f"apply: residual {m}" for m in (1, 2, 3)]
    + ["apply: avg-pool residual, odd res_T", "apply: mask", "apply: ROUND_OUT", "apply: strided cond",
       "apply: non-dense out / res / mask", "apply: Tout = 1", "apply: Tn >= 2000", "apply: warps not a multiple of 8",
       "apply: constant and DC-offset channels", "apply: no norm"]
    + [("fold K", k) for k in range(1, 9)] + [f"fold: residual {m}" for m in range(4)]
    + ["fold: avg-pool residual, odd Tin", "fold: overlapping reflect regions", "fold: non-dense dres / dx",
       "fold: grid-stride loop wraps"]
    + [("bias T", t) for t in (1, 16, 37, 128, 300, 1024)]
    + ["bias: B = 1", "bias: B = 256", "bias: channel sub-range", "bias: groups (bank layout)", "bias: idle threads"]
    + ["nbw: norm + AdaIN + ReLU", "nbw: ReLU only (bias gradient)", "nbw: out null", "nbw: Tf <= 16", "nbw: Tf > 16",
       "nbw: tiles wrap the CTAs"])


@dataclass(frozen=True)
class Case:
    """kind "bwd" (avc_norm_bwd) / "apply" (avc_norm_apply_fwd): C = conv rows Cout, T = Tout.  "fold"
    (avc_fold_add_fwd): C channels, T = Tin, K the forward conv's width.  "bias" (avc_bias_grad, or _groups with
    group_c): C channels, T steps.  "nbw": the data-gradient conv of a K-wide 128 -> 128 conv over T steps with the
    upstream block's norm backward in its epilogue (AVC_F_NORMBWD).  res: residual mode (the adjoint one for fold /
    nbw); strided: model strides (cond rows 12 apart, channel sub-range views)."""
    group: str
    kind: str
    B: int
    C: int
    T: int
    K: int = 0
    shuffle: bool = False
    norm: bool = False
    cond: bool = False
    relu: bool = False
    rnd: bool = False
    dbias: str = ""
    res: int = 0
    res_odd: bool = False
    mask: bool = False
    strided: bool = False
    edge: bool = False
    need_dx: bool = True
    group_c: int = 0

    @property
    def id(self):
        return (f"{self.kind}-B{self.B}-C{self.C}-T{self.T}" + (f"-k{self.K}" if self.K else "")
                + ("-shuf" if self.shuffle else "") + ("-norm" if self.norm else "") + ("-cond" if self.cond else "")
                + ("-relu" if self.relu else "") + ("-tf32out" if self.rnd else "") + (f"-db{self.dbias}" if self.dbias else "")
                + (f"-res{self.res}" if self.res else "") + ("odd" if self.res_odd else "") + ("-mask" if self.mask else "")
                + ("-strided" if self.strided else "") + ("-edge" if self.edge else "") + ("" if self.need_dx else "-nodx")
                + (f"-g{self.group_c}" if self.group_c else ""))


def cases(sms):
    c = []
    bw = lambda g, B, Co, T, **k: c.append(Case(g, "bwd", B, Co, T, **k))      # noqa: E731
    # cached kernel (no shuffle, Tout <= 128)
    bw("bwd cached", 256, 128, 128, norm=True, cond=True, relu=True, rnd=True, strided=True)
    bw("bwd cached", 5, 128, 37, relu=True, rnd=True, dbias="part", strided=True)      # speaker encoder: ReLU only
    bw("bwd cached", 9, 128, 20, relu=True, dbias="atomic", strided=True)
    bw("bwd cached", 257, 128, 64, relu=True, rnd=True, dbias="part")
    bw("bwd cached", 1, 128, 128, relu=True, dbias="part")
    bw("bwd cached", 9, 128, 100, norm=True, cond=True, relu=True, strided=True, edge=True)
    bw("bwd cached", 3, 128, 1, norm=True, relu=True)
    bw("bwd cached", 5, 128, 48, norm=True, rnd=True)
    # norm_bwd_kernel<false> (Tout > 128)
    bw("bwd plain", 2, 128, 129, norm=True, cond=True, relu=True, rnd=True, strided=True)
    bw("bwd plain", 257, 128, 129, relu=True, dbias="atomic")
    bw("bwd plain", 5, 128, 300, relu=True, dbias="part", strided=True)
    bw("bwd plain", 1, 128, 2000, norm=True, cond=True, relu=True, edge=True)
    bw("bwd plain", 9, 128, 150, norm=True, edge=True)
    # norm_bwd_kernel<true> (pixel shuffle: 256 conv rows -> 128 channels)
    bw("bwd shuffle", 256, 256, 16, shuffle=True, norm=True, cond=True, relu=True, rnd=True, dbias="part", strided=True)
    bw("bwd shuffle", 5, 256, 64, shuffle=True, norm=True, cond=True, relu=True, dbias="atomic")
    bw("bwd shuffle", 1, 256, 8, shuffle=True, norm=True, cond=True, relu=True, dbias="part")
    bw("bwd shuffle", 9, 256, 129, shuffle=True, norm=True, dbias="part", strided=True, edge=True)
    bw("bwd shuffle", 3, 256, 37, shuffle=True, relu=True, rnd=True, dbias="part")
    bw("bwd shuffle", 2, 256, 300, shuffle=True, norm=True, cond=True, relu=True, dbias="atomic", edge=True)
    ap = lambda g, B, Co, T, **k: c.append(Case(g, "apply", B, Co, T, **k))    # noqa: E731
    ap("apply plain", 1, 128, 600, norm=True, cond=True, relu=True, res=1, strided=True, rnd=True)
    ap("apply plain", 2, 128, 1, norm=True, relu=True)
    ap("apply plain", 3, 128, 37, norm=True, relu=True, res=2, res_odd=True, mask=True)
    ap("apply plain", 5, 128, 2000, norm=True, relu=True, res=1, edge=True)
    ap("apply plain", 7, 128, 145, relu=True, res=2, rnd=True)
    ap("apply plain", 1, 128, 33, norm=True, cond=True, mask=True, strided=True)
    ap("apply plain", 1, 80, 301, norm=True, relu=True, res=2)                             # 20 warps
    ap("apply plain", 3, 80, 129, norm=True, cond=True, relu=True, res=1, mask=True, strided=True, rnd=True)
    ap("apply shuffle", 1, 256, 300, shuffle=True, norm=True, cond=True, relu=True, res=3, strided=True, rnd=True)
    ap("apply shuffle", 2, 256, 1000, shuffle=True, norm=True, cond=True, relu=True, res=3, mask=True, edge=True)
    ap("apply shuffle", 3, 256, 1, shuffle=True, norm=True, relu=True, res=3)
    ap("apply shuffle", 5, 256, 73, shuffle=True, norm=True, cond=True, relu=True, res=1, strided=True, edge=True)
    ap("apply shuffle", 1, 256, 77, shuffle=True, relu=True, res=2, res_odd=True, rnd=True)
    ap("apply shuffle", 1, 40, 50, shuffle=True, norm=True, cond=True, relu=True, res=2)   # 5 warps
    for K in range(1, 9):
        pl = K // 2
        c.append(Case("fold", "fold", 2, 64, pl + 1, K=K, res=K % 4, strided=K % 2 == 0))   # smallest legal Tin
        c.append(Case("fold", "fold", 3, 128, 37, K=K, res=(K + 2) % 4, strided=K % 2 == 1))
    c.append(Case("fold", "fold", 256, 128, 128, K=5, res=1))
    c.append(Case("fold", "fold", 256, 128, 37, K=8, res=2, strided=True))
    for B, Cc, T, st in ((256, 128, 16, False), (1, 128, 1, False), (256, 128, 37, True), (1, 128, 128, False),
                         (3, 128, 300, True), (2, 64, 1024, False), (256, 128, 1, True)):
        c.append(Case("bias", "bias", B, Cc, T, strided=st))
    for B, T, st in ((256, 16, True), (5, 128, True), (2, 300, False)):
        c.append(Case("bias", "bias", B, 1024, T, strided=st, group_c=128))
    c.append(Case("nbw", "nbw", 3 * sms + 2, 128, 16, K=5, norm=True, cond=True, relu=True, res=1, strided=True))
    c.append(Case("nbw", "nbw", 7, 128, 37, K=5, relu=True, res=2))
    c.append(Case("nbw", "nbw", sms + 3, 128, 128, K=5, norm=True, relu=True, need_dx=False))   # one sample per tile
    c.append(Case("nbw", "nbw", sms + 5, 128, 64, K=3, norm=True, cond=True, relu=True, res=3, strided=True))
    c.append(Case("nbw", "nbw", 19, 128, 16, K=5, relu=True, res=1, need_dx=False))
    return c


# ------------------------------------------------------------------ helpers
def place(x, strided):
    """planar [B][C][T] -> (A4 device tensor, address of x's first channel, batch stride in floats).  strided: x is
    the channel sub-range [PAD_C, PAD_C + C) of a tensor 8 channels wider, the rest SENTINEL."""
    B, Cc, T = x.shape
    if not strided:
        a = to_a4(x)
        return a, a.data_ptr(), Cc * T
    wide = torch.full((B, Cc + 2 * PAD_C, T), SENTINEL)
    wide[:, PAD_C:PAD_C + Cc] = x
    a = to_a4(wide)
    return a, a.data_ptr() + (PAD_C // 4) * T * 16, (Cc + 2 * PAD_C) * T


def take(a, Cc, strided):
    """planar view back from place(); asserts the SENTINEL outside it survived."""
    p = from_a4(a)
    if not strided:
        return p
    assert bool((p[:, :PAD_C] == SENTINEL).all() and (p[:, PAD_C + Cc:] == SENTINEL).all()), "write outside the view"
    return p[:, PAD_C:PAD_C + Cc]


def rows(x, strided):
    """[B][W] rows -> a device tensor whose stride(0) is the model's: strided = conds[:, 5] of a [B][12][W] tensor."""
    if not strided:
        return x.cuda()
    big = torch.full((x.shape[0], 12, x.shape[1]), SENTINEL)
    big[:, 5] = x
    return big.cuda()[:, 5]


def rows_back(v, strided):
    """the rows of rows() on the host; asserts the SENTINEL in the other 11 rows of each sample survived."""
    if not strided:
        return v.cpu()
    big = v._base.cpu()
    assert bool((big[:, :5] == SENTINEL).all() and (big[:, 6:] == SENTINEL).all()), "write outside the AdaIN rows"
    return big[:, 5]


def tf32_exact(y):
    return bool(((y.contiguous().view(torch.int32) & 0x1FFF) == 0).all())


def ulp_excess(y, ref):
    """max over elements of (|y - ref| - one TF32 ulp of ref), clamped at 0, over max |ref|."""
    r = ref.abs()
    ulp = torch.where(r > 0, torch.ldexp(torch.ones_like(r), torch.frexp(r)[1] - 11), torch.zeros_like(r))
    return float(((y.double() - ref).abs() - ulp).clamp_min(0).max() / r.max().clamp_min(1e-30))


def out_err(y, ref, rounded, name):
    if rounded:
        assert tf32_exact(y), f"{name}: a stored value is not TF32-exact"
        return ulp_excess(y, ref)
    return relerr(y, ref)


def conv_inputs(case, gen, Co, T):
    """raw conv output c [B][Co][T]; edge: normalised channel 0 constant over time (a bias seen through an all-zero
    input), channel 2 (shuffle) / 4 and 5 offset by 100x their spread."""
    c = torch.randn((case.B, Co, T), generator=gen) + 0.5 * torch.randn((1, Co, 1), generator=gen)
    if case.edge:
        c[:, 0:2] = c[0, 0, 0].item()
        c[:, 4:6] = 100.0 + torch.randn((case.B, 2, T), generator=gen)
    return c


def ada_rows(case, gen, Cn):
    cd = 0.5 * torch.randn((case.B, 2 * Cn), generator=gen)
    cd[:, Cn:] += 1.0
    return cd


def relu_rows_kept(c, mean, rstd, cond, shuffle):
    """[B][Cn] rows whose reference pre-activation stays clear of 0 (see the module docstring)."""
    y = c.double()
    if shuffle:
        y = y.reshape(y.shape[0], y.shape[1] // 2, 2, y.shape[2]).transpose(2, 3).reshape(y.shape[0], y.shape[1] // 2, -1)
    pre = (y - mean.double()[:, :, None]) * rstd.double()[:, :, None]
    if cond is not None:
        Cn = pre.shape[1]
        pre = pre * cond.double()[:, Cn:, None] + cond.double()[:, :Cn, None]
    a = pre.abs()
    near = a.amin(dim=2) < NEAR * a.amax(dim=2)
    assert float(near.double().mean()) < 0.01, f"{int(near.sum())} of {near.numel()} rows have a pre-activation near 0"
    return ~near


@pytest.fixture(scope="module")
def eng():
    import oracle.ae_oracle as orc
    from adaptive_voice_conversion_b200.engine import Engine
    e = Engine(orc.default_config(80), torch.device("cuda", 0))
    e.precision = "tf32"
    return e


def _sms():
    return torch.cuda.get_device_properties(0).multi_processor_count if torch.cuda.is_available() else 132


RESULTS = {}     # case id -> (group, features, {output: error})
_T0 = []


# ------------------------------------------------------------------ avc_norm_bwd
def run_bwd(eng, case, gen):
    from adaptive_voice_conversion_b200 import _lib as L
    B, Co, T = case.B, case.C, case.T
    Cn, Tn = (Co // 2, 2 * T) if case.shuffle else (Co, T)
    c = conv_inputs(case, gen, Co, T)
    cond = ada_rows(case, gen, Cn) if case.cond else None
    dy = torch.randn((B, Cn, Tn), generator=gen)
    mean = rstd = stats = None
    if case.norm:
        _, m64, r64 = norm_apply(c, shuffle=case.shuffle, norm=True, eps=EPS)
        mean, rstd = m64.float(), r64.float()          # the fp32 statistics the kernel reads, and the reference too
        stats = torch.stack([mean, rstd], 2).cuda()
    ca = to_a4(c)
    dya, dy_ptr, dy_bs = place(dy, case.strided)
    dc = torch.full((B, Co // 4, T, 4), SENTINEL, device="cuda")
    d = L.ConvDesc()
    d.B, d.Cin, d.Cout, d.K, d.stride, d.in_ups, d.Tin, d.Tout = B, 4, Co, 1, 1, 1, T, T
    d.shuffle, d.norm, d.relu, d.eps = int(case.shuffle), int(case.norm), int(case.relu), EPS
    d.save_c, d.stats = ca.data_ptr(), stats.data_ptr() if stats is not None else None
    d.dy, d.dy_bstride, d.dc = dy_ptr, dy_bs, dc.data_ptr()
    dcond = None
    if case.cond:
        cv = rows(cond, case.strided)
        dcond = rows(torch.full((B, 2 * Cn), SENTINEL), case.strided)
        d.cond, d.cond_bstride = cv.data_ptr(), cv.stride(0)
        d.dcond, d.dcond_bstride = dcond.data_ptr(), dcond.stride(0)
    db0 = torch.randn((Co,), generator=gen)
    dbias = db0.cuda() if case.dbias else None
    if case.dbias:
        d.dbias = dbias.data_ptr()
        if case.dbias == "part":
            part = torch.full((B * Co,), SENTINEL, device="cuda")
            d.dbias_part = part.data_ptr()
    d.flags = L.F_ROUND_OUT if case.rnd else 0
    eng._ck(eng.lib.avc_norm_bwd(C.byref(d), eng.stream), f"norm_bwd[{case.id}]")
    dc_k = from_a4(dc)
    dc_r, dcond_r, db_r = norm_bwd(c, mean, rstd, cond, dy, shuffle=case.shuffle, norm=case.norm, relu=case.relu)
    keep = torch.ones((B, Cn), dtype=torch.bool)
    if case.norm and case.relu:
        keep = relu_rows_kept(c, mean, rstd, cond, case.shuffle)
    keep_c = keep.repeat_interleave(2, dim=1) if case.shuffle else keep
    kk = keep_c[:, :, None].expand_as(dc_r)
    errs = {"dc": out_err(dc_k[kk], dc_r[kk], case.rnd, "dc")}
    if case.cond:
        dk, dr = rows_back(dcond, case.strided), dcond_r
        k2 = torch.cat([keep, keep], 1)
        errs["dcond"] = relerr(dk[k2], dr[k2])
    if case.dbias:
        full = keep_c.all(dim=0)
        sums = bias_sums(dc_r)
        errs["dbias"] = float(((dbias.cpu().double() - db0.double() - sums)[full]).abs().max() / sums.abs().max())
    feats = set()
    cached = not case.shuffle and T <= 128            # avc_norm_bwd's kernel selection
    kname = "shuffle" if case.shuffle else "cached" if cached else "plain"
    feats.add(("bwd kernel", kname))
    if cached and T == 128:
        feats.add("bwd: cached at Tout = 128")
    if kname == "plain" and T == 129:
        feats.add("bwd: plain at Tout = 129")
    feats.add("bwd: ReLU only" if not case.norm else "bwd: norm without ReLU" if not case.relu else "")
    if case.norm:
        feats.add("bwd: AdaIN" if case.cond else "bwd: norm without AdaIN")
    feats.add("bwd: ROUND_OUT" if case.rnd else "bwd: fp32 dc")
    feats.add({"": "bwd: dbias null", "part": "bwd: dbias partials", "atomic": "bwd: dbias atomics"}[case.dbias])
    if case.dbias:
        feats.add(f"bwd: B = {B} with dbias")
        if cached and B % 8:
            feats.add("bwd: cached, dead warps with dbias")
    if T < 32:
        feats.add("bwd: Tout < 32")
    if T % 32:
        feats.add("bwd: Tout % 32 != 0")
    if case.strided:
        feats.add("bwd: non-dense dy")
        if case.cond:
            feats.add("bwd: strided cond / dcond")
    if case.edge:
        feats.add("bwd: constant and DC-offset channels")
    return feats, errs


# ------------------------------------------------------------------ avc_norm_apply_fwd
def run_apply(eng, case, gen):
    from adaptive_voice_conversion_b200 import _lib as L
    B, Co, T = case.B, case.C, case.T
    Cn, Tn = (Co // 2, 2 * T) if case.shuffle else (Co, T)
    c = conv_inputs(case, gen, Co, T)
    cond = ada_rows(case, gen, Cn) if case.cond else None
    rT = {0: 0, 1: Tn, 2: 2 * Tn - (1 if case.res_odd else 0), 3: Tn // 2}[case.res]
    res = torch.randn((B, Cn, rT), generator=gen) if rT else None
    mask = (torch.randn((B, Cn, Tn), generator=gen) > -0.5).float() if case.mask else None
    ca = to_a4(c)
    out, out_ptr, out_bs = place(torch.full((B, Cn, Tn), SENTINEL), case.strided)
    stats = torch.full((B, Cn, 2), SENTINEL, device="cuda") if case.norm else None
    d = L.ConvDesc()
    d.B, d.Cin, d.Cout, d.K, d.stride, d.in_ups, d.Tin, d.Tout = B, 4, Co, 1, 1, 1, T, T
    d.shuffle, d.norm, d.relu, d.eps = int(case.shuffle), int(case.norm), int(case.relu), EPS
    d.save_c, d.out, d.out_bstride = ca.data_ptr(), out_ptr, out_bs
    d.stats = stats.data_ptr() if stats is not None else None
    keep = []
    if case.cond:
        cv = rows(cond, case.strided)
        keep.append(cv)
        d.cond, d.cond_bstride = cv.data_ptr(), cv.stride(0)
    if res is not None:
        ra, d.res, d.res_bstride = place(res, case.strided)
        keep.append(ra)
        d.res_mode, d.res_T = case.res, rT
    if mask is not None:
        ma, d.mask, d.mask_bstride = place(mask, case.strided)
        keep.append(ma)
    d.flags = L.F_ROUND_OUT if case.rnd else 0
    eng._ck(eng.lib.avc_norm_apply_fwd(C.byref(d), eng.stream), f"norm_apply_fwd[{case.id}]")
    y_r, m_r, r_r = norm_apply(c, shuffle=case.shuffle, norm=case.norm, eps=EPS, cond=cond, relu=case.relu, res=res,
                               res_mode=case.res, mask=mask)
    errs = {"out": out_err(take(out, Cn, case.strided), y_r, case.rnd, "out")}
    if case.norm:
        s = stats.cpu().double()
        errs["mean"] = float(((s[:, :, 0] - m_r).abs() * r_r).max())
        errs["rstd"] = float(((s[:, :, 1] - r_r).abs() / r_r).max())
    feats = {("apply kernel", "shuffle" if case.shuffle else "plain")}
    if case.res:
        feats.add(f"apply: residual {case.res}")
        if case.res == RES_POOL and rT % 2:
            feats.add("apply: avg-pool residual, odd res_T")
    if case.mask:
        feats.add("apply: mask")
    if case.rnd:
        feats.add("apply: ROUND_OUT")
    if case.strided:
        if case.cond:
            feats.add("apply: strided cond")
        if case.res and case.mask:
            feats.add("apply: non-dense out / res / mask")
    if T == 1:
        feats.add("apply: Tout = 1")
    if Tn >= 2000:
        feats.add("apply: Tn >= 2000")
    if (B * Cn // 4) % 8:
        feats.add("apply: warps not a multiple of 8")
    if case.edge:
        feats.add("apply: constant and DC-offset channels")
    if not case.norm:
        feats.add("apply: no norm")
    return feats, errs


# ------------------------------------------------------------------ avc_fold_add_fwd
def run_fold(eng, case, gen):
    from adaptive_voice_conversion_b200 import _lib as L
    B, Cc, T, K = case.B, case.C, case.T, case.K
    pl, pr = K // 2, K // 2 - (1 if K % 2 == 0 else 0)
    dxp = torch.randn((B, Cc, T + pl + pr), generator=gen)
    rT = {0: 0, 1: T, 2: (T + 1) // 2, 3: 2 * T}[case.res]
    dres = torch.randn((B, Cc, rT), generator=gen) if rT else None
    xa = to_a4(dxp)
    dx, dx_ptr, dx_bs = place(torch.full((B, Cc, T), SENTINEL), case.strided)
    f = L.FoldDesc()
    f.B, f.C, f.Tin, f.pad_left, f.pad_right = B, Cc, T, pl, pr
    f.dxp, f.dx, f.dx_bstride = xa.data_ptr(), dx_ptr, dx_bs
    if dres is not None:
        ra, f.dres, f.dres_bstride = place(dres, case.strided)
        f.res_mode, f.res_T = case.res, rT
    eng._ck(eng.lib.avc_fold_add_fwd(C.byref(f), eng.stream), f"fold_add[{case.id}]")
    errs = {"dx": relerr(take(dx, Cc, case.strided), fold_add(dxp, pl, pr, dres, case.res))}
    feats = {("fold K", K), f"fold: residual {case.res}"}
    if case.res == RES_POOL and T % 2:
        feats.add("fold: avg-pool residual, odd Tin")
    if pr >= 1 and max(1, T - 1 - pr) <= min(pl, T - 2):
        feats.add("fold: overlapping reflect regions")
    if case.strided and case.res:
        feats.add("fold: non-dense dres / dx")
    if B * (Cc // 4) * T > 148 * 16 * 256:
        feats.add("fold: grid-stride loop wraps")
    return feats, errs


# ------------------------------------------------------------------ avc_bias_grad / avc_bias_grad_groups
def run_bias(eng, case, gen):
    B, Cc, T = case.B, case.C, case.T
    dc = torch.randn((B, Cc, T), generator=gen)
    a, ptr, bs = place(dc, case.strided)
    db0 = torch.randn((Cc,), generator=gen)
    if case.group_c:
        outs = [db0[i:i + case.group_c].clone().cuda() for i in range(0, Cc, case.group_c)]
        tab = torch.tensor([o.data_ptr() for o in outs], dtype=torch.int64).cuda()
        eng._ck(eng.lib.avc_bias_grad_groups(ptr, bs, tab.data_ptr(), case.group_c, B, Cc, T, eng.stream), f"bias_grad_groups[{case.id}]")
        got = torch.cat([o.cpu() for o in outs])
    else:
        out = db0.cuda()
        eng._ck(eng.lib.avc_bias_grad(ptr, bs, out.data_ptr(), B, Cc, T, eng.stream), f"bias_grad[{case.id}]")
        got = out.cpu()
    sums = bias_sums(dc, case.group_c or None).reshape(-1)
    errs = {"dbias": float((got.double() - db0.double() - sums).abs().max() / sums.abs().max())}
    feats = {("bias T", T)}
    if B in (1, 256):
        feats.add(f"bias: B = {B}")
    if case.strided:
        feats.add("bias: channel sub-range")
    if case.group_c:
        feats.add("bias: groups (bank layout)")
    if 1024 % T:
        feats.add("bias: idle threads")
    return feats, errs


# ------------------------------------------------------------------ AVC_F_NORMBWD epilogue of avc_conv_block_tc
def run_nbw(eng, case, gen):
    import test_gpu_tc2_exact as tc2
    from adaptive_voice_conversion_b200 import _lib as L
    B, Cc, T, K = case.B, case.C, case.T, case.K
    pl, pr = K // 2, K // 2 - (1 if K % 2 == 0 else 0)
    c2 = tc2.Case("nbw", "fold", B, Cc, Cc, K, T, in_tf32=True, fres=case.res)
    x = tf32(torch.randn((B, Cc, T), generator=gen))                   # the downstream dc, TF32-exact like the engine's
    w = torch.randn((Cc, Cc, K), generator=gen) / math.sqrt(Cc * K)   # forward layer [Ci][Co][K]
    rT = tc2.res_len(c2)
    res = torch.randn((B, Cc, rT), generator=gen) if rT else None
    name = "blk"
    P = {name + ".weight": w.cuda(), name + ".bias": torch.zeros(Cc).cuda()}
    eng.conv_names = lambda: [name]
    eng.packed.pop(name, None)
    eng.pack_weights(P, need_dgrad=True)
    out = torch.full((B, Cc // 4, T, 4), SENTINEL, device="cuda")
    dev = dict(x=to_a4(x), out=out, res=to_a4(res) if res is not None else None, w=eng.packed[name]["dgrad_tc"])
    ptr = {k: (v.data_ptr() if v is not None else None) for k, v in dev.items()} | {"mask": None}
    g, par = tc2.geometry(c2)[0]
    d = tc2.make_desc(c2, g, par, ptr)
    # the upstream block: raw conv output c, its fp32 statistics and AdaIN rows
    c = conv_inputs(case, gen, Cc, T)
    cond = ada_rows(case, gen, Cc) if case.cond else None
    mean = rstd = None
    d.flags = int(d.flags) | L.F_NORMBWD | L.F_ROUND_OUT
    d.norm, d.relu, d.eps = int(case.norm), int(case.relu), EPS
    ca = to_a4(c)
    d.save_c = ca.data_ptr()
    if case.norm:
        _, m64, r64 = norm_apply(c, norm=True, eps=EPS)
        mean, rstd = m64.float(), r64.float()
        stats = torch.stack([mean, rstd], 2).cuda()
        d.stats = stats.data_ptr()
    dcond = None
    if case.cond:
        cv = rows(cond, case.strided)
        dcond = rows(torch.full((B, 2 * Cc), SENTINEL), case.strided)
        d.cond, d.cond_bstride = cv.data_ptr(), cv.stride(0)
        d.dcond, d.dcond_bstride = dcond.data_ptr(), dcond.stride(0)
    dc = torch.full((B, Cc // 4, T, 4), SENTINEL, device="cuda")
    d.dc = dc.data_ptr()
    db0 = torch.randn((Cc,), generator=gen)
    dbias = None
    if not case.norm:
        dbias = db0.cuda()
        d.dbias = dbias.data_ptr()
    if not case.need_dx:
        d.out = None
    sms = _sms()
    rc, plan = tc2.plan_of(eng.lib, d, sms)
    assert rc == 0, L.last_error()
    eng._ck(eng.lib.avc_conv_block_tc(C.byref(d), eng.tc_status.data_ptr(), eng.stream), f"conv_block_tc[{case.id}]")
    eng.check_tc_status()
    full = F.conv_transpose1d(tf32(x).double(), tf32(w).double())     # [B][Co][T + K - 1]
    dx_r = fold_add(full, pl, pr, res, case.res)
    dc_r, dcond_r, db_r = norm_bwd(c, mean, rstd, cond, dx_r, norm=case.norm, relu=case.relu)
    keep = relu_rows_kept(c, mean, rstd, cond, False) if case.norm and case.relu else torch.ones((B, Cc), dtype=torch.bool)
    kk = keep[:, :, None].expand_as(dc_r)
    errs = {"dc": out_err(from_a4(dc)[kk], dc_r[kk], True, "dc")}
    if case.need_dx:
        errs["dx"] = relerr(from_a4(out), dx_r)
    else:
        assert bool((from_a4(out) == SENTINEL).all()), "out is null: nothing may be written"
    if case.cond:
        k2 = torch.cat([keep, keep], 1)
        errs["dcond"] = relerr(rows_back(dcond, case.strided)[k2], dcond_r[k2])
    if dbias is not None:
        sums = bias_sums(dc_r)
        errs["dbias"] = float((dbias.cpu().double() - db0.double() - sums).abs().max() / sums.abs().max())
    feats = {"nbw: Tf <= 16" if T <= 16 else "nbw: Tf > 16"}
    if case.norm and case.cond and case.relu:
        feats.add("nbw: norm + AdaIN + ReLU")
    if not case.norm:
        feats.add("nbw: ReLU only (bias gradient)")
    if not case.need_dx:
        feats.add("nbw: out null")
    if plan.ntiles > sms:
        feats.add("nbw: tiles wrap the CTAs")
    return feats, errs


RUN = {"bwd": run_bwd, "apply": run_apply, "fold": run_fold, "bias": run_bias, "nbw": run_nbw}


@pytest.mark.parametrize("case", cases(_sms()), ids=lambda c: c.id)
def test_norm_exact(eng, case):
    if not _T0:
        _T0.append(time.time())
    gen = torch.Generator().manual_seed(zlib.crc32(case.id.encode()))
    feats, errs = RUN[case.kind](eng, case, gen)
    feats.discard("")
    RESULTS[case.id] = (case.group, feats, errs)
    for k, e in errs.items():
        tol = TOL_MEAN if k == "mean" else TOL_TC if case.kind == "nbw" else TOL
        assert e < tol, f"{k}: error {e:.3e} (tolerance {tol:.0e})"


def test_deterministic_bias_gradients(eng):
    """avc_norm_bwd with dbias_part (every kernel) and both bias-gradient entry points give the same bits twice."""
    from adaptive_voice_conversion_b200 import _lib as L
    gen = torch.Generator().manual_seed(5)
    for Co, T, shuffle in ((128, 64, False), (128, 300, False), (256, 37, True)):
        B = 257
        c, dy = to_a4(torch.randn((B, Co, T), generator=gen)), torch.randn((B, Co // (2 if shuffle else 1), T * (2 if shuffle else 1)), generator=gen)
        dya = to_a4(dy)
        got = []
        for _ in range(2):
            dc = torch.zeros_like(c)
            db = torch.zeros(Co, device="cuda")
            part = torch.zeros(B * Co, device="cuda")
            d = L.ConvDesc()
            d.B, d.Cin, d.Cout, d.K, d.stride, d.in_ups, d.Tin, d.Tout = B, 4, Co, 1, 1, 1, T, T
            d.shuffle, d.relu, d.eps = int(shuffle), 1, EPS
            d.save_c, d.dy, d.dy_bstride, d.dc = c.data_ptr(), dya.data_ptr(), dy[0].numel(), dc.data_ptr()
            d.dbias, d.dbias_part = db.data_ptr(), part.data_ptr()
            eng._ck(eng.lib.avc_norm_bwd(C.byref(d), eng.stream), "norm_bwd")
            got.append((db.cpu(), dc.cpu()))
        assert torch.equal(got[0][0], got[1][0]) and torch.equal(got[0][1], got[1][1]), (Co, T, shuffle)
    dc = to_a4(torch.randn((256, 1104, 16), generator=gen))
    bank = dc.data_ptr()
    got = []
    for _ in range(2):
        outs = [torch.zeros(128, device="cuda") for _ in range(8)]
        tab = torch.tensor([o.data_ptr() for o in outs], dtype=torch.int64).cuda()
        one = torch.zeros(1024, device="cuda")
        eng._ck(eng.lib.avc_bias_grad_groups(bank, 1104 * 16, tab.data_ptr(), 128, 256, 1024, 16, eng.stream), "bias_grad_groups")
        eng._ck(eng.lib.avc_bias_grad(bank, 1104 * 16, one.data_ptr(), 256, 1024, 16, eng.stream), "bias_grad")
        got.append((torch.cat([o.cpu() for o in outs]), one.cpu()))
    assert torch.equal(got[0][0], got[1][0]) and torch.equal(got[0][1], got[1][1])
    assert torch.equal(got[0][0], got[0][1])       # one order of summation for both entry points


@pytest.mark.parametrize("shuffle", [False, True], ids=["same", "shuffle-up"])
def test_engine_long_sample_fills_descriptors(eng, shuffle):
    """Engine.conv in tf32 mode on a 600-frame sample with InstanceNorm, AdaIN rows of the decoder's [B][12][256]
    tensor, ReLU and a residual: the plain tensor-core conv followed by avc_norm_apply_fwd, against the float64
    reference on the TF32-rounded x and w."""
    from adaptive_voice_conversion_b200 import _lib as L
    from adaptive_voice_conversion_b200.engine import A4
    gen = torch.Generator().manual_seed(600 + shuffle)
    B, Ci, K, T = 2, 128, 5, 600
    Co = 256 if shuffle else 128
    Cn, Tn = (Co // 2, 2 * T) if shuffle else (Co, T)
    x = torch.randn((B, Ci, T), generator=gen)
    w = torch.randn((Co, Ci, K), generator=gen) / math.sqrt(Ci * K)
    bias = 0.1 * torch.randn((Co,), generator=gen)
    conds = 0.5 * torch.randn((B, 12, 2 * Cn), generator=gen)
    conds[:, :, Cn:] += 1.0
    res = torch.randn((B, Cn, Tn // 2 if shuffle else Tn), generator=gen)
    mode = L.RES_UP if shuffle else L.RES_SAME
    name = "blk"
    P = {name + ".weight": w.cuda(), name + ".bias": bias.cuda()}
    eng.conv_names = lambda: [name]
    eng.packed.pop(name, None)
    eng.pack_weights(P, need_dgrad=False)
    xt, rt, cd = to_a4(x), to_a4(res), conds.cuda()
    n0 = L.launch_count()
    out, rec = eng.conv(P, name, A4(xt, xt.data_ptr(), B, Ci, T, Ci * T), shuffle=shuffle, norm=True, cond=cd[:, 7], relu=True,
                        res=A4(rt, rt.data_ptr(), B, Cn, res.shape[2], Cn * res.shape[2]), res_mode=mode, train=True)
    eng.check_tc_status()
    assert L.launch_count() - n0 == 2       # conv_tc_plain + norm_apply_fwd
    c_r = F.conv1d(F.pad(tf32(x).double(), (2, 2), mode="reflect"), tf32(w).double(), bias.double())
    y_r, m_r, r_r = norm_apply(c_r, shuffle=shuffle, norm=True, eps=EPS, cond=conds[:, 7], relu=True, res=res, res_mode=mode)
    errs = {"c": relerr(from_a4(rec["c"].t), c_r), "out": relerr(from_a4(out.t), y_r),
            "mean": float(((rec["stats"].cpu().double()[:, :, 0] - m_r).abs() * r_r).max()),
            "rstd": float(((rec["stats"].cpu().double()[:, :, 1] - r_r).abs() / r_r).max())}
    print(f"\nengine {'shuffle-up' if shuffle else 'same'}: " + ", ".join(f"{k} {e:.2e}" for k, e in errs.items()))
    for k, e in errs.items():
        tol = TOL_MEAN if k == "mean" else TOL_TC
        assert e < tol, f"{k}: error {e:.3e} (tolerance {tol:.0e})"


def test_norm_exact_coverage():
    """The cases reached every entry of FEATURES; reports the worst error per group."""
    all_ids = [c.id for c in cases(_sms())]
    if any(i not in RESULTS for i in all_ids):
        pytest.skip("only part of the module ran")
    worst, covered = {}, set()
    for grp, feats, errs in RESULTS.values():
        covered |= feats
        worst[grp] = max(worst.get(grp, 0.0), *(e for k, e in errs.items() if k != "mean"))
        if "mean" in errs:
            worst["mean"] = max(worst.get("mean", 0.0), errs["mean"])
    print(f"\nnorm exact: {len(all_ids)} cases in {time.time() - _T0[0]:.1f} s on {torch.cuda.get_device_name(0)}; worst error "
          f"per group (tolerance {TOL:.0e}, mean {TOL_MEAN:.0e}, nbw {TOL_TC:.0e}): "
          + ", ".join(f"{g} {e:.2e}" for g, e in sorted(worst.items())))
    for cid in all_ids:
        print(f"  {cid}: " + ", ".join(f"{k} {e:.2e}" for k, e in RESULTS[cid][2].items()))
    missing = [f for f in FEATURES if f not in covered]
    assert not missing, missing
