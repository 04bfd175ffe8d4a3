"""GPU: the persistent tensor-core conv kernel (conv_block_tc2_kernel, csrc/conv_tc2.cu) against a float64 reference
computed on the SAME TF32-rounded operands.

The kernel rounds both MMA operands to TF32 with cvt.rna (the weight packs, and the input in its patch warps unless the
producer already did: AVC_F_IN_TF32).  The reference rounds them the same way, then convolves, normalises, folds, ... in
float64 on the CPU, so what is left of the difference is the kernel's fp32 accumulation and epilogue.  A kernel that
skipped a rounding, dropped a tap or mis-folded a halo row is off by far more than the tolerance.

Every case is driven through the C entry point with a hand-built descriptor.  Before the launch the plan query
(avc_conv_block_tc_plan) reports the tile plan the launch uses; the last test asserts that the union of those plans
reaches every kernel instance and every plan feature in FEATURES, so a planner change cannot silently drop coverage.
The cases follow from the SM count (tests/test_conv_tc2_plan.py checks the coverage for 132 and 114 SMs on the CPU).

Tolerance: max |kernel - reference| / max |reference| per output tensor (`out`, and the raw conv `c` of a forward
block).  Worst observed on 1x NVIDIA H100 80GB HBM3 (132 SMs, 400 W power limit), per group of cases:
    width 2.8e-6, stacked 1.1e-6, time-tiled 1.9e-6, dgrad 1.6e-6, fold 3.0e-6, fold chunked 1.8e-6.
TOL is about 3x the worst of them.  For scale: when the patch warps skip the TF32 rounding of the input, the cases that
round in the kernel are off by 2.8e-4 .. 5.7e-4; a dropped tap or a dropped reflect term of the fold, by 0.18 .. 0.55.
The module takes about 10 s on that GPU (the float64 reference on the CPU included).
"""
import ctypes as C
import math
import time
import zlib
from dataclasses import dataclass

import pytest
import torch
import torch.nn.functional as F

pytestmark = pytest.mark.gpu

TOL = 1e-5

# every (N, NL) instance of conv_block_tc2_kernel: the single-chunk widths and the last-chunk widths of a chunked sample
INSTANCES = [(n, n) for n in range(16, 161, 16)] + [(128, nl) for nl in range(32, 113, 16)]
FEATURES = ([("instance", n, nl) for n, nl in INSTANCES] + [("hs", 1), ("hs", 2), ("hs", 4)] + [
    "short last stage", "nst == 1", "nst < nstage", "tiles wrap the CTAs", "G > 1, ragged batch tail",
    "partial M tile", "mtiles > 1, partial last M tile (data gradient)", "ntt > 1, ragged last time tile",
    "patch: rounding", "patch: reflect rows only", "patch: off", "forward stride 2",
    "stride-2 parity data gradient", "stride-2 parity data gradient, time-tiled",
    "fold, residual 0", "fold, residual 1", "fold, residual 2", "fold, residual 3", "fold at Lp + K - 1 == 256",
    "pixel shuffle + AdaIN"])


@dataclass(frozen=True)
class Case:
    """One launch (two for kind "s2").  Channel counts are the KERNEL's: Ci input, Co output channels.
    kind "fwd": conv block (reflect or zero padding), nn.Conv1d weight [Co][Ci][K], FWD pack.
    kind "dgrad": data gradient of a stride-1 conv (zero padding K-1, Tout = T + K - 1); the forward layer's weight is
    [Ci][Co][K] and the kernel reads its DGRAD pack.  "fold": the same with AVC_F_FOLD (reflect / residual adjoint of
    the forward block, fres = its residual mode).  "s2": data gradient of a stride-2 K = 5 conv of input length T as the
    two tap-parity convs (out_tstride 2)."""
    group: str
    kind: str
    B: int
    Ci: int
    Co: int
    K: int
    T: int
    stride: int = 1
    zero_pad: bool = False
    in_tf32: bool = False
    shuffle: bool = False
    norm: bool = False
    cond: bool = False
    relu: bool = False
    res: int = 0
    fres: int = 0
    mask: bool = False

    @property
    def id(self):
        return (f"{self.kind}-B{self.B}-{self.Ci}to{self.Co}-k{self.K}-T{self.T}-s{self.stride}" + ("-zero" if self.zero_pad else "")
                + ("-tf32in" if self.in_tf32 else "") + ("-shuf" if self.shuffle else "") + ("-norm" if self.norm else "")
                + ("-cond" if self.cond else "") + ("-relu" if self.relu else "") + (f"-res{self.res}" if self.res else "")
                + (f"-fres{self.fres}" if self.kind == "fold" else "") + ("-mask" if self.mask else ""))


def cases(sms):
    """The case list for a device of `sms` SMs."""
    c = [
        # single-chunk widths, one sample per tile (inference: B = 1, one utterance)
        Case("width", "fwd", 1, 16, 128, 5, 12, relu=True),                                   # N = 16, nst = 1
        Case("width", "fwd", 1, 128, 80, 1, 32, in_tf32=True),                                 # N = 32, out_conv: partial M tile
        Case("width", "fwd", 1, 128, 128, 5, 48, stride=2, relu=True, res=2),                  # N = 48 (stride 2: 47 columns)
        Case("width", "fwd", 1, 128, 128, 5, 75, norm=True, relu=True, res=1),                 # N = 80
        Case("width", "fwd", 1, 1104, 128, 1, 90, in_tf32=True, norm=True, relu=True),         # N = 96, in_conv: short last stage
        Case("width", "fwd", 1, 128, 256, 5, 100, in_tf32=True, shuffle=True, norm=True, cond=True, relu=True, res=3),  # N = 112
        Case("width", "fwd", 1, 80, 128, 8, 128, relu=True),                                  # N = 128, bank conv: short last stage
        Case("width", "fwd", 1, 128, 128, 3, 141, zero_pad=True, in_tf32=True, relu=True),      # N = 144, patch off
        # stacked samples
        Case("stacked", "fwd", 8 * sms, 16, 128, 5, 16, relu=True),                            # N = 160: G = 8, one round
        Case("stacked", "fwd", 8 * sms - 5, 32, 128, 3, 16, in_tf32=True, norm=True, cond=True, relu=True, res=1),  # ragged tail
        Case("stacked", "fwd", 2 * sms + 3, 64, 128, 5, 32, in_tf32=True, norm=True, relu=True, res=1),
        Case("stacked", "fwd", sms + 5, 16, 128, 5, 128, norm=True, relu=True, res=1),          # one sample per tile: tiles wrap
        Case("stacked", "fwd", 3 * sms + 1, 32, 256, 5, 16, in_tf32=True, shuffle=True, norm=True, cond=True, relu=True, res=3),
        Case("stacked", "fwd", sms + 7, 64, 128, 5, 64, stride=2, norm=True, relu=True, res=2),
        # time-tiled long samples (no InstanceNorm)
        Case("time-tiled", "fwd", 2, 32, 128, 8, 300, relu=True),                              # hs = 1, ragged last time tile
        Case("time-tiled", "fwd", 1, 128, 128, 5, 600, stride=2, in_tf32=True, relu=True, res=2),
        Case("time-tiled", "fwd", 1, 128, 80, 1, 333, in_tf32=True),
        # data gradients
        Case("dgrad", "dgrad", 2, 128, 1104, 1, 64, mask=True),                                # in_conv -> bank: 9 M tiles
        Case("dgrad", "dgrad", 3, 128, 128, 5, 120, in_tf32=True),
        Case("dgrad", "s2", 5, 128, 128, 5, 128, in_tf32=True),
        Case("dgrad", "s2", sms + 9, 128, 128, 5, 32, in_tf32=True),
        Case("dgrad", "s2", 2, 128, 128, 5, 400, in_tf32=True),                                # Lp = 404: time-tiled
        Case("dgrad", "s2", 1, 128, 128, 5, 507),
        # folded data gradients
        Case("fold", "fold", 3 * sms + 2, 128, 128, 5, 16, in_tf32=True, fres=1),
        Case("fold", "fold", 7, 128, 128, 5, 37, fres=2),
        Case("fold", "fold", 5, 128, 128, 3, 64, in_tf32=True, fres=3),
        Case("fold", "fold", 3, 128, 128, 8, 96, in_tf32=True, fres=0),
    ]
    # chunked folded samples: Lp = T + K - 1 just above each 16-column boundary of the last chunk (NL = 32 .. 128), and
    # one at the tensor-map limit Lp + K - 1 == 256
    for i, lp in enumerate([145, 161, 177, 193, 209, 225, 241]):
        c.append(Case("fold chunked", "fold", 2, 128, 128, 5, lp - 4, in_tf32=(i % 2 == 0), fres=i % 4))
    c.append(Case("fold chunked", "fold", 2, 128, 128, 5, 248, in_tf32=True, fres=1))
    c.append(Case("fold chunked", "fold", 2, 128, 128, 8, 242, fres=3))
    return c


def geometry(case):
    """[(desc fields, par)] of the launches of a case: par is the output parity of an "s2" launch, else None."""
    K, T = case.K, case.T
    pl, pr = K // 2, K // 2 - (1 if K % 2 == 0 else 0)
    if case.kind == "fwd":
        Tout = (T + pl + pr - K) // case.stride + 1
        return [(dict(K=K, stride=case.stride, pad_left=pl, zero=case.zero_pad, Tin=T, Tout=Tout), None)]
    if case.kind in ("dgrad", "fold"):
        return [(dict(K=K, stride=1, pad_left=K - 1, zero=True, Tin=T, Tout=T + K - 1, fpl=pl, fpr=pr), None)]
    assert case.kind == "s2" and K == 5
    Tdc, Lp = (T - 1) // 2 + 1, T + 4
    return [(dict(K=kk, stride=1, pad_left=pl_, zero=True, Tin=Tdc, Tout=(Lp + 1 - par) // 2, out_T=Lp), par)
            for par, kk, pl_ in ((0, 3, 2), (1, 2, 1))]


def out_shape(case):
    """(channels, time) of the tensor the kernel writes to `out`."""
    g = geometry(case)[0][0]
    if case.kind == "fwd":
        return (case.Co // 2, 2 * g["Tout"]) if case.shuffle else (case.Co, g["Tout"])
    if case.kind == "fold":
        return case.Co, case.T
    if case.kind == "s2":
        return case.Co, case.T + 4
    return case.Co, g["Tout"]


def res_len(case):
    """time steps of the residual input: the forward block's residual (res) or the gradient it receives (fold)."""
    if case.kind == "fwd":
        Tn = out_shape(case)[1]
        return {0: 0, 1: Tn, 2: case.T, 3: Tn // 2}[case.res]
    if case.kind == "fold":
        return {0: 0, 1: case.T, 2: (case.T + 1) // 2, 3: 2 * case.T}[case.fres]
    return 0


def make_desc(case, g, par, ptr):
    """The descriptor of one launch; ptr maps a tensor name to its device address (stand-ins on the CPU)."""
    from adaptive_voice_conversion_b200 import _lib as L
    d = L.ConvDesc()
    d.B, d.Cin, d.Cout, d.K, d.stride = case.B, case.Ci, case.Co, g["K"], g["stride"]
    d.pad_left, d.pad_mode, d.in_ups, d.Tin, d.Tout = g["pad_left"], L.PAD_ZERO if g["zero"] else L.PAD_REFLECT, 1, g["Tin"], g["Tout"]
    d.in_, d.in_bstride = ptr["x"], case.Ci * g["Tin"]
    d.w_tc = ptr["w_even" if par == 0 else "w_odd" if par == 1 else "w"]
    Cn, Tn = out_shape(case)
    d.out, d.out_bstride = ptr["out"], Cn * Tn
    d.eps = 1e-5
    d.flags = L.F_IN_TF32 if case.in_tf32 else 0
    if case.kind == "fwd":
        d.bias = ptr["bias"]
        d.shuffle, d.norm, d.relu = int(case.shuffle), int(case.norm), int(case.relu)
        d.save_c = ptr["c"]
        d.stats = ptr["stats"] if case.norm else None
        if case.cond:
            d.cond, d.cond_bstride = ptr["cond"], 2 * Cn
        if case.res:
            d.res, d.res_bstride, d.res_mode, d.res_T = ptr["res"], Cn * res_len(case), case.res, res_len(case)
    elif case.kind == "fold":
        d.flags = int(d.flags) | L.F_FOLD | (g["fpl"] << 8) | (g["fpr"] << 16)
        d.out_T = case.T
        if case.fres:
            d.res, d.res_bstride, d.res_mode, d.res_T = ptr["res"], case.Co * res_len(case), case.fres, res_len(case)
    elif case.kind == "s2":
        d.out_tstride, d.out_toff, d.out_T = 2, par, g["out_T"]
    if case.mask:
        d.mask, d.mask_bstride = ptr["mask"], Cn * Tn
    return d


def features(case, g, par, plan, sms):
    """The plan features (FEATURES) one launch exercises."""
    nl = plan.N_last if plan.nchunk > 1 else plan.N
    f = {("instance", plan.N, nl), ("hs", plan.hs)}
    if (case.Ci // 8) % plan.hs:
        f.add("short last stage")
    if plan.nst == 1:
        f.add("nst == 1")
    if plan.nst < plan.nstage:
        f.add("nst < nstage")
    if plan.ntiles > sms:
        f.add("tiles wrap the CTAs")
    if plan.G > 1 and case.B % plan.G:
        f.add("G > 1, ragged batch tail")
    if case.Co % 128:
        f.add("partial M tile")
        if plan.mtiles > 1 and case.kind != "fwd":
            f.add("mtiles > 1, partial last M tile (data gradient)")
    if plan.ntt > 1 and g["Tout"] % plan.TT:
        f.add("ntt > 1, ragged last time tile")
    if not plan.patch:
        f.add("patch: off")
    elif case.in_tf32:
        f.add("patch: reflect rows only")
    else:
        f.add("patch: rounding")
    if case.kind == "fwd" and case.stride == 2:
        f.add("forward stride 2")
    if case.kind == "s2":
        f.add("stride-2 parity data gradient")
        if plan.ntt > 1:
            f.add("stride-2 parity data gradient, time-tiled")
    if case.kind == "fold":
        f.add(f"fold, residual {case.fres}")
        if g["Tout"] + g["K"] - 1 == 256:
            f.add("fold at Lp + K - 1 == 256")
    if case.shuffle and case.cond:
        f.add("pixel shuffle + AdaIN")
    return f


def plan_of(lib, d, sms):
    from adaptive_voice_conversion_b200 import _lib as L
    p = L.TcPlan()
    rc = lib.avc_conv_block_tc_plan(C.byref(d), sms, C.byref(p))
    return rc, p


# ------------------------------------------------------------------ reference (float64 on the CPU)
def tf32(x):
    """cvt.rna.tf32.f32: round the fp32 bit pattern to nearest (ties away from zero) at 10 mantissa bits."""
    b = x.contiguous().view(torch.int32)
    return ((b + 0x1000) & -0x2000).view(torch.float32)


def reference(case, x, w, bias, cond, res, mask):
    """-> (out, raw conv + bias or None) in float64.  x, w: the fp32 tensors the kernel reads (before its rounding)."""
    xr, wr = tf32(x).double(), tf32(w).double()
    if case.kind == "fwd":
        g = geometry(case)[0][0]
        K, pl = case.K, g["pad_left"]
        pr = K // 2 - (1 if K % 2 == 0 else 0)
        xp = F.pad(xr, (pl, pr)) if case.zero_pad else F.pad(xr, (pl, pr), mode="reflect")
        c = F.conv1d(xp, wr, bias.double(), stride=case.stride)
        y = c
        if case.shuffle:
            b_, ch, t = y.shape
            y = y.reshape(b_, ch // 2, 2, t).transpose(2, 3).reshape(b_, ch // 2, 2 * t)
        if case.norm:
            mu = y.mean(dim=2, keepdim=True)
            y = (y - mu) / torch.sqrt(y.var(dim=2, unbiased=False, keepdim=True) + 1e-5)
        if case.cond:
            cn = y.shape[1]
            cd = cond.double()
            y = y * cd[:, cn:, None] + cd[:, :cn, None]
        if case.relu:
            y = F.relu(y)
        if case.res:
            r = res.double()
            y = y + {1: lambda: r, 2: lambda: F.avg_pool1d(r, 2, ceil_mode=True), 3: lambda: F.interpolate(r, scale_factor=2, mode="nearest")}[case.res]()
        if case.mask:
            y = y * (mask > 0)
        return y, c
    # data gradients: x is the gradient of the forward conv's output, w the forward conv's weight [Ci][Co][K]
    stride = 2 if case.kind == "s2" else 1
    Lp = case.T + case.K - 1 if case.kind != "s2" else case.T + 4
    full = F.conv_transpose1d(xr, wr, stride=stride)
    dxp = torch.zeros(case.B, case.Co, Lp, dtype=torch.float64)
    n = min(Lp, full.shape[2])
    dxp[:, :, :n] = full[:, :, :n]
    if case.kind != "fold":
        y = dxp
        if case.mask:
            y = y * (mask > 0)
        return y, None
    # adjoint of the forward block's reflect padding and of its residual branch, by autograd in float64
    K = case.K
    pl, pr = K // 2, K // 2 - (1 if K % 2 == 0 else 0)
    xi = torch.zeros(case.B, case.Co, case.T, dtype=torch.float64, requires_grad=True)
    obj = (F.pad(xi, (pl, pr), mode="reflect") * dxp).sum()
    if case.fres:
        r = res.double()
        br = {1: lambda: xi, 2: lambda: F.avg_pool1d(xi, 2, ceil_mode=True), 3: lambda: F.interpolate(xi, scale_factor=2, mode="nearest")}[case.fres]()
        obj = obj + (br * r).sum()
    obj.backward()
    return xi.grad, None


# ------------------------------------------------------------------ the GPU run
def to_a4(t):
    """planar [B][C][T] -> A4 [B][C/4][T][4] on the device, bit-exact (no rounding)."""
    B, Cc, T = t.shape
    return t.reshape(B, Cc // 4, 4, T).permute(0, 1, 3, 2).contiguous().cuda()


def from_a4(a):
    B, Q, T, _ = a.shape
    return a.cpu().permute(0, 1, 3, 2).reshape(B, 4 * Q, T)


def relerr(y, ref):
    return float((y.double() - ref).abs().max() / ref.abs().max().clamp_min(1e-30))


@pytest.fixture(scope="module")
def eng():
    import oracle.ae_oracle as orc
    from adaptive_voice_conversion_b200.engine import Engine
    e = Engine(orc.default_config(80), torch.device("cuda", 0))
    e.precision = "tf32"
    return e


def _sms():
    return torch.cuda.get_device_properties(0).multi_processor_count if torch.cuda.is_available() else 132


RESULTS = {}     # case id -> (group, plan features, {output: error})
_T0 = []


@pytest.mark.parametrize("case", cases(_sms()), ids=lambda c: c.id)
def test_tc2_exact(eng, case):
    from adaptive_voice_conversion_b200 import _lib as L
    if not _T0:
        _T0.append(time.time())
    sms = _sms()
    gen = torch.Generator().manual_seed(zlib.crc32(case.id.encode()))
    B, Ci, Co, K, T = case.B, case.Ci, case.Co, case.K, case.T
    geo = geometry(case)
    Tin = geo[0][0]["Tin"]
    x = torch.randn((B, Ci, Tin), generator=gen)
    if case.in_tf32:
        x = tf32(x)     # a rounding producer's output
    fwd = case.kind == "fwd"
    wshape = (Co, Ci, K) if fwd else (Ci, Co, K)
    w = torch.randn(wshape, generator=gen) / math.sqrt(Ci * K)
    bias = torch.randn((Co,), generator=gen) * 0.1
    Cn, Tn = out_shape(case)
    cond = (torch.randn((B, 2 * Cn), generator=gen) * 0.5 + 0.7) if case.cond else None
    rT = res_len(case)
    res = torch.randn((B, Cn if fwd else Co, rT), generator=gen) if rT else None
    mask = (torch.randn((B, Cn, Tn), generator=gen) > -0.5).float() if case.mask else None

    # weight packs exactly as the engine makes them; a stride-2 layer of the default config gets the tap-parity packs
    name = "speaker_encoder.second_conv_layers.1" if case.kind == "s2" else "blk"
    P = {name + ".weight": w.cuda(), name + ".bias": bias.cuda()}
    eng.conv_names = lambda: [name]
    eng.packed.pop(name, None)
    eng.pack_weights(P, need_dgrad=not fwd)
    pk = eng.packed[name]
    xa = to_a4(x)
    out = torch.zeros((B, Cn // 4, Tn, 4), device="cuda")
    c = torch.zeros((B, Co // 4, geo[0][0]["Tout"], 4), device="cuda") if fwd else None
    stats = torch.zeros((B, Cn, 2), device="cuda") if case.norm else None
    dev = dict(x=xa, out=out, c=c, stats=stats, bias=P[name + ".bias"], cond=cond.cuda() if cond is not None else None,
               res=to_a4(res) if res is not None else None, mask=to_a4(mask) if mask is not None else None,
               w=pk.get("fwd_tc" if fwd else "dgrad_tc"), w_even=pk.get("dgrad_tc_even"), w_odd=pk.get("dgrad_tc_odd"))
    ptr = {k: (v.data_ptr() if v is not None else None) for k, v in dev.items()}
    feats = set()
    for g, par in geo:
        d = make_desc(case, g, par, ptr)
        rc, plan = plan_of(eng.lib, d, sms)
        assert rc == 0, L.last_error()
        assert plan.instance >= 0, (plan.N, plan.N_last)
        feats |= features(case, g, par, plan, sms)
        eng._ck(eng.lib.avc_conv_block_tc(C.byref(d), eng.tc_status.data_ptr(), eng.stream), f"conv_block_tc[{case.id}]")
        eng.check_tc_status()
    y_ref, c_ref = reference(case, x, w, bias, cond, res, mask)
    errs = {"out": relerr(from_a4(out), y_ref)}
    if c_ref is not None:
        errs["c"] = relerr(from_a4(c), c_ref)
    RESULTS[case.id] = (case.group, feats, errs)
    for k, e in errs.items():
        assert e < TOL, f"{k}: max error {e:.3e} of the reference max (tolerance {TOL:.0e})"


def test_plan_and_launch_reject_alike(eng):
    """A descriptor the plan query rejects is rejected by the launch with the same code and message."""
    from adaptive_voice_conversion_b200 import _lib as L
    case = Case("reject", "fwd", 2, 128, 128, 5, 200, norm=True)      # InstanceNorm over a sample that needs time tiles
    g, par = geometry(case)[0]
    t = torch.zeros(4 << 20, device="cuda")
    d = make_desc(case, g, par, {k: t.data_ptr() for k in ("x", "out", "c", "stats", "bias", "w")} | {"cond": None, "res": None, "mask": None})
    rc, _ = plan_of(eng.lib, d, _sms())
    msg = L.last_error()
    assert rc == L.ERR_UNSUPPORTED and "time tiles" in msg
    assert eng.lib.avc_conv_block_tc(C.byref(d), eng.tc_status.data_ptr(), eng.stream) == rc and L.last_error() == msg


def test_tc2_exact_coverage():
    """The recorded plans reach every kernel instance and every feature; reports the worst error per group."""
    all_ids = [c.id for c in cases(_sms())]
    if any(i not in RESULTS for i in all_ids):
        pytest.skip("only part of the module ran")
    worst = {}
    covered = set()
    for grp, feats, errs in RESULTS.values():
        covered |= feats
        worst[grp] = max(worst.get(grp, 0.0), *errs.values())
    print(f"\ntc2 exact: {len(all_ids)} cases in {time.time() - _T0[0]:.1f} s; worst error per group (tolerance {TOL:.0e}): "
          + ", ".join(f"{g} {e:.2e}" for g, e in sorted(worst.items())))
    for cid in all_ids:
        print(f"  {cid}: " + ", ".join(f"{k} {e:.2e}" for k, e in RESULTS[cid][2].items()))
    missing = [f for f in FEATURES if f not in covered]
    assert not missing, missing
