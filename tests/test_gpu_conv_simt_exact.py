"""GPU: the exact-fp32 FFMA conv-block kernel (conv_block_fwd_kernel, csrc/conv_simt.cu) against a float64 reference
computed on the SAME fp32 operands.

The kernel multiplies the fp32 operands as stored (no rounding), so the reference convolves, normalises, adds the
residual ... in float64 on the CPU from exactly the values the kernel reads; what is left of the difference is the
kernel's fp32 accumulation and epilogue.  Weights come from the engine's own FFMA packs (avc_pack_conv_weight); the first
test checks those packs bit for bit against the permutations of include/avc_b200.h, for the single-layer and the batched
pack kernel.

Every case is driven through avc_conv_block_fwd with a hand-built descriptor.  Before the launch the plan query
(avc_conv_block_fwd_plan) reports the tile plan the launch uses; the coverage test asserts that the union of those plans
reaches every kernel instance and every entry of FEATURES (tests/test_conv_simt_plan.py checks the same on the CPU, and
that the plans the engine's own launches reach are a subset of the case list's).

Error measures, per case:
* `c` (raw conv + bias) and unnormalised `out`: max over elements of |kernel - ref| / (sum |w||x| + |bias|), the sum
  over the same gather and carried through the epilogue with absolute values (|gamma|, |beta|, |residual|), so that
  cancellation in a reference entry cannot hide an error; max |kernel - ref| / max |ref| is reported beside it;
* normalised `out`: max |kernel - ref| / max |ref|;
* `stats`: max of |mean error| * rstd (the shift of the normalised output) and |rstd error| / rstd;
* AVC_F_ROUND_OUT: `out` must be TF32-exact (low 13 bits zero), and its error is measured after taking off half a TF32
  ulp of the reference (2^-11 |ref|).
NaN fills every sample-stride gap of in / res / mask (and the other channels of a strided `in`); a sentinel surrounds
`out` (and the other channels of a strided `out`), `c` and `stats`, and must survive the launch.

Worst measured on 1x NVIDIA H100 80GB HBM3 (132 SMs, 700 W power limit), per measure and group of cases:
    bound (c, unnormalised out, data gradients): bank 2.9e-7, packed 2.9e-7, tile 256 2.9e-7, tiled 3.2e-7,
        misc 2.5e-7, dgrad 3.2e-7 (max-relative beside it at most 1.5e-6);
    normalised out: packed 1.2e-6, tile 256 1.3e-6, misc 9.9e-8;
    stats: packed 2.4e-6 (InstanceNorm over 5 steps), tile 256 3.0e-7, misc 3.0e-7.
TOL is about 3-4x the worst of each measure.  For scale, mutations of the kernel (scratch copies, never committed) each
fail cases of this module, the smallest failing error far above TOL:
    tap K - 1 dropped from the FMA loop: 66 of 66 cases fail, from 0.28;
    every segment after the first staged 4 floats late (s * segp + 4): 16 cases (every packed plan), from 1.2;
    the last step (o = nlanes / 2) of the Welford shuffle skipped: 14 cases (every norm with seg_out >= 16), from 0.13;
    the 4-channel half stage of Cin % 8 == 4 skipped: 2 cases (both Cin % 8 == 4 cases), from 0.29;
    the input of every time tile after the first staged one step late: 12 cases (every time-tiled plan), from 1.2.
The module takes about 3 s on that GPU (the float64 reference on the CPU included).
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

TOL = {"bound": 1e-6, "norm": 5e-6, "stats": 8e-6}
GAP = 36               # floats of NaN after every sample of in / res / mask
GUARD = 1024           # floats of sentinel after out, c and stats
SENTINEL = -1.5e30
HALF_TF32_ULP = 2.0 ** -11


@dataclass(frozen=True)
class Case:
    """One launch.  Channel counts are the KERNEL's: Ci input, Co output channels.
    kind "fwd": conv block, nn.Conv1d weight [Co][Ci][K], FWD pack, input length T, conv stride `stride`.
    kind "dgrad": data gradient of a conv of input length T, kernel K, stride `stride` (the launch's in_ups) whose weight
    is [Ci][wld or Co][K]: zero padding K - 1, DGRAD pack; w_ld = wld > Co computes the first Co channels only."""
    group: str
    kind: str
    B: int
    Ci: int
    Co: int
    K: int
    T: int
    stride: int = 1
    zero_pad: bool = False
    shuffle: bool = False
    norm: bool = False
    cond: bool = False
    relu: bool = False
    res: int = 0
    res_odd: bool = False   # residual 2: res_T = 2 Tn - 1 (avg_pool's lone last element)
    mask: bool = False
    round_out: bool = False
    in_tf32: bool = False   # AVC_F_IN_TF32 set (a hint the FFMA kernel ignores); operands are still raw fp32
    wld: int = 0
    in_wide: int = 0        # 4-channel chunks of a wider tensor before and after `in` (strided in)
    out_wide: int = 0       # ... before and after `out` (strided out: the conv-bank concat)

    @property
    def id(self):
        return (f"{self.kind}-B{self.B}-{self.Ci}to{self.Co}-k{self.K}-T{self.T}-s{self.stride}" + ("-zero" if self.zero_pad else "")
                + ("-shuf" if self.shuffle else "") + ("-norm" if self.norm else "") + ("-cond" if self.cond else "")
                + ("-relu" if self.relu else "") + (f"-res{self.res}" if self.res else "") + ("odd" if self.res_odd else "")
                + ("-mask" if self.mask else "") + ("-round" if self.round_out else "") + ("-tf32in" if self.in_tf32 else "")
                + (f"-ld{self.wld}" if self.wld else "") + (f"-inw{self.in_wide}" if self.in_wide else "")
                + (f"-outw{self.out_wide}" if self.out_wide else ""))


def _pads(K):
    return K // 2, K // 2 - (1 if K % 2 == 0 else 0)


def geometry(case):
    """Descriptor fields of the launch: K, stride, pad_left, pad_mode zero?, in_ups, Tin, Tout."""
    K, T, S = case.K, case.T, case.stride
    pl, pr = _pads(K)
    Tconv = (T + pl + pr - K) // S + 1
    if case.kind == "fwd":
        return dict(stride=S, pad_left=pl, zero=case.zero_pad, in_ups=1, Tin=T, Tout=Tconv)
    return dict(stride=1, pad_left=K - 1, zero=True, in_ups=S, Tin=Tconv, Tout=T + pl + pr)


def out_shape(case):
    Tout = geometry(case)["Tout"]
    return (case.Co // 2, 2 * Tout) if case.shuffle else (case.Co, Tout)


def res_len(case):
    Tn = out_shape(case)[1]
    return {0: 0, 1: Tn, 2: 2 * Tn - (1 if case.res_odd else 0), 3: Tn // 2}[case.res]


def in_bstride(case):
    g = geometry(case)
    return case.Ci * g["Tin"] + 2 * case.in_wide * 4 * g["Tin"] + GAP


def out_bstride(case):
    Cn, Tn = out_shape(case)
    return Cn * Tn + 2 * case.out_wide * 4 * Tn


def make_desc(case, ptr):
    """The descriptor of the launch; ptr maps a tensor name to its device address (stand-ins on the CPU)."""
    from adaptive_voice_conversion_b200 import _lib as L
    g = geometry(case)
    Cn, Tn = out_shape(case)
    d = L.ConvDesc()
    d.B, d.Cin, d.Cout, d.K, d.stride = case.B, case.Ci, case.Co, case.K, g["stride"]
    d.pad_left, d.pad_mode, d.in_ups, d.Tin, d.Tout = g["pad_left"], L.PAD_ZERO if g["zero"] else L.PAD_REFLECT, g["in_ups"], g["Tin"], g["Tout"]
    d.in_, d.in_bstride = ptr["x"], in_bstride(case)
    d.w_packed, d.w_ld = ptr["w"], case.wld or case.Co
    d.out, d.out_bstride = ptr["out"], out_bstride(case)
    d.eps = 1e-5
    d.flags = (L.F_ROUND_OUT if case.round_out else 0) | (L.F_IN_TF32 if case.in_tf32 else 0)
    if case.kind == "fwd":
        d.bias, d.save_c = ptr["bias"], ptr["c"]
        d.shuffle, d.norm, d.relu = int(case.shuffle), int(case.norm), int(case.relu)
        d.stats = ptr["stats"] if case.norm else None
        if case.cond:
            d.cond, d.cond_bstride = ptr["cond"], 2 * Cn
        if case.res:
            d.res, d.res_bstride, d.res_mode, d.res_T = ptr["res"], Cn * res_len(case) + GAP, case.res, res_len(case)
    if case.mask:
        d.mask, d.mask_bstride = ptr["mask"], Cn * Tn + GAP
    return d


def plan_of(lib, d):
    from adaptive_voice_conversion_b200 import _lib as L
    p = L.SimtPlan()
    rc = lib.avc_conv_block_fwd_plan(C.byref(d), C.byref(p))
    return rc, p


# ------------------------------------------------------------------ plan features
INSTANCES = list(range(12))
FEATURES = ([("instance", i) for i in INSTANCES]
            + [("seg_out", s, "B % nseg != 0") for s in (8, 16, 32, 64)] + [("seg_out", 128), "packed tile, B = 1"]
            + [("tile 256", 1, 1), ("tile 256", 5, 1), ("tile 256", 5, 2), "tile 256: shuffle + AdaIN + residual 3"]
            + [("tiled, ragged last tile", 8, 1), ("tiled, ragged last tile", 5, 1), ("tiled, ragged last tile", 5, 2)]
            + ["dgrad, in_ups 1", "dgrad, in_ups 2, tiled", "dgrad, w_ld > Cout, mask", ("partial Cout tile", 128),
               ("partial Cout tile", 64), "Cin % 8 == 4", "strided in", "strided out", "zero-padded forward",
               "residual 1", "residual 2", "residual 2, odd res_T", "residual 3", "round out", "pixel shuffle", "AdaIN",
               "stats", "mask"])


def launch_kind(d):
    """'fwd', or 'dgrad ups N' for a data gradient (zero padding K - 1, no bias) -- how the engine builds them."""
    from adaptive_voice_conversion_b200 import _lib as L
    if d.pad_mode == L.PAD_ZERO and d.pad_left == d.K - 1 and not d.bias:
        return f"dgrad ups {d.in_ups}"
    return "fwd"


def launch_keys(d, p):
    """The features one launch exercises: FEATURES entries, plus (instance, tile plan) and (instance, kind) pairs."""
    from adaptive_voice_conversion_b200 import _lib as L
    inst, kind = p.instance, launch_kind(d)
    plan = "tiled" if p.tiled else f"seg {p.seg_out}"
    f = {("instance", inst), ("instance", inst, plan), ("instance", inst, kind)}
    if p.tiled:
        if d.Tout % p.TT:
            f.add(("tiled, ragged last tile", d.K, d.stride if kind == "fwd" else d.in_ups))
    elif p.nseg == 1:
        f.add(("seg_out", p.seg_out))
    else:
        if d.B % p.nseg:
            f.add(("seg_out", p.seg_out, "B % nseg != 0"))
        if d.B == 1:
            f.add("packed tile, B = 1")
    if p.TT == 256:
        f.add(("tile 256", d.K, d.stride))
        if d.shuffle and d.cond and d.res_mode == L.RES_UP and d.res:
            f.add("tile 256: shuffle + AdaIN + residual 3")
    if kind.startswith("dgrad"):
        if d.in_ups == 1:
            f.add("dgrad, in_ups 1")
        elif p.tiled:
            f.add("dgrad, in_ups 2, tiled")
        if d.w_ld > d.Cout and d.mask:
            f.add("dgrad, w_ld > Cout, mask")
    elif d.pad_mode == L.PAD_ZERO:
        f.add("zero-padded forward")
    if d.Cout % p.TCO:
        f.add(("partial Cout tile", p.TCO))
    if d.Cin % 8 == 4:
        f.add("Cin % 8 == 4")
    Cn, Tn = (d.Cout // 2, 2 * d.Tout) if d.shuffle else (d.Cout, d.Tout)
    if d.in_bstride >= (d.Cin + 4) * d.Tin:
        f.add("strided in")
    if d.out_bstride > Cn * Tn:
        f.add("strided out")
    if d.res:
        f.add(f"residual {d.res_mode}")
        if d.res_mode == L.RES_POOL and d.res_T % 2:
            f.add("residual 2, odd res_T")
    for flag, name in ((d.flags & L.F_ROUND_OUT, "round out"), (d.shuffle, "pixel shuffle"), (d.cond, "AdaIN"),
                       (d.stats, "stats"), (d.mask, "mask"), (d.norm, "norm"), (d.relu, "relu"), (d.save_c, "save_c")):
        if flag:
            f.add(name)
    return f


# ------------------------------------------------------------------ the case list
def bank_cases():
    """The conv bank (80 -> 128, K = 1..8, ReLU) reading its input from, and writing its output into, a wider tensor,
    at one utterance of 16, 40, 128 and 300 frames: packed, single-sample and time-tiled plans of every K."""
    return [Case("bank", "fwd", 1, 80, 128, k, t, relu=True, in_wide=1, out_wide=2) for k in range(1, 9) for t in (16, 40, 128, 300)]


CASES = bank_cases() + [
    # packed tiles: nseg samples of seg_out columns per CTA, ragged batch tails
    Case("packed", "fwd", 21, 32, 128, 5, 7, norm=True, relu=True, res=1),                  # seg_out 8, nseg 16
    Case("packed", "fwd", 1, 64, 128, 5, 8, norm=True, relu=True),                          # seg_out 8, B = 1
    Case("packed", "fwd", 13, 64, 128, 5, 16, norm=True, relu=True, res=1),                 # seg_out 16
    Case("packed", "fwd", 7, 128, 128, 5, 32, stride=2, relu=True, res=2),                  # seg_out 16, stride 2
    Case("packed", "fwd", 6, 128, 128, 5, 29, norm=True, relu=True),                        # seg_out 32
    Case("packed", "fwd", 5, 128, 128, 5, 33, stride=2, norm=True, relu=True, res=2, res_odd=True),  # seg_out 32, res_T 33
    Case("packed", "fwd", 3, 128, 128, 3, 64, relu=True),                                   # seg_out 64
    Case("packed", "fwd", 5, 128, 128, 5, 128, stride=2, norm=True, relu=True, res=2),      # seg_out 64, stride 2
    Case("packed", "fwd", 5, 128, 256, 5, 16, shuffle=True, norm=True, cond=True, relu=True, res=3),  # decoder upsampling
    Case("packed", "fwd", 1, 128, 128, 5, 10, stride=2, norm=True, relu=True, res=2),       # seg_out 8, stride 2
    Case("packed", "fwd", 3, 128, 128, 5, 250, stride=2, norm=True, relu=True, res=2),      # seg_out 128, stride 2
    Case("packed", "fwd", 1, 128, 128, 1, 5),                                               # mean / std heads: seg_out 8
    Case("packed", "fwd", 5, 128, 128, 1, 25, relu=True),                                   # seg_out 32, K = 1
    Case("packed", "fwd", 3, 128, 128, 5, 100, norm=True, cond=True, relu=True, res=1),     # seg_out 128
    Case("packed", "fwd", 3, 128, 80, 1, 100),                                              # out_conv: partial Cout tile
    Case("packed", "fwd", 4, 1104, 128, 1, 64, norm=True, relu=True),                       # in_conv
    # the 256-column tile (InstanceNorm over 129..256 steps)
    Case("tile 256", "fwd", 2, 1104, 128, 1, 200, norm=True, relu=True),                    # in_conv
    Case("tile 256", "fwd", 2, 128, 128, 5, 256, norm=True, relu=True, res=1),
    Case("tile 256", "fwd", 3, 128, 128, 5, 301, stride=2, norm=True, relu=True, res=2, res_odd=True),  # Tout 151
    Case("tile 256", "fwd", 2, 128, 256, 5, 150, shuffle=True, norm=True, cond=True, relu=True, res=3),  # Tn 300
    Case("tile 256", "fwd", 2, 128, 96, 5, 140, norm=True, relu=True),                      # partial Cout tile of 64
    # time-tiled samples (no InstanceNorm)
    Case("tiled", "fwd", 2, 80, 128, 8, 300, relu=True, in_wide=2, out_wide=1),
    Case("tiled", "fwd", 1, 128, 128, 5, 333),                                              # plain conv before avc_norm_apply_fwd
    Case("tiled", "fwd", 2, 128, 128, 5, 601, stride=2, relu=True, res=2, res_odd=True),    # Tout 301
    # layouts, padding, rounding
    Case("misc", "fwd", 3, 84, 128, 5, 40, relu=True),                                      # Cin % 8 == 4
    Case("misc", "fwd", 2, 36, 128, 3, 50, zero_pad=True, relu=True, in_wide=1),            # zero padding, Cin % 8 == 4
    Case("misc", "fwd", 4, 128, 128, 3, 48, relu=True, round_out=True),
    Case("misc", "fwd", 3, 128, 128, 5, 60, norm=True, relu=True, res=1, round_out=True, mask=True),
    # data gradients
    Case("dgrad", "dgrad", 3, 128, 128, 5, 64),                                             # Lp 68
    Case("dgrad", "dgrad", 5, 128, 128, 5, 29),                                             # Lp 33: seg_out 64, ragged
    Case("dgrad", "dgrad", 3, 128, 128, 5, 64, stride=2),                                   # in_ups 2, Lp 68
    Case("dgrad", "dgrad", 2, 128, 128, 5, 300, stride=2, in_tf32=True),                    # in_ups 2, Lp 304: time-tiled
    Case("dgrad", "dgrad", 2, 128, 1024, 1, 64, mask=True, wld=1104),                       # in_conv -> bank channels
    Case("dgrad", "dgrad", 3, 80, 128, 1, 128),                                             # out_conv
]


# ------------------------------------------------------------------ reference (float64 on the CPU)
def _shuffle(y):
    b_, ch, t = y.shape
    return y.reshape(b_, ch // 2, 2, t).transpose(2, 3).reshape(b_, ch // 2, 2 * t)


def _res_term(case, r, Tn):
    if case.res == 1:
        return r
    if case.res == 3:
        return r[:, :, torch.arange(Tn) // 2]
    i = torch.arange(Tn)
    a, b = r[:, :, 2 * i], r[:, :, (2 * i + 1).clamp(max=r.shape[2] - 1)]
    lone = (2 * i + 1 >= r.shape[2])
    return torch.where(lone, a, 0.5 * (a + b))


def reference(case, x, w, bias, cond, res, mask):
    """float64: out, its bound (None when normalised), c and its bound, mean, rstd.  x, w: the fp32 operands."""
    xd, wd = x.double(), w.double()
    Cn, Tn = out_shape(case)
    if case.kind == "dgrad":
        wt = wd[:, :case.Co]
        Lp = geometry(case)["Tout"]
        full = F.conv_transpose1d(xd, wt, stride=case.stride)
        fullb = F.conv_transpose1d(xd.abs(), wt.abs(), stride=case.stride)
        n = min(Lp, full.shape[2])
        y, yb = torch.zeros(case.B, case.Co, Lp, dtype=torch.float64), torch.zeros(case.B, case.Co, Lp, dtype=torch.float64)
        y[:, :, :n], yb[:, :, :n] = full[:, :, :n], fullb[:, :, :n]
        if case.mask:
            y, yb = y * (mask > 0), yb * (mask > 0)
        return dict(out=y, out_bound=yb)
    pl, pr = _pads(case.K)
    xp = F.pad(xd, (pl, pr)) if case.zero_pad else F.pad(xd, (pl, pr), mode="reflect")
    bd = bias.double()
    c = F.conv1d(xp, wd, bd, stride=case.stride)
    cb = F.conv1d(xp.abs(), wd.abs(), bd.abs(), stride=case.stride)
    y, yb = (_shuffle(c), _shuffle(cb)) if case.shuffle else (c, cb)
    r = dict(c=c, c_bound=cb)
    if case.norm:
        mu = y.mean(dim=2, keepdim=True)
        rstd = 1.0 / torch.sqrt(((y - mu) ** 2).mean(dim=2, keepdim=True) + 1e-5)
        y, yb = (y - mu) * rstd, None
        r["mean"], r["rstd"] = mu[:, :, 0], rstd[:, :, 0]
    if case.cond:
        cd = cond.double()
        y = y * cd[:, Cn:, None] + cd[:, :Cn, None]
        if yb is not None:
            yb = yb * cd[:, Cn:, None].abs() + cd[:, :Cn, None].abs()
    if case.relu:
        y = F.relu(y)
    if case.res:
        rt = _res_term(case, res.double(), Tn)
        y = y + rt
        if yb is not None:
            yb = yb + rt.abs()
    if case.mask:
        y = y * (mask > 0)
        if yb is not None:
            yb = yb * (mask > 0)
    r["out"], r["out_bound"] = y, yb
    return r


# ------------------------------------------------------------------ device buffers
def a4_rows(t, wide, gap, fill):
    """planar [B][C][T] -> A4 rows of a device buffer: per sample `wide` 4-channel chunks of `fill`, the tensor, `wide`
    chunks and `gap` floats of `fill`; GUARD floats of `fill` after the last sample.  -> (buffer, address, bstride)."""
    B, Cc, T = t.shape
    lead = wide * 4 * T
    bstride = Cc * T + 2 * lead + gap
    buf = torch.full((B * bstride + GUARD,), fill, device="cuda")
    rows = buf[:B * bstride].view(B, bstride)
    rows[:, lead:lead + Cc * T] = t.reshape(B, Cc // 4, 4, T).permute(0, 1, 3, 2).reshape(B, Cc * T).cuda()
    return buf, buf.data_ptr() + 4 * lead, bstride


def a4_read(buf, B, Cc, T, wide, gap):
    """-> (planar [B][C][T] on the CPU, everything else of the buffer)."""
    lead = wide * 4 * T
    bstride = Cc * T + 2 * lead + gap
    h = buf.cpu()
    rows = h[:B * bstride].view(B, bstride)
    y = rows[:, lead:lead + Cc * T].reshape(B, Cc // 4, T, 4).permute(0, 1, 3, 2).reshape(B, Cc, T)
    rest = torch.cat([rows[:, :lead].reshape(-1), rows[:, lead + Cc * T:].reshape(-1), h[B * bstride:]])
    return y, rest


def sentinel_intact(rest):
    return bool((rest.view(torch.int32) == torch.tensor([SENTINEL]).view(torch.int32)).all())


def pack(lib, w, mode):
    """The engine's FFMA pack of an nn.Conv1d weight [Cout][Cin][K] (w on the device)."""
    from adaptive_voice_conversion_b200 import _lib as L
    p = torch.empty(w.numel(), device="cuda")
    Co, Ci, K = w.shape
    rc = lib.avc_pack_conv_weight(w.data_ptr(), p.data_ptr(), Co, Ci, K, mode, torch.cuda.current_stream().cuda_stream)
    assert rc == 0, L.last_error()
    return p


def operands(case):
    """The case's fp32 operands on the CPU, seeded by its id."""
    gen = torch.Generator().manual_seed(zlib.crc32(case.id.encode()))
    g = geometry(case)
    Cn, Tn = out_shape(case)
    x = torch.randn((case.B, case.Ci, g["Tin"]), generator=gen)
    wshape = (case.Co, case.Ci, case.K) if case.kind == "fwd" else (case.Ci, case.wld or case.Co, case.K)
    w = torch.randn(wshape, generator=gen) / math.sqrt(case.Ci * case.K)
    bias = torch.randn((case.Co,), generator=gen) * 0.1
    cond = (torch.randn((case.B, 2 * Cn), generator=gen) * 0.5 + 0.7) if case.cond else None
    res = torch.randn((case.B, Cn, res_len(case)), generator=gen) if case.res else None
    mask = (torch.randn((case.B, Cn, Tn), generator=gen) > -0.5).float() if case.mask else None
    return x, w, bias, cond, res, mask


def run_case(lib, case, x, w, bias, cond, res, mask):
    """Launch the case on the device -> dict of planar CPU outputs, and whether every guard survived."""
    from adaptive_voice_conversion_b200 import _lib as L
    g = geometry(case)
    Cn, Tn = out_shape(case)
    xbuf, xptr, _ = a4_rows(x, case.in_wide, GAP, float("nan"))
    wdev = w.cuda()
    wp = pack(lib, wdev, L.PACK_FWD if case.kind == "fwd" else L.PACK_DGRAD)
    obuf, optr, _ = a4_rows(torch.zeros(case.B, Cn, Tn), case.out_wide, 0, SENTINEL)
    obuf[:] = SENTINEL
    dev = dict(x=xptr, w=wp.data_ptr(), out=optr)
    keep = [xbuf, wdev, wp, obuf]
    if case.kind == "fwd":
        cbuf = torch.full((case.B * case.Co * g["Tout"] + GUARD,), SENTINEL, device="cuda")
        sbuf = torch.full((case.B * Cn * 2 + GUARD,), SENTINEL, device="cuda")
        bd = bias.cuda()
        dev.update(c=cbuf.data_ptr(), stats=sbuf.data_ptr(), bias=bd.data_ptr())
        keep += [cbuf, sbuf, bd]
        if case.cond:
            cdev = cond.cuda()
            dev["cond"] = cdev.data_ptr()
            keep.append(cdev)
        if case.res:
            rbuf, dev["res"], _ = a4_rows(res, 0, GAP, float("nan"))
            keep.append(rbuf)
    if case.mask:
        mbuf, dev["mask"], _ = a4_rows(mask, 0, GAP, float("nan"))
        keep.append(mbuf)
    d = make_desc(case, dev)
    rc, plan = plan_of(lib, d)
    assert rc == 0, L.last_error()
    rc = lib.avc_conv_block_fwd(C.byref(d), torch.cuda.current_stream().cuda_stream)
    assert rc == 0, L.last_error()
    torch.cuda.synchronize()
    out = {}
    out["out"], rest = a4_read(obuf, case.B, Cn, Tn, case.out_wide, 0)
    intact = sentinel_intact(rest)
    if case.kind == "fwd":
        n = case.B * case.Co * g["Tout"]
        cb = cbuf.cpu()
        out["c"] = cb[:n].view(case.B, case.Co // 4, g["Tout"], 4).permute(0, 1, 3, 2).reshape(case.B, case.Co, g["Tout"])
        intact = intact and sentinel_intact(cb[n:])
        sb = sbuf.cpu()
        if case.norm:
            st = sb[:case.B * Cn * 2].view(case.B, Cn, 2)
            out["mean"], out["rstd"] = st[:, :, 0], st[:, :, 1]
            intact = intact and sentinel_intact(sb[case.B * Cn * 2:])
        else:
            intact = intact and sentinel_intact(sb)      # stats is not asked for without norm: nothing is written
    return out, intact, d, plan


def bound_err(y, ref, bound):
    err = (y.double() - ref).abs()
    return float((err / bound.clamp_min(1e-30)).max()), float(err.max() / ref.abs().max().clamp_min(1e-30))


def errors(case, got, ref):
    """{measure name: (measure class, error, max-relative error or None)}."""
    e = {}
    y = got["out"]
    if case.round_out:
        assert bool(((y.view(torch.int32) & 0x1FFF) == 0).all()), "AVC_F_ROUND_OUT: output not TF32-exact"
    slack = HALF_TF32_ULP * ref["out"].abs() * (1 + 2 ** -10) if case.round_out else 0.0
    err = ((y.double() - ref["out"]).abs() - slack).clamp_min(0)
    rel = float(err.max() / ref["out"].abs().max().clamp_min(1e-30))
    if ref["out_bound"] is not None:
        e["out"] = ("bound", float((err / ref["out_bound"].clamp_min(1e-30)).max()), rel)
    else:
        e["out"] = ("norm", rel, None)
    if "c" in ref:
        eb, er = bound_err(got["c"], ref["c"], ref["c_bound"])
        e["c"] = ("bound", eb, er)
    if "mean" in ref:
        dm = float(((got["mean"].double() - ref["mean"]).abs() * ref["rstd"]).max())
        dr = float(((got["rstd"].double() - ref["rstd"]).abs() / ref["rstd"]).max())
        e["stats"] = ("stats", max(dm, dr), None)
    return e


@pytest.fixture(scope="module")
def lib():
    from adaptive_voice_conversion_b200 import _lib as L
    return L.load()


RESULTS = {}    # case id -> (group, launch keys, {output: (class, error, relative error)})
_T0 = []


def test_ffma_weight_packs_are_exact_permutations(lib):
    """avc_pack_conv_weight and the simt_fwd / simt_dgrad outputs of avc_pack_conv_weights_batch move the weights bit
    for bit: P[ci][j][co] = W[co][ci][j] (FWD), P[co][j][ci] = W[co][ci][K-1-j] (DGRAD)."""
    from adaptive_voice_conversion_b200 import _lib as L
    gen = torch.Generator().manual_seed(3)
    shapes = [(128, 80, 8), (128, 1104, 1), (128, 128, 5), (80, 128, 1), (256, 128, 5), (128, 84, 3), (96, 36, 7)]
    ws = []
    for co, ci, k in shapes:
        w = torch.randn((co, ci, k), generator=gen)
        w.view(-1)[:4] = torch.tensor([-0.0, 1e-40, float("inf"), -3e38])   # signed zero, subnormal, extremes
        ws.append(w.cuda())
    bits = lambda t: t.contiguous().view(torch.int32).cpu()
    fwd_ref = [w.permute(1, 2, 0) for w in ws]                 # [ci][j][co]
    dg_ref = [w.flip(2).permute(0, 2, 1) for w in ws]          # [co][j][ci]
    for w, fr, dr in zip(ws, fwd_ref, dg_ref):
        assert torch.equal(bits(pack(lib, w, L.PACK_FWD)), bits(fr).view(-1))
        assert torch.equal(bits(pack(lib, w, L.PACK_DGRAD)), bits(dr).view(-1))
    items = (L.PackItem * len(ws))()
    outs = []
    for it, w in zip(items, ws):
        f, g = torch.full((w.numel(),), float("nan"), device="cuda"), torch.full((w.numel(),), float("nan"), device="cuda")
        it.w, it.simt_fwd, it.simt_dgrad = w.data_ptr(), f.data_ptr(), g.data_ptr()
        it.Cout, it.Cin, it.K = w.shape
        outs.append((f, g))
    table = torch.frombuffer(bytearray(bytes(items)), dtype=torch.uint8).cuda()
    rc = lib.avc_pack_conv_weights_batch(table.data_ptr(), len(ws), max(w.numel() for w in ws), torch.cuda.current_stream().cuda_stream)
    assert rc == 0, L.last_error()
    torch.cuda.synchronize()
    for (f, g), fr, dr in zip(outs, fwd_ref, dg_ref):
        assert torch.equal(bits(f), bits(fr).view(-1))
        assert torch.equal(bits(g), bits(dr).view(-1))


@pytest.mark.parametrize("case", CASES, ids=lambda c: c.id)
def test_conv_simt_exact(lib, case):
    if not _T0:
        _T0.append(time.time())
    ops = operands(case)
    got, intact, d, plan = run_case(lib, case, *ops)
    assert plan.instance >= 0
    keys = launch_keys(d, plan)
    ref = reference(case, *ops)
    errs = errors(case, got, ref)
    RESULTS[case.id] = (case.group, keys, errs)
    assert intact, "a write outside out / c / stats"
    for k, (cls, e, rel) in errs.items():
        assert e < TOL[cls], f"{k}: error {e:.3e} ({cls}; max-relative {rel}) over the tolerance {TOL[cls]:.0e}"


@pytest.mark.parametrize("Tin,seg_out", [(5, 8), (27, 32)])
def test_sample_bits_do_not_depend_on_its_place_in_a_packed_tile(lib, Tin, seg_out):
    """A sample's out / c / stats bits are the same launched alone and at every segment position of a packed tile (and
    in the ragged tile after it), with random samples as neighbours."""
    base = Case("prop", "fwd", 1, 64, 128, 5, Tin, norm=True, relu=True, res=1)
    x1, w, bias, cond, res1, mask = operands(base)
    alone, ok, d, plan = run_case(lib, base, x1, w, bias, cond, res1, mask)
    assert ok and plan.seg_out == seg_out and plan.nseg == 128 // seg_out
    nseg = plan.nseg
    B = nseg + 3
    gen = torch.Generator().manual_seed(11)
    for pos in list(range(nseg)) + [nseg + 1]:
        case = Case("prop", "fwd", B, 64, 128, 5, Tin, norm=True, relu=True, res=1)
        x = torch.randn((B, 64, Tin), generator=gen)
        r = torch.randn((B, 128, res_len(base)), generator=gen)
        x[pos], r[pos] = x1[0], res1[0]
        got, ok, _, p = run_case(lib, case, x, w, bias, cond, r, mask)
        assert ok and p.nseg == nseg
        for k in ("out", "c", "mean", "rstd"):
            assert torch.equal(got[k][pos].view(torch.int32), alone[k][0].view(torch.int32)), (pos, k)


def test_two_launches_are_bit_identical(lib):
    for case in (Case("prop", "fwd", 13, 64, 128, 5, 16, norm=True, relu=True, res=1),
                 Case("prop", "dgrad", 2, 128, 128, 5, 300, stride=2)):
        ops = operands(case)
        a, _, _, _ = run_case(lib, case, *ops)
        b, _, _, _ = run_case(lib, case, *ops)
        for k in a:
            assert torch.equal(a[k].view(torch.int32), b[k].view(torch.int32)), (case.id, k)


def rejected_descs(ptr):
    """(what, descriptor) pairs the plan query and the launch must refuse with AVC_ERR_UNSUPPORTED."""
    from adaptive_voice_conversion_b200 import _lib as L
    out = [("norm, Tout > 256", make_desc(Case("r", "fwd", 2, 128, 128, 5, 300, norm=True), ptr)),
           ("norm, Tout 200 at K = 3", make_desc(Case("r", "fwd", 2, 128, 128, 3, 200, norm=True), ptr))]
    base = Case("r", "dgrad", 2, 128, 128, 5, 64)
    for what, field, val in (("AVC_F_FOLD", "flags", L.F_FOLD | (2 << 8) | (2 << 16)), ("AVC_F_NORMBWD", "flags", L.F_NORMBWD),
                             ("out_tstride", "out_tstride", 2), ("out_toff", "out_toff", 1), ("out_T", "out_T", 68)):
        d = make_desc(base, ptr)
        setattr(d, field, val)
        out.append((what, d))
    return out


def test_plan_and_launch_reject_alike(lib):
    """Every refused descriptor is refused by the launch with the same code and message; AVC_F_IN_TF32 is accepted."""
    from adaptive_voice_conversion_b200 import _lib as L
    t = torch.zeros(1 << 20, device="cuda")
    ptr = {k: t.data_ptr() for k in ("x", "w", "out", "c", "stats", "bias", "cond", "res", "mask")}
    for what, d in rejected_descs(ptr):
        rc, _ = plan_of(lib, d)
        msg = L.last_error()
        assert rc == L.ERR_UNSUPPORTED and msg.startswith("avc_conv_block_fwd"), (what, rc, msg)
        assert lib.avc_conv_block_fwd(C.byref(d), torch.cuda.current_stream().cuda_stream) == rc, what
        assert L.last_error() == msg, what
    d = make_desc(Case("r", "dgrad", 2, 128, 128, 5, 64, in_tf32=True), ptr)
    assert plan_of(lib, d)[0] == 0 and lib.avc_conv_block_fwd(C.byref(d), torch.cuda.current_stream().cuda_stream) == 0
    torch.cuda.synchronize()


def test_conv_simt_exact_coverage():
    """The recorded plans reach every kernel instance and every feature; reports the worst error per measure and group."""
    if any(c.id not in RESULTS for c in CASES):
        pytest.skip("only part of the module ran")
    covered, worst, worst_grp = set(), {}, {}
    for grp, keys, errs in RESULTS.values():
        covered |= keys
        for k, (cls, e, rel) in errs.items():
            worst[cls] = max(worst.get(cls, 0.0), e)
            worst_grp[(grp, cls)] = max(worst_grp.get((grp, cls), 0.0), e)
    print(f"\nconv simt exact: {len(CASES)} cases in {time.time() - _T0[0]:.1f} s; worst error per measure (tolerances {TOL}): "
          + ", ".join(f"{c} {e:.2e}" for c, e in sorted(worst.items())))
    print("  per group: " + ", ".join(f"{g}/{c} {e:.2e}" for (g, c), e in sorted(worst_grp.items())))
    for cid, (_, _, errs) in RESULTS.items():
        print(f"  {cid}: " + ", ".join(f"{k} {e:.2e}" + (f" (rel {r:.2e})" if r is not None else "") for k, (_, e, r) in errs.items()))
    missing = [f for f in FEATURES if f not in covered]
    assert not missing, missing
