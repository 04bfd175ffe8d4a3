"""GPU: the conv weight-gradient kernels against a float64 reference computed on the operands the kernel multiplies.

    dW[co][ci][j] += sum_{b,t} dc[b][co][t] * x[b][ci][reflect(t * stride + j - pad_left)]

* avc_conv_wgrad_tc (conv_wgrad_split_kernel + wgrad_tc_reduce_kernel, the default TF32 path): x and dc are rounded to
  TF32 on the host (round to nearest), so the tensor core's reading of its operands changes nothing and the products
  are exact in fp32; what is left is the order of the fp32 accumulation.  One case passes raw fp32 operands and its
  reference reads them truncated toward zero to TF32's 19 bits, which is what the tensor core does with the low bits.
* avc_conv_wgrad_tc_acc + avc_wgrad_acc_flush (AVC_WGRAD_ACC=1): the same cases accumulated in place, then ONE flush
  over a device item table that holds every layer of the list, twice.
* avc_conv_wgrad (conv_wgrad_kernel, exact fp32; the TF32 engine's fall-back for the shapes the tensor-core kernel
  does not take): raw fp32 operands.

The reference gathers the input with one reflection, as src_pos does (the descriptor carries no right padding).  dw is
preloaded with non-zero content (the kernels add), and NaN guard bands sit before and after dw and after the scratch
region the size query asks for; operands with a sample stride larger than their own C*T have NaN in the gap.

Error measure: max over elements of |kernel - reference| / sum_{b,t} |dc| * |x| (the same gather), so cancellation in a
reference entry cannot hide an error; max |kernel - reference| / max |reference| is reported beside it.
Worst measured on 1x NVIDIA H100 80GB HBM3 (132 SMs, 700 W power limit), as the elementwise bound / relative to the
max: tc stride 1 5.2e-7 / 1.8e-6, tc stride 2 1.2e-7 / 2.8e-7, tc raw operands 9.8e-8 / 4.0e-7 (so the truncation
model holds), acc + flush 5.2e-7 / 1.8e-6, simt stride 1 2.8e-7 / 1.0e-6, simt stride 2 2.6e-7 / 8.9e-7.  The
tolerances are about 4x the worst of each kernel.  For scale, arithmetic-only mutations of the kernels (odd stride-2
taps reading the even parity block, a dropped slice in the reduction, one sample fewer staged in a partial tile, the
MMA's row r0 + 4 replaced by r0, a skipped last partial time chunk of the FFMA kernel) each fail cases of this module.
The module's checks take about 1 s on that GPU, 20 s with start-up.

The tile plan of the tensor-core kernel (samples per tile G, batch slices) and the slice count of the FFMA kernel are
mirrored by tc_plan / simt_plan below; the scratch size queries pin the mirrors to the library, and the last test
asserts that the case list reaches every feature in FEATURES.  Kernel-level determinism (two launches from the same
preloaded dw are bit-identical) and step-level determinism of a training step follow.
"""
import ctypes as C
import time
import zlib
from dataclasses import dataclass

import pytest
import torch

from _layer_ref import tf32_rna  # noqa: F401  (cvt.rna.tf32.f32 on the bit pattern; also imported from here by _small_ref)

pytestmark = pytest.mark.gpu

TOL = {"tc": 2e-6, "acc": 2e-6, "simt": 1e-6}
GUARD = 1024          # floats of NaN guard band
WG_SMS = 132          # the slice count of the tensor-core plan is computed for 132 SMs (wgrad_tc_plan)


def cdiv(a, b):
    return -(-a // b)


@dataclass(frozen=True)
class Case:
    kernel: str       # "tc" or "simt"
    B: int
    Cin: int
    Cout: int
    K: int
    Tin: int
    stride: int = 1
    strided: bool = False   # x_bstride / dc_bstride larger than the operand's own C*T (the conv bank's channel ranges)
    raw: bool = False       # tc: raw fp32 operands (not TF32-rounded on the host)

    @property
    def pad_left(self):
        return self.K // 2

    @property
    def Tout(self):
        pl, pr = self.K // 2, self.K // 2 - (1 if self.K % 2 == 0 else 0)
        return (self.Tin + pl + pr - self.K) // self.stride + 1

    @property
    def x_bstride(self):
        return self.Cin * self.Tin + (52 if self.strided else 0)

    @property
    def dc_bstride(self):
        return self.Cout * self.Tout + (36 if self.strided else 0)

    @property
    def id(self):
        return (f"{self.kernel}-B{self.B}-{self.Cin}to{self.Cout}-k{self.K}-T{self.Tin}-s{self.stride}"
                + ("-strided" if self.strided else "") + ("-raw" if self.raw else ""))


TC_CASES = [
    Case("tc", 3, 16, 128, 1, 8),                        # G = 16 > B: one partial tile, nslices = 1
    Case("tc", 203, 16, 128, 2, 24),                     # G = 5, ragged last tile, nslices = 41
    Case("tc", 30, 80, 128, 8, 128, strided=True),       # bank conv: nslices = 30
    Case("tc", 256, 80, 128, 5, 128, strided=True),      # bank conv at B = 256: nslices = 43
    Case("tc", 7, 128, 80, 3, 72),                       # partial co tile
    Case("tc", 64, 128, 80, 1, 64),                      # out_conv: G = 2, nslices = 32
    Case("tc", 9, 1104, 128, 1, 128, strided=True),      # in_conv: 35 ci tiles, ci tail, nslices = 3
    Case("tc", 3, 1536, 256, 1, 128),                    # 96 CTAs per slice: nslices = 1
    Case("tc", 5, 128, 512, 4, 64),                      # G = 2, ragged, 4 co tiles
    Case("tc", 11, 128, 256, 6, 40),                     # G = 3, ragged
    Case("tc", 6, 64, 128, 7, 16),                       # G = 8 > B
    Case("tc", 19, 128, 128, 5, 63, stride=2),           # odd Tin: Tout = 32, G = 2, ragged
    Case("tc", 4, 128, 128, 5, 128, stride=2, strided=True),   # Tout = 64
    Case("tc", 37, 128, 128, 4, 15, stride=2),           # even K, odd Tin: Tout = 8, G = 8, ragged
    Case("tc", 5, 128, 128, 5, 128, raw=True),
]
SIMT_CASES = [
    Case("simt", 3, 128, 128, 5, 37),                    # Tout % 16 != 0, nsl = 1
    Case("simt", 16, 128, 128, 5, 244),                  # nsl = 8
    Case("simt", 4, 1104, 80, 1, 200),                   # ci and co tails of 128-wide tiles
    Case("simt", 6, 80, 256, 8, 300, strided=True),
    Case("simt", 5, 128, 128, 5, 200, stride=2),         # stride 2, Tout = 100
    Case("simt", 9, 80, 128, 2, 200, strided=True),
    Case("simt", 2, 80, 128, 3, 244, strided=True),
    Case("simt", 3, 80, 128, 4, 200, strided=True),
    Case("simt", 4, 80, 128, 6, 244, strided=True),
    Case("simt", 5, 80, 128, 7, 200, strided=True),
    Case("simt", 2, 128, 128, 1, 25),
]
CASES = TC_CASES + SIMT_CASES

FEATURES = ([("tc", "K", k) for k in range(1, 9)] + [("tc", "Tout", 1, t) for t in (8, 24, 72, 128)]
            + [("tc", "Tout", 2, t) for t in (8, 32, 64)]
            + [("tc", "stride 2, odd Tin"), ("tc", "G > 1, B % G != 0"), ("tc", "nslices", "1"), ("tc", "nslices", "2-24"),
               ("tc", "nslices", "> 24, % 8 != 0"), ("tc", "Cout", 80), ("tc", "Cout", 256), ("tc", "Cout", 512),
               ("tc", "strided operands"), ("tc", "raw operands")]
            + [("tc", "Cin", c) for c in (16, 80, 1104, 1536)]
            + [("simt", "K", k) for k in range(1, 9)] + [("simt", "Tout", t) for t in (37, 244, 200, 300)]
            + [("simt", "stride 2, Tout > 64"), ("simt", "Cin", 1104), ("simt", "Cout", 80), ("simt", "nsl", "1"),
               ("simt", "nsl", ">= 3"), ("simt", "strided operands")])


# ------------------------------------------------------------------ the launch plans, mirrored
def tc_supported(B, Cin, Cout, K, Tin, Tout, stride):
    """wgrad_tc_supported: the shapes avc_wgrad_tc_scratch_floats accepts."""
    return (stride in (1, 2) and Tout % 8 == 0 and Tout <= 128 and 1 <= K <= 8 and Cin % 4 == 0 and Cout % 4 == 0
            and Tin + K - 1 >= (Tout - 1) * stride + 1 and (stride == 1 or Tout <= 64))


def tc_plan(B, Cin, Cout, K, Tout, stride):
    """wgrad_tc_plan -> (samples per tile G, batch slices, Cout rounded up to 128)."""
    G = (1 if Tout >= 128 else 128 // Tout) if stride == 1 else (1 if Tout >= 64 else 64 // Tout)
    ntiles = cdiv(B, G)
    nsl = min(max(WG_SMS // (cdiv(Cin, 32) * cdiv(Cout, 128)), 1), ntiles)
    return G, cdiv(ntiles, cdiv(ntiles, nsl)), cdiv(Cout, 128) * 128


def simt_plan(B, Cin, Cout, K, Tout):
    """avc_conv_wgrad's batch slices -> (slices, Cout rounded up to 128)."""
    tiles = cdiv(Cin, 128) * cdiv(Cout, 128) * K
    nsl = max(min(cdiv(2 * 148 * 2, tiles), max(B * Tout // 256, 1), B), 1)
    return cdiv(B, cdiv(B, nsl)), cdiv(Cout, 128) * 128


def nslices_bucket(kernel, n):
    if kernel == "tc":
        return "1" if n == 1 else "2-24" if n <= 24 else "> 24, % 8 != 0" if n % 8 else "> 24, % 8 == 0"
    return "1" if n == 1 else "2" if n == 2 else ">= 3"


def desc_keys(kernel, B, Cin, Cout, K, Tin, Tout, stride, strided):
    """Feature keys of one weight-gradient launch, as tests/test_wgrad_plan.py records them from the engine."""
    keys = {(kernel, "stride", stride), (kernel, "K", K), (kernel, "strided", strided), (kernel, "Cout % 128", Cout % 128 != 0),
            (kernel, "Cout > 128", Cout > 128)}
    if kernel == "tc":
        G, ns, _ = tc_plan(B, Cin, Cout, K, Tout, stride)
        keys |= {("tc", "G > 1", G > 1), ("tc", "B % G", B % G != 0), ("tc", "nslices", nslices_bucket("tc", ns)),
                 ("tc", "Cin % 32", Cin % 32 != 0), ("tc", "Cin > 32", Cin > 32)}
    else:
        ns, _ = simt_plan(B, Cin, Cout, K, Tout)
        keys |= {("simt", "nsl", nslices_bucket("simt", ns)), ("simt", "Cin % 128", Cin % 128 != 0),
                 ("simt", "Cin > 128", Cin > 128), ("simt", "Tout % 16", Tout % 16 != 0), ("simt", "Tout > 128", Tout > 128)}
    return keys


def case_keys(case):
    return desc_keys(case.kernel, case.B, case.Cin, case.Cout, case.K, case.Tin, case.Tout, case.stride, case.strided)


def features(case):
    """The FEATURES one case reaches."""
    k, T = case.kernel, case.Tout
    f = {(k, "K", case.K)}
    if case.strided:
        f.add((k, "strided operands"))
    if k == "tc":
        G, ns, _ = tc_plan(case.B, case.Cin, case.Cout, case.K, T, case.stride)
        f |= {("tc", "Tout", case.stride, T), ("tc", "nslices", nslices_bucket("tc", ns)), ("tc", "Cin", case.Cin),
              ("tc", "Cout", case.Cout)}
        if case.stride == 2 and case.Tin % 2:
            f.add(("tc", "stride 2, odd Tin"))
        if G > 1 and case.B % G:
            f.add(("tc", "G > 1, B % G != 0"))
        if case.raw:
            f.add(("tc", "raw operands"))
    else:
        ns, _ = simt_plan(case.B, case.Cin, case.Cout, case.K, T)
        f |= {("simt", "Tout", T), ("simt", "nsl", nslices_bucket("simt", ns)), ("simt", "Cin", case.Cin), ("simt", "Cout", case.Cout)}
        if case.stride == 2 and T > 64:
            f.add(("simt", "stride 2, Tout > 64"))
    return f


def make_desc(case, x, dc, dw):
    from adaptive_voice_conversion_b200 import _lib as L
    d = L.WgradDesc()
    d.B, d.Cin, d.Cout, d.K, d.stride = case.B, case.Cin, case.Cout, case.K, case.stride
    d.pad_left, d.Tin, d.Tout = case.pad_left, case.Tin, case.Tout
    d.x, d.x_bstride, d.dc, d.dc_bstride, d.dw = x, case.x_bstride, dc, case.dc_bstride, dw
    return d


# ------------------------------------------------------------------ reference
def tf32_trunc(x):
    """The top 19 bits of the fp32 pattern (sign, exponent, 10 mantissa bits): truncation toward zero."""
    return (x.contiguous().view(torch.int32) & -0x2000).view(torch.float32)


def reference(x, dc, K, stride, pad_left):
    """(dW, sum |dc| |x|) in float64 on the device; x [B][Cin][Tin], dc [B][Cout][Tout] as the kernel multiplies them."""
    Tin, Tout = x.shape[2], dc.shape[2]
    u = torch.arange(Tout, device=x.device)[None, :] * stride + torch.arange(K, device=x.device)[:, None] - pad_left
    p = torch.where(u < 0, -u, u)
    p = torch.where(p >= Tin, 2 * (Tin - 1) - p, p)
    valid = ((p >= 0) & (p < Tin)).double()
    xg = x.double()[:, :, p.clamp(0, Tin - 1)] * valid          # [B][Cin][K][Tout]
    dcd = dc.double()
    return torch.einsum("bot,bcjt->ocj", dcd, xg), torch.einsum("bot,bcjt->ocj", dcd.abs(), xg.abs())


def to_a4(t, bstride):
    """planar [B][C][T] -> A4 [B][C/4][T][4] on the device, samples bstride floats apart, NaN in the gap."""
    B, Cc, T = t.shape
    buf = torch.full((B, bstride), float("nan"), device="cuda")
    buf[:, :Cc * T] = t.reshape(B, Cc // 4, 4, T).permute(0, 1, 3, 2).reshape(B, Cc * T).cuda()
    return buf


_DATA = {}


def data(case):
    """Device operands of a case: (x A4, dc A4, dW reference, sum |dc||x|, preload), made once per module."""
    if case.id not in _DATA:
        gen = torch.Generator().manual_seed(zlib.crc32(case.id.encode()))
        x = torch.randn((case.B, case.Cin, case.Tin), generator=gen)
        dc = torch.randn((case.B, case.Cout, case.Tout), generator=gen)
        pre = torch.randn((case.Cout, case.Cin, case.K), generator=gen)
        if case.kernel == "tc" and not case.raw:
            x, dc = tf32_rna(x), tf32_rna(dc)
        xr, dcr = (tf32_trunc(x), tf32_trunc(dc)) if case.raw else (x, dc)
        ref, aref = reference(xr.cuda(), dcr.cuda(), case.K, case.stride, case.pad_left)
        _DATA[case.id] = (to_a4(x, case.x_bstride), to_a4(dc, case.dc_bstride), ref, aref, pre.cuda())
    return _DATA[case.id]


def guarded(n, fill=float("nan")):
    """(buffer, view of n floats): GUARD NaN floats on either side."""
    buf = torch.full((n + 2 * GUARD,), float("nan"), device="cuda")
    v = buf[GUARD:GUARD + n]
    v.fill_(fill)
    return buf, v


def guards_intact(buf):
    return bool(torch.isnan(buf[:GUARD]).all()) and bool(torch.isnan(buf[-GUARD:]).all())


def errors(dw, pre, ref, aref, scale=1.0):
    """(max |err| / sum|dc||x|, max |err| / max |ref|) of dw - pre against scale * ref."""
    err = (dw.double() - pre.double() - scale * ref).abs()
    return float((err / (scale * aref)).max()), float(err.max() / (scale * ref.abs().max()))


@pytest.fixture(scope="module")
def eng():
    import oracle.ae_oracle as orc
    from adaptive_voice_conversion_b200.engine import Engine
    e = Engine(orc.default_config(80), torch.device("cuda", 0))
    e.precision = "tf32"
    return e


RESULTS = {}      # case id or "acc:" + id -> (class, bound error, relative error)
_T0 = []


def _group(case):
    return f"{case.kernel} stride {case.stride}" + (" raw operands" if case.raw else "")


def launch(eng, case, x, dc, dw):
    """One launch of the case's kernel; returns the scratch buffer (guarded)."""
    d = make_desc(case, x.data_ptr(), dc.data_ptr(), dw.data_ptr())
    if case.kernel == "tc":
        n = int(eng.lib.avc_wgrad_tc_scratch_floats(C.byref(d)))
        G, ns, coutp = tc_plan(case.B, case.Cin, case.Cout, case.K, case.Tout, case.stride)
        assert n == ns * case.K * case.Cin * coutp, (n, ns, coutp)
        sbuf, s = guarded(n)
        eng._ck(eng.lib.avc_conv_wgrad_tc(C.byref(d), s.data_ptr(), eng.tc_status.data_ptr(), eng.stream), case.id)
        eng.check_tc_status()
    else:
        n = int(eng.lib.avc_conv_wgrad_scratch_floats(C.byref(d)))
        ns, coutp = simt_plan(case.B, case.Cin, case.Cout, case.K, case.Tout)
        assert n == ns * case.K * case.Cin * coutp, (n, ns, coutp)
        sbuf, s = guarded(n)
        eng._ck(eng.lib.avc_conv_wgrad(C.byref(d), s.data_ptr(), eng.stream), case.id)
    return sbuf


@pytest.mark.parametrize("case", CASES, ids=lambda c: c.id)
def test_wgrad_exact(eng, case):
    if not _T0:
        _T0.append(time.time())
    x, dc, ref, aref, pre = data(case)
    dbuf, dw = guarded(pre.numel())
    dw.copy_(pre.flatten())
    sbuf = launch(eng, case, x, dc, dw)
    torch.cuda.synchronize()
    assert guards_intact(dbuf), "write outside dw"
    assert guards_intact(sbuf), "write outside the scratch region"
    eb, er = errors(dw.view_as(pre), pre, ref, aref)
    RESULTS[case.id] = (_group(case), eb, er)
    assert eb < TOL[case.kernel], f"max error {eb:.3e} of sum |dc||x| (relative to max |ref|: {er:.3e}; tolerance {TOL[case.kernel]:.0e})"


def test_wgrad_acc_and_one_flush_of_every_layer(eng):
    """avc_conv_wgrad_tc_acc for every tensor-core case into its own zeroed region, then ONE avc_wgrad_acc_flush over a
    device table of all of them; twice (the flush must leave every region zeroed)."""
    from adaptive_voice_conversion_b200 import _lib as L
    rows = []
    for case in TC_CASES:
        x, dc, ref, aref, pre = data(case)
        nf = int(eng.lib.avc_wgrad_acc_floats(case.Cout, case.Cin, case.K))
        assert nf == case.K * case.Cin * tc_plan(case.B, case.Cin, case.Cout, case.K, case.Tout, case.stride)[2]
        abuf, acc = guarded(nf, 0.0)
        dbuf, dw = guarded(pre.numel())
        dw.copy_(pre.flatten())
        rows.append((case, abuf, acc, dbuf, dw))
    items = (L.WgradAccItem * len(rows))()
    for it, (case, _, acc, _, dw) in zip(items, rows):
        it.acc, it.dw, it.Cout, it.Cin, it.K = acc.data_ptr(), dw.data_ptr(), case.Cout, case.Cin, case.K
    table = torch.frombuffer(bytearray(bytes(items)), dtype=torch.uint8).cuda()
    max_units = max(acc.numel() // 4 for _, _, acc, _, _ in rows)
    for cycle in (1, 2):
        for case, _, acc, _, dw in rows:
            x, dc = data(case)[:2]
            d = make_desc(case, x.data_ptr(), dc.data_ptr(), 0)
            eng._ck(eng.lib.avc_conv_wgrad_tc_acc(C.byref(d), acc.data_ptr(), eng.tc_status.data_ptr(), eng.stream), case.id)
        eng._ck(eng.lib.avc_wgrad_acc_flush(table.data_ptr(), len(rows), max_units, eng.stream), "wgrad_acc_flush")
        eng.check_tc_status()
        for case, abuf, acc, dbuf, dw in rows:
            _, _, ref, aref, pre = data(case)
            assert guards_intact(abuf) and guards_intact(dbuf), case.id
            assert float(acc.abs().max()) == 0.0, case.id
            eb, er = errors(dw.view_as(pre), pre, ref, aref, scale=cycle)
            RESULTS[f"acc{cycle}:{case.id}"] = ("acc + flush" + (" raw operands" if case.raw else ""), eb, er)
            assert eb < TOL["acc"], (case.id, cycle, eb, er)


def test_wgrad_exact_coverage():
    """The case list reaches every feature; reports the worst error per kernel and stride class."""
    if any(c.id not in RESULTS for c in CASES):
        pytest.skip("only part of the module ran")
    covered = set().union(*(features(c) for c in CASES))
    worst = {}
    for grp, eb, er in RESULTS.values():
        wb, wr = worst.get(grp, (0.0, 0.0))
        worst[grp] = (max(wb, eb), max(wr, er))
    print(f"\nwgrad exact: {len(RESULTS)} checks in {time.time() - _T0[0]:.1f} s; worst error per class "
          f"(of sum |dc||x| / of max |ref|; tolerances {TOL}):")
    for g, (eb, er) in sorted(worst.items()):
        print(f"  {g}: {eb:.2e} / {er:.2e}")
    for cid, (g, eb, er) in RESULTS.items():
        print(f"  {cid}: {eb:.2e} / {er:.2e}")
    missing = [f for f in FEATURES if f not in covered]
    assert not missing, missing


# ------------------------------------------------------------------ run-to-run determinism
@pytest.mark.parametrize("kernel,T", [("simt", 200), ("tc", 128)])
def test_wgrad_kernel_is_deterministic(eng, kernel, T):
    """Two launches from the same preloaded dw give the same bits: B = 256, 128 -> 128 channels, K = 5."""
    case = Case(kernel, 256, 128, 128, 5, T)
    gen = torch.Generator().manual_seed(7)
    x = to_a4(torch.randn((case.B, case.Cin, case.Tin), generator=gen), case.x_bstride)
    dc = to_a4(torch.randn((case.B, case.Cout, case.Tout), generator=gen), case.dc_bstride)
    pre = torch.randn((case.Cout * case.Cin * case.K,), generator=gen).cuda()
    if kernel == "simt":
        assert simt_plan(case.B, case.Cin, case.Cout, case.K, case.Tout)[0] >= 3
    outs = []
    for _ in range(2):
        dw = pre.clone()
        launch(eng, case, x, dc, dw)
        outs.append(dw)
    torch.cuda.synchronize()
    assert torch.equal(outs[0], outs[1]), int((outs[0] != outs[1]).sum())


def _step_flat_g(tmp_path, precision, T, B=32):
    import types
    import oracle.ae_oracle as orc
    from adaptive_voice_conversion_b200.solver import Solver
    cfg = orc.default_config(80)
    cfg["data_loader"]["batch_size"] = B
    args = types.SimpleNamespace(data_dir="synthetic", train_set="train", train_index_file="", logdir=str(tmp_path / "log"),
                                 load_model=False, load_opt=False, store_model_path=str(tmp_path / "model"),
                                 load_model_path=str(tmp_path / "model"), summary_steps=1, save_steps=1000, tag="t", iters=0)
    solver = Solver(cfg, args)
    solver.model.load_state_dict(orc.init_state(cfg, seed=0), strict=True)
    tr = solver.trainer
    tr.eng.precision = precision            # the engine is cached per model/device: set explicitly
    tr.eng.wgrad_acc = False
    tr.eng.prepare_wgrad_acc(tr.P, tr.G)
    tr.eng.pack_weights(tr.P, need_dgrad=True)
    g = torch.Generator().manual_seed(1)
    x = torch.randn((B, 80, T), generator=g).cuda()
    eps = torch.randn((B, 128, T // 8), generator=g).cuda()
    outs = []
    for _ in range(2):
        tr._fwd_bwd(x, eps)
        torch.cuda.synchronize()
        outs.append(solver.opt.flat_g.clone())
    tr.eng.precision = "tf32"
    tr.eng.pack_weights(tr.P, need_dgrad=True)
    return outs


@pytest.mark.parametrize("precision,T", [("fp32", 128), ("tf32", 200)])
def test_training_step_gradient_is_deterministic(tmp_path, precision, T):
    """The whole gradient of a training step is bit-identical across two runs from the same state: the exact-fp32 path,
    and TF32 at a segment length whose weight gradients partly fall back to the FFMA kernel.  B = 32 so that the FFMA
    weight gradients of 128 -> 128 convs split the batch into 16 slices (at B = 4 two slices added onto zeros would give
    the same bits in either order)."""
    assert simt_plan(32, 128, 128, 5, T)[0] >= 3
    g0, g1 = _step_flat_g(tmp_path, precision, T)
    assert torch.equal(g0, g1), int((g0 != g1).sum())
