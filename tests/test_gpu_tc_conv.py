"""GPU: the tensor-core (TF32) fused conv block and its data-gradient use against the CPU oracle.
TF32 inputs are rounded to nearest (10-bit mantissa): tolerance 3e-3 of the tensor max for a
single block (fp32 path: 2e-4, tests/test_gpu_kernels.py)."""
import math

import pytest
import torch

import oracle.ae_oracle as orc
from test_gpu_kernels import ref_block, relerr, rnd, to_a4, from_a4

pytestmark = pytest.mark.gpu
TOL = 3e-3


@pytest.fixture(scope="module")
def eng():
    from adaptive_voice_conversion_b200.engine import Engine
    e = Engine(orc.default_config(80), torch.device("cuda", 0))
    e.precision = "tf32"
    return e


CASES = [
    # B, Cin, Cout, K, T, shuffle, norm, cond, relu, res_mode
    (5, 128, 128, 5, 128, 0, 1, 0, 1, 0),
    (5, 128, 128, 5, 64, 0, 1, 0, 1, 1),
    (19, 128, 128, 5, 16, 0, 0, 0, 1, 1),
    (300, 128, 128, 5, 16, 0, 1, 1, 1, 0),    # several samples per CTA, ragged tail
    (9, 128, 256, 5, 16, 1, 1, 1, 1, 3),      # pixel shuffle: two M tiles
    (3, 128, 256, 5, 64, 1, 1, 1, 1, 3),
    (3, 80, 128, 8, 128, 0, 0, 0, 1, 0),      # bank conv, even kernel
    (3, 80, 128, 1, 128, 0, 0, 0, 1, 0),
    (3, 80, 128, 3, 128, 0, 0, 0, 1, 0),
    (2, 1104, 128, 1, 128, 0, 1, 0, 1, 0),    # in_conv: 69 slabs through the ring
    (2, 128, 80, 1, 128, 0, 0, 0, 0, 0),      # out_conv: partial M tile
    (2, 128, 128, 5, 37, 0, 1, 0, 1, 1),      # odd length
    (2, 128, 128, 5, 200, 0, 1, 0, 1, 1),     # N = 208 columns
    (2, 128, 128, 5, 256, 0, 1, 1, 1, 1),
    # persistent kernel (conv_tc2.cu): more tiles than SMs (stage barrier phases wrap)
    (301, 128, 128, 5, 128, 0, 1, 0, 1, 1),
    (601, 128, 128, 5, 64, 0, 1, 1, 1, 1),    # 2 samples per tile, odd tail
    (450, 128, 256, 5, 32, 1, 1, 1, 1, 3),    # stacked samples + pixel shuffle, two M tiles
    (3, 128, 128, 5, 512, 0, 0, 0, 1, 1),     # time-tiled long sample (no InstanceNorm): 4 tiles of 128 columns
    (2, 128, 128, 5, 300, 0, 0, 0, 1, 0),     # ragged last time tile
    (2, 80, 128, 8, 333, 0, 0, 0, 1, 0),      # even kernel, time-tiled
]
CASES_S2 = [(5, 128, 128, 5, 128, 1), (19, 128, 128, 5, 32, 0), (3, 128, 128, 5, 37, 1), (300, 128, 128, 5, 64, 1), (333, 128, 128, 5, 128, 1),
            (3, 128, 128, 5, 512, 0)]


@pytest.mark.parametrize("B,Cin,Cout,K,T,norm", CASES_S2)
def test_tc_conv_stride2(eng, B, Cin, Cout, K, T, norm):
    """Stride-2 block (encoder second convs, model.py:243-249): full-resolution MMAs, even
    columns kept, pooled residual."""
    x = rnd((B, Cin, T), 1)
    w = rnd((Cout, Cin, K), 2) / math.sqrt(Cin * K)
    b = rnd((Cout,), 3) * 0.1
    res = rnd((B, Cout, T), 5)
    yr = ref_block(x, w, b, 2, 0, norm, None, 1, res, 2)
    P = {"blk.weight": w.cuda(), "blk.bias": b.cuda()}
    eng.packed.pop("blk", None)
    eng.conv_names = lambda: ["blk"]
    eng.pack_weights(P, need_dgrad=False)
    out, rec = eng.conv(P, "blk", to_a4(eng, x), stride=2, norm=bool(norm), relu=True, res=to_a4(eng, res), res_mode=2, train=True)
    eng.check_tc_status()
    assert relerr(from_a4(eng, out), yr) < TOL, relerr(from_a4(eng, out), yr)
    assert relerr(from_a4(eng, rec["c"]), orc.reflect_conv1d(x, w, b, 2)) < TOL



@pytest.mark.parametrize("case", CASES, ids=[str(c) for c in CASES])
def test_tc_conv_block(eng, case):
    from adaptive_voice_conversion_b200 import _lib as L
    B, Cin, Cout, K, T, shuffle, norm, use_cond, relu, res_mode = case
    x = rnd((B, Cin, T), 1)
    w = rnd((Cout, Cin, K), 2) / math.sqrt(Cin * K)
    b = rnd((Cout,), 3) * 0.1
    Tout = T
    Cn, Tn = (Cout // 2, 2 * Tout) if shuffle else (Cout, Tout)
    cond = (rnd((B, 2 * Cn), 4) * 0.5 + 0.7) if use_cond else None
    res_T = {0: 0, 1: Tn, 3: Tn // 2}[res_mode]
    res = rnd((B, Cn, res_T), 5) if res_mode else None
    xr, wr = x.clone().requires_grad_(True), w.clone().requires_grad_(True)
    cr = cond.clone().requires_grad_(True) if cond is not None else None
    yr = ref_block(xr, wr, b, 1, shuffle, norm, cr, relu, res, res_mode)
    dy = rnd(tuple(yr.shape), 6)
    yr.backward(dy)

    P = {"blk.weight": w.cuda(), "blk.bias": b.cuda()}
    G = {k: torch.zeros_like(v) for k, v in P.items()}
    eng.packed.pop("blk", None)
    eng.conv_names = lambda: ["blk"]
    eng.pack_weights(P, need_dgrad=True)
    assert "fwd_tc" in eng.packed["blk"]
    xa = to_a4(eng, x)
    ra = to_a4(eng, res) if res is not None else None
    cg = cond.cuda() if cond is not None else None
    out, rec = eng.conv(P, "blk", xa, shuffle=bool(shuffle), norm=bool(norm), cond=cg, relu=bool(relu), res=ra,
                        res_mode=res_mode, train=True)
    eng.check_tc_status()
    y = from_a4(eng, out)
    assert relerr(y, yr) < TOL, f"forward {relerr(y, yr)}"
    if rec["c"] is not None:
        c_ref = orc.reflect_conv1d(x, w, b)
        assert relerr(from_a4(eng, rec["c"]), c_ref) < TOL
    dcond = torch.zeros_like(cg) if cg is not None else None
    dx = eng.conv_bwd(P, G, rec, to_a4(eng, dy), dcond=dcond)
    eng.check_tc_status()
    # TF32 moves pre-activations by ~1e-3, so ~0.1% of the ReLU masks differ from the fp32
    # reference and the gradient differs by O(1) at those elements: assert in relative L2
    # (sqrt(1e-3) ~ 3e-2 expected); the linear case below pins the dgrad kernel tightly.
    def rl2(a, b):
        a, b = a.double().cpu().flatten(), b.double().flatten()
        return float((a - b).norm() / b.norm())
    lim = 1e-1 if relu else 2 * TOL
    assert rl2(from_a4(eng, dx), xr.grad) < lim, f"dx {rl2(from_a4(eng, dx), xr.grad)}"
    assert rl2(G["blk.weight"], wr.grad) < lim, f"dW {rl2(G['blk.weight'], wr.grad)}"


@pytest.mark.parametrize("B,Cin,Cout,K,T", [(5, 128, 128, 5, 128), (7, 128, 256, 5, 32), (3, 256, 128, 5, 64), (2, 128, 1104, 1, 128), (3, 128, 128, 5, 200)])
def test_tc_dgrad_linear(eng, B, Cin, Cout, K, T):
    """Data gradient of a plain conv (no norm / ReLU): exact transposed conv, max-norm check.
    Cout=256 -> 2 K-slab groups in the transposed problem; Cout=1104 with dx restricted to
    1024 channels is the in_conv -> bank gradient."""
    x = rnd((B, Cin, T), 1).requires_grad_(True)
    w = rnd((Cout, Cin, K), 2) / math.sqrt(Cin * K)
    y = orc.reflect_conv1d(x, w, None)
    dy = rnd(tuple(y.shape), 3)
    y.backward(dy)
    P = {"blk.weight": w.cuda(), "blk.bias": torch.zeros(Cout).cuda()}
    G = {k: torch.zeros_like(v) for k, v in P.items()}
    eng.packed.pop("blk", None)
    eng.conv_names = lambda: ["blk"]
    eng.pack_weights(P, need_dgrad=True)
    pl, pr = K // 2, K // 2 - (1 if K % 2 == 0 else 0)
    rec = dict(name="blk", xin=to_a4(eng, x.detach()), c=None, stats=None, cond=None, out=None, stride=1, shuffle=False, norm=False,
               relu=False, K=K, Cin=Cin, Cout=Cout, Tout=T, pl=pl, pr=pr)
    dx = eng.conv_bwd(P, G, rec, to_a4(eng, dy))
    eng.check_tc_status()
    assert relerr(from_a4(eng, dx), x.grad) < TOL, relerr(from_a4(eng, dx), x.grad)


@pytest.mark.parametrize("B,Cin,Cout,K,T", [(5, 128, 128, 5, 128), (37, 128, 128, 5, 16), (9, 128, 256, 5, 32), (3, 80, 128, 8, 128),
                                             (3, 80, 128, 1, 128), (2, 1104, 128, 1, 128), (3, 128, 80, 1, 64), (300, 128, 128, 5, 16)])
def test_tc_wgrad(eng, B, Cin, Cout, K, T):
    """Weight gradient on the tensor cores (MN-major operands staged from the A4 layout) vs autograd."""
    import ctypes as C
    from adaptive_voice_conversion_b200 import _lib as L
    x = rnd((B, Cin, T), 1)
    w = (rnd((Cout, Cin, K), 2) / math.sqrt(Cin * K)).requires_grad_(True)
    y = orc.reflect_conv1d(x, w, None)
    dc = rnd(tuple(y.shape), 3)
    y.backward(dc)
    xa, da = to_a4(eng, x), to_a4(eng, dc)
    dw = torch.full((Cout, Cin, K), 0.25, device="cuda")     # accumulates (+=) into existing content
    wd = L.WgradDesc()
    wd.B, wd.Cin, wd.Cout, wd.K, wd.stride, wd.pad_left, wd.Tin, wd.Tout = B, Cin, Cout, K, 1, K // 2, T, T
    wd.x, wd.x_bstride, wd.dc, wd.dc_bstride, wd.dw = xa.ptr, xa.bstride, da.ptr, da.bstride, dw.data_ptr()
    assert int(eng.lib.avc_wgrad_tc_scratch_floats(C.byref(wd))) > 0
    eng.wgrad(wd, "t")
    eng.check_tc_status()
    assert relerr(dw.cpu() - 0.25, w.grad) < TOL, relerr(dw.cpu() - 0.25, w.grad)


@pytest.mark.parametrize("B,C_,T", [(5, 128, 128), (19, 128, 32), (3, 128, 64)])
def test_tc_stride2_backward_linear(eng, B, C_, T):
    """Stride-2 conv (encoder second convs): data gradient as two tap-parity convs and the weight
    gradient with parity-split staging, both on the tensor cores, vs autograd of the plain conv."""
    K = 5
    x = rnd((B, C_, T), 1).requires_grad_(True)
    w = (rnd((C_, C_, K), 2) / math.sqrt(C_ * K)).requires_grad_(True)
    y = orc.reflect_conv1d(x, w, None, 2)
    dy = rnd(tuple(y.shape), 3)
    y.backward(dy)
    P = {"speaker_encoder.second_conv_layers.1.weight": w.detach().cuda(), "speaker_encoder.second_conv_layers.1.bias": torch.zeros(C_).cuda()}
    name = "speaker_encoder.second_conv_layers.1"     # a stride-2 layer of the default config
    G = {k: torch.zeros_like(v) for k, v in P.items()}
    eng.packed.pop(name, None)
    eng.conv_names = lambda: [name]
    eng.pack_weights(P, need_dgrad=True)
    assert "dgrad_tc_even" in eng.packed[name]
    rec = dict(name=name, xin=to_a4(eng, x.detach()), c=None, stats=None, cond=None, out=None, stride=2, shuffle=False, norm=False,
               relu=False, K=K, Cin=C_, Cout=C_, Tout=y.shape[-1], pl=2, pr=2)
    n0 = __import__("adaptive_voice_conversion_b200._lib", fromlist=["x"]).launch_count()
    dx = eng.conv_bwd(P, G, rec, to_a4(eng, dy))
    eng.check_tc_status()
    assert relerr(from_a4(eng, dx), x.grad) < TOL, relerr(from_a4(eng, dx), x.grad)
    assert relerr(G[name + ".weight"], w.grad) < TOL, relerr(G[name + ".weight"], w.grad)
