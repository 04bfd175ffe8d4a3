"""GPU: the data-gradient conv with the reflect-padding / residual adjoint folded into its epilogue
(AVC_F_FOLD, csrc/conv_tc2.cu) against the two-pass path (conv + avc_fold_add_fwd) and autograd.
Default path."""
import math
import os

import pytest
import torch
import torch.nn.functional as F

import oracle.ae_oracle as orc
from test_gpu_kernels import relerr, rnd, to_a4, from_a4

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def eng():
    from adaptive_voice_conversion_b200.engine import Engine
    e = Engine(orc.default_config(80), torch.device("cuda", 0))
    e.precision = "tf32"
    return e


# B, C, K, T, residual mode of the block this conv opens (0 none, 1 same, 2 avg-pool, 3 nearest-upsample)
CASES = [(5, 128, 5, 128, 0), (5, 128, 5, 128, 1), (19, 128, 5, 64, 2), (3, 128, 5, 37, 2), (7, 128, 5, 32, 3), (300, 128, 5, 16, 1),
         (3, 128, 3, 64, 1), (3, 128, 8, 48, 0), (2, 128, 1, 64, 1), (2, 256, 5, 200, 1)]


@pytest.mark.parametrize("B,C_,K,T,mode", CASES)
def test_fold_fused_matches_two_pass_and_autograd(eng, B, C_, K, T, mode):
    from adaptive_voice_conversion_b200 import _lib as L
    x = rnd((B, C_, T), 1).requires_grad_(True)
    w = (rnd((C_, C_, K), 2) / math.sqrt(C_ * K))
    y = orc.reflect_conv1d(x, w, None)
    res_T = {0: 0, 1: T, 2: (T + 1) // 2, 3: 2 * T}[mode]
    dres = rnd((B, C_, res_T), 4) if mode else None
    # the block output is conv2(...) + shortcut(x): shortcut = identity / avg_pool1d(ceil) / nearest upsample
    out = y.sum() * 0
    if mode == 1:
        out = (x * dres).sum()
    elif mode == 2:
        out = (F.avg_pool1d(x, kernel_size=2, ceil_mode=True) * dres).sum()
    elif mode == 3:
        out = (F.interpolate(x, scale_factor=2, mode="nearest") * dres).sum()
    dy = rnd(tuple(y.shape), 3)
    ((y * dy).sum() + out).backward()

    name = "blk"
    P = {"blk.weight": w.cuda(), "blk.bias": torch.zeros(C_).cuda()}
    eng.conv_names = lambda: [name]
    eng.packed.pop(name, None)
    eng.pack_weights(P, need_dgrad=True)
    pl = K // 2
    pr = K // 2 - 1 if K % 2 == 0 else K // 2
    res = {}
    for fused in (False, True):
        eng.fold_fused = fused
        G = {k: torch.zeros_like(v) for k, v in P.items()}
        rec = dict(name=name, xin=to_a4(eng, x.detach()), c=None, stats=None, cond=None, out=None, stride=1, shuffle=False, norm=False,
                   relu=False, K=K, Cin=C_, Cout=C_, Tout=T, pl=pl, pr=pr)
        n0 = L.launch_count()
        dx = eng.conv_bwd(P, G, rec, to_a4(eng, dy), dres=to_a4(eng, dres) if dres is not None else None,
                          dres_mode={0: L.RES_NONE, 1: L.RES_SAME, 2: L.RES_POOL, 3: L.RES_UP}[mode])
        eng.check_tc_status()
        res[fused] = (from_a4(eng, dx), L.launch_count() - n0)
    eng.fold_fused = False
    assert relerr(res[False][0], x.grad) < 3e-3
    assert relerr(res[True][0], x.grad) < 3e-3
    assert relerr(res[True][0], res[False][0]) < 1e-6        # same products and the same order of additions
    if not (K == 1 and mode == 0):
        assert res[True][1] == res[False][1] - 1               # one launch fewer: no avc_fold_add_fwd
