"""GPU: conv weight gradients accumulated in place (vector atomics + one flush launch,
csrc/wgrad_tc.cu ATOMIC / avc_wgrad_acc_flush) against the two-stage deterministic path and
against autograd.  Default path."""
import math
import os

import pytest
import torch

import oracle.ae_oracle as orc
from test_gpu_kernels import relerr, rnd, to_a4

pytestmark = pytest.mark.gpu
TOL = 3e-3


@pytest.fixture(scope="module")
def eng():
    from adaptive_voice_conversion_b200.engine import Engine
    e = Engine(orc.default_config(80), torch.device("cuda", 0))
    e.precision = "tf32"
    return e


CASES = [(5, 128, 128, 5, 128, 1), (37, 128, 128, 5, 16, 1), (9, 128, 256, 5, 32, 1), (3, 80, 128, 8, 128, 1), (2, 1104, 128, 1, 128, 1),
         (3, 128, 80, 1, 64, 1), (300, 128, 128, 5, 16, 1), (19, 128, 128, 5, 32, 2)]


@pytest.mark.parametrize("B,Cin,Cout,K,T,stride", CASES)
def test_wgrad_acc_matches_inline_and_autograd(eng, B, Cin, Cout, K, T, stride):
    import ctypes as C
    from adaptive_voice_conversion_b200 import _lib as L
    x = rnd((B, Cin, T), 1)
    w = (rnd((Cout, Cin, K), 2) / math.sqrt(Cin * K)).requires_grad_(True)
    y = orc.reflect_conv1d(x, w, None, stride)
    dc = rnd(tuple(y.shape), 3)
    y.backward(dc)
    xa, da = to_a4(eng, x), to_a4(eng, dc)
    P = {"blk.weight": w.detach().cuda(), "blk.bias": torch.zeros(Cout).cuda()}
    res = {}
    for mode in ("inline", "acc"):
        G = {k: torch.full_like(v, 0.25) for k, v in P.items()}     # accumulates (+=) into existing content
        eng.conv_names = lambda: ["blk"]
        eng.wgrad_acc = mode == "acc"
        eng._wg_acc = None
        eng.prepare_wgrad_acc(P, G)
        assert (eng._wg_acc is not None) == (mode == "acc")
        wd = L.WgradDesc()
        wd.B, wd.Cin, wd.Cout, wd.K, wd.stride, wd.pad_left, wd.Tin, wd.Tout = B, Cin, Cout, K, stride, K // 2, T, y.shape[-1]
        wd.x, wd.x_bstride, wd.dc, wd.dc_bstride, wd.dw = xa.ptr, xa.bstride, da.ptr, da.bstride, G["blk.weight"].data_ptr()
        assert int(eng.lib.avc_wgrad_tc_scratch_floats(C.byref(wd))) > 0
        for _ in range(2):      # twice: the flush must leave the accumulation buffer zeroed
            eng.wgrad(wd, "blk")
            eng.flush_wgrad()
        eng.check_tc_status()
        if mode == "acc":
            assert float(eng._wg_acc["arena"].abs().max()) == 0.0
        res[mode] = (G["blk.weight"].cpu() - 0.25) / 2
    eng.wgrad_acc, eng._wg_acc = False, None
    assert relerr(res["inline"], w.grad) < TOL
    assert relerr(res["acc"], w.grad) < TOL
    assert relerr(res["acc"], res["inline"]) < 1e-5      # same products, different summation order


def test_trainer_step_with_wgrad_acc(tmp_path):
    """Whole step: in-place accumulation vs the deterministic path, same weights / data / eps."""
    import types
    from adaptive_voice_conversion_b200.solver import Solver
    outs = {}
    for mode in ("0", "1"):
        os.environ["AVC_WGRAD_ACC"] = mode
        try:
            cfg = orc.default_config(80)
            cfg["data_loader"]["batch_size"] = 4
            args = types.SimpleNamespace(data_dir="synthetic", train_set="train", train_index_file="", logdir=str(tmp_path / "log"),
                                         load_model=False, load_opt=False, store_model_path=str(tmp_path / "model"),
                                         load_model_path=str(tmp_path / "model"), summary_steps=1, save_steps=1000, tag="t", iters=0)
            solver = Solver(cfg, args)
            solver.model.load_state_dict(orc.init_state(cfg, seed=0), strict=True)
            solver.trainer.eng.wgrad_acc = mode == "1"      # the engine is cached per model/device: set explicitly
            solver.trainer.eng.prepare_wgrad_acc(solver.trainer.P, solver.trainer.G)
            solver.trainer.eng.pack_weights(solver.trainer.P, need_dgrad=True)
            g = torch.Generator().manual_seed(1)
            x = torch.randn((4, 80, 128), generator=g).cuda()
            eps = torch.randn((4, 128, 16), generator=g).cuda()
            solver.trainer._fwd_bwd(x, eps)
            torch.cuda.synchronize()
            outs[mode] = solver.opt.flat_g.clone()
        finally:
            os.environ.pop("AVC_WGRAD_ACC", None)
    num = float((outs["1"] - outs["0"]).double().norm() / outs["0"].double().norm())
    assert num < 1e-5, num
