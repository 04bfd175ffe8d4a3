"""GPU diagnostic: per-CTA phase cycles of the tensor-core weight-gradient kernels (avc_wgrad_tc_set_debug), TMA-staged vs round-1 -staged."""
import os, sys, ctypes as C
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch
from adaptive_voice_conversion_b200.engine import A4, Engine
from adaptive_voice_conversion_b200.config import default_config
from adaptive_voice_conversion_b200 import _lib as L
dev = torch.device("cuda", 0)
eng = Engine(default_config(80), dev)
B = 256
for (Cin, Cout, K, T, S, tag) in [(128, 128, 5, 128, 1, "k5 T128"), (128, 128, 5, 64, 1, "k5 T64"), (128, 128, 5, 16, 1, "k5 T16"),
                                  (1104, 128, 1, 128, 1, "in_conv"), (80, 128, 8, 128, 1, "bank k8"), (128, 128, 5, 64, 2, "k5 s2 Tout64")]:
    Tin = T * S
    x = A4.empty(B, Cin, Tin, dev); x.t.normal_()
    dc = A4.empty(B, Cout, T, dev); dc.t.normal_()
    acc = torch.zeros(int(eng.lib.avc_wgrad_acc_floats(Cout, Cin, K)), device=dev)
    wd = L.WgradDesc()
    wd.B, wd.Cin, wd.Cout, wd.K, wd.stride, wd.pad_left, wd.Tin, wd.Tout = B, Cin, Cout, K, S, K // 2, Tin, T
    wd.x, wd.x_bstride, wd.dc, wd.dc_bstride = x.ptr, x.bstride, dc.ptr, dc.bstride
    st = torch.cuda.current_stream().cuda_stream
    res = {}
    for mode in (1, 0):
        L.set_option("wgrad_split", bool(mode))
        acc.zero_()
        for _ in range(3):
            L.check(eng.lib.avc_conv_wgrad_tc_acc(C.byref(wd), acc.data_ptr(), eng.tc_status.data_ptr(), st), "wgrad")
        torch.cuda.synchronize()
        res[mode] = acc.clone()
        dbg = torch.zeros(8 * 1024, dtype=torch.int64, device=dev)
        eng.lib.avc_wgrad_tc_set_debug(dbg.data_ptr())
        L.check(eng.lib.avc_conv_wgrad_tc_acc(C.byref(wd), acc.data_ptr(), eng.tc_status.data_ptr(), st), "wgrad")
        torch.cuda.synchronize()
        eng.lib.avc_wgrad_tc_set_debug(None)
        t = dbg.view(-1, 8).cpu()
        t = t[t[:, 0] != 0]
        f = lambda i: float(t[:, i].float().mean())
        life = (t[:, 1] - t[:, 0]).float()
        print(f"{tag:13s} {'split   ' if mode else 'round-1 '} CTAs {len(t):4d} tiles/CTA {f(7):5.2f}  life mean {life.mean():7.0f} max {life.max():7.0f} cyc = {life.max() / 1965:5.1f} us | staging/wait {f(2):7.0f} wait-free {f(3):6.0f}"
              f" mma-issue {f(4):6.0f} drain {f(5):6.0f} epilogue {f(6):6.0f}", flush=True)
    L.set_option("wgrad_split", True)
    print(f"{tag:13s} split vs round-1 accumulated result: rel-L2 diff {float((res[1] - res[0]).norm() / res[0].norm()):.2e}", flush=True)
eng.check_tc_status()
