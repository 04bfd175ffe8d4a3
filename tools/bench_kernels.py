"""GPU micro-benchmark (CUDA-graph timed) of the main kernels at the B=256 training shapes."""
import os, sys
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch
from adaptive_voice_conversion_b200.engine import A4, Engine
from adaptive_voice_conversion_b200.config import default_config
from adaptive_voice_conversion_b200 import _lib as L
from _harness import graph_us

B = 256


def main():
    dev = torch.device("cuda", 0)
    for prec in ("tf32", "fp32"):
        eng = Engine(default_config(80), dev); eng.precision = prec
        print(f"--- precision {prec}")
        for (Cin, Cout, K, T, norm, tag) in [(128, 128, 5, 128, True, "conv5 T128"), (128, 128, 5, 64, True, "conv5 T64"), (128, 128, 5, 16, True, "conv5 T16"),
                                             (1104, 128, 1, 128, True, "in_conv"), (80, 128, 8, 128, False, "bank k8"), (128, 256, 5, 64, True, "shuffle conv T64")]:
            w = torch.randn(Cout, Cin, K, device=dev) * 0.05
            P = {"r.weight": w, "r.bias": torch.zeros(Cout, device=dev)}
            G = {k: torch.zeros_like(v) for k, v in P.items()}
            eng.packed.pop("r", None); eng.conv_names = lambda: ["r"]; eng.pack_weights(P, need_dgrad=True)
            x = A4.empty(B, Cin, T, dev); x.t.normal_()
            shuffle = Cout == 256
            out, rec = eng.conv(P, "r", x, shuffle=shuffle, norm=norm, relu=True, train=True)
            dy = A4.empty(out.B, out.C, out.T, dev); dy.t.normal_()
            t_fwd = graph_us(lambda: eng.conv(P, "r", x, shuffle=shuffle, norm=norm, relu=True, train=True), 10, 3)
            flops = 2.0 * Cin * Cout * K * T * B
            # backward pieces
            dc = A4.empty(B, Cout, T, dev); dc.t.normal_()
            wd = L.WgradDesc()
            wd.B, wd.Cin, wd.Cout, wd.K, wd.stride, wd.pad_left, wd.Tin, wd.Tout = B, Cin, Cout, K, 1, K // 2, T, T
            wd.x, wd.x_bstride, wd.dc, wd.dc_bstride, wd.dw = x.ptr, x.bstride, dc.ptr, dc.bstride, G["r.weight"].data_ptr()
            t_wg = graph_us(lambda: eng.wgrad(wd, "r"), 10, 3)
            t_bwd = graph_us(lambda: eng.conv_bwd(P, G, rec, dy), 10, 3)
            print(f"{tag:18s} fwd {t_fwd:8.1f} us ({flops / t_fwd / 1e6:7.1f} TF/s)  wgrad {t_wg:8.1f} us ({flops / t_wg / 1e6:7.1f} TF/s)  full conv_bwd {t_bwd:8.1f} us")
        eng.check_tc_status()


if __name__ == "__main__":
    main()
