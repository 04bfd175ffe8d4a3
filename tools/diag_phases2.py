"""GPU diagnostic: per-role wait / work cycles of the persistent conv kernel (conv_tc2.cu, avc_tc2_set_debug)."""
import os, sys
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch
from adaptive_voice_conversion_b200.engine import A4, Engine
from adaptive_voice_conversion_b200.config import default_config
dev = torch.device("cuda", 0)
eng = Engine(default_config(80), dev)
B = int(os.environ.get("DIAG_B", "256"))
for (Cin, Cout, K, T, kw, tag) in [(128, 128, 5, 128, dict(norm=True, relu=True), "conv5 T128 IN"), (128, 128, 5, 128, dict(), "conv5 T128 plain"),
                                   (1104, 128, 1, 128, dict(norm=True, relu=True), "in_conv"), (128, 128, 5, 64, dict(norm=True, relu=True), "conv5 T64"),
                                   (128, 128, 5, 16, dict(norm=True, relu=True), "conv5 T16"), (80, 128, 8, 128, dict(relu=True), "bank k8")]:
    w = torch.randn(Cout, Cin, K, device=dev) * 0.05
    P = {"r.weight": w, "r.bias": torch.zeros(Cout, device=dev)}
    eng.packed.pop("r", None); eng.conv_names = lambda: ["r"]; eng.pack_weights(P, need_dgrad=False)
    x = A4.empty(B, Cin, T, dev); x.t.normal_()
    x.tf32 = True   # as in the real model (producers round): the kernel skips its rounding pass
    train = bool(kw)
    for _ in range(3):
        eng.conv(P, "r", x, train=train, **kw)
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(10):
        eng.conv(P, "r", x, train=train, **kw)
    e1.record(); torch.cuda.synchronize()
    us = e0.elapsed_time(e1) * 100
    dbg = torch.zeros(16 * 256, dtype=torch.int64, device=dev)
    eng.lib.avc_tc2_set_debug(dbg.data_ptr())
    eng.conv(P, "r", x, train=train, **kw)
    torch.cuda.synchronize()
    eng.lib.avc_tc2_set_debug(None)
    t = dbg.view(-1, 16).cpu()
    t = t[t[:, 0] != 0]
    f = lambda i: float(t[:, i].float().mean())
    life = (t[:, 1] - t[:, 0]).float()
    print(f"{tag:18s} {us:6.1f} us/launch incl. python (hot L2)  CTAs {len(t)}  tiles/CTA {f(12):.2f}")
    print(f"  CTA life mean {life.mean():7.0f} max {life.max():7.0f} cyc = {life.max() / 1965:5.1f} us | producer wait-empty {f(2):6.0f} | patch wait-full {f(3):6.0f} work {f(4):6.0f}"
          f" | mma wait-ready {f(5):6.0f} wait-acc {f(6):5.0f} issue {f(7):6.0f} | epi wait-acc {f(8):6.0f} acc-pass {f(9):5.0f} params {f(10):5.0f} c-rows {f(11):5.0f} out-rows {f(13):5.0f} end-bar {f(14):5.0f}", flush=True)
eng.check_tc_status()
