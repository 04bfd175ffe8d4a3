"""GPU diagnostic: per-CTA phase timing (main loop vs epilogue) of the tensor-core conv kernel."""
import os, sys
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch
from adaptive_voice_conversion_b200.engine import A4, Engine
from adaptive_voice_conversion_b200.config import default_config
dev = torch.device("cuda", 0)
eng = Engine(default_config(80), dev)
for (Cin, Cout, K, T, tag) in [(128, 128, 5, 128, "conv5 T128"), (1104, 128, 1, 128, "in_conv"), (128, 128, 5, 16, "conv5 T16")]:
    w = torch.randn(Cout, Cin, K, device=dev) * 0.05
    P = {"r.weight": w, "r.bias": torch.zeros(Cout, device=dev)}
    eng.packed.pop("r", None); eng.conv_names = lambda: ["r"]; eng.pack_weights(P, need_dgrad=False)
    x = A4.empty(256, Cin, T, dev); x.t.normal_()
    x.tf32 = True   # as in the real model (producers round): the kernel skips its rounding pass
    for _ in range(3):
        eng.conv(P, "r", x, norm=True, relu=True, train=True)
    dbg = torch.zeros(12 * 1024, dtype=torch.int64, device=dev)
    eng.lib.avc_tc_set_debug(dbg.data_ptr())
    eng.conv(P, "r", x, norm=True, relu=True, train=True)
    torch.cuda.synchronize()
    eng.lib.avc_tc_set_debug(None)
    t = dbg.view(-1, 12).cpu()
    t = t[t[:, 0] != 0]
    main, epi = (t[:, 1] - t[:, 0]).float(), (t[:, 2] - t[:, 1]).float()
    span = float(t[:, 2].max() - t[:, 0].min())
    f = lambda i: float(t[:, i].float().mean())
    print(f"{tag:12s} producer wait-empty {f(4):8.0f} | patcher wait-full {f(6):8.0f} work {f(7):8.0f} | mma wait-ready {f(8):8.0f} issue {f(9):8.0f}")
    print(f"{tag:12s} CTAs {len(t):4d}  main loop {main.mean():8.0f} cyc (max {main.max():8.0f})  epilogue {epi.mean():8.0f} cyc (max {epi.max():8.0f})  first-start->last-end {span:8.0f}")
