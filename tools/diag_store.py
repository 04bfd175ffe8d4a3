"""GPU diagnostic: how fast can one SM push bytes to L2 / HBM?  (avc_probe_store)"""
import os, sys
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch
from adaptive_voice_conversion_b200 import _lib as L
lib = L.load()
dev = torch.device("cuda", 0)
st = torch.cuda.current_stream().cuda_stream
for ctas in (132, 32, 1):
    for kb in (64, 256, 2048):
        nbytes = kb * 1024
        dst = torch.empty(ctas * nbytes // 4, device=dev)
        cyc = torch.zeros(ctas, dtype=torch.int64, device=dev)
        for mode, name in ((0, "STG.128"), (1, "bulk 2KB"), (2, "both")):
            for _ in range(2):
                L.check(lib.avc_probe_store(dst.data_ptr(), nbytes, ctas, mode, cyc.data_ptr(), st), "probe")
            torch.cuda.synchronize()
            c = cyc.float()
            print(f"ctas {ctas:4d}  {kb:5d} KB/CTA  {name:9s}  {nbytes / float(c.mean()):6.1f} B/clk/SM (mean)  {nbytes / float(c.max()):6.1f} (slowest)  total {ctas * nbytes / float(c.max()) * 1.965 / 1e3:6.2f} TB/s", flush=True)
