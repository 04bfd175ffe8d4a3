"""GPU diagnostic: ablation timing of the persistent conv kernel (conv_tc2.cu, AVC_T2_VARIANT bits 16..256).

Each probe removes ONE resource user from the kernel (results are wrong, only the time is read): what the launch
time falls to tells which resource the real kernel is waiting for.  Timed like bench.py's roofline leg: a CUDA graph
of 20 back-to-back launches on rotating >L2 inputs, CUDA events on the launching stream.
"""
import os, sys
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch
from adaptive_voice_conversion_b200.engine import A4, Engine
from adaptive_voice_conversion_b200.config import default_config

dev = torch.device("cuda", 0)
eng = Engine(default_config(80), dev)
B = int(os.environ.get("DIAG_B", "256"))
PROBES = [(0, "full kernel"), (16, "weights 1 KB/stage"), (256, "no input rows"), (16 + 256, "no copies"), (64, "no MMAs"),
          (128, "no accumulator pass"), (32, "no store pass"), (32 + 128, "no epilogue"), (16 + 256 + 32 + 128, "MMAs only"),
          (64 + 32 + 128, "copies only"), (16 + 256 + 64 + 128, "stores only"), (16 + 256 + 64 + 32 + 128, "empty pipeline"),
          (2048, "full, one patch warp"), (2048 + 496, "empty, one patch warp")]
if os.environ.get("DIAG_PROBES"):
    keep = {int(v) for v in os.environ["DIAG_PROBES"].split(",")}
    PROBES = [p for p in PROBES if p[0] in keep]
SHAPES = [(128, 128, 5, 128, dict(norm=True, relu=True), "conv5 T128 IN"), (128, 128, 5, 32, dict(norm=True, relu=True), "conv5 T32 IN"),
          (1104, 128, 1, 128, dict(norm=True, relu=True), "in_conv 1104")]


def time_graph(fn, reps=20):
    side = torch.cuda.Stream(dev)
    g = torch.cuda.CUDAGraph()
    keep = []
    with torch.cuda.stream(side):
        with torch.cuda.graph(g, stream=side):
            for i in range(reps):
                keep.append(fn(i))
        g.replay(); side.synchronize()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record(side)
        for _ in range(3):
            g.replay()
        e1.record(side); side.synchronize()
    return e0.elapsed_time(e1) / (3 * reps) * 1e3


for (Cin, Cout, K, T, kw, tag) in SHAPES:
    w = torch.randn(Cout, Cin, K, device=dev) * 0.05
    P = {"r.weight": w, "r.bias": torch.zeros(Cout, device=dev)}
    eng.packed.pop("r", None); eng.conv_names = lambda: ["r"]; eng.pack_weights(P, need_dgrad=False)
    nbuf = max(2, int(200e6 // (B * Cin * T * 4)) + 1)
    xs = [A4.empty(B, Cin, T, dev) for _ in range(nbuf)]
    for x in xs:
        x.t.normal_()
    for pre in (True, False):
        for x in xs:
            x.tf32 = pre
        row = []
        for v, name in PROBES:
            eng.lib.avc_tc2_set_variant(v)
            for i in range(2):
                eng.conv(P, "r", xs[i % nbuf], train=True, **kw)
            torch.cuda.synchronize()
            us = time_graph(lambda i: eng.conv(P, "r", xs[i % nbuf], train=True, **kw))
            row.append(f"{name} {us:6.2f}")
        eng.lib.avc_tc2_set_variant(0)
        print(f"{tag:14s} B={B} input {'pre-rounded' if pre else 'fp32 (rounding pass)'}: " + " | ".join(row), flush=True)
torch.cuda.synchronize()
# the probes leave garbage in the status word's neighbourhood only if a wait timed out: report it
print("tc status:", int(eng.tc_status.item()))
