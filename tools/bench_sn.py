"""Cost of the decoder's spectral norm (Decoder.sn) on the GPU.

    python tools/bench_sn.py [--out result.json]

1. Kernel times: avc_spectral_norm (iterate, fixed) and avc_spectral_norm_bwd on the 26 decoder layers of the
   c_in 80 and c_in 512 models, each call captured 50 times into a CUDA graph and timed with CUDA events over replays
   (so the time is the device's, launch gaps included, without Python's enqueue cost).
2. Step time of the fused training step (Solver.run_steps on synthetic batches, graph replay) with sn False and
   sn True, alternated window by window in this one process, at c_in 80 B 256 and c_in 512 B 128.
Prints one JSON line with the card's name and power limit beside the numbers.
"""
from __future__ import annotations

import argparse
import contextlib
import io
import json
import os
import sys
import tempfile
import types

import torch

from _harness import card, graph_us, median_wall_s

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import oracle.ae_oracle as orc  # noqa: E402


def config(c_in, sn, batch=None):
    cfg = orc.default_config(c_in)
    cfg["Decoder"]["sn"] = sn
    if batch is not None:
        cfg["data_loader"]["batch_size"] = batch
    return cfg


def kernel_times(c_in):
    from adaptive_voice_conversion_b200.model import AE
    torch.manual_seed(0)
    model = AE(config(c_in, True)).cuda()
    eng = model.engine(torch.device("cuda", torch.cuda.current_device()))
    P = dict(model.named_parameters())
    P.update(model.named_buffers())
    eng.bind_spectral_norm(P)
    G = {n: torch.randn_like(p) for n, p in model.named_parameters() if n.endswith(".weight_orig")}
    eng.bind_spectral_norm(P, G)
    names = eng.sn_names()
    floats = sum(P[n + ".weight_orig"].numel() for n in names)
    with torch.no_grad():
        out = {"layers": len(names), "weight_MB": round(4 * floats / 1e6, 2),
               "iterate_us": graph_us(lambda: eng.spectral_norm(P, True), 50, 20),
               "fixed_us": graph_us(lambda: eng.spectral_norm(P, False), 50, 20),
               "bwd_us": graph_us(lambda: eng.spectral_norm_bwd(P, G), 50, 20)}
    return out


def step_times(c_in, batch, steps, windows):
    from adaptive_voice_conversion_b200.solver import Solver
    solvers = {}
    td = tempfile.mkdtemp()
    for sn in (False, True):
        args = types.SimpleNamespace(data_dir="synthetic", train_set="train", train_index_file="", logdir=os.path.join(td, "log"),
                                     load_model=False, load_opt=False, store_model_path=os.path.join(td, f"m{int(sn)}"),
                                     load_model_path=os.path.join(td, f"m{int(sn)}"), summary_steps=1, save_steps=10 ** 9,
                                     tag="t", iters=0)
        with contextlib.redirect_stdout(io.StringIO()):
            s = Solver(config(c_in, sn, batch), args)
        s.run_steps(10)            # eager warm-up, graph capture, replays
        torch.cuda.synchronize()
        solvers[sn] = s
    ms = {False: [], True: []}
    for _ in range(windows):
        for sn in (False, True):
            ms[sn].append(1000.0 * median_wall_s(lambda: solvers[sn].run_steps(steps), 1, warmup=0) / steps)
    med = {sn: sorted(v)[len(v) // 2] for sn, v in ms.items()}
    return {"c_in": c_in, "batch": batch, "steps_per_window": steps, "sn_false_ms": ms[False], "sn_true_ms": ms[True],
            "median_sn_false_ms": med[False], "median_sn_true_ms": med[True],
            "overhead_ms": med[True] - med[False], "overhead_frac": med[True] / med[False] - 1.0}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", default=None)
    ap.add_argument("--steps", type=int, default=50)
    ap.add_argument("--windows", type=int, default=5)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_sn.py needs a GPU")
    res = {"card": card(), "kernels": {f"c{c}": kernel_times(c) for c in (80, 512)},
           "steps": [step_times(80, 256, a.steps, a.windows), step_times(512, 128, a.steps, a.windows)]}
    line = json.dumps(res)
    print(line)
    if a.out:
        with open(a.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
