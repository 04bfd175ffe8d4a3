"""Cost of the held-out evaluation (adaptive_voice_conversion_b200/evaluate.py) on the GPU.

    python tools/bench_eval.py [--dir DATA_ROOT] [--out result.json]

For c_in 512 at B 128 and c_in 80 at B 256, on a generated data directory whose `in_test` set has 10 000 index entries
(the size preprocess.py's --testing_samples gives by default):
1. One Solver.evaluate(): host clock around a call that ends in a device synchronise, median of 3 (after one warm-up).
2. avc_eval_losses alone on one full batch: CUDA events over 200 launches on inputs rotated past the L2, its bytes
   (dec and x once, mu and ls, the 16-byte rows) and their share of the H100 SXM's 3.35 TB/s.
3. The training step of the same Solver (run_steps, graph replay; median of 3 windows of 40 steps), so that the
   evaluation is also given in steps.
Each model is saved as <DATA_ROOT>/c<c_in>/model.ckpt, the input of `python evaluate.py -m ... -d <DATA_ROOT>/c<c_in>`.
Prints one JSON line with the card's name and power limit beside the numbers.
"""
from __future__ import annotations

import argparse
import contextlib
import io
import itertools
import json
import os
import pickle
import sys
import tempfile
import types

import numpy as np
import torch

from _harness import card, events_ms, median_wall_s

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

HBM_BYTES_PER_S = 3.35e12
SEG = 128


def write_set(root, name, n_mels, n_entries, seed, n_speakers=20, utts_per_speaker=10):
    """VCTK-like: 20 speakers x 10 utterances of 129-600 frames, N(0,1) mels, n_entries random crops."""
    rng = np.random.default_rng(seed)
    data = {f"p{400 + s}_{u:03d}": rng.standard_normal((int(rng.integers(SEG + 1, 601)), n_mels)).astype(np.float32)
            for s in range(n_speakers) for u in range(utts_per_speaker)}
    utts = list(data)
    index = []
    for _ in range(n_entries):
        utt = utts[int(rng.integers(len(utts)))]
        index.append([utt, int(rng.integers(0, len(data[utt]) - SEG + 1))])
    with open(os.path.join(root, f"{name}.pkl"), "wb") as f:
        pickle.dump(data, f)
    with open(os.path.join(root, f"{name}_samples_{SEG}.json"), "w") as f:
        json.dump(index, f)


def kernel_time(c_in, B, reps=200, rotate_bytes=256 << 20):
    """avc_eval_losses on one full batch, rotating over enough input sets (>= 256 MB) that they do not stay in the 50 MB
    L2: the time is that of reading HBM."""
    from adaptive_voice_conversion_b200 import _lib as L
    g = torch.Generator(device="cuda").manual_seed(0)
    C_lat, T_lat = 128, SEG // 8
    nbytes = 4 * B * (2 * c_in * SEG + 2 * C_lat * T_lat) + 16 * B
    descs, keep = [], []
    for _ in range(-(-rotate_bytes // nbytes)):
        dec = torch.randn((B, c_in // 4, SEG, 4), device="cuda", generator=g)
        x = torch.randn((B, c_in, SEG), device="cuda", generator=g)
        mu = torch.randn((B, C_lat // 4, T_lat, 4), device="cuda", generator=g)
        ls = torch.randn((B, C_lat // 4, T_lat, 4), device="cuda", generator=g)
        out = torch.zeros((B, 2), dtype=torch.float64, device="cuda")
        keep.append((dec, x, mu, ls, out))
        descs.append(L.EvalDesc(B=B, C=c_in, T=SEG, C_lat=C_lat, T_lat=T_lat, dec=dec.data_ptr(), x=x.data_ptr(),
                                mu=mu.data_ptr(), ls=ls.data_ptr(), out=out.data_ptr(), first=0))
    lib, st = L.load(), torch.cuda.current_stream().cuda_stream
    for d in descs:
        L.check(lib.avc_eval_losses(d, st))
    n = itertools.count()
    us = 1e3 * events_ms(lambda: lib.avc_eval_losses(descs[next(n) % len(descs)], st), reps, 0)
    return {"us": round(us, 2), "bytes": nbytes, "input_sets_rotated": len(descs), "GB_per_s": round(nbytes / us / 1e3, 1),
            "share_of_3.35TB_per_s": round(nbytes / (us * 1e-6) / HBM_BYTES_PER_S, 3)}


def bench(root, c_in, B, n_entries):
    from adaptive_voice_conversion_b200.config import default_config
    from adaptive_voice_conversion_b200.solver import Solver
    d = os.path.join(root, f"c{c_in}")
    os.makedirs(d, exist_ok=True)
    write_set(d, "train", c_in, 4 * B, seed=1)
    write_set(d, "in_test", c_in, n_entries, seed=2)
    cfg = default_config(c_in)
    cfg["data_loader"]["batch_size"] = B
    args = types.SimpleNamespace(data_dir=d, train_set="train", train_index_file=f"train_samples_{SEG}.json",
                                 logdir=os.path.join(d, "log"), load_model=False, load_opt=False,
                                 store_model_path=os.path.join(d, "model"), load_model_path=os.path.join(d, "model"),
                                 summary_steps=10 ** 9, save_steps=10 ** 9, tag="bench", iters=0, eval_steps=0,
                                 eval_sets="in_test")
    torch.manual_seed(0)
    with contextlib.redirect_stdout(io.StringIO()):
        s = Solver(cfg, args)
        s.run_steps(8)                      # capture and warm the training graph
        s.evaluate()                        # warm-up: loads the set, allocator, packs
    times, results = [], []
    eval_s = median_wall_s(lambda: results.append(s.evaluate()), 3, warmup=0, samples=times)
    res = results[-1]
    n_steps, windows = 40, []
    step_s = median_wall_s(lambda: s.run_steps(n_steps), 3, warmup=0, samples=windows) / n_steps
    s.save_model(s.iteration - 1)          # <d>/model.ckpt for `python evaluate.py`
    return {"c_in": c_in, "batch": B, "entries": n_entries, "batches": -(-n_entries // B),
            "evaluate_s_median_of_3": round(eval_s, 4), "evaluate_s_all": [round(t, 4) for t in times],
            "segments_per_s": round(n_entries / eval_s), "train_step_ms": round(step_s * 1e3, 3),
            "train_step_ms_windows": [round(w * 1e3 / n_steps, 3) for w in windows],
            "evaluate_in_train_steps": round(eval_s / step_s, 1), "kernel": kernel_time(c_in, B),
            "in_test": res["in_test"]}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--dir", default=None, help="where the data directories are written (default: a temporary one)")
    ap.add_argument("--entries", type=int, default=10000)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_eval.py measures on the GPU; no CUDA device is visible")
    root = a.dir or tempfile.mkdtemp(prefix="avc_bench_eval_")
    result = {"card": card(), "runs": [bench(root, 512, 128, a.entries), bench(root, 80, 256, a.entries)], "dir": root}
    line = json.dumps(result)
    print(line)
    if a.out:
        with open(a.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
