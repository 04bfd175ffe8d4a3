"""Cost of the MCD-DTW evaluation (adaptive_voice_conversion_b200/mcd.py) on the GPU.

    python tools/bench_mcd.py [--pairs 10000] [--out result.json]

1. avc_mel_cepstrum and avc_dtw alone on synthetic VCTK-like pairs (lengths uniform in 100-600 frames, 512 mels,
   24 coefficients): CUDA events around each launch, median of 3 after one warm-up.  Cells (sum of Tx Ty) per second
   and FP64 operations per second are computed from the shapes: a DTW cell is 3D + 2 operations (D subtractions,
   multiplications and additions, the square root, the accumulation), a cepstrum row n_mels (2D + 4) (the
   multiply-adds of the DCT and the four operations of the log amplitude).
2. `evaluate.py -mcd` end to end on a generated out_test-like set (10 speakers reading 40 shared sentences, each line
   read with probability 0.6, and 10 lines of their own; 100-600 frames) with a random-init c_in 512 model: the
   evaluate_mcd call timed with a host clock around a call that ends in a device synchronise (its result is copied to
   the host), after one warm-up, and the CLI run once.
3. The float64 numpy restatement (tests/_mcd_ref.py) on a subset of the pairs, as the host comparison.
Generated data lives in a temporary directory.  Prints one JSON line with the card's name and power limit.
"""
from __future__ import annotations

import argparse
import contextlib
import io
import json
import os
import pickle
import sys
import tempfile
import time

import numpy as np
import torch

from _harness import card, median_events_s

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))


def kernels(n_pairs, dims, n_mels, host_pairs):
    from _mcd_ref import dtw64
    from adaptive_voice_conversion_b200 import mcd as M
    rng = np.random.default_rng(0)
    tx, ty = rng.integers(100, 601, n_pairs), rng.integers(100, 601, n_pairs)
    lengths = [int(v) for v in np.concatenate([tx, ty])]
    attr = {"mean": rng.uniform(0.3, 0.7, n_mels).astype(np.float32), "std": rng.uniform(0.1, 0.3, n_mels).astype(np.float32)}
    g = torch.Generator(device="cuda").manual_seed(0)
    mels = torch.randn((sum(lengths), n_mels), generator=g, device="cuda")
    parts = list(torch.split(mels, lengths))
    t_cep = median_events_s(lambda: M.mel_cepstrum(parts, attr, dims=dims), 3)
    ceps = M.mel_cepstrum(parts, attr, dims=dims)
    del mels, parts
    xs, ys = ceps[:n_pairs], ceps[n_pairs:]
    t_dtw = median_events_s(lambda: M.dtw(xs, ys), 3)
    rows = sum(lengths)
    cells = int((tx * ty).sum())
    sub = range(host_pairs)
    t0 = time.perf_counter()
    for i in sub:
        dtw64(xs[i].cpu().numpy(), ys[i].cpu().numpy())
    t_host = time.perf_counter() - t0
    host_cells = int((tx[:host_pairs] * ty[:host_pairs]).sum())
    return {
        "pairs": n_pairs, "dims": dims, "n_mels": n_mels, "cells": cells, "rows": rows,
        "mel_cepstrum_s": t_cep, "mel_cepstrum_rows_per_s": rows / t_cep,
        "mel_cepstrum_fp64_ops_per_s": rows * n_mels * (2 * dims + 4) / t_cep,
        "dtw_s": t_dtw, "dtw_cells_per_s": cells / t_dtw, "dtw_fp64_ops_per_s": cells * (3 * dims + 2) / t_dtw,
        "numpy_dtw_pairs": host_pairs, "numpy_dtw_s": t_host, "numpy_dtw_cells_per_s": host_cells / t_host,
    }


def write_out_test(root, n_mels, seed=0, n_speakers=10, n_shared=40, n_own=10):
    rng = np.random.default_rng(seed)
    data = {}
    for s in range(n_speakers):
        for k in range(n_shared + n_own):
            if k < n_shared and rng.random() > 0.6:
                continue
            u = f"p{400 + s}_{k:03d}"
            data[u + ".wav"] = rng.standard_normal((int(rng.integers(100, 601)), n_mels)).astype(np.float32)
            text = f"Shared sentence number {k}." if k < n_shared else f"Speaker {s} says line {k}."
            os.makedirs(os.path.join(root, "txt", f"p{400 + s}"), exist_ok=True)
            with open(os.path.join(root, "txt", f"p{400 + s}", u + ".txt"), "w") as f:
                f.write(text + "\n")
    with open(os.path.join(root, "out_test.pkl"), "wb") as f:
        pickle.dump(data, f)
    keys = sorted(u for u in data if len(data[u]) > 128)       # HeldOut's segments of 128 frames
    index = [[keys[int(rng.integers(len(keys)))], 0] for _ in range(256)]
    with open(os.path.join(root, "out_test_samples_128.json"), "w") as f:
        json.dump(index, f)
    with open(os.path.join(root, "attr.pkl"), "wb") as f:
        pickle.dump({"mean": rng.uniform(0.3, 0.7, n_mels).astype(np.float32),
                     "std": rng.uniform(0.1, 0.3, n_mels).astype(np.float32)}, f)
    return data


def end_to_end(tmp):
    import evaluate as cli
    from adaptive_voice_conversion_b200 import mcd as M
    from adaptive_voice_conversion_b200.config import load_config
    from adaptive_voice_conversion_b200.model import AE
    cfg = load_config(os.path.join(ROOT, "config.yaml"))
    data = write_out_test(tmp, cfg["ContentEncoder"]["c_in"])
    torch.manual_seed(0)
    model = AE(cfg).cuda()
    ckpt = os.path.join(tmp, "model.ckpt")
    torch.save(model.state_dict(), ckpt)
    model.eval()
    with open(os.path.join(tmp, "attr.pkl"), "rb") as f:
        attr = pickle.load(f)
    texts = M.read_transcripts(os.path.join(tmp, "txt"), data)
    M.evaluate_mcd(model, data, attr, texts)
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    res = M.evaluate_mcd(model, data, attr, texts)
    t_mcd = time.perf_counter() - t0
    out = io.StringIO()
    t0 = time.perf_counter()
    with contextlib.redirect_stdout(out):
        cli.main(["-c", os.path.join(ROOT, "config.yaml"), "-m", ckpt, "-d", tmp, "-eval_sets", "out_test", "-mcd",
                  "-transcripts", os.path.join(tmp, "txt"), "-o", os.path.join(tmp, "eval.json")])
    t_cli = time.perf_counter() - t0
    return {"utterances": len(data), "triplets": res["n"], "n_short": res["n_short"], "mcd": res["mcd"],
            "mcd_source": res["mcd_source"], "evaluate_mcd_s": t_mcd, "triplets_per_s": res["n"] / t_mcd,
            "cli_s": t_cli, "cli_output": out.getvalue().strip().splitlines()}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--pairs", type=int, default=10000)
    ap.add_argument("--host_pairs", type=int, default=20)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    res = {"card": card()}
    res["kernels_d24"] = kernels(a.pairs, 24, 512, a.host_pairs)
    print(json.dumps(res), file=sys.stderr)
    torch.cuda.empty_cache()
    with tempfile.TemporaryDirectory() as tmp:
        res["evaluate_mcd_c512"] = end_to_end(tmp)
    line = json.dumps(res)
    print(line)
    if a.out:
        with open(a.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
