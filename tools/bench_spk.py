"""Cost of the speaker measures (adaptive_voice_conversion_b200/speaker_eval.py) on the GPU.

    python tools/bench_spk.py [--n 8000] [--out result.json]

1. avc_spk_eer alone for N vectors (8 000 by default: a VCTK out_test set) at D = 128 (speaker), 256 (content) and
   1024 (mel of 512 bins): CUDA events around the call, median of 3 after one warm-up, and one profiled call
   (torch.profiler) for the time of each kernel.  Trials/s over the whole call.  The score kernel's FP64 rate counts
   2 D operations per trial (a multiply and an add per coordinate, each rounded on its own: no FMA, so at most half
   the data sheet's 33.5 TFLOP/s FP64 vector rate, which counts an FMA as two).  Each counting pass reads every stored
   key once (12 passes, or 18 when the third search runs), so their bound is HBM bandwidth (3.35 TB/s data sheet).
2. avc_time_stats_varlen on a padded batch of 64 mels of 512 bins, lengths 100-600 (extent 640): bytes read (two passes
   over the valid frames) per second.
3. `evaluate.py -spk` end to end on a generated out_test-like set (20 speakers, 20 utterances each, 100-600 frames) with
   a random-init c_in 512 model: the evaluate_speakers call timed with a host clock around a call that ends in a copy
   to the host, after one warm-up, and the CLI run once.
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

FP64_PEAK = 33.5e12      # H100 SXM data sheet, FP64 (non-tensor), FMA counted as two
HBM_PEAK = 3.35e12


def kernel_times(fn):
    """{kernel name: seconds} of one call of fn, from torch.profiler."""
    from torch.profiler import ProfilerActivity, profile
    fn()
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        fn()
        torch.cuda.synchronize()
    out = {}
    for e in prof.key_averages():
        t = getattr(e, "self_device_time_total", 0)
        if t > 0:
            out[e.key] = out.get(e.key, 0.0) + t / 1e6
    return out


def eer_kernel(n, d):
    from adaptive_voice_conversion_b200 import speaker_eval as S
    rng = np.random.default_rng(d)
    labels = rng.integers(0, 100, n).astype(np.int32)
    centres = rng.standard_normal((100, d)) * 0.7 * d ** -0.25
    V = torch.from_numpy((centres[labels] + rng.standard_normal((n, d))).astype(np.float32)).cuda()
    ws = S.eer_workspace(n, "cuda")
    res = S.eer(V, labels, ws)
    t = median_events_s(lambda: S.eer(V, labels, ws), 3)
    k = kernel_times(lambda: S.eer(V, labels, ws))
    pick = lambda name: sum(v for kk, v in k.items() if name in kk)
    trials = n * (n - 1) // 2
    t_score, t_hist = pick("spk_score_kernel"), pick("spk_hist_kernel")
    nt = -(-n // 64)
    key_bytes = nt * (nt + 1) // 2 * 4096 * 8
    # the third search runs only after a non-target rank selection (SpkState.after_q, 32 784 bytes into the state);
    # otherwise its six histogram launches return at once
    passes = 12 + 6 * int(ws[32784:32788].cpu().numpy().view(np.int32)[0])
    return {"n": n, "d": d, "trials": trials, "eer": res["eer"], "call_s": t, "trials_per_s": trials / t,
            "score_kernel_s": t_score, "score_fp64_ops_per_s": 2 * d * trials / t_score,
            "score_share_of_fp64_peak": 2 * d * trials / t_score / FP64_PEAK, "counting_passes": passes,
            "hist_kernels_s": t_hist, "hist_bytes_per_s": passes * key_bytes / t_hist,
            "hist_share_of_hbm_peak": passes * key_bytes / t_hist / HBM_PEAK,
            "step_kernels_s": pick("spk_step_kernel"), "norm_kernel_s": pick("spk_norm_kernel")}


def pooling():
    from adaptive_voice_conversion_b200 import speaker_eval as S
    rng = np.random.default_rng(0)
    lens = rng.integers(100, 601, 64)
    x = torch.randn(64, 512, 640, device="cuda")
    t = median_events_s(lambda: S.time_stats(x, lens), 5)
    lx = torch.from_numpy(lens.astype(np.int32)).cuda()
    from adaptive_voice_conversion_b200 import _lib as L
    out = torch.empty(64, 1024, device="cuda")
    launch = lambda: L.load().avc_time_stats_varlen(x.data_ptr(), out.data_ptr(), 64, 512, 640, lx.data_ptr(),
                                                    torch.cuda.current_stream().cuda_stream)
    t_k = median_events_s(launch, 5)
    read = 2 * int(lens.sum()) * 512 * 4
    return {"batch": 64, "channels": 512, "extent": 640, "wrapper_s": t, "kernel_s": t_k,
            "bytes_read_per_s": read / t_k}


def write_out_test(root, n_mels, n_speakers=20, per_speaker=20, seed=0):
    rng = np.random.default_rng(seed)
    data = {f"p{400 + s}_{k:03d}.wav": rng.standard_normal((int(rng.integers(100, 601)), n_mels)).astype(np.float32)
            for s in range(n_speakers) for k in range(per_speaker)}
    with open(os.path.join(root, "out_test.pkl"), "wb") as f:
        pickle.dump(data, f)
    keys = sorted(u for u in data if len(data[u]) > 128)       # HeldOut's segments of 128 frames
    with open(os.path.join(root, "out_test_samples_128.json"), "w") as f:
        json.dump([[keys[int(rng.integers(len(keys)))], 0] for _ in range(256)], f)
    return data


def end_to_end(tmp):
    import evaluate as cli
    from adaptive_voice_conversion_b200 import speaker_eval as S
    from adaptive_voice_conversion_b200.config import load_config
    from adaptive_voice_conversion_b200.model import AE
    cfg = load_config(os.path.join(ROOT, "config.yaml"))
    data = write_out_test(tmp, cfg["ContentEncoder"]["c_in"])
    torch.manual_seed(0)
    model = AE(cfg).cuda()
    ckpt = os.path.join(tmp, "model.ckpt")
    torch.save(model.state_dict(), ckpt)
    model.eval()
    S.evaluate_speakers(model, data)
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    res = S.evaluate_speakers(model, data)
    t_spk = time.perf_counter() - t0
    out = io.StringIO()
    t0 = time.perf_counter()
    with contextlib.redirect_stdout(out):
        cli.main(["-c", os.path.join(ROOT, "config.yaml"), "-m", ckpt, "-d", tmp, "-eval_sets", "out_test", "-spk",
                  "-o", os.path.join(tmp, "eval.json")])
    t_cli = time.perf_counter() - t0
    return {"utterances": len(data), "pairs": res["conversion"]["n"], "eer": {k: v["eer"] for k, v in res["eer"].items()},
            "evaluate_speakers_s": t_spk, "cli_s": t_cli, "cli_output": out.getvalue().strip().splitlines()}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--n", type=int, default=8000)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    res = {"card": card()}
    res["eer"] = [eer_kernel(a.n, d) for d in (128, 256, 1024)]
    torch.cuda.empty_cache()
    res["pooling"] = pooling()
    print(json.dumps(res), file=sys.stderr)
    with tempfile.TemporaryDirectory() as tmp:
        res["evaluate_spk_c512"] = end_to_end(tmp)
    line = json.dumps(res)
    print(line)
    if a.out:
        with open(a.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
