"""Cost of the YIN F0 tracker and of the F0 evaluation (adaptive_voice_conversion_b200/f0.py) on the GPU.

    python tools/bench_f0.py [--signals 64] [--frames 512] [--out result.json]

1. avc_yin alone on --signals harmonic signals of --frames frames each (hop 300 at 24 kHz) at the default parameters
   (W 1024, lags 1..480): CUDA events around each call, median of 5 after one warm-up.  FP64 operations are counted
   from the definition: each (frame, tau, j) term of the difference function is a subtraction and a fused multiply-add
   (3 operations), over the data-sheet FP64 rate of the H100 SXM (34 TFLOP/s without tensor cores).
2. evaluate_f0 on a generated set (20 speakers x 20 utterances of 200-600 frames, N(0, 1) mels, random-init model) at
   c_in 80 and 512, with Griffin-Lim at its default 100 iterations: conversion, synthesis, tracking and host seconds,
   each ended by a device synchronise, after one warm-up call.
3. Copy-synthesis F0 fidelity: harmonic test signals (60-400 Hz, vibrato) -> wav_to_mel -> mel_to_signal -> tracker at
   80 and 512 mels; the median relative F0 error over the frames voiced in both the original and the synthesis.
Prints one JSON line with the card's name and power limit.
"""
from __future__ import annotations

import argparse
import json
import os
import sys

import numpy as np
import torch

from _harness import card, median_events_s

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

FP64_PEAK = 34e12   # H100 SXM data sheet, FP64 without tensor cores


def tracker(n_signals, n_frames):
    from _f0_ref import harmonic
    from adaptive_voice_conversion_b200 import f0 as F
    p = F.F0Params()
    hop, sr = 300, 24000
    rng = np.random.default_rng(0)
    sigs = [torch.from_numpy(harmonic(float(rng.uniform(60, 400)), (n_frames - 1) * hop / sr, phase_seed=i)).cuda()
            for i in range(n_signals)]
    frames = sum(1 + s.numel() // hop for s in sigs)
    t = median_events_s(lambda: F.yin(sigs, sr, hop, p), 5)
    ops = 3.0 * frames * p.tau_max(sr) * p.win
    return {"signals": n_signals, "frames": frames, "seconds_per_call": t, "frames_per_second": frames / t,
            "fp64_flops": ops / t, "fp64_share_of_datasheet": ops / t / FP64_PEAK}


def evaluation(c_in):
    from adaptive_voice_conversion_b200 import f0 as F
    from adaptive_voice_conversion_b200.config import default_config
    from adaptive_voice_conversion_b200.model import AE
    rng = np.random.default_rng(c_in)
    data = {f"p{300 + s}_{u:03d}.wav": rng.standard_normal((int(rng.integers(200, 601)), c_in)).astype(np.float32)
            for s in range(20) for u in range(20)}
    attr = {"mean": rng.uniform(0.3, 0.7, c_in).astype(np.float32), "std": rng.uniform(0.1, 0.3, c_in).astype(np.float32)}
    torch.manual_seed(0)
    model = AE(default_config(c_in)).cuda()
    F.evaluate_f0(model, data, attr, max_pairs=20)
    tm = {}
    res = F.evaluate_f0(model, data, attr, timings=tm)
    return {"c_in": c_in, "utterances": len(data), "pairs": res["n"] + res["n_unvoiced"], "n": res["n"],
            "frames": int(sum(len(v) for v in data.values())), "seconds": tm, "total": sum(tm.values())}


def fidelity(n_mels):
    from _f0_ref import harmonic
    from adaptive_voice_conversion_b200 import f0 as F
    from adaptive_voice_conversion_b200.vocoder import Vocoder
    p, sr, hop = F.F0Params(), 24000, 300
    voc = Vocoder(n_mels=n_mels)
    rng = np.random.default_rng(1)
    errs, f0s = [], np.linspace(60, 400, 24)
    wavs = []
    for i, f in enumerate(f0s):
        rate = float(rng.uniform(3, 6))
        wavs.append(torch.from_numpy(harmonic(lambda t: f * (1 + 0.03 * np.sin(2 * np.pi * rate * t)), 1.5,
                                              phase_seed=i)).cuda())
    mels = [m for m, _ in voc.wav_to_mel(wavs)]
    ref = F.track([w[: hop * (m.shape[0] - 1)] for w, m in zip(wavs, mels)], sr, hop, p)
    syn = F.track(voc.mel_to_signal(mels), sr, hop, p)
    per = []
    for (fa, va), (fb, vb) in zip(ref, syn):
        both = va & vb
        e = np.abs(fb[both] / fa[both] - 1)
        errs.append(e)
        per.append(float(np.median(e)) if len(e) else None)
    allerr = np.concatenate(errs)
    return {"n_mels": n_mels, "median_rel_f0_error": float(np.median(allerr)),
            "p90_rel_f0_error": float(np.quantile(allerr, 0.9)), "frames_voiced_in_both": int(len(allerr)),
            "frames": int(sum(len(v) for _, v in ref))}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--signals", type=int, default=64)
    ap.add_argument("--frames", type=int, default=512)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    out = {"card": card(), "yin": tracker(args.signals, args.frames),
           "evaluate_f0": [evaluation(c) for c in (80, 512)], "copy_synthesis": [fidelity(m) for m in (80, 512)]}
    line = json.dumps(out)
    print(line)
    if args.out:
        with open(args.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
