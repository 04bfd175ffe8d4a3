"""Cost of the speaker-classifier probes (adaptive_voice_conversion_b200/speaker_probe.py) on the GPU.

    python tools/bench_probe.py [--speakers 100] [--utts 64] [--frames 300] [--out result.json]

At a VCTK-like size (100 speakers x 64 utterances of 250-350 frames, about 300 on average, so about 240 000 latent
frames), with a random-init model at c_in 80 and 512:
1. the features of the fit set (speaker_eval.representations plus the content-code frame rows): host clock around a
   call that ends in a synchronise;
2. fitting each of the four probes with the default (untuned) ProbeParams, and scoring it on its own fit rows: host
   clock, each call ending in a copy to the host;
3. the kernel split of one training step at each probe's batch size (the frame probe at 4096 x 128 -> 256 -> 256 -> S):
   CUDA events around 200 repetitions of each part (linear forward, cross-entropy, gradient zeroing, linear backward,
   norm and Adam), after a warm-up.
Random-init models separate nothing, so the accuracies are not meaningful here; only the times are.  Prints one JSON
line with the card's name and power limit.
"""
from __future__ import annotations

import argparse
import ctypes as C
import json
import os
import sys

import numpy as np
import torch

from _harness import card, events_ms, median_wall_s

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def step_split(D, S, Bt, H=256):
    """{part: ms per step} of one training step of a probe with batch Bt (CUDA events)."""
    from adaptive_voice_conversion_b200 import _lib as L
    from adaptive_voice_conversion_b200 import speaker_probe as P
    from adaptive_voice_conversion_b200.utils import _stream
    dev = torch.device("cuda")
    lib, st = L.load(), _stream(dev)
    flat = P.init_params(D, S, P.ProbeParams(hidden=H), 0).to(dev)
    grad = torch.zeros_like(flat)
    m, v, vmax = (torch.zeros_like(flat) for _ in range(3))
    hp = torch.tensor([0, 0, 1, 1e-3, 0.9, 0.999, 1e-8, 0, float("inf"), 0], dtype=torch.float32, device=dev)
    step, sq, sqs = torch.zeros(1, device=dev), torch.zeros(1, device=dev), torch.empty(1024, device=dev)
    Pv, Gv = P.unflatten(flat, D, H, S), P.unflatten(grad, D, H, S)
    net = P._Mlp(D, H, S, Bt, dev)
    x = torch.randn(Bt, D, device=dev)
    lab = torch.randint(0, S, (Bt,), dtype=torch.int32, device=dev)
    tot = torch.zeros(1, dtype=torch.float64, device=dev)
    scratch = torch.empty(L.PROBE_SUM_SCRATCH, dtype=torch.float64, device=dev)
    n = flat.numel()

    def zero():
        L.check(lib.avc_fill_zero(grad.data_ptr(), n * 4, st))

    def update():
        L.check(lib.avc_sqnorm(grad.data_ptr(), n, sqs.data_ptr(), sq.data_ptr(), st))
        L.check(lib.avc_adam_step(flat.data_ptr(), grad.data_ptr(), m.data_ptr(), v.data_ptr(), vmax.data_ptr(), n,
                                  hp.data_ptr(), sq.data_ptr(), step.data_ptr(), st))
    net.forward(Pv, x, Bt)
    out = {"linear_fwd": events_ms(lambda: net.forward(Pv, x, Bt), 200, 5),
           "xent": events_ms(lambda: P.xent(net.z, lab, 1.0 / Bt, dlogits=net.dz, loss_sum=tot, scratch=scratch),
                             200, 5),
           "fill_zero": events_ms(zero, 200, 5),
           "linear_bwd": events_ms(lambda: net.backward(Pv, Gv, x, Bt), 200, 5),
           "sqnorm_adam": events_ms(update, 200, 5)}
    out["step"] = sum(out.values())
    flops = 2 * Bt * (D * H + H * H + H * S) * 3        # forward, data and weight gradients
    out["linear_tflops"] = flops / ((out["linear_fwd"] + out["linear_bwd"]) * 1e-3) / 1e12
    return out


def run(c_in, n_spk, n_utts, frames, seed=0):
    from adaptive_voice_conversion_b200 import speaker_probe as P
    from adaptive_voice_conversion_b200.config import default_config
    from adaptive_voice_conversion_b200.model import AE
    torch.manual_seed(c_in)
    model = AE(default_config(c_in)).cuda().eval()
    rng = np.random.default_rng(seed)
    lens = rng.integers(frames - 50, frames + 51, n_spk * n_utts)
    mels = [torch.randn(int(T), c_in, device="cuda") for T in lens]
    labels = np.repeat(np.arange(n_spk), n_utts)
    P.features(model, mels[:8])                          # warm-up
    feats = {}
    t_feat = median_wall_s(lambda: feats.update(P.features(model, mels)), 1, warmup=0)
    res = {"c_in": c_in, "utterances": len(mels), "mel_frames": int(lens.sum()),
           "latent_frames": int(feats["offsets"][-1]), "features_s": t_feat, "probes": {}}
    frame_lab = np.repeat(labels, np.diff(feats["offsets"]))
    for k in P.REPRESENTATIONS:
        fr = k == "content_frames"
        lab = frame_lab if fr else labels
        fitted, scored = [], []
        t_fit = median_wall_s(lambda: fitted.append(P.fit_probe(feats[k], lab, seed=seed, n_classes=n_spk, frames=fr)),
                              1, warmup=0)
        probe = fitted[0]
        t_score = median_wall_s(lambda: scored.append(P.score_probe(probe, feats[k], lab)), 1, warmup=0)
        sc = scored[0]
        res["probes"][k] = {"rows": int(feats[k].shape[0]), "dims": int(feats[k].shape[1]), "fit_s": t_fit,
                            "score_s": t_score, "fit_acc": float((sc["rank"] == 0).mean()),
                            "last_loss": probe.losses[-1]}
    return res


def main(argv=None):
    ap = argparse.ArgumentParser()
    ap.add_argument("--speakers", type=int, default=100)
    ap.add_argument("--utts", type=int, default=64)
    ap.add_argument("--frames", type=int, default=300)
    ap.add_argument("--out", default=None)
    a = ap.parse_args(argv)
    if not torch.cuda.is_available():
        raise SystemExit("bench_probe needs a CUDA device")
    out = {"card": card(), "runs": [run(c, a.speakers, a.utts, a.frames) for c in (80, 512)],
           "step_split_ms": {"frame_probe_4096x128": step_split(128, a.speakers, 4096),
                             "speaker_probe_256x128": step_split(128, a.speakers, 256),
                             "mel_probe_256x1024": step_split(1024, a.speakers, 256)}}
    line = json.dumps(out)
    print(line)
    if a.out:
        with open(a.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
