"""Speaker adaptation: one adaptation step (AdaptTrainer) against one training step (FusedTrainer) at the same shape.

    python tools/bench_adapt.py [--batch 128] [--mels 80 512] [--steps 50] [--reps 3]

For each c_in of --mels, at B = --batch segments of 128 frames (seed-0 weights, N(0,1) inputs from torch seed 0), both
trainers run eager (AVC_GRAPH=0 path) and replayed from their CUDA graph: three warm-up steps, then --steps steps
between CUDA events, repeated --reps times with the two trainers alternated; the minimum ms per step is reported with
every repetition.  The adaptation step runs no speaker encoder and no encoder backward.  Reads the card name and power
limit in the same run; prints one JSON line and writes nothing.
"""
import argparse
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import torch  # noqa: E402

from _harness import card, events_ms  # noqa: E402


def trainers(n_mels, B, graph):
    import oracle.ae_oracle as orc
    from adaptive_voice_conversion_b200 import adapt as A
    from adaptive_voice_conversion_b200.model import AE
    from adaptive_voice_conversion_b200.optim import FusedAdam
    from adaptive_voice_conversion_b200.trainer import FusedTrainer
    cfg = orc.default_config(n_mels)
    cfg["data_loader"]["batch_size"] = B
    o = cfg["optimizer"]
    out = {}
    for kind in ("train", "adapt"):
        m = AE(cfg)
        m.load_state_dict(orc.init_state(cfg, seed=0), strict=True)
        m = m.cuda()
        if kind == "train":
            m.flatten_parameters()
            opt = FusedAdam(m, lr=o["lr"], betas=(o["beta1"], o["beta2"]), amsgrad=o["amsgrad"],
                            weight_decay=o["weight_decay"], max_norm=o["grad_norm"])
            t = FusedTrainer(m, opt, cfg)
        else:
            t = A.make_trainer(m, torch.zeros(cfg["SpeakerEncoder"]["c_out"]), cfg)
        t.auto_graph = graph
        out[kind] = t
    return out


def time_steps(t, x, lam, n):
    ms = events_ms(lambda: t.step(x, lam), n, 0)
    t.losses()      # raises on a tensor-core pipeline time-out
    return ms


def bench(n_mels, B, steps, reps):
    torch.manual_seed(0)
    x = torch.randn(B, n_mels, 128, device="cuda")
    res = {"c_in": n_mels, "batch": B}
    for mode, graph in (("eager", False), ("graph", True)):
        ts = trainers(n_mels, B, graph)
        for t in ts.values():
            for _ in range(3):
                t.step(x, 1.0)
        torch.cuda.synchronize()
        ms = {k: [] for k in ts}
        for _ in range(reps):
            for k, t in ts.items():
                ms[k].append(time_steps(t, x, 1.0, steps))
        res[mode] = {f"{k}_ms_per_step": min(v) for k, v in ms.items()}
        res[mode].update({f"{k}_ms_reps": v for k, v in ms.items()})
        res[mode]["adapt_over_train"] = min(ms["adapt"]) / min(ms["train"])
        res[mode]["launches_per_step"] = {k: t.launches_per_step for k, t in ts.items()} if mode == "eager" else None
        del ts
        torch.cuda.empty_cache()
    return res


def main():
    p = argparse.ArgumentParser()
    p.add_argument("--batch", type=int, default=128)
    p.add_argument("--mels", type=int, nargs="+", default=[80, 512])
    p.add_argument("--steps", type=int, default=50)
    p.add_argument("--reps", type=int, default=3)
    a = p.parse_args()
    print(json.dumps({"card": card(), "runs": [bench(n, a.batch, a.steps, a.reps) for n in a.mels]}))


if __name__ == "__main__":
    main()
