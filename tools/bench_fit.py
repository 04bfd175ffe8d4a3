"""Speaker-code fitting: one wave step (CodeFitTrainer) against speaker adaptation's step (AdaptTrainer) at the same B.

    python tools/bench_fit.py [--shapes 1x128 16x8 32x4] [--mels 80 512] [--steps 50] [--reps 5] [--fit_steps 300]

For each c_in of --mels and each S_w x m of --shapes (B = S_w m segments of 128 frames, seed-0 weights, N(0,1) crops
from torch seed 0 gathered on the device as a run gathers them), both trainers replay their CUDA graph: three warm-up
steps, then --steps steps between CUDA events, repeated --reps times with the two alternated; the minimum ms per step is
reported with every repetition.  The wave step includes its crop gather.  "speakers_per_s" is S_w / (--fit_steps x the
wave step): speakers fitted per second by a run of --fit_steps steps, waves back to back.  The launch counts are of one
eager step (the fitting step's without its gather).  Reads the card name and power limit in the same run; prints one
JSON line and writes nothing.
"""
import argparse
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import numpy as np  # noqa: E402
import torch  # noqa: E402

from _harness import card, events_ms  # noqa: E402


def model_of(cfg):
    import oracle.ae_oracle as orc
    from adaptive_voice_conversion_b200.model import AE
    m = AE(cfg)
    m.load_state_dict(orc.init_state(cfg, seed=0), strict=True)
    return m.cuda()


def bench(n_mels, S, m, steps, reps, fit_steps):
    import oracle.ae_oracle as orc
    from adaptive_voice_conversion_b200 import adapt as A
    from adaptive_voice_conversion_b200 import fit as F
    cfg = orc.default_config(n_mels)
    B = S * m
    torch.manual_seed(0)
    names = [f"p{300 + s}" for s in range(S)]
    mels = {f"{s}_{k}": torch.randn(400, n_mels).numpy() for s in names for k in range(2)}
    per, _ = F.plan(names, [[f"{s}_0", f"{s}_1"] for s in names], {u: 400 for u in mels}, 128, m)
    n_warm = 3 + reps * steps
    corpus = F.WaveCorpus(mels, [e for s in names for e in per[s]["index"]],
                          F.order_table([per[s]["n_crops"] for s in names], m, n_warm + 1, 0, names), cfg, "cuda")
    fit = F.CodeFitTrainer(model_of(cfg), cfg, S, m)
    fit.reset(torch.zeros(S, cfg["SpeakerEncoder"]["c_out"], device="cuda"))
    ad = A.make_trainer(model_of(cfg), torch.zeros(cfg["SpeakerEncoder"]["c_out"]), cfg)
    x = torch.empty(B, n_mels, 128, device="cuda")
    corpus.gather(x, 0, B)
    k = [0]

    def fit_step():
        fit.run_step(corpus, k[0])
        k[0] += 1

    def ad_step():
        ad.step(x, 0.0)
    for _ in range(3):
        fit_step()
        ad_step()
    launches = {"fit": fit.launches_per_step, "adapt": ad.launches_per_step}
    torch.cuda.synchronize()
    ms = {"fit": [], "adapt": []}
    for _ in range(reps):
        for key, fn in (("fit", fit_step), ("adapt", ad_step)):
            ms[key].append(events_ms(fn, steps, 0))
    fit.eng.check_tc_status()
    ad.losses()     # raises on a tensor-core pipeline time-out
    best = {key: min(v) for key, v in ms.items()}
    return {"c_in": n_mels, "S_w": S, "m": m, "batch": B, "fit_ms_per_step": best["fit"],
            "adapt_ms_per_step": best["adapt"], "fit_ms_reps": ms["fit"], "adapt_ms_reps": ms["adapt"],
            "fit_over_adapt": best["fit"] / best["adapt"], "launches_per_step": launches,
            "speakers_per_s": S / (fit_steps * best["fit"] / 1e3), "fit_steps": fit_steps}


def main():
    p = argparse.ArgumentParser()
    p.add_argument("--shapes", nargs="+", default=["1x128", "16x8", "32x4"])
    p.add_argument("--mels", type=int, nargs="+", default=[80, 512])
    p.add_argument("--steps", type=int, default=50)
    p.add_argument("--reps", type=int, default=5)
    p.add_argument("--fit_steps", type=int, default=300)
    a = p.parse_args()
    shapes = [tuple(int(v) for v in s.split("x")) for s in a.shapes]
    runs = []
    for n in a.mels:
        for S, m in shapes:
            runs.append(bench(n, S, m, a.steps, a.reps, a.fit_steps))
            torch.cuda.empty_cache()
    print(json.dumps({"card": card(), "runs": runs}))


if __name__ == "__main__":
    main()
