"""Time-varying speaker morphs: Inferencer.inference_morph against inference_with_codes on the same sources.

    python tools/bench_morph.py [--sources 64] [--frames 512] [--mels 80 512] [--ks 1 2 8] [--reps 5]

--sources sources of --frames frames each (one padded batch), CUDA graphs on (AVC_INFER_GRAPH=1): inference_with_codes
with one code per source, and inference_morph with K anchors per source whose weights glide between them over the
utterance.  Each shape is captured by a warm-up call; then the best of --reps calls of each, alternated, timed with a
device synchronise.  Seed-0 weights and inputs.  Reads the card name and power limit in the same run; prints one JSON
line and writes nothing.
"""
import argparse
import json
import os
import sys
import types

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import torch  # noqa: E402

from _harness import card, median_wall_s  # noqa: E402


def run(n_mels, n_src, frames, ks, reps):
    import oracle.ae_oracle as orc
    from adaptive_voice_conversion_b200.inference import Inferencer
    cfg = orc.default_config(n_mels)
    args = types.SimpleNamespace(attr=None, model=None, source=None, target=None, output=None, sample_rate=24000)
    inf = Inferencer(cfg, args)
    inf.model.load_state_dict(orc.init_state(cfg, seed=0), strict=True)
    g = torch.Generator().manual_seed(0)
    xs = [torch.randn((frames, n_mels), generator=g).cuda() for _ in range(n_src)]
    codes = torch.randn((n_src, cfg["SpeakerEncoder"]["c_out"]), generator=g).cuda()
    out = {"n_mels": n_mels, "sources": n_src, "frames": frames}
    plain = lambda: inf.inference_with_codes(xs, codes)     # noqa: E731
    plain()
    morphs = {}
    for K in ks:
        cs = [torch.randn((K, cfg["SpeakerEncoder"]["c_out"]), generator=g).cuda() for _ in range(n_src)]
        t = torch.linspace(0, K - 1, frames)
        w = torch.clamp(1 - (t[None, :] - torch.arange(K, dtype=torch.float32)[:, None]).abs(), min=0).cuda()
        ws = [w.clone() for _ in range(n_src)]
        morphs[K] = lambda cs=cs, ws=ws: inf.inference_morph(xs, cs, ws)
        morphs[K]()
    best = {"codes": float("inf"), **{K: float("inf") for K in ks}}
    for _ in range(reps):
        best["codes"] = min(best["codes"], median_wall_s(plain, 1, warmup=0))
        for K in ks:
            best[K] = min(best[K], median_wall_s(morphs[K], 1, warmup=0))
    out["inference_with_codes_ms"] = best["codes"] * 1e3
    for K in ks:
        out[f"inference_morph_K{K}_ms"] = best[K] * 1e3
        out[f"inference_morph_K{K}_over_codes"] = best[K] / best["codes"]
    return out


def main():
    p = argparse.ArgumentParser()
    p.add_argument("--sources", type=int, default=64)
    p.add_argument("--frames", type=int, default=512)
    p.add_argument("--mels", type=int, nargs="+", default=[80, 512])
    p.add_argument("--ks", type=int, nargs="+", default=[1, 2, 8])
    p.add_argument("--reps", type=int, default=5)
    a = p.parse_args()
    os.environ["AVC_INFER_GRAPH"] = "1"
    print(json.dumps({"card": card(), "runs": [run(n, a.sources, a.frames, a.ks, a.reps) for n in a.mels]}))


if __name__ == "__main__":
    main()
