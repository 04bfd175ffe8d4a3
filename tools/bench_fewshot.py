"""Few-shot conversion: the grouped pooling kernel, Inferencer.embed_speakers and inference_padded with reference sets.

    python tools/bench_fewshot.py [--sets 64] [--refs 1 4 16] [--pairs 512] [--mels 80 512] [--reps 5]

* avc_time_mean_grouped_fwd on the speaker encoder's last activation (128 channels) of 64 x 16 references of 13-75
  frames (100-600 input frames / 8): CUDA events over 200 launches, with the bytes it reads over that time;
* embed_speakers for --sets sets of K references of 100-600 frames, for each K of --refs (seed-0 weights);
* inference_padded of --pairs pairs (100-600 frames) with 4-reference sets against single references, after one
  warm-up call each (graph captures), alternated, --reps calls each ending in a device synchronise.
Lengths and mels come from numpy default_rng(0) / torch seed 0.  Reads the card name and power limit in the same run;
prints one JSON line and writes nothing.
"""
import argparse
import json
import os
import statistics
import sys
import types

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import numpy as np  # noqa: E402
import torch  # noqa: E402

from _harness import card, events_ms, median_wall_s  # noqa: E402


def kernel(iters=200):
    from adaptive_voice_conversion_b200 import _lib as L
    lib = L.load()
    rng = np.random.default_rng(0)
    sizes, Cc, div = [16] * 64, 128, 8
    B = sum(sizes)
    lens = rng.integers(100, 601, B)
    T = -(-600 // div)
    x = torch.randn(B, Cc // 4, T, 4, device="cuda")
    lt = torch.tensor(lens, dtype=torch.int32, device="cuda")
    offs = torch.tensor([0] + sizes).cumsum(0).to(torch.int32).cuda()
    out = torch.empty(len(sizes), Cc, device="cuda")

    def launch():
        L.check(lib.avc_time_mean_grouped_fwd(x.data_ptr(), x[0].numel(), out.data_ptr(), B, Cc, T, lt.data_ptr(), div, 1,
                                              offs.data_ptr(), len(sizes), None), "avc_time_mean_grouped_fwd")
    us = 1e3 * events_ms(launch, iters, 10)
    frames = int(sum(-(-int(v) // div) for v in lens))
    nbytes = frames * Cc * 4 + B * 4 + len(sizes) * Cc * 4
    return {"groups": len(sizes), "members": B, "channels": Cc, "valid_frames": frames, "us_per_launch": us,
            "read_GB_per_s": nbytes / (us * 1e-6) / 1e9}


def inferencer(n_mels):
    import oracle.ae_oracle as orc
    from adaptive_voice_conversion_b200.inference import Inferencer
    cfg = orc.default_config(n_mels)
    args = types.SimpleNamespace(attr=None, model=None, source=None, target=None, output=None, sample_rate=24000)
    inf = Inferencer(cfg, args)
    inf.model.load_state_dict(orc.init_state(cfg, seed=0), strict=True)
    return inf


def embedding(inf, n_mels, n_sets, ks, reps):
    rng = np.random.default_rng(0)
    g = torch.Generator().manual_seed(0)
    out = []
    for k in ks:
        sets = [[torch.randn((int(t), n_mels), generator=g).cuda() for t in rng.integers(100, 601, k)] for _ in range(n_sets)]
        t = []
        med = median_wall_s(lambda: inf.embed_speakers(sets), reps, samples=t)
        out.append({"K": k, "sets": n_sets, "sets_per_s": n_sets / med, "s": t})
    return out


def conversion(inf, n_mels, n_pairs, reps, k=4):
    rng = np.random.default_rng(0)
    g = torch.Generator().manual_seed(0)
    xs = [torch.randn((int(t), n_mels), generator=g).cuda() for t in rng.integers(100, 601, n_pairs)]
    cs = [torch.randn((int(t), n_mels), generator=g).cuda() for t in rng.integers(100, 601, n_pairs)]
    sets = [[cs[(i + j) % n_pairs] for j in range(k)] for i in range(n_pairs)]
    inf.inference_padded(xs, cs)
    inf.inference_padded(xs, sets)
    caps = inf.padded_captures
    t1, tk = [], []
    for _ in range(reps):
        t1.append(median_wall_s(lambda: inf.inference_padded(xs, cs), 1, warmup=0))
        tk.append(median_wall_s(lambda: inf.inference_padded(xs, sets), 1, warmup=0))
    return {"pairs": n_pairs, "K": k, "single_pairs_per_s": n_pairs / statistics.median(t1),
            "sets_pairs_per_s": n_pairs / statistics.median(tk), "single_s": t1, "sets_s": tk,
            "captures_in_timed_calls": inf.padded_captures - caps}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--sets", type=int, default=64)
    ap.add_argument("--refs", type=int, nargs="+", default=[1, 4, 16])
    ap.add_argument("--pairs", type=int, default=512)
    ap.add_argument("--mels", type=int, nargs="+", default=[80, 512])
    ap.add_argument("--reps", type=int, default=5)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_fewshot needs a GPU")
    res = {"card": card(), "grouped_pool_kernel": kernel(), "models": []}
    for n in a.mels:
        inf = inferencer(n)
        res["models"].append({"mels": n, "embed_speakers": embedding(inf, n, a.sets, a.refs, a.reps),
                              "inference_padded": conversion(inf, n, a.pairs, a.reps)})
    print(json.dumps(res))


if __name__ == "__main__":
    main()
