"""Inferencer.inference_padded against Inferencer.inference_ragged, and wav to wav through `inference.py -pairs`.

    python tools/bench_padded.py [--pairs 512] [--mels 80 512] [--reps 3] [--wav-pairs 32]

Per mel count: --pairs random mel pairs, lengths uniform in 100..600 frames (numpy default_rng(0), as bench_mcd.py),
seed-0 weights.  After one warm-up call each (graph captures), the two methods are timed alternately, --reps calls each
ending in a device synchronise; pairs/s from the median.  Also: padded frames per valid frame, the largest relative
difference of the outputs, and the wall time of one `inference.py -pairs` process on --wav-pairs seeded synthetic wavs
of 1-6 s (start-up, captures and 100 Griffin-Lim iterations included).  Reads the card name and power limit in the
same run; prints one JSON line and writes only under a temporary directory.
"""
import argparse
import json
import os
import statistics
import subprocess
import sys
import tempfile
import time
import types

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import numpy as np  # noqa: E402
import torch  # noqa: E402

from _harness import card, median_wall_s  # noqa: E402


def conversion(n_mels, n_pairs, reps):
    import oracle.ae_oracle as orc
    from adaptive_voice_conversion_b200.inference import Inferencer, padded_batches
    cfg = orc.default_config(n_mels)
    args = types.SimpleNamespace(attr=None, model=None, source=None, target=None, output=None, sample_rate=24000)
    inf = Inferencer(cfg, args)
    inf.model.load_state_dict(orc.init_state(cfg, seed=0), strict=True)
    rng = np.random.default_rng(0)
    src = rng.integers(100, 601, n_pairs).tolist()
    ref = rng.integers(100, 601, n_pairs).tolist()
    g = torch.Generator().manual_seed(0)
    xs = [torch.randn((t, n_mels), generator=g).cuda() for t in src]
    cs = [torch.randn((t, n_mels), generator=g).cuda() for t in ref]
    a, b = inf.inference_ragged(xs, cs), inf.inference_padded(xs, cs)
    diff = max(float((p - q).abs().max() / (q.abs().max() + 1e-12)) for p, q in zip(b, a))
    caps = inf.padded_captures
    t_r, t_p = [], []
    for _ in range(reps):
        t_r.append(median_wall_s(lambda: inf.inference_ragged(xs, cs), 1, warmup=0))
        t_p.append(median_wall_s(lambda: inf.inference_padded(xs, cs), 1, warmup=0))
    plan = padded_batches(src, ref)
    pad_src = sum(B * T for _, T, _, B in plan) / sum(src)
    pad_ref = sum(B * Tc for _, _, Tc, B in plan) / sum(ref)
    return {"mels": n_mels, "ragged_pairs_per_s": n_pairs / statistics.median(t_r),
            "padded_pairs_per_s": n_pairs / statistics.median(t_p), "ragged_s": t_r, "padded_s": t_p, "batches": len(plan),
            "captures_in_timed_calls": inf.padded_captures - caps, "padded_per_valid_frame": [pad_src, pad_ref],
            "max_relerr_padded_vs_ragged": diff}


def wav_to_wav(n_pairs):
    import oracle.ae_oracle as orc
    import yaml
    from scipy.io.wavfile import write
    from adaptive_voice_conversion_b200.model import AE
    with tempfile.TemporaryDirectory() as td:
        cfg = orc.default_config(80)
        with open(os.path.join(td, "config.yaml"), "w") as f:
            yaml.safe_dump(cfg, f)
        m = AE(cfg)
        m.load_state_dict(orc.init_state(cfg, seed=0))
        torch.save(m.state_dict(), os.path.join(td, "model.ckpt"))
        rng = np.random.default_rng(0)
        wavs, secs = [os.path.join(td, f"w{i}.wav") for i in range(n_pairs)], rng.uniform(1.0, 6.0, n_pairs)
        for i, (p, d) in enumerate(zip(wavs, secs)):
            t = np.arange(int(d * 24000)) / 24000
            y = 0.3 * np.sin(2 * np.pi * (100 + 5 * i) * t * (1 + 0.1 * t)) + 0.02 * rng.standard_normal(t.size)
            write(p, 24000, (y * 32767).astype(np.int16))
        with open(os.path.join(td, "pairs.txt"), "w") as f:
            f.writelines(f"{wavs[i]} {wavs[(i + 1) % n_pairs]}\n" for i in range(n_pairs))
        cmd = [sys.executable, os.path.join(ROOT, "inference.py"), "-c", os.path.join(td, "config.yaml"),
               "-m", os.path.join(td, "model.ckpt"), "-pairs", os.path.join(td, "pairs.txt"), "-o", os.path.join(td, "out")]
        t0 = time.perf_counter()
        subprocess.run(cmd, check=True, env=dict(os.environ, PYTHONPATH=ROOT), stdout=subprocess.DEVNULL)
        wall = time.perf_counter() - t0
        n_out = len([f for f in os.listdir(os.path.join(td, "out")) if f.endswith(".wav")])
    return {"pairs": n_pairs, "source_audio_s": float(secs.sum()), "wall_s": wall, "wavs_written": n_out}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--pairs", type=int, default=512)
    ap.add_argument("--mels", type=int, nargs="+", default=[80, 512])
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--wav-pairs", type=int, default=32)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_padded needs a GPU")
    res = {"card": card(), "conversion": [conversion(n, a.pairs, a.reps) for n in a.mels]}
    if a.wav_pairs > 0:
        res["wav_to_wav"] = wav_to_wav(a.wav_pairs)
    print(json.dumps(res))


if __name__ == "__main__":
    main()
