"""Training throughput from a real data directory: the device-resident corpus (data_utils.DeviceSegments) against the
stock DataLoader path, beside the synthetic arm bench.py times.

    python tools/bench_corpus.py [--utts 1000] [--configs 512:128 80:256] [--steps 100] [--windows 3]

For each --configs entry (mels:batch) a seeded VCTK-like corpus is written to a temporary directory: --utts
utterances of 129-600 N(0,1) frames (per-mel z-normalised features) and an index of every crop of 128 frames.  Then:
  - peak device memory of the trainer alone (torch.cuda.max_memory_allocated over Solver construction, graph capture and
    --steps steps of the synthetic arm, less what was allocated before);
  - Solver.run_steps(--steps) is timed for three Solvers -- synthetic pinned batches (bench.py's e2e arm), the device
    corpus, the DataLoader (4 workers) -- alternating in a rotating order, over --windows windows each, every window
    bracketed by a device synchronise; the median window is reported;
  - avc_segment_gather's time per launch from CUDA events over --launches launches, and the bytes it moves
    (one read and one write of the batch) per second against 3.35 TB/s (H100 SXM HBM3).
The card's name, power limit and max SM clock are read in the same run.  Prints one JSON line per config; writes
nothing outside the temporary directory.
"""
import argparse
import contextlib
import io
import itertools
import json
import os
import pickle
import statistics
import sys
import tempfile
import types

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import numpy as np  # noqa: E402
import torch  # noqa: E402

from _harness import card, events_ms  # noqa: E402

HBM_BPS = 3.35e12
SEG = 128


def write_corpus(path, n_utt, n_mels, seed=0):
    rng = np.random.default_rng(seed)
    data = {f"p{i // 400:03d}_{i:05d}": rng.standard_normal((int(rng.integers(129, 601)), n_mels), dtype=np.float32)
            for i in range(n_utt)}
    index = [[u, t] for u, a in data.items() for t in range(len(a) - SEG + 1)]
    with open(os.path.join(path, "train.pkl"), "wb") as f:
        pickle.dump(data, f, protocol=4)
    with open(os.path.join(path, "train_samples_128.json"), "w") as f:
        json.dump(index, f)
    return sum(len(a) for a in data.values()), len(index)


def make_solver(cfg, data_dir, tmp):
    from adaptive_voice_conversion_b200.solver import Solver
    args = types.SimpleNamespace(data_dir=data_dir, train_set="train", train_index_file="train_samples_128.json",
                                 logdir=os.path.join(tmp, "log"), load_model=False, load_opt=False, store_model_path=None,
                                 load_model_path=None, summary_steps=10 ** 9, save_steps=10 ** 9, tag="bench", iters=0)
    out = io.StringIO()
    torch.manual_seed(0)
    with contextlib.redirect_stdout(out):
        s = Solver(cfg, args)
    s.data_line = next((ln for ln in out.getvalue().splitlines() if ln.startswith("training data:")), None)
    return s


def gather_time(ds, launches):
    ds.seek(0)
    next(ds)                                   # loads epoch 0's order
    B = ds.sampler.batch_size
    xs = [ds.gather(0, B) for _ in range(3)]
    n = itertools.count()

    def launch():
        i = next(n)
        xs[i % 3] = ds.gather((i * B) % max(1, ds.sampler.n - B), B)
    us = 1e3 * events_ms(launch, launches, 0, sync=True)
    nbytes = 2 * B * ds.c_in * ds.T * 4 + B * 12      # batch read + written; order and starts entries
    return {"us_per_launch": us, "bytes_per_launch": nbytes, "achieved_TBps": nbytes / us / 1e6,
            "share_of_3.35TBps": nbytes / us / 1e6 / (HBM_BPS / 1e12)}


def run_config(n_mels, batch, a):
    from adaptive_voice_conversion_b200.config import default_config
    from adaptive_voice_conversion_b200 import data_utils as D
    from torch.utils.data import DataLoader
    cfg = default_config(n_mels)
    cfg["data_loader"]["batch_size"] = batch
    K = a.steps
    res = {"config": f"c{n_mels} B={batch} T={SEG}", "card": card()}
    with tempfile.TemporaryDirectory() as tmp:
        ddir = os.path.join(tmp, "data")
        os.makedirs(ddir)
        frames, entries = write_corpus(ddir, a.utts, n_mels, seed=n_mels)
        res["corpus"] = {"utterances": a.utts, "frames": frames, "entries": entries,
                         "device_bytes": D.corpus_device_bytes(frames, n_mels, entries)}
        # the trainer's own peak, before any other arm allocates
        torch.cuda.synchronize()
        torch.cuda.reset_peak_memory_stats()
        base = torch.cuda.memory_allocated()
        syn = make_solver(cfg, "synthetic", tmp)
        syn.run_steps(K, lambda_of=lambda it: 1.0)
        torch.cuda.synchronize()
        res["trainer_peak_bytes"] = torch.cuda.max_memory_allocated() - base
        dev = make_solver(cfg, ddir, tmp)
        assert isinstance(dev.train_loader, D.DeviceSegments), dev.data_line
        import adaptive_voice_conversion_b200.solver as S
        real_total = S._device_total_memory
        S._device_total_memory = lambda d: 0        # force the DataLoader path for the third arm
        try:
            dl = make_solver(cfg, ddir, tmp)
        finally:
            S._device_total_memory = real_total
        assert isinstance(dl.train_loader, DataLoader)
        res["data_line"] = dev.data_line
        arms = {"synthetic": syn, "device_corpus": dev, "dataloader": dl}
        for s in arms.values():                     # graph capture + warm-up of every arm
            s.run_steps(max(a.warmup, 4), lambda_of=lambda it: 1.0)
        torch.cuda.synchronize()
        wins = {k: [] for k in arms}
        names = list(arms)
        for w in range(a.windows):
            for name in names[w % 3:] + names[:w % 3]:    # rotated: no arm always follows the same one
                s, metas = arms[name], []
                wins[name].append(events_ms(lambda: metas.append(s.run_steps(K, lambda_of=lambda it: 1.0)), 1, 0))
                assert all(np.isfinite(v) for v in metas[0].values()), (name, metas[0])
        res["run_steps"] = {k: {"seg_per_s": batch * K / (statistics.median(v) * 1e-3), "ms_per_step": statistics.median(v) / K,
                                "window_ms": v} for k, v in wins.items()}
        syn_rate = res["run_steps"]["synthetic"]["seg_per_s"]
        res["device_vs_synthetic"] = res["run_steps"]["device_corpus"]["seg_per_s"] / syn_rate
        res["dataloader_vs_synthetic"] = res["run_steps"]["dataloader"]["seg_per_s"] / syn_rate
        res["gather"] = gather_time(dev.train_loader, a.launches)
        del arms, syn, dev, dl
        torch.cuda.synchronize()
        torch.cuda.empty_cache()
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--utts", type=int, default=1000, help="utterances of 129-600 frames in the generated corpus")
    ap.add_argument("--configs", nargs="+", default=["512:128", "80:256"], help="mels:batch")
    ap.add_argument("--steps", type=int, default=100, help="steps per timed window")
    ap.add_argument("--warmup", type=int, default=10)
    ap.add_argument("--windows", type=int, default=3)
    ap.add_argument("--launches", type=int, default=500)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_corpus needs a CUDA device")
    from adaptive_voice_conversion_b200 import _lib as L
    L.load(build_if_missing=False)
    for c in a.configs:
        n_mels, batch = (int(v) for v in c.split(":"))
        print(json.dumps(run_config(n_mels, batch, a)), flush=True)


if __name__ == "__main__":
    main()
