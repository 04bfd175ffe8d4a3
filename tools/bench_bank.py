"""Speaker banks: the two pooling kernels, avc_spk_identify and a whole bank build.

    python tools/bench_bank.py [--m 100000] [--s 2000] [--dims 128] [--speakers 100] [--utts 40] [--mels 80 512]

* avc_time_sum_varlen on the speaker encoder's last activation (128 channels) of 64 utterances of 13-75 frames
  (100-600 input frames / 8), and avc_pooled_group_mean of a table of --speakers x --utts rows into --speakers codes:
  CUDA events over 200 launches each, with the bytes each reads over that time;
* avc_spk_identify of --m queries against a bank of --s codes of --dims dimensions: CUDA events over 5 launches, with
  the float64 multiply-adds it performs (2 per coordinate of every query-row pair: the dot and the row's norm);
* build_bank of --speakers speakers x --utts utterances of 100-600 frames (seed-0 weights) at each c_in of --mels,
  after one warm-up build, timed with a device synchronise.
Inputs come from numpy default_rng(0) / torch seed 0.  Reads the card name and power limit in the same run; prints one
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

from _harness import card, events_ms, median_wall_s  # noqa: E402


def pooling(n_spk, n_utts, iters=200):
    from adaptive_voice_conversion_b200 import _lib as L
    lib = L.load()
    rng = np.random.default_rng(0)
    B, Cc, div = 64, 128, 8
    lens = rng.integers(100, 601, B)
    T = -(-600 // div)
    x = torch.randn(B, Cc // 4, T, 4, device="cuda")
    lt = torch.tensor(lens, dtype=torch.int32, device="cuda")
    sums = torch.empty(B, Cc, device="cuda")
    counts = torch.empty(B, dtype=torch.int32, device="cuda")

    def time_sum():
        L.check(lib.avc_time_sum_varlen(x.data_ptr(), x[0].numel(), sums.data_ptr(), counts.data_ptr(), B, Cc, T,
                                        lt.data_ptr(), div, 1, None), "avc_time_sum_varlen")
    us_sum = 1e3 * events_ms(time_sum, iters, min(iters, 10))
    frames = int(sum(-(-int(v) // div) for v in lens))
    N = n_spk * n_utts
    tab = torch.randn(N, Cc, device="cuda")
    cnt = torch.tensor(rng.integers(13, 76, N), dtype=torch.int32, device="cuda")
    offs = torch.arange(0, N + 1, n_utts, dtype=torch.int64, device="cuda")
    out = torch.empty(n_spk, Cc, device="cuda")

    def group_mean():
        L.check(lib.avc_pooled_group_mean(tab.data_ptr(), cnt.data_ptr(), N, Cc, offs.data_ptr(), n_spk, out.data_ptr(),
                                          None), "avc_pooled_group_mean")
    us_pool = 1e3 * events_ms(group_mean, iters, min(iters, 10))
    return {"time_sum_varlen": {"utterances": B, "channels": Cc, "valid_frames": frames, "us_per_launch": us_sum,
                                "read_GB_per_s": (frames * Cc * 4 + B * 4) / (us_sum * 1e-6) / 1e9},
            "pooled_group_mean": {"groups": n_spk, "rows": N, "channels": Cc, "us_per_launch": us_pool,
                                  "read_GB_per_s": (N * Cc * 4 + N * 4 + (n_spk + 1) * 8) / (us_pool * 1e-6) / 1e9}}


def identify(m, s, d, iters=5):
    from adaptive_voice_conversion_b200 import speaker_eval as S
    from adaptive_voice_conversion_b200 import _lib as L
    import ctypes as C
    lib = L.load()
    q = torch.randn(m, d, device="cuda")
    bank = torch.randn(s, d, device="cuda")
    tg = torch.randint(0, s, (m,), dtype=torch.int32, device="cuda")
    best = torch.empty(m, dtype=torch.int32, device="cuda")
    rank = torch.empty(m, dtype=torch.int32, device="cuda")
    bs = torch.empty(m, dtype=torch.float64, device="cuda")
    ts = torch.empty(m, dtype=torch.float64, device="cuda")
    desc = L.SpkIdentifyDesc(m=m, s=s, dims=d, queries=q.data_ptr(), bank=bank.data_ptr(), q_target=tg.data_ptr(),
                             best=best.data_ptr(), best_score=bs.data_ptr(), target_score=ts.data_ptr(),
                             target_rank=rank.data_ptr())
    S.identify(q[:4], bank)    # the Python path once
    us = 1e3 * events_ms(lambda: L.check(lib.avc_spk_identify(C.byref(desc), None), "avc_spk_identify"), iters,
                         min(iters, 10))
    fma = 2 * m * s * d
    return {"m": m, "s": s, "dims": d, "ms_per_launch": us / 1e3, "fp64_fma_per_s": fma / (us * 1e-6)}


def build(n_mels, n_spk, n_utts, reps=3):
    import oracle.ae_oracle as orc
    from adaptive_voice_conversion_b200.model import AE
    from adaptive_voice_conversion_b200.speaker_bank import build_bank
    cfg = orc.default_config(n_mels)
    model = AE(cfg)
    model.load_state_dict(orc.init_state(cfg, seed=0), strict=True)
    model = model.cuda().eval()
    rng = np.random.default_rng(0)
    torch.manual_seed(0)
    mels = {f"p{s:03d}_{k:03d}": torch.randn(int(rng.integers(100, 601)), n_mels, device="cuda")
            for s in range(n_spk) for k in range(n_utts)}
    frames = sum(int(v.shape[0]) for v in mels.values())
    ts = []
    median_wall_s(lambda: build_bank(model, mels), reps, samples=ts)
    t = min(ts)
    return {"c_in": n_mels, "speakers": n_spk, "utterances": len(mels), "input_frames": frames, "seconds": ts,
            "utterances_per_s": len(mels) / t, "input_frames_per_s": frames / t}


def main():
    p = argparse.ArgumentParser()
    p.add_argument("--m", type=int, default=100000)
    p.add_argument("--s", type=int, default=2000)
    p.add_argument("--dims", type=int, default=128)
    p.add_argument("--speakers", type=int, default=100)
    p.add_argument("--utts", type=int, default=40)
    p.add_argument("--mels", type=int, nargs="+", default=[80, 512])
    a = p.parse_args()
    res = {"card": card(), "pooling": pooling(a.speakers, a.utts), "identify": identify(a.m, a.s, a.dims),
           "build": [build(n, a.speakers, a.utts) for n in a.mels]}
    print(json.dumps(res))


if __name__ == "__main__":
    main()
