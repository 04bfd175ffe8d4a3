"""Corpus preparation throughput: preprocess.py's (or preprocess_libri.py's) pipeline on a seeded synthetic corpus,
stage by stage, against today's single-file path (Vocoder.get_spectrograms per file: host resample_poly, then GPU
analysis).

    python tools/bench_prepare.py [--corpus vctk|libri] [--utts 2000] [--speakers 40] [--n_mels 512]
        [--chunk_seconds 1800] [--out DIR]

--corpus vctk (default): VCTK-shaped, 48 kHz int16 mono, so the resampler halves the rate.  --corpus libri:
LibriTTS-shaped (train-clean-100 and dev-clean, speaker / chapter / file, a tenth of the speakers in dev-clean), 24 kHz
int16 mono, so the resampler only converts the format.  Each file is 2-5 s of tone and noise between leading and
trailing silence, written to a temporary directory (deleted afterwards).  Host stages are wall-clock; device stages
are CUDA events around their launches, summed over chunks.  End to end is one run of all four stages; stage 0 is that
run less the timed stages 1-3 (reduce, index sampling).  "headers" is the first pass over the files (their lengths,
for the chunk planner); "decode" is the full read of each chunk's files.  avc_resample_poly's traffic is 2 bytes read
per input sample and 4 written per output sample (plus its tap table and the staged windows' overlap, not counted).
"resample_pairs" times avc_resample_poly alone on 10 minutes of 3 s int16 files at 48 kHz -> 24 kHz, whose tap table
is staged in shared memory, and at 11.025 kHz -> 48 kHz, whose table (13 440 floats) does not fit beside the window and
is read through L1: the median of 7 calls of Preparer.resample's launches, CUDA events.
The card's name, power limit and clock are read in the same run.
"""
import argparse
import contextlib
import functools
import json
import os
import shutil
import sys
import tempfile
import time
from collections import defaultdict

import numpy as np
import torch
from scipy.io import wavfile

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from adaptive_voice_conversion_b200 import prepare as P   # noqa: E402
from adaptive_voice_conversion_b200 import vocoder as V   # noqa: E402
from _harness import card   # noqa: E402

HBM_BYTES_PER_S = 3.35e12   # H100 SXM data sheet


class Timer:
    def __init__(self):
        self.host_s = defaultdict(float)
        self.events = defaultdict(list)

    @contextlib.contextmanager
    def host(self, name):
        t0 = time.perf_counter()
        yield
        self.host_s[name] += time.perf_counter() - t0

    @contextlib.contextmanager
    def device(self, name):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        yield
        b.record()
        self.events[name].append((a, b))

    def device_s(self):
        torch.cuda.synchronize()
        return {k: sum(a.elapsed_time(b) for a, b in v) / 1e3 for k, v in self.events.items()}


def synth_pcm(rng, sr):
    n = int(sr * rng.uniform(2.0, 5.0))
    t = np.arange(n) / sr
    f0 = rng.uniform(100, 250)
    y = sum(rng.uniform(0.05, 0.2) / k * np.sin(2 * np.pi * k * f0 * t + rng.uniform(0, 6.3)) for k in range(1, 5))
    y += 0.02 * rng.standard_normal(n)
    y = np.concatenate([np.zeros(int(0.3 * sr)), y, np.zeros(int(0.4 * sr))])
    return np.round(np.clip(y, -1, 1 - 2 ** -15) * 32768).astype(np.int16)


def write_corpus(root, n_utts, n_speakers, seed):
    rng = np.random.default_rng(seed)
    wav = os.path.join(root, "wav48")
    speakers = [str(225 + i) for i in range(n_speakers)]
    n_in = []
    for u in range(n_utts):
        spk = speakers[u % n_speakers]
        os.makedirs(os.path.join(wav, f"p{spk}"), exist_ok=True)
        pcm = synth_pcm(rng, 48000)
        wavfile.write(os.path.join(wav, f"p{spk}", f"p{spk}_{u // n_speakers + 1:03d}.wav"), 48000, pcm)
        n_in.append(pcm.size)
    info = os.path.join(root, "speaker-info.txt")
    with open(info, "w") as f:
        f.write("ID  AGE  GENDER  ACCENTS  REGION\n")
        f.writelines(f"{s}  23  F  English  Somewhere\n" for s in speakers)
    return wav, info, np.array(n_in, np.int64)


def write_libri_corpus(root, n_utts, n_speakers, seed):
    """<root>/LibriTTS/{train-clean-100,dev-clean}/<speaker>/<chapter>/<speaker>_<chapter>_<p>_<s>.wav, two chapters
    per speaker, the last tenth of the speakers (at least one) in dev-clean."""
    rng = np.random.default_rng(seed)
    libri = os.path.join(root, "LibriTTS")
    speakers = [str(100 + 7 * i) for i in range(n_speakers)]
    n_dev = max(1, n_speakers // 10)
    n_in = []
    for u in range(n_utts):
        i = u % n_speakers
        spk, ch, k = speakers[i], str(1000 + 10 * i + (u // n_speakers) % 2), u // n_speakers
        d = os.path.join(libri, "dev-clean" if i >= n_speakers - n_dev else "train-clean-100", spk, ch)
        os.makedirs(d, exist_ok=True)
        pcm = synth_pcm(rng, 24000)
        wavfile.write(os.path.join(d, f"{spk}_{ch}_{k:06d}_{k + 1:06d}.wav"), 24000, pcm)
        n_in.append(pcm.size)
    return libri, np.array(n_in, np.int64)


RESAMPLE_PAIRS = [(48000, 24000), (11025, 48000)]


def resample_pairs(seed, seconds=600.0, reps=7):
    """{"<rate>-><target>": ms, traffic and whether the tap table is staged} of avc_resample_poly per RESAMPLE_PAIRS."""
    out = {}
    for rate, sr in RESAMPLE_PAIRS:
        rng = np.random.default_rng(seed)
        items = [(rate, synth_pcm(rng, rate)[:3 * rate]) for _ in range(int(seconds // 3))]
        prep = P.Preparer(80, sr)
        prep.resample(items)
        ts = []
        for _ in range(reps):
            prep.timer = Timer()
            prep.resample(items)
            ts.append(prep.timer.device_s()["resample"])
        up, down = P.rate_pair(rate, sr)
        half, tab = P.resample_taps(up, down)
        window = 511 * down // up + tab.shape[1] + 1
        n_in = sum(a.size for _, a in items)
        n_bytes = 2 * n_in + 4 * sum(P.n_resampled(a.size, up, down) for _, a in items)
        t = float(np.median(ts))
        out[f"{rate}->{sr}"] = {"up_down": [up, down], "taps": int(tab.size), "staged_taps": 4 * (tab.size + window) <= 48 * 1024,
                                "ms": round(1e3 * t, 3), "GB_per_s": round(n_bytes / t / 1e9, 1)}
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--corpus", choices=("vctk", "libri"), default="vctk")
    ap.add_argument("--utts", type=int, default=2000)
    ap.add_argument("--speakers", type=int, default=40)
    ap.add_argument("--n_mels", type=int, default=512)
    ap.add_argument("--chunk_seconds", type=float, default=1800.0)
    ap.add_argument("--seed", type=int, default=0)
    ap.add_argument("--out", default=None, help="write the JSON result here as well")
    a = ap.parse_args()
    assert torch.cuda.is_available(), "bench_prepare needs a GPU"
    root = tempfile.mkdtemp(prefix="bench_prepare_")
    opts = dict(n_mels=a.n_mels, n_utts_attr=5000, training_samples=100000, testing_samples=10000,
                chunk_seconds=a.chunk_seconds, log=lambda *x: None)
    if a.corpus == "vctk":
        rate = 48000

        def corpus(d, n_utts, n_speakers, seed):
            wav, info, n_in = write_corpus(d, n_utts, n_speakers, seed)
            paths = sorted(os.path.join(wav, s, f) for s in os.listdir(wav) for f in os.listdir(os.path.join(wav, s)))
            prepare = functools.partial(P.run, wav, info, n_out_speakers=max(1, n_speakers // 10), **opts)
            return prepare, paths, n_in
    else:
        rate = 24000

        def corpus(d, n_utts, n_speakers, seed):
            libri, n_in = write_libri_corpus(d, n_utts, n_speakers, seed)
            paths = P.read_libri_paths(libri, "train-clean-100") + P.read_libri_paths(libri, "dev-clean")
            return functools.partial(P.run_libri, libri, test_prop=0.05, **opts), paths, n_in
    try:
        t0 = time.perf_counter()
        prepare, paths, n_in = corpus(root, a.utts, a.speakers, a.seed)
        print(f"corpus: {a.corpus}, {a.utts} files, {n_in.sum() / rate / 3600:.2f} h at {rate // 1000} kHz, written in "
              f"{time.perf_counter() - t0:.1f} s", flush=True)
        # warm-up: modules, tap tables and the allocator, on a small tree of its own
        warm = os.path.join(root, "warm")
        prepare_w, _, _ = corpus(warm, 40, 4, a.seed + 1)
        prepare_w(os.path.join(warm, "out"))
        torch.cuda.synchronize()

        # one preprocess run (stage 0 runs every stage, as the shell script's -le rule does)
        timer = Timer()
        t0 = time.perf_counter()
        prepare(os.path.join(root, "out"), stage=0, timer=timer)
        torch.cuda.synchronize()
        t_all = time.perf_counter() - t0
        t_index = timer.host_s["reduce_and_index"]
        t_features = t_all - t_index
        t_no_pickle = t_features - timer.host_s["pickle"]
        dev = timer.device_s()
        skipped = open(os.path.join(root, "out", "skipped_files.txt")).read().count("\n")

        n_out = -(-n_in * 24000 // rate)
        rs_bytes = 2 * int(n_in.sum()) + 4 * int(n_out.sum())
        audio_s = n_in.sum() / rate

        # today's path: one file at a time through Vocoder.get_spectrograms
        voc = V.Vocoder(n_mels=a.n_mels)
        voc.get_spectrograms(paths[0])
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        for p in paths:
            voc.get_spectrograms(p)
        t_base = time.perf_counter() - t0

        pairs = resample_pairs(a.seed)
        res = {
            "card": card(),
            "corpus": a.corpus, "files": a.utts, "audio_hours": round(float(audio_s) / 3600, 3), "n_mels": a.n_mels,
            "chunk_seconds": a.chunk_seconds, "skipped": skipped,
            "host_s": {k: round(v, 3) for k, v in timer.host_s.items()},
            "device_s": {k: round(v, 4) for k, v in dev.items()},
            "resample": {"bytes": rs_bytes, "GB_per_s": round(rs_bytes / dev["resample"] / 1e9, 1),
                         "share_of_3.35TB_per_s": round(rs_bytes / dev["resample"] / HBM_BYTES_PER_S, 3)},
            "resample_pairs": pairs,
            "stage0_s": round(t_features, 2),
            "stage0_without_pickling_s": round(t_no_pickle, 2),
            "stages1_3_s": round(t_index, 2),
            "end_to_end": {"s": round(t_all, 2), "utts_per_s": round(a.utts / t_all, 1),
                           "audio_s_per_s": round(float(audio_s) / t_all, 1)},
            "stage0": {"utts_per_s": round(a.utts / t_features, 1), "audio_s_per_s": round(float(audio_s) / t_features, 1)},
            "baseline_get_spectrograms": {"s": round(t_base, 2), "utts_per_s": round(a.utts / t_base, 1),
                                          "audio_s_per_s": round(float(audio_s) / t_base, 1)},
        }
        print(json.dumps(res, indent=1))
        if a.out:
            os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
            with open(a.out, "w") as f:
                json.dump(res, f, indent=1)
    finally:
        shutil.rmtree(root, ignore_errors=True)


if __name__ == "__main__":
    main()
