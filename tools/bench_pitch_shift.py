"""Cost and accuracy of the formant-preserving pitch shift (avc_pitch_shift, Vocoder.mel_to_signal(semitones=)).

    python tools/bench_pitch_shift.py [--signals 64] [--frames 512] [--utts 16] [--out result.json]

1. avc_pitch_shift alone on --signals x --frames rows of mel pseudo-inverse magnitudes at the default lifter (40),
   shift +4 semitones: CUDA events around each call, median of 5 after one warm-up.  Bytes: each row's 1025 floats
   read and written (2 x 4100).  FLOPs: the two Q x 1025 cosine sums per row (cepstrum and envelope), 2 per fused
   multiply-add.  The shares are of the H100 SXM data sheet's 3.35 TB/s and 67 TFLOP/s FP32; the larger bound applies.
2. Wav-to-wav cost at 512 mels: mel_to_wav of --utts formant-shaped harmonic tones of 300-600 frames with shift 0, a
   fixed +4 and match (match_shifts against one reference tone each, then mel_to_wav with its shifts), at the default
   100 Griffin-Lim iterations and at the PGHI start with 8: wall seconds ended by a device synchronise, median of 3
   after one warm-up.
3. Pitch accuracy: formant-shaped tones (100, 150 and 220 Hz, 2 % vibrato, 1.5 s) -> wav_to_mel -> mel_to_signal with
   shift s and with 0 -> tracker, at 80 and 512 mels; the median over the frames voiced in both of
   |12 log2(f0_shifted / f0_unshifted) - s|, and how many frames that is.
Prints one JSON line with the card's name and power limit.
"""
from __future__ import annotations

import argparse
import json
import os
import sys

import numpy as np
import torch

from _harness import card, median_events_s, median_wall_s

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

HBM_PEAK = 3.35e12    # H100 SXM data sheet, bytes/s
FP32_PEAK = 67e12     # H100 SXM data sheet, FP32 FLOP/s without tensor cores
SHIFTS = (-12.0, -7.0, -3.0, 4.0, 7.0, 12.0)


def dev(a):
    return torch.from_numpy(np.ascontiguousarray(a, np.float32)).cuda()


def tones(voc, f0s, seconds, seed=0):
    from _pshift_ref import formant_tone
    return [m for m, _ in voc.wav_to_mel([dev(formant_tone(f, s, phase_seed=seed + i, vibrato=0.02))
                                          for i, (f, s) in enumerate(zip(f0s, seconds))])]


def kernel(n_signals, n_frames):
    from adaptive_voice_conversion_b200 import vocoder as V
    from adaptive_voice_conversion_b200 import _lib as L
    voc = V.Vocoder(n_mels=512)
    rng = np.random.default_rng(0)
    mels = tones(voc, rng.uniform(80, 300, 8), [n_frames * 300 / 24000 + 0.1] * 8)
    mag = torch.cat(voc.mel_to_mag(mels))
    rows = n_signals * n_frames
    S = mag[torch.arange(rows, device="cuda") % mag.shape[0]].contiguous()
    ratio = torch.full((rows,), float(np.float32(2 ** (4 / 12))), device="cuda")
    out = torch.empty_like(S)
    lifter = voc.hp.ps_lifter
    lib = L.load()

    def call():
        L.check(lib.avc_pitch_shift(S.data_ptr(), ratio.data_ptr(), out.data_ptr(), rows, 1025, lifter,
                                    torch.cuda.current_stream().cuda_stream), "avc_pitch_shift")
    t = median_events_s(call, 5)
    bytes_ = 2 * 4100 * rows
    flops = 2 * 2 * lifter * 1025 * rows
    t_hbm, t_fp32 = bytes_ / HBM_PEAK, flops / FP32_PEAK
    return {"rows": rows, "lifter": lifter, "seconds": t, "bytes": bytes_, "flops": flops,
            "GB_per_s": bytes_ / t / 1e9, "TFLOP_per_s": flops / t / 1e12,
            "share_of_hbm_bound": t_hbm / t, "share_of_fp32_bound": t_fp32 / t,
            "bound": "hbm" if t_hbm >= t_fp32 else "fp32", "share_of_bound": max(t_hbm, t_fp32) / t}


def wav_to_wav(n_utts):
    from adaptive_voice_conversion_b200 import f0 as F
    from adaptive_voice_conversion_b200 import vocoder as V
    rng = np.random.default_rng(1)
    secs = rng.uniform(300, 600, n_utts) * 300 / 24000
    out = {}
    for label, kw in (("gl100_zero", dict(n_iter=100)), ("gl8_pghi", dict(n_iter=8, gl_init="pghi"))):
        voc = V.Vocoder(n_mels=512, hp=V.AudioParams(**kw))
        convs = tones(voc, rng.uniform(90, 150, n_utts), secs)
        refs = tones(voc, rng.uniform(180, 260, n_utts), secs[::-1], seed=100)

        def match():
            shifts, _ = F.match_shifts(voc, convs, [[r] for r in refs], voc.hp)
            return voc.mel_to_wav(convs, semitones=shifts)
        r = {"utterances": n_utts, "frames": int(sum(m.shape[0] for m in convs)),
             "shift_0_s": median_wall_s(lambda: voc.mel_to_wav(convs), 3),
             "shift_+4_s": median_wall_s(lambda: voc.mel_to_wav(convs, semitones=4.0), 3),
             "match_s": median_wall_s(match, 3)}
        r["match_over_shift_0"] = r["match_s"] / r["shift_0_s"]
        r["fixed_over_shift_0"] = r["shift_+4_s"] / r["shift_0_s"]
        out[label] = r
    return out


def accuracy():
    from adaptive_voice_conversion_b200 import f0 as F
    from adaptive_voice_conversion_b200 import vocoder as V
    out = {}
    for n_mels in (80, 512):
        voc = V.Vocoder(n_mels=n_mels)
        mels = tones(voc, (100.0, 150.0, 220.0), (1.5, 1.5, 1.5), seed=7)
        base = F.track(voc.mel_to_signal(mels), 24000, 300)
        res = {}
        for s in SHIFTS:
            shifted = F.track(voc.mel_to_signal(mels, semitones=s), 24000, 300)
            errs, frames = [], 0
            for (fa, va), (fb, vb) in zip(base, shifted):
                both = va & vb
                errs.append(np.abs(12 * np.log2(fb[both] / fa[both]) - s))
                frames += len(va)
            e = np.concatenate(errs)
            res[f"{s:+g}"] = {"median_abs_error_semitones": float(np.median(e)) if e.size else None,
                              "voiced_in_both": int(e.size), "frames": frames}
        out[str(n_mels)] = res
    return out


def main():
    p = argparse.ArgumentParser()
    p.add_argument("--signals", type=int, default=64)
    p.add_argument("--frames", type=int, default=512)
    p.add_argument("--utts", type=int, default=16)
    p.add_argument("--out", default=None)
    a = p.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_pitch_shift needs a GPU")
    res = {"card": card(), "kernel": kernel(a.signals, a.frames), "wav_to_wav_512": wav_to_wav(a.utts),
           "pitch_accuracy": accuracy()}
    line = json.dumps(res)
    print(line)
    if a.out:
        with open(a.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
