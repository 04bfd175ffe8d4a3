"""Cost and accuracy of banked pitch profiles and the mean-and-variance log-F0 transform (-pitch_shift mv).

    python tools/bench_pitch_profile.py [--utts 1000] [--frames 512] [--convs 64] [--out result.json]

1. Profile stage of a bank (speaker_bank.build_pitch_profiles) on --utts utterances of --frames frames at 512 mels
   (formant-shaped harmonic tones, 10 utterances per speaker), at the default 100 Griffin-Lim iterations: the wall
   seconds of synthesis, tracking and host work (each ended by a device synchronise), one call after a warm-up on 16
   utterances, and the same scaled to 1000 utterances.
2. Wav-to-wav cost of --convs conversions of --frames frames at 512 mels: mel_to_wav unshifted; match (match_shifts
   against one reference each, then mel_to_wav with its shifts); mv toward one reference each (mv_match, then
   mel_to_wav with the per-frame shifts); and mv toward a banked profile (no reference to synthesise).  Wall seconds,
   median of 3 after one warm-up; the host share of mv is the mv_shifts call alone.
3. Accuracy on tones with a known vibrato at 80 and 512 mels: a 150 Hz tone with 1 % vibrato moved by mv toward the
   profile of a 220 Hz tone with 4 % vibrato (both tracked as synthesised): the tracked log2 std after mv against the
   target's and before, and the mean's distance in semitones, against match's.  Then a glide: a per-frame target mean
   rising linearly by 7 semitones over the utterance (sigma_t = sigma_c): the median over the frames voiced in both of
   |12 log2(f0_out / f0_in) - s(f)|, and how many frames that is.
Prints one JSON line with the card's name and power limit.
"""
from __future__ import annotations

import argparse
import json
import os
import sys
import time

import numpy as np
import torch

from _harness import card, median_wall_s

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

SR, HOP = 24000, 300


def dev(a):
    return torch.from_numpy(np.ascontiguousarray(a, np.float32)).cuda()


def tone_mels(voc, specs, frames=None):
    """wav_to_mel of formant tones (f0, seconds, vibrato), cropped to `frames` when given."""
    from _pshift_ref import formant_tone
    mels = [m for m, _ in voc.wav_to_mel([dev(formant_tone(f, s, phase_seed=i, vibrato=v))
                                          for i, (f, s, v) in enumerate(specs)])]
    return [m[:frames].contiguous() for m in mels] if frames else mels


def profile_stage(n_utts, frames):
    from adaptive_voice_conversion_b200 import speaker_bank as SB
    from adaptive_voice_conversion_b200.vocoder import AudioParams, Vocoder
    voc = Vocoder(n_mels=512)
    secs = (frames + 40) * HOP / SR
    base = tone_mels(voc, [(90.0 + 7.0 * k, secs, 0.02) for k in range(20)], frames)
    attr = {"mean": np.zeros(512, np.float32), "std": np.ones(512, np.float32)}

    def bank_of(n):
        mels = {f"s{i // 10:04d}_{i % 10:03d}": base[i % len(base)] for i in range(n)}
        speakers, utts, _ = SB.bank_order(list(mels), {u: frames for u in mels}, 0, lambda u: u.split("_")[0])
        bank = SB.SpeakerBank(speakers, torch.zeros(len(speakers), 4, device="cuda"), [len(u) for u in utts], utts,
                              "f" * 64)
        return bank, mels
    SB.build_pitch_profiles(*bank_of(16), attr, AudioParams())
    bank, mels = bank_of(n_utts)
    t = {}
    SB.build_pitch_profiles(bank, mels, attr, AudioParams(), timings=t)
    total = sum(t.values())
    return {"utts": n_utts, "frames": frames, "seconds": t, "total_s": total,
            "per_1000_utts_s": {k: v * 1000.0 / n_utts for k, v in t.items()},
            "host_share": t["host"] / total}


def wav_to_wav(n_convs, frames):
    from adaptive_voice_conversion_b200 import f0 as F
    from adaptive_voice_conversion_b200.vocoder import Vocoder
    voc = Vocoder(n_mels=512)
    secs = (frames + 40) * HOP / SR
    convs = tone_mels(voc, [(100.0 + 3.0 * k, secs, 0.01) for k in range(n_convs)], frames)
    refs = tone_mels(voc, [(180.0 + 2.0 * k, secs, 0.04) for k in range(n_convs)], frames)
    hp = voc.hp
    prof = (float(np.log2(200.0)), 0.05)

    def match():
        s, _ = F.match_shifts(voc, convs, [[r] for r in refs], hp)
        voc.mel_to_wav(convs, semitones=s)

    def mv_refs():
        s, _ = F.mv_match(voc, convs, hp, ref_sets=[[r] for r in refs])
        voc.mel_to_wav(convs, semitones=s)

    def mv_bank():
        s, _ = F.mv_match(voc, convs, hp, profiles=[prof] * n_convs)
        voc.mel_to_wav(convs, semitones=s)
    res = {"convs": n_convs, "frames": frames, "unshifted_s": median_wall_s(lambda: voc.mel_to_wav(convs), 3),
           "match_s": median_wall_s(match, 3), "mv_refs_s": median_wall_s(mv_refs, 3),
           "mv_bank_s": median_wall_s(mv_bank, 3)}
    tracks = F.track_chunks(F.synthesize(voc, convs, hp), SR, HOP, F.F0Params())
    t0 = time.perf_counter()
    F.mv_shifts(tracks, [prof] * n_convs)
    res["mv_shifts_host_s"] = time.perf_counter() - t0
    return res


def accuracy(n_mels):
    from adaptive_voice_conversion_b200 import f0 as F
    from adaptive_voice_conversion_b200.vocoder import Vocoder
    voc = Vocoder(n_mels=n_mels)
    conv, ref = tone_mels(voc, [(150.0, 2.0, 0.01), (220.0, 2.0, 0.04)])
    tracks = F.track_chunks(F.synthesize(voc, [conv, ref], voc.hp), SR, HOP, F.F0Params())
    target = F.track_profile(tracks[1:])
    before = F.track_profile(tracks[:1])
    out = {"n_mels": n_mels, "target": target, "before": before}
    if target is None or before is None:
        out["note"] = "no voiced frame"
        return out
    mv, info = F.mv_shifts(tracks[:1], [target])
    match, _ = F.shifts_from_tracks(tracks[:1], [tracks[1:]])
    shifted = F.track_chunks(voc.mel_to_signal([conv, conv], semitones=[mv[0], match[0]]), SR, HOP, F.F0Params())
    after, matched = F.track_profile(shifted[:1]), F.track_profile(shifted[1:])
    out.update(after_mv=after, after_match=matched, info=info[0])
    if after is not None:
        out["sd_gap_st"] = {"before": 12 * abs(before[1] - target[1]), "mv": 12 * abs(after[1] - target[1])}
        out["mean_gap_st"] = {"mv": 12 * abs(after[0] - target[0]),
                              "match": None if matched is None else 12 * abs(matched[0] - target[0])}
    # a glide: the target mean rises 7 semitones over the utterance, the std kept
    T = conv.shape[0]
    mu = before[0] + np.linspace(0.0, 7.0 / 12.0, T)
    glide, _ = F.mv_shifts(tracks[:1], [(mu, np.full(T, before[1]))])
    (fa, va), (fb, vb) = F.track_chunks(voc.mel_to_signal([conv, conv], semitones=[0.0, glide[0]]), SR, HOP,
                                        F.F0Params())
    both = va & vb
    err = np.abs(12 * np.log2(fb[both] / fa[both]) - glide[0][both])
    out["glide"] = {"median_abs_err_st": float(np.median(err)) if both.any() else None,
                    "voiced_in_both": int(both.sum()), "frames": int(T)}
    return out


def main():
    ap = argparse.ArgumentParser(description=__doc__.splitlines()[0])
    ap.add_argument("--utts", type=int, default=1000)
    ap.add_argument("--frames", type=int, default=512)
    ap.add_argument("--convs", type=int, default=64)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    res = {"card": card(), "profile_stage": profile_stage(a.utts, a.frames),
           "wav_to_wav": wav_to_wav(a.convs, a.frames), "accuracy": [accuracy(80), accuracy(512)]}
    line = json.dumps(res)
    print(line)
    if a.out:
        with open(a.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
