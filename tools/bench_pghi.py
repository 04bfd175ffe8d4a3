"""The PGHI start phase of the GPU vocoder (avc_pghi, ``init="pghi"``): its cost and what it buys Griffin-Lim.

    python tools/bench_pghi.py [--utts 64] [--frames 512] [--long 10000] [--mels 80 512] [--momentum 0.99]
                               [--sc-iters 0 8 16 32 64 100] [--windows 3]

Reports, in one JSON line (and a summary on stderr):
  - the avc_pghi launch alone (CUDA events around the C call on prebuilt buffers, median of --windows windows) for
    --utts utterances of --frames frames, and for one utterance of --long frames: the integration is serial in frames,
    so a long single utterance is its worst case;
  - the median over the batch of the spectral convergence ||S - |STFT(y)||| / ||S|| after each --sc-iters count,
    for the zero and pghi starts, at momentum 0 and --momentum, on the consistent magnitudes |STFT| of
    tools/bench_vocoder.py's synthetic signals and on the mel pseudo-inverse magnitudes mel_to_wav feeds Griffin-Lim
    (their mels, mel_to_mag) at each --mels count;
  - per mel count and momentum, the fewest iterations of the --sc-iters grid whose pghi-start median on the mel input
    is at or below that of 100 plain zero-phase iterations (the true count lies between it and the grid's previous
    entry), and the wav-to-wav rate (wav -> mel, Inferencer.inference_ragged, mel -> wav with that start) at that
    count.
The card name and power limit are read in the same run.  The signals are synthetic (vibrato tones with harmonics and a
noise floor); speech is not measured.  Writes nothing.
"""
import argparse
import ctypes as C
import json
import os
import statistics
import sys
import types

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))

import torch  # noqa: E402

from bench_vocoder import card, convergence_table, event_time, fewest_iterations, timed, utterances  # noqa: E402

INITS = ("zero", "pghi")


def pghi_time(V, mags, hp, windows, reps=5):
    """The avc_pghi launch alone: the magnitudes, the utterance table and X are built once, outside the timing."""
    S = torch.cat(mags).contiguous()
    r = V._Ragged([0] * len(mags), [m.shape[0] for m in mags], S.device)
    X = torch.empty(S.shape[0], hp.n_bins, 2, device=S.device)
    d = r.desc(hp, mag=S, X=X)
    tol = C.c_float(hp.pghi_tol)
    return statistics.median(event_time(lambda: V._call("avc_pghi", d, S.device, tol, None), reps)
                             for _ in range(windows))


def tables(V, mags, hp, iters, momenta):
    """{init: {momentum: {n_iter: median spectral convergence over the batch}}}"""
    return {init: convergence_table(V, mags, hp, iters, momenta, init) for init in INITS}


def fewest_pghi_iterations(table, momentum, plain_iters=100):
    """The fewest grid iterations whose pghi-start median at this momentum is at or below zero phase's without
    momentum at plain_iters."""
    return fewest_iterations(table["pghi"], momentum, target=table["zero"][0.0][plain_iters])


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--utts", type=int, default=64)
    ap.add_argument("--frames", type=int, default=512)
    ap.add_argument("--long", type=int, default=10000)
    ap.add_argument("--mels", type=int, nargs="+", default=[80, 512])
    ap.add_argument("--momentum", type=float, default=0.99)
    ap.add_argument("--sc-iters", type=int, nargs="+", default=[0, 8, 16, 32, 64, 100])
    ap.add_argument("--windows", type=int, default=3)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_pghi needs a CUDA device")
    os.environ.setdefault("AVC_INFER_GRAPH", "1")
    import oracle.ae_oracle as orc
    from adaptive_voice_conversion_b200 import vocoder as V
    from adaptive_voice_conversion_b200.inference import Inferencer

    hp0 = V.AudioParams()
    n_samples = hp0.hop_length * (a.frames - 1)
    audio_s = a.utts * n_samples / hp0.sr
    wavs = utterances(a.utts, n_samples)
    res = {"card": card(), "utts": a.utts, "frames": a.frames, "long_frames": a.long, "momentum": a.momentum,
           "pghi_tol": hp0.pghi_tol, "signals": "synthetic (vibrato tones with harmonics and a noise floor)"}
    print(f"card (name, power limit, max SM clock): {res['card']}", file=sys.stderr)
    iters = sorted(set(a.sc_iters) | {100})
    momenta = (0.0, a.momentum)
    consistent = [A for A, _ in V.magnitude(wavs, hp0)]
    res["pghi_ms"] = pghi_time(V, consistent, hp0, a.windows) * 1e3
    long_mag = [A for A, _ in V.magnitude(utterances(1, hp0.hop_length * (a.long - 1), seed=1), hp0)]
    res["pghi_long_ms"] = pghi_time(V, long_mag, hp0, a.windows, reps=2) * 1e3
    print(f"avc_pghi: {a.utts} x {a.frames} frames {res['pghi_ms']:.3f} ms, 1 x {a.long} frames "
          f"{res['pghi_long_ms']:.3f} ms", file=sys.stderr)
    res["sc_consistent"] = tables(V, consistent, hp0, iters, momenta)
    print(f"median spectral convergence, consistent |STFT|: {res['sc_consistent']}", file=sys.stderr)
    for n_mels in a.mels:
        voc = V.Vocoder(n_mels=n_mels)
        hp = voc.hp
        mels = [m for m, _ in voc.wav_to_mel(wavs)]
        assert all(m.shape[0] == a.frames for m in mels), [m.shape[0] for m in mels]
        mags = voc.mel_to_mag(mels)
        table = tables(V, mags, hp, iters, momenta)
        out = {"sc_mel_pseudo_inverse": table}
        cfg = orc.default_config(n_mels)
        inf = Inferencer(cfg, types.SimpleNamespace(attr=None, model=None, source=None, target=None, output=None,
                                                    sample_rate=hp.sr))
        inf.model.load_state_dict(orc.init_state(cfg, seed=0), strict=True)

        def convert(n_iter=None, momentum=None, init=None):
            src = [m for m, _ in voc.wav_to_mel(wavs)]
            tgt = src[1:] + src[:1]
            return voc.mel_to_wav(inf.inference_ragged(src, tgt), n_iter, momentum, init)

        t_plain, _ = timed(convert, a.windows, 1)
        out["conversion_zero_100"] = {"utt_per_s": a.utts / t_plain, "audio_s_per_s": audio_s / t_plain}
        for m in momenta:
            n_fast = fewest_pghi_iterations(table, m)
            rec = {"fewest_pghi_grid_iters_at_or_below_zero_100": n_fast}
            if n_fast is not None:
                t_fast, w_fast = timed(lambda: convert(n_fast, m, "pghi"), a.windows, 1)
                rec["conversion"] = {"n_iter": n_fast, "utt_per_s": a.utts / t_fast, "audio_s_per_s": audio_s / t_fast,
                                     "windows_s": w_fast}
            out[f"momentum_{m}"] = rec
            print(f"[mels={n_mels}] momentum {m}: fewest pghi-start grid iterations at or below 100 plain: {n_fast}"
                  + (f", wav to wav {rec['conversion']['utt_per_s']:.1f} utt/s" if n_fast is not None else ""),
                  file=sys.stderr)
        print(f"[mels={n_mels}] median spectral convergence, mel pseudo-inverse: {table}; wav to wav with 100 plain "
              f"iterations {a.utts / t_plain:.1f} utt/s", file=sys.stderr)
        res[f"mels{n_mels}"] = out
    print(json.dumps(res))


if __name__ == "__main__":
    main()
