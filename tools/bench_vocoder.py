"""Throughput of the GPU vocoder (csrc/audio.cu, adaptive_voice_conversion_b200/vocoder.py).

    python tools/bench_vocoder.py [--utts 64] [--frames 512] [--mels 80 512] [--windows 3] [--reps 3]
                                  [--momentum 0.99] [--sc-iters 8 16 32 64 100]

Workload: --utts utterances of --frames frames each (512 frames = 6.4 s at 24 kHz, hop 300), for each mel count.
Times, as the median over --windows windows of --reps calls each, every window ending in a device synchronise:
  - analysis   Vocoder.wav_to_mel (trim, pre-emphasis, STFT, mel projection);
  - synthesis  Vocoder.mel_to_wav (mel-to-linear, 100 Griffin-Lim iterations, de-emphasis, trim);
  - conversion wav -> mel (source and target), Inferencer.inference_ragged, mel -> wav.
Griffin-Lim kernel time per iteration comes from CUDA events around avc_griffin_lim with n_iter = 100 and 0, without
momentum and with --momentum (fast Griffin-Lim); the bytes an iteration must move are computed from the shapes below
and reported against 3.35 TB/s (H100 SXM HBM3).
Fast Griffin-Lim's effect: the median over the batch of the spectral convergence ||S - |STFT(y)||| / ||S|| for each
--sc-iters count, momentum 0 and --momentum, on two inputs: the consistent magnitudes |STFT| of the synthetic signals,
and the mel pseudo-inverse magnitudes mel_to_wav feeds Griffin-Lim (the signals' mels, mel_to_mag).  Then the wav-to-wav
rate at the fewest --sc-iters iterations whose median with --momentum on the mel input is at or below that of 100
plain iterations, if there is such a count.  The signals are synthetic (no speech is read), so these are
synthetic-signal numbers.
The card name and power limit are read in the same run.  The float64 numpy oracle's Griffin-Lim time for one
utterance on the host is printed for context.  Prints one JSON line; writes nothing.
"""
import argparse
import json
import os
import statistics
import subprocess
import sys
import time
import types

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import numpy as np  # noqa: E402
import torch  # noqa: E402

HBM_BPS = 3.35e12


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True).stdout.strip().splitlines()
    return q[torch.cuda.current_device()] if q else torch.cuda.get_device_name()


def utterances(n_utt, n_samples, seed=0):
    """Steady vibrato tones with harmonics and a noise floor: nothing is trimmed, so every utterance keeps its frames."""
    rng = np.random.default_rng(seed)
    t = np.arange(n_samples) / 24000
    out = []
    for _ in range(n_utt):
        f0 = rng.uniform(100, 250) * (1 + 0.03 * np.sin(2 * np.pi * 5 * t))
        ph = 2 * np.pi * np.cumsum(f0) / 24000
        y = sum(0.2 / k * np.sin(k * ph) for k in range(1, 7)) + 0.01 * rng.standard_normal(n_samples)
        out.append(torch.from_numpy(y.astype(np.float32)).cuda())
    return out


def timed(fn, windows, reps):
    fn()
    torch.cuda.synchronize()
    ts = []
    for _ in range(windows):
        t0 = time.perf_counter()
        for _ in range(reps):
            fn()
        torch.cuda.synchronize()
        ts.append((time.perf_counter() - t0) / reps)
    return statistics.median(ts), ts


def gl_bytes_per_iteration(F, n_samples, win, bins, momentum=False):
    """Least HBM traffic of one iteration: iSTFT frames read X and write the windowed frames, the overlap-add reads
    them and writes the signal, the projecting STFT reads the signal and S and writes the next X; with momentum it
    also reads and writes the previous spectrum P."""
    return (F * bins * 8 + F * win * 4 + F * win * 4 + n_samples * 4 + n_samples * 4 + F * bins * 4 + F * bins * 8
            + (2 * F * bins * 8 if momentum else 0))


def event_time(fn, reps):
    fn()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(reps):
        fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / 1e3 / reps


def gl_kernel_time(V, mags, hp, n_iter, momentum=0.0, reps=5):
    plan = V.GriffinLim(mags, hp, n_iter, momentum)
    return event_time(plan.run, reps)


def spectral_convergence(V, mags, ys):
    """||S - |STFT(y)||| / ||S|| per utterance, in float64 on the device."""
    out = []
    for S, (A, _) in zip(mags, V.magnitude(ys)):
        S = S.double()
        out.append(float(torch.linalg.norm(S - A.double()) / torch.linalg.norm(S)))
    return out


def convergence_table(V, mags, hp, iters, momenta, init=None):
    """{momentum: {n_iter: median spectral convergence over the batch}}, from the start ``init`` (default hp's)."""
    return {m: {n: statistics.median(spectral_convergence(V, mags, V.griffin_lim(mags, hp, n, m, init)))
                for n in iters} for m in momenta}


def fewest_iterations(table, momentum, plain_iters=100, target=None):
    """The fewest iterations of the table's grid whose median with momentum is at or below ``target``, by default
    plain Griffin-Lim's at plain_iters in the same table."""
    target = table[0.0][plain_iters] if target is None else target
    ok = [n for n, sc in sorted(table[momentum].items()) if sc <= target]
    return ok[0] if ok else None


def gl_stage_times(V, L, mags, hp, reps=20):
    """The two halves of an iteration on the Griffin-Lim buffers: iSTFT (frames + overlap-add) and projecting STFT."""
    plan = V.GriffinLim(mags, hp, 1).run()
    d_istft = L.AudioDesc.from_buffer_copy(plan.desc)
    d_stft = L.AudioDesc.from_buffer_copy(plan.desc)
    d_stft.mode = L.STFT_PROJECT
    t_istft = event_time(lambda: V._call("avc_istft", d_istft, plan.dev), reps)
    t_stft = event_time(lambda: V._call("avc_stft", d_stft, plan.dev), reps)
    return t_istft, t_stft


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--utts", type=int, default=64)
    ap.add_argument("--frames", type=int, default=512)
    ap.add_argument("--mels", type=int, nargs="+", default=[80, 512])
    ap.add_argument("--windows", type=int, default=3)
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--momentum", type=float, default=0.99)
    ap.add_argument("--sc-iters", type=int, nargs="+", default=[8, 16, 32, 64, 100])
    ap.add_argument("--skip-oracle", action="store_true")
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_vocoder needs a CUDA device")
    os.environ.setdefault("AVC_INFER_GRAPH", "1")
    import oracle.ae_oracle as orc
    import oracle.audio_oracle as ao
    from adaptive_voice_conversion_b200 import _lib as L
    from adaptive_voice_conversion_b200 import vocoder as V
    from adaptive_voice_conversion_b200.inference import Inferencer

    hp0 = V.AudioParams()
    n_samples = hp0.hop_length * (a.frames - 1)      # 1 + n // hop = frames
    audio_s = a.utts * n_samples / hp0.sr
    wavs = utterances(a.utts, n_samples)
    res = {"card": card(), "utts": a.utts, "frames": a.frames, "audio_seconds": round(audio_s, 3), "n_iter": hp0.n_iter,
           "momentum": a.momentum, "signals": "synthetic (vibrato tones with harmonics and a noise floor)"}
    print(f"card (name, power limit, max SM clock): {res['card']}", file=sys.stderr)
    iters = sorted(set(a.sc_iters) | {100})
    momenta = (0.0, a.momentum)
    consistent = [A for A, _ in V.magnitude(wavs, hp0)]
    res["sc_consistent"] = convergence_table(V, consistent, hp0, iters, momenta)
    print(f"median spectral convergence, consistent |STFT|: {res['sc_consistent']}", file=sys.stderr)
    for n_mels in a.mels:
        voc = V.Vocoder(n_mels=n_mels)
        hp = voc.hp
        pairs = voc.wav_to_mel(wavs)
        mels = [m for m, _ in pairs]
        assert all(m.shape[0] == a.frames for m in mels), [m.shape[0] for m in mels]
        cfg = orc.default_config(n_mels)
        inf = Inferencer(cfg, types.SimpleNamespace(attr=None, model=None, source=None, target=None, output=None,
                                                    sample_rate=hp.sr))
        inf.model.load_state_dict(orc.init_state(cfg, seed=0), strict=True)

        def convert(n_iter=None, momentum=None):
            src = [m for m, _ in voc.wav_to_mel(wavs)]
            tgt = src[1:] + src[:1]
            return voc.mel_to_wav(inf.inference_ragged(src, tgt), n_iter, momentum)

        t_ana, w_ana = timed(lambda: voc.wav_to_mel(wavs), a.windows, a.reps)
        t_syn, w_syn = timed(lambda: voc.mel_to_wav(mels), a.windows, a.reps)
        t_cnv, w_cnv = timed(convert, a.windows, 1)
        mags = voc.mel_to_mag(mels)
        t100 = gl_kernel_time(V, mags, hp, hp.n_iter)
        t0 = gl_kernel_time(V, mags, hp, 0)
        per_it = (t100 - t0) / hp.n_iter
        t_istft, t_stft = gl_stage_times(V, L, mags, hp)
        F = a.utts * a.frames
        nbytes = gl_bytes_per_iteration(F, a.utts * n_samples, hp.win_length, hp.n_bins)
        t100_m = gl_kernel_time(V, mags, hp, hp.n_iter, a.momentum)
        t0_m = gl_kernel_time(V, mags, hp, 0, a.momentum)
        per_it_m = (t100_m - t0_m) / hp.n_iter
        nbytes_m = gl_bytes_per_iteration(F, a.utts * n_samples, hp.win_length, hp.n_bins, momentum=True)
        sc_mel = convergence_table(V, mags, hp, iters, momenta)
        n_fast = fewest_iterations(sc_mel, a.momentum)
        fast = {"gl_iteration_us": per_it_m * 1e6, "gl_iteration_bytes": nbytes_m,
                "gl_iteration_TBps": nbytes_m / per_it_m / 1e12, "gl_iteration_vs_plain": per_it_m / per_it,
                "sc_mel_pseudo_inverse": sc_mel, "fewest_iters_at_or_below_plain_100": n_fast}
        if n_fast is not None:
            t_fast, w_fast = timed(lambda: convert(n_fast, a.momentum), a.windows, 1)
            fast["conversion"] = {"n_iter": n_fast, "utt_per_s": a.utts / t_fast, "audio_s_per_s": audio_s / t_fast,
                                  "windows_s": w_fast}
        res[f"mels{n_mels}"] = {
            "gl_istft_us": t_istft * 1e6, "gl_project_stft_us": t_stft * 1e6,
            "analysis": {"utt_per_s": a.utts / t_ana, "audio_s_per_s": audio_s / t_ana, "windows_s": w_ana},
            "synthesis": {"utt_per_s": a.utts / t_syn, "audio_s_per_s": audio_s / t_syn, "windows_s": w_syn},
            "conversion": {"utt_per_s": a.utts / t_cnv, "audio_s_per_s": audio_s / t_cnv, "windows_s": w_cnv},
            "gl_call_ms": t100 * 1e3, "gl_istft_only_ms": t0 * 1e3,
            "gl_iteration_us": per_it * 1e6, "gl_iteration_bytes": nbytes,
            "gl_iteration_TBps": nbytes / per_it / 1e12, "gl_iteration_frac_of_3.35TBps": nbytes / per_it / HBM_BPS,
            f"momentum_{a.momentum}": fast,
        }
        print(f"[mels={n_mels}] analysis {a.utts / t_ana:.1f} utt/s, synthesis {a.utts / t_syn:.2f} utt/s, "
              f"conversion {a.utts / t_cnv:.2f} utt/s; GL iteration {per_it * 1e6:.1f} us "
              f"({nbytes / per_it / 1e12:.2f} TB/s), with momentum {per_it_m * 1e6:.1f} us "
              f"({nbytes_m / per_it_m / 1e12:.2f} TB/s)", file=sys.stderr)
        print(f"[mels={n_mels}] median spectral convergence, mel pseudo-inverse: {sc_mel}; fewest iterations with "
              f"momentum at or below 100 plain: {n_fast}"
              + (f", wav to wav {fast['conversion']['utt_per_s']:.1f} utt/s" if n_fast is not None else ""),
              file=sys.stderr)
    if not a.skip_oracle:
        S = np.abs(ao.stft(wavs[0].cpu().numpy().astype(np.float64)))
        t = time.perf_counter()
        ao.griffin_lim(S, hp0.n_iter)
        res["oracle_numpy_griffin_lim_one_utt_s"] = time.perf_counter() - t
    print(json.dumps(res))


if __name__ == "__main__":
    main()
