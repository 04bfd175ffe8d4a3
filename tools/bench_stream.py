"""Streaming conversion (adaptive_voice_conversion_b200/streaming.py): update time per stage and how many streams fit
in real time.

    python tools/bench_stream.py [--streams 1 64 1024 4096] [--updates 20] [--config config.yaml] [-m ckpt -a attr]
                                 [-pitch {0,SEMITONES,match,mv}] [-retarget]

Reports, in one JSON line (and a summary on stderr):
  - per stream count S, at the default StreamParams (H = 8 frames = 100 ms per block): the mean wall time of one
    steady-state update (every stream pushes H hop samples, so every stream emits one block) split into analysis,
    conversion and RTISI-LA, each stage ended by a device synchronise; and the largest measured S whose update fits
    in the H frames' duration;
  - the avc_rtisi_la kernel alone (CUDA events around the C call on tables prepared beforehand, each launch from the
    same steady-state state of the largest S, median of 7) and its rate of 2048-point FFTs against offline
    Griffin-Lim's (avc_griffin_lim, 16 iterations on the same number of frames, median of 7);
  - with -m and -a: the frame-aligned mel L1 and cepstral distance (avc_mel_cepstrum, no DTW: the same frame grid)
    between the streamed mel and the offline conversion of the same untrimmed input.
  - with -pitch: every stream opened with that pitch setting (a fixed shift, or match / mv toward log2 F0 mean
    log2(200 Hz), std 0.15), the stages then include shadow, tracking, tracking_copy (the YIN outputs' one
    device-to-host copy) and shift; the latency with tracking; the avc_yin_window kernel alone (CUDA events on tables
    prepared beforehand, median of 7) at 64 and 1 024 streams x 8 frames; and for match / mv the output's voiced log2
    F0 mean and std error (semitones, median over 5 synthetic glides, seeds 0-4) after warm-up, tracked offline, for
    glides pushed as magnitudes through PitchStage toward the GPU test's target (log2(220 Hz), 0.15), the test's
    seeds 0-2 among them;
  - with -retarget: before every update (start-up and timed alike) each stream is retargeted (at=None) to the next of
    four codes over a ramp of H frames, so every window of every stream in steady state is a morph window (up to
    four anchors, K = 4) and every frame lies in a ramp: the worst case.  The host time of the retarget calls is the
    stage "retarget".
The model has random weights unless -m is given; the input is synthetic (harmonic tones).  The card name and power
limit are read in the same run.  Writes nothing.
"""
import argparse
import ctypes as C
import dataclasses
import json
import math
import os
import sys
import types

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

import numpy as np  # noqa: E402
import torch  # noqa: E402

from _harness import card, median_events_s  # noqa: E402
from adaptive_voice_conversion_b200 import _lib as L  # noqa: E402


def harmonic(n, sr, seed):
    from _rtisi_ref import harmonic as h
    return torch.from_numpy(h(n, sr, seed=seed).astype(np.float32))


def yin_window_ms(n_streams, hp, dev, frames=8, origin=40):
    """avc_yin_window alone: n_streams entries of `frames` frames each at a steady-state origin, the table and buffers
    prepared beforehand, CUDA events around the C call (median of 7 after a warm-up)."""
    import ctypes as C
    from adaptive_voice_conversion_b200 import _lib as L
    from adaptive_voice_conversion_b200.f0 import F0Params
    from adaptive_voice_conversion_b200.streaming import yin_last_sample
    from adaptive_voice_conversion_b200.utils import _stream
    from adaptive_voice_conversion_b200.vocoder import _SEG, _ptr
    fp = F0Params()
    span = fp.win + fp.tau_max(hp.sr)
    first = max(0, origin * hp.hop_length - span // 2 - 1)
    n = yin_last_sample(origin + frames - 1, hp.hop_length, span) + 1 - first
    y = torch.randn(n_streams * n, device=dev)
    tab = np.zeros(n_streams, _SEG)
    for k in range(n_streams):
        tab[k] = (k * n, n, k * frames, frames, origin)
    table = torch.from_numpy(tab.view(np.uint8)).to(dev)
    out = torch.empty(3, n_streams * frames, dtype=torch.float64, device=dev)
    d = L.AudioDesc(hop=hp.hop_length, n_seg=n_streams, n_frames=n_streams * frames, n_samples=int(y.numel()),
                    segs=_ptr(table), y=_ptr(y))

    def launch():
        L.check(L.load().avc_yin_window(C.byref(d), fp.win, fp.tau_min(hp.sr), fp.tau_max(hp.sr),
                                        C.c_float(fp.threshold), _ptr(out[0]), _ptr(out[1]), _ptr(out[2]),
                                        _stream(dev)), "avc_yin_window")
    return 1e3 * median_events_s(launch, 7)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--streams", type=int, nargs="+", default=[1, 64, 1024, 4096])
    ap.add_argument("--updates", type=int, default=20)
    ap.add_argument("--config", "-c", default=os.path.join(ROOT, "config.yaml"))
    ap.add_argument("-m", "--model")
    ap.add_argument("-a", "--attr")
    ap.add_argument("--quality-seconds", type=float, default=6.0)
    ap.add_argument("-pitch", "--pitch", default="0", help="pitch setting of every stream: 0, SEMITONES, match or mv")
    ap.add_argument("-retarget", "--retarget", action="store_true",
                    help="retarget every stream before every update (a ramp of H frames through four codes)")
    ap.add_argument("-stream_gl_init", "--stream-gl-init", default="estimate", choices=["estimate", "pghi"],
                    help="RTISI-LA's start phase (StreamParams.gl_init); pghi also times avc_pghi_stream alone")
    args = ap.parse_args()
    target = (math.log2(200.0), 0.15)
    pitch = (args.pitch, *target) if args.pitch in ("match", "mv") else (float(args.pitch) or None)
    if not torch.cuda.is_available():
        raise SystemExit("bench_stream.py needs a CUDA device")
    from adaptive_voice_conversion_b200.config import load_config
    from adaptive_voice_conversion_b200.inference import Inferencer
    from adaptive_voice_conversion_b200.streaming import StreamingConverter, StreamParams
    from adaptive_voice_conversion_b200.vocoder import GriffinLim, Vocoder

    cfg = load_config(args.config)
    torch.manual_seed(0)
    inf = Inferencer(cfg, types.SimpleNamespace(model=args.model, attr=args.attr))
    dev = torch.device("cuda:0")
    voc = Vocoder(n_mels=cfg["SpeakerEncoder"]["c_in"], device=dev)
    hp = voc.hp
    p = StreamParams(gl_init=args.stream_gl_init)
    block = p.hop * hp.hop_length
    budget_ms = 1e3 * block / hp.sr
    c_out = cfg["SpeakerEncoder"]["c_out"]
    res = {"card": card(), "params": p.__dict__, "block_ms": budget_ms, "n_mels": hp.n_mels, "pitch": args.pitch,
           "retarget": args.retarget, "stages": {}}
    import time
    from adaptive_voice_conversion_b200.streaming import KEEP
    pool = [torch.randn(c_out, generator=torch.Generator().manual_seed(10 ** 6 + k)).to(dev) for k in range(4)]

    def push(conv, ids, chunk, k):
        """One update, after retargeting every stream with -retarget (its host time added to stage "retarget")."""
        if args.retarget:
            t0 = time.perf_counter()
            for i, sid in enumerate(ids):
                conv.retarget(sid, pool[(k + i) % len(pool)], ramp=p.hop, pitch=KEEP)
            if conv.stage_ms is not None:
                conv.stage_ms["retarget"] = conv.stage_ms.get("retarget", 0.0) + 1e3 * (time.perf_counter() - t0)
        conv.push({sid: chunk for sid in ids})
    rt_ms = None
    for S in args.streams:
        conv = StreamingConverter(inf, voc, p)
        ids = [conv.open(torch.randn(c_out, generator=torch.Generator().manual_seed(i)).to(dev), pitch)
               for i in range(S)]
        res["latency_samples"], res["tracked_latency_samples"] = conv.latency_samples, conv.tracked_latency_samples
        sig = harmonic(block * (args.updates + 40), hp.sr, seed=S).to(dev)
        # start-up (the first block needs m frames, start-up windows of every length) and graph captures
        pos = 0
        for k in range(20):
            push(conv, ids, sig[pos:pos + block], k)
            pos += block
        conv.stage_ms = {}
        torch.cuda.synchronize()
        for k in range(20, 20 + args.updates):
            push(conv, ids, sig[pos:pos + block], k)
            pos += block
        st = {k: v / args.updates for k, v in conv.stage_ms.items()}
        st["update"] = sum(st.values())
        res["stages"][S] = st
        parts = ", ".join(f"{k} {v:.2f}" for k, v in st.items() if k != "update")
        print(f"S={S:5d}: update {st['update']:.2f} ms ({parts}); block {budget_ms:.0f} ms", file=sys.stderr)
        if S == max(args.streams):
            # the avc_rtisi_la kernel alone: one steady-state update's tables and buffers prepared once, then the C
            # call timed by CUDA events, each launch from a copy of the same state (the copy outside the events)
            conv.stage_ms = None
            mags = {sid: voc.mel_to_mag([torch.rand(p.hop, hp.n_mels, device=dev)])[0] for sid in ids}
            pghi = p.gl_init == "pghi"
            state0, count0 = conv.rt.state.clone(), conv.rt.count.clone()
            pstate0 = conv.rt.pstate.clone() if pghi else None
            desc, _, keep = conv.rt.prepare(mags)
            ev = [torch.cuda.Event(enable_timing=True) for _ in range(3)]
            times, ptimes = [], []
            lib = L.load()
            for _ in range(7):
                conv.rt.state.copy_(state0)
                conv.rt.count.copy_(count0)
                if pghi:
                    conv.rt.pstate.copy_(pstate0)
                torch.cuda.synchronize()
                ev[0].record()
                if pghi:   # the two launches of Rtisi.launch, with an event between them
                    L.check(lib.avc_pghi_stream(C.byref(desc[0]), C.c_float(hp.pghi_tol), None, None), "avc_pghi_stream")
                    ev[2].record()
                    L.check(lib.avc_rtisi_la_from(C.byref(desc[1]), desc[0].X, None), "avc_rtisi_la_from")
                else:
                    conv.rt.launch(desc)
                ev[1].record()
                torch.cuda.synchronize()
                times.append(ev[0].elapsed_time(ev[1]))
                if pghi:
                    ptimes.append(ev[0].elapsed_time(ev[2]))
            rt_ms = sorted(times)[len(times) // 2]
            if pghi:
                pg_ms = sorted(ptimes)[len(ptimes) // 2]
                res["pghi_stream_kernel"] = {"streams": S, "ms": pg_ms}
                print(f"avc_pghi_stream kernel alone, {S} streams x {p.hop} frames: {pg_ms:.3f} ms (of {rt_ms:.3f} ms "
                      f"with avc_rtisi_la_from)", file=sys.stderr)
            del keep
            ffts = S * p.hop * (1 + p.gl_iters * (p.gl_lookahead + 1)) * 2
            # offline Griffin-Lim on the same number of frames: 2 FFTs per frame per iteration
            frames = S * p.hop
            n_iter = 16
            utts = [torch.rand(max(8, frames // 64), hp.n_bins, device=dev) for _ in range(64)]
            gl = GriffinLim(utts, hp, n_iter=n_iter)
            gl_ms = 1e3 * median_events_s(gl.run, 7)
            gl_ffts = sum(u.shape[0] for u in utts) * (2 * n_iter + 1)
            res["rtisi_kernel"] = {"streams": S, "ms": rt_ms, "fft_per_s": ffts / (rt_ms * 1e-3),
                                   "gl_ms": gl_ms, "gl_fft_per_s": gl_ffts / (gl_ms * 1e-3)}
            print(f"avc_rtisi_la kernel, {S} streams x {p.hop} frames: {rt_ms:.3f} ms, {ffts / rt_ms / 1e6:.2f} G FFT/s; "
                  f"offline Griffin-Lim {gl_ffts / gl_ms / 1e6:.2f} G FFT/s", file=sys.stderr)
        del conv
        torch.cuda.empty_cache()
    fits = [S for S, st in res["stages"].items() if st["update"] <= budget_ms]
    res["max_realtime_streams_measured"] = max(fits) if fits else 0
    if args.pitch in ("match", "mv"):
        res["yin_window_kernel"] = {n: yin_window_ms(n, hp, dev) for n in (64, 1024)}
        for n, ms in res["yin_window_kernel"].items():
            print(f"avc_yin_window kernel, {n} streams x 8 frames: {ms:.3f} ms", file=sys.stderr)
        from test_gpu_stream_pitch import GLIDE_TARGET, glide_errors
        errs = [glide_errors((args.pitch, *GLIDE_TARGET), seed, warmup=p.pitch_warmup) for seed in range(5)]
        res["glide"] = {"mean_error_st": float(np.median([e[0] for e in errs])),
                        "std_error_st": float(np.median([e[1] for e in errs])),
                        "per_glide": [[float(a), float(b), int(c)] for a, b, c in errs]}
        print(f"glide after warm-up: median error of the voiced mean {res['glide']['mean_error_st']:.3f} st, of the "
              f"std {res['glide']['std_error_st']:.3f} st", file=sys.stderr)
    if args.model and args.attr:
        from adaptive_voice_conversion_b200.mcd import mel_cepstrum
        conv = StreamingConverter(inf, voc, dataclasses.replace(p, keep_mels=True))
        code = torch.randn(c_out, generator=torch.Generator().manual_seed(0)).to(dev)
        y = harmonic(int(args.quality_seconds * hp.sr), hp.sr, seed=1).to(dev)
        sid = conv.open(code)
        for k in range(0, y.numel(), 480):
            conv.push({sid: y[k:k + 480]})
        conv.close(sid)
        streamed = conv.take_mels(sid)
        mel = voc.wav_to_mel([y], trim=False)[0][0]
        mean = torch.as_tensor(np.asarray(inf.attr["mean"], np.float32)).to(dev)
        std = torch.as_tensor(np.asarray(inf.attr["std"], np.float32)).to(dev)
        x = ((mel - mean) / std).t()[None].contiguous()
        off = inf.model.inference_from_embeddings(x, code[None])[0, :, :mel.shape[0]].t()
        cs, co = mel_cepstrum([streamed, off], inf.attr, hp)
        res["quality"] = {"mel_l1": float((streamed - off).abs().mean()),
                          "cepstral_distance": float((cs[:, 1:] - co[:, 1:]).pow(2).sum(1).sqrt().mean()),
                          "frames": int(mel.shape[0])}
        print(f"quality vs offline: {res['quality']}", file=sys.stderr)
    print(f"card: {res['card']}; largest measured S in real time: {res['max_realtime_streams_measured']}; latency "
          f"{res.get('latency_samples')} samples, tracked {res.get('tracked_latency_samples')}", file=sys.stderr)
    print(json.dumps(res))


if __name__ == "__main__":
    main()
