"""Streaming conversion (adaptive_voice_conversion_b200/streaming.py): update time per stage and how many streams fit
in real time.

    python tools/bench_stream.py [--streams 1 64 1024 4096] [--updates 20] [--config config.yaml] [-m ckpt -a attr]

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
The model has random weights unless -m is given; the input is synthetic (harmonic tones).  The card name and power
limit are read in the same run.  Writes nothing.
"""
import argparse
import dataclasses
import json
import os
import subprocess
import sys
import types

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

import numpy as np  # noqa: E402
import torch  # noqa: E402


def card():
    try:
        return subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                              capture_output=True, text=True, timeout=30).stdout.strip().splitlines()[0]
    except Exception as e:   # noqa: BLE001
        return f"unknown ({e})"


def harmonic(n, sr, seed):
    from _rtisi_ref import harmonic as h
    return torch.from_numpy(h(n, sr, seed=seed).astype(np.float32))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--streams", type=int, nargs="+", default=[1, 64, 1024, 4096])
    ap.add_argument("--updates", type=int, default=20)
    ap.add_argument("--config", "-c", default=os.path.join(ROOT, "config.yaml"))
    ap.add_argument("-m", "--model")
    ap.add_argument("-a", "--attr")
    ap.add_argument("--quality-seconds", type=float, default=6.0)
    args = ap.parse_args()
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
    p = StreamParams()
    block = p.hop * hp.hop_length
    budget_ms = 1e3 * block / hp.sr
    c_out = cfg["SpeakerEncoder"]["c_out"]
    res = {"card": card(), "params": p.__dict__, "block_ms": budget_ms, "n_mels": hp.n_mels, "stages": {}}
    rt_ms = None
    for S in args.streams:
        conv = StreamingConverter(inf, voc, p)
        ids = [conv.open(torch.randn(c_out, generator=torch.Generator().manual_seed(i)).to(dev)) for i in range(S)]
        sig = harmonic(block * (args.updates + 40), hp.sr, seed=S).to(dev)
        # start-up (the first block needs m frames, start-up windows of every length) and graph captures
        pos = 0
        for _ in range(20):
            conv.push({sid: sig[pos:pos + block] for sid in ids})
            pos += block
        conv.stage_ms = {}
        torch.cuda.synchronize()
        for _ in range(args.updates):
            conv.push({sid: sig[pos:pos + block] for sid in ids})
            pos += block
        st = {k: v / args.updates for k, v in conv.stage_ms.items()}
        st["update"] = sum(st.values())
        res["stages"][S] = st
        print(f"S={S:5d}: update {st['update']:.2f} ms (analysis {st['analysis']:.2f}, conversion "
              f"{st['conversion']:.2f}, rtisi {st['rtisi']:.2f}); block {budget_ms:.0f} ms", file=sys.stderr)
        if S == max(args.streams):
            # the avc_rtisi_la kernel alone: one steady-state update's tables and buffers prepared once, then the C
            # call timed by CUDA events, each launch from a copy of the same state (the copy outside the events)
            conv.stage_ms = None
            mags = {sid: voc.mel_to_mag([torch.rand(p.hop, hp.n_mels, device=dev)])[0] for sid in ids}
            state0, count0 = conv.rt.state.clone(), conv.rt.count.clone()
            desc, _, keep = conv.rt.prepare(mags)
            ev = [torch.cuda.Event(enable_timing=True) for _ in range(2)]
            times = []
            for _ in range(7):
                conv.rt.state.copy_(state0)
                conv.rt.count.copy_(count0)
                torch.cuda.synchronize()
                ev[0].record()
                conv.rt.launch(desc)
                ev[1].record()
                torch.cuda.synchronize()
                times.append(ev[0].elapsed_time(ev[1]))
            rt_ms = sorted(times)[len(times) // 2]
            del keep
            ffts = S * p.hop * (1 + p.gl_iters * (p.gl_lookahead + 1)) * 2
            # offline Griffin-Lim on the same number of frames: 2 FFTs per frame per iteration
            frames = S * p.hop
            n_iter = 16
            utts = [torch.rand(max(8, frames // 64), hp.n_bins, device=dev) for _ in range(64)]
            gl = GriffinLim(utts, hp, n_iter=n_iter)
            gl.run()
            times = []
            for _ in range(7):
                torch.cuda.synchronize()
                ev[0].record()
                gl.run()
                ev[1].record()
                torch.cuda.synchronize()
                times.append(ev[0].elapsed_time(ev[1]))
            gl_ms = sorted(times)[len(times) // 2]
            gl_ffts = sum(u.shape[0] for u in utts) * (2 * n_iter + 1)
            res["rtisi_kernel"] = {"streams": S, "ms": rt_ms, "fft_per_s": ffts / (rt_ms * 1e-3),
                                   "gl_ms": gl_ms, "gl_fft_per_s": gl_ffts / (gl_ms * 1e-3)}
            print(f"avc_rtisi_la kernel, {S} streams x {p.hop} frames: {rt_ms:.3f} ms, {ffts / rt_ms / 1e6:.2f} G FFT/s; "
                  f"offline Griffin-Lim {gl_ffts / gl_ms / 1e6:.2f} G FFT/s", file=sys.stderr)
        del conv
        torch.cuda.empty_cache()
    fits = [S for S, st in res["stages"].items() if st["update"] <= budget_ms]
    res["max_realtime_streams_measured"] = max(fits) if fits else 0
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
    print(f"card: {res['card']}; largest measured S in real time: {res['max_realtime_streams_measured']}", file=sys.stderr)
    print(json.dumps(res))


if __name__ == "__main__":
    main()
