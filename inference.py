"""One-shot voice conversion entry point with the reference's flags (inference.py:95-109).

Mels ending in .wav are read and written through the GPU Griffin-Lim vocoder (adaptive_voice_conversion_b200.vocoder),
as the reference does:

    python inference.py -c config.yaml -m model.ckpt -a attr.pkl -s src.wav -t tgt.wav -o out.wav

-gl_iters (default 100) and -gl_momentum (default 0, plain Griffin-Lim) set the synthesis of a .wav output; a
momentum such as 0.99 runs fast Griffin-Lim.

Any of the three may instead be a .npy mel ([T, n_mels], already normalised when -attr is omitted):

    python inference.py -c config.yaml -m model.ckpt -s src.npy -t tgt.npy -o out.npy

Many pairs in one call: -pairs FILE names one pair per line, ``source target [output_name]`` (blank lines and lines
starting with # are skipped), and -o is the output directory:

    python inference.py -c config.yaml -m model.ckpt -a attr.pkl -pairs pairs.txt -o out_dir

output_name defaults to ``<source stem>_to_<target stem>.wav``; a name ending in .npy saves the converted mel, any other
name gets a .wav.  The sources and targets are analysed in one batched Vocoder.wav_to_mel call (.npy mels are read
as in the single-pair mode), converted by Inferencer.inference_padded, and the .wav outputs synthesised in one batched
Vocoder.mel_to_wav call (-gl_iters, -gl_momentum).  A missing file, a malformed line or an utterance shorter than the
model accepts is reported with its line number before anything runs on the GPU.
"""
import os
from argparse import ArgumentParser

import numpy as np
import torch

from adaptive_voice_conversion_b200.config import load_config
from adaptive_voice_conversion_b200.inference import Inferencer
from adaptive_voice_conversion_b200.utils import local_device


def is_wav(path):
    return str(path).lower().endswith(".wav")


def read_pairs(path):
    """[(line number, source, target, output name)] of a pairs file; ValueError naming the line of a malformed entry
    or a missing input."""
    out = []
    with open(path) as f:
        for n, line in enumerate(f, 1):
            parts = line.split()
            if not parts or parts[0].startswith("#"):
                continue
            err = lambda msg: ValueError(f"{path} line {n}: {msg}")  # noqa: E731
            if len(parts) not in (2, 3):
                raise err(f"expected 'source target [output_name]', got {len(parts)} fields")
            for fp in parts[:2]:
                if not os.path.isfile(fp) or not (is_wav(fp) or fp.lower().endswith(".npy")):
                    raise err(f"{fp} is not an existing .wav or .npy file")
            stem = lambda p: os.path.splitext(os.path.basename(p))[0]  # noqa: E731
            name = parts[2] if len(parts) == 3 else f"{stem(parts[0])}_to_{stem(parts[1])}"
            ext = os.path.splitext(name)[1].lower()
            if os.path.basename(name) != name or ext not in ("", ".wav", ".npy"):
                raise err(f"output_name {name} must be a file name ending in .wav, .npy or nothing")
            out.append((n, parts[0], parts[1], name if ext else name + ".wav"))
    if not out:
        raise ValueError(f"{path}: no pairs")
    return out


def check_frames(pairs, src_frames, tgt_frames, minimum):
    """ValueError naming the line of the first pair whose source / target is shorter than (min_src, min_ref)."""
    for (n, src, tgt, _), ts, tt in zip(pairs, src_frames, tgt_frames):
        if ts < minimum[0]:
            raise ValueError(f"line {n}: source {src} has {ts} frames; the model needs at least {minimum[0]}")
        if tt < minimum[1]:
            raise ValueError(f"line {n}: target {tgt} has {tt} frames; the model needs at least {minimum[1]}")


def run_pairs(args, config):
    """The -pairs mode: every pair of the file, batched (see the module docstring)."""
    from adaptive_voice_conversion_b200.mcd import min_frames
    from adaptive_voice_conversion_b200.vocoder import AudioParams, Vocoder, load_wav
    pairs = read_pairs(args.pairs)
    os.makedirs(args.output, exist_ok=True)
    dev = local_device()
    files = sorted({p for _, s, t, _ in pairs for p in (s, t)})
    need_voc = any(is_wav(f) for f in files) or any(is_wav(name) for *_, name in pairs)
    vocoder = Vocoder(n_mels=config["SpeakerEncoder"]["c_in"] // config["data_loader"]["frame_size"],
                      hp=AudioParams(n_iter=args.gl_iters, momentum=args.gl_momentum)) if need_voc else None
    wavs = [f for f in files if is_wav(f)]
    mels = {}
    if wavs:
        sigs = [torch.from_numpy(load_wav(f, vocoder.hp.sr)).to(dev) for f in wavs]
        mels.update((f, m) for f, (m, _) in zip(wavs, vocoder.wav_to_mel(sigs)))
    mels.update((f, torch.from_numpy(np.load(f).astype(np.float32)).to(dev)) for f in files if not is_wav(f))
    check_frames(pairs, [mels[s].shape[0] for _, s, _, _ in pairs], [mels[t].shape[0] for _, _, t, _ in pairs],
                 min_frames(config))
    inf = Inferencer(config=config, args=args, vocoder=vocoder)
    if inf.attr is not None:
        mean = torch.as_tensor(np.asarray(inf.attr["mean"], np.float32)).to(dev)
        std = torch.as_tensor(np.asarray(inf.attr["std"], np.float32)).to(dev)
        mels = {f: (m - mean) / std for f, m in mels.items()}
    decs = inf.inference_padded([mels[s] for _, s, _, _ in pairs], [mels[t] for _, _, t, _ in pairs])
    if inf.attr is not None:
        decs = [d * std + mean for d in decs]
    to_wav = [i for i, (*_, name) in enumerate(pairs) if is_wav(name)]
    ys = vocoder.mel_to_wav([decs[i].contiguous() for i in to_wav]) if to_wav else []
    for i, y in zip(to_wav, ys):
        inf.write_wav_to_file(y.cpu().numpy(), os.path.join(args.output, pairs[i][3]))
    for i, (*_, name) in enumerate(pairs):
        if not is_wav(name):
            np.save(os.path.join(args.output, name), decs[i].cpu().numpy())


if __name__ == "__main__":
    p = ArgumentParser()
    p.add_argument("-attr", "-a", help="attr file path")
    p.add_argument("-config", "-c", help="config file path")
    p.add_argument("-model", "-m", help="model path")
    p.add_argument("-source", "-s", help="source .wav or mel .npy")
    p.add_argument("-target", "-t", help="target .wav or mel .npy")
    p.add_argument("-output", "-o", help="output .wav or mel .npy")
    p.add_argument("-sample_rate", "-sr", default=24000, type=int)
    p.add_argument("-gl_iters", default=100, type=int, help="Griffin-Lim iterations of a .wav output")
    p.add_argument("-gl_momentum", default=0.0, type=float,
                   help="fast Griffin-Lim momentum in [0, 1) of a .wav output (0: plain Griffin-Lim)")
    p.add_argument("-pairs", help="file of 'source target [output_name]' lines: convert them all, into the -o directory")
    args = p.parse_args()
    config = load_config(args.config)
    if args.pairs:
        run_pairs(args, config)
        raise SystemExit(0)
    vocoder = None
    if any(is_wav(f) for f in (args.source, args.target, args.output)):
        from adaptive_voice_conversion_b200.vocoder import AudioParams, Vocoder
        vocoder = Vocoder(n_mels=config["SpeakerEncoder"]["c_in"] // config["data_loader"]["frame_size"],
                          hp=AudioParams(n_iter=args.gl_iters, momentum=args.gl_momentum))
    inf = Inferencer(config=config, args=args, vocoder=vocoder if is_wav(args.output) else None)

    def read(path):
        return vocoder.get_spectrograms(path)[0] if is_wav(path) else np.load(path).astype(np.float32)

    src, tgt = read(args.source), read(args.target)
    if inf.attr is not None:
        src, tgt = inf.normalize(src), inf.normalize(tgt)
    dev = local_device()
    wav, mel = inf.inference_one_utterance(torch.from_numpy(src).to(dev), torch.from_numpy(tgt).to(dev))
    if is_wav(args.output):
        inf.write_wav_to_file(wav, args.output)
    else:
        np.save(args.output, mel)
