"""One-shot voice conversion entry point with the reference's flags (inference.py:95-109).

Mels ending in .wav are read and written through the GPU Griffin-Lim vocoder (adaptive_voice_conversion_b200.vocoder),
as the reference does:

    python inference.py -c config.yaml -m model.ckpt -a attr.pkl -s src.wav -t tgt.wav -o out.wav

-gl_iters (default 100) and -gl_momentum (default 0, plain Griffin-Lim) set the synthesis of a .wav output; a
momentum such as 0.99 runs fast Griffin-Lim.

Any of the three may instead be a .npy mel ([T, n_mels], already normalised when -attr is omitted):

    python inference.py -c config.yaml -m model.ckpt -s src.npy -t tgt.npy -o out.npy
"""
from argparse import ArgumentParser

import numpy as np
import torch

from adaptive_voice_conversion_b200.config import load_config
from adaptive_voice_conversion_b200.inference import Inferencer
from adaptive_voice_conversion_b200.utils import local_device


def is_wav(path):
    return str(path).lower().endswith(".wav")


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
    args = p.parse_args()
    config = load_config(args.config)
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
