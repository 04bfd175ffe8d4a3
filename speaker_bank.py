"""Build a speaker bank: every usable utterance of each speaker pooled into one speaker code, saved for
inference.py -bank and evaluate.py -spk -bank (adaptive_voice_conversion_b200/speaker_bank.py gives the definitions).

From a prepared set (``<data_dir>/<set>.pkl``, attr-normalised mels; optionally only some speakers):

    python speaker_bank.py -c config.yaml -m model.ckpt -d data/ -set train -o bank.pt [-speakers p225,p226]

From your own recordings, analysed by the GPU vocoder and normalised with -a (repeat -wav for every speaker):

    python speaker_bank.py -c config.yaml -m model.ckpt -a attr.pkl -wav alice a1.wav a2.wav -wav bob b1.wav -o bank.pt

Prints the number of speakers, the utterances pooled and the utterances skipped (shorter than the model accepts).
data_loader.frame_size 1 only.
"""
import os
import pickle
from argparse import ArgumentParser

import numpy as np
import torch

from adaptive_voice_conversion_b200.config import load_config


def parser():
    p = ArgumentParser(description="Pool each speaker's utterances into a saved speaker code")
    p.add_argument("-config", "-c", default="config.yaml", help="config file path")
    p.add_argument("-model", "-m", required=True, help="model checkpoint (.ckpt)")
    p.add_argument("-output", "-o", required=True, help="bank file to write")
    p.add_argument("-data_dir", "-d", help="data directory written by preprocess.py (with -set)")
    p.add_argument("-set", help="set name: <data_dir>/<set>.pkl (with -d)")
    p.add_argument("-speakers", help="comma-separated speakers of the set to bank (default: all)")
    p.add_argument("-attr", "-a", help="mel statistics for -wav recordings")
    p.add_argument("-wav", nargs="+", action="append", metavar=("NAME", "FILE"),
                   help="a speaker's name and recordings (repeatable)")
    return p


def check_args(p, args):
    """Argument errors (p.error): exactly one source, -d with -set, -a with -wav, two or more words per -wav."""
    if bool(args.wav) == bool(args.data_dir or args.set):
        p.error("give either -d DIR -set NAME or -wav NAME FILE [FILE ...]")
    if args.wav:
        if not args.attr:
            p.error("-wav needs -a attr.pkl to normalise the recordings")
        if args.speakers:
            p.error("-speakers selects speakers of a -set; with -wav name the speakers themselves")
        names = [w[0] for w in args.wav]
        if any(len(w) < 2 for w in args.wav):
            p.error("-wav needs a speaker name and at least one file")
        if len(set(names)) != len(names):
            p.error("-wav: a speaker is named twice")
        for w in args.wav:
            for f in w[1:]:
                if not os.path.isfile(f):
                    p.error(f"-wav {w[0]}: {f} is not a file")
    elif not (args.data_dir and args.set):
        p.error("-d and -set go together")


def set_mels(args):
    """(mels, speaker_of) of -d/-set: the set's utterances (restricted to -speakers)."""
    from adaptive_voice_conversion_b200.evaluate import speaker_of
    with open(os.path.join(args.data_dir, f"{args.set}.pkl"), "rb") as f:
        data = pickle.load(f)
    if args.speakers:
        want = [s for s in args.speakers.split(",") if s]
        have = {speaker_of(u) for u in data}
        missing = [s for s in want if s not in have]
        if missing:
            raise SystemExit(f"speaker_bank.py: {', '.join(missing)} not in {args.set}")
        data = {u: v for u, v in data.items() if speaker_of(u) in set(want)}
    return data, speaker_of


def wav_mels(args, config, dev):
    """(mels, speaker_of) of the -wav recordings: one batched analysis, attr-normalised; utterance ids NAME/k."""
    from adaptive_voice_conversion_b200.vocoder import Vocoder, load_wav
    with open(args.attr, "rb") as f:
        attr = pickle.load(f)
    voc = Vocoder(n_mels=config["SpeakerEncoder"]["c_in"])
    ids, owner, sigs = [], {}, []
    for name, *files in args.wav:
        for k, path in enumerate(files):
            u = f"{name}/{k:05d}"
            ids.append(u)
            owner[u] = name
            sigs.append(torch.from_numpy(load_wav(path, voc.hp.sr)).to(dev))
    mean = torch.as_tensor(np.asarray(attr["mean"], np.float32)).to(dev)
    std = torch.as_tensor(np.asarray(attr["std"], np.float32)).to(dev)
    mels = {u: (m - mean) / std for u, (m, _) in zip(ids, voc.wav_to_mel(sigs))}
    return mels, owner.__getitem__


def main(argv=None):
    p = parser()
    args = p.parse_args(argv)
    check_args(p, args)
    config = load_config(args.config)
    if int(config["data_loader"]["frame_size"]) != 1:
        p.error(f"speaker banks support data_loader.frame_size 1 only (got {config['data_loader']['frame_size']})")
    from adaptive_voice_conversion_b200.model import AE
    from adaptive_voice_conversion_b200.speaker_bank import build_bank
    from adaptive_voice_conversion_b200.utils import local_device
    dev = local_device()
    model = AE(config).to(dev)
    model.load_state_dict(torch.load(args.model, map_location=dev), strict=True)
    model.eval()
    mels, speaker_of = wav_mels(args, config, dev) if args.wav else set_mels(args)
    bank = build_bank(model, mels, speaker_of=speaker_of)
    bank.save(args.output)
    print(f"bank: {len(bank)} speakers, {sum(bank.n_utts)} utterances pooled, {bank.n_skipped} skipped -> {args.output}")
    return bank


if __name__ == "__main__":
    main()
