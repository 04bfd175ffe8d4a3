"""Adapt a trained model to one speaker: fine-tune the decoder and the speaker's code on their recordings, with both
encoders frozen (adaptive_voice_conversion_b200/adapt.py gives the definitions).

From your own recordings, analysed by the GPU vocoder and normalised with -a (held-out recordings optional):

    python adapt.py -c config.yaml -m base.ckpt -a attr.pkl -speaker alice -wav a1.wav a2.wav ... \\
        [-holdout h1.wav h2.wav] -o alice_model [-steps 500] [-lr LR] [-batch_size B] [-seed 0]

From a prepared set (the speaker's utterances of <data_dir>/<set>.pkl), held out on another set, with MCD-DTW on its
parallel utterances when -transcripts is given:

    python adapt.py -c config.yaml -m base.ckpt -d data/ -set train -speaker p225 -o p225_model \\
        [-eval_set in_test] [-transcripts VCTK-Corpus/txt] [-steps ...]

Writes <o>.ckpt (the full AE state_dict; the encoders' entries are the base checkpoint's), <o>.bank.pt (a one-speaker
bank of the adapted code) and <o>.json (settings, the training loss every 100 steps, the clips used and skipped, the
held-out results before and after).  Convert with

    python inference.py -c config.yaml -m <o>.ckpt -a attr.pkl -s src.wav -bank <o>.bank.pt -speaker NAME -o out.wav

The defaults of -steps, -lr (the config's rate) and -batch_size (the config's) are not tuned.
data_loader.frame_size 1 only.
"""
import os
import pickle
import types
from argparse import ArgumentParser

import torch

from adaptive_voice_conversion_b200.config import load_config


def parser():
    p = ArgumentParser(description="Fine-tune the decoder and one speaker's code on that speaker's recordings")
    p.add_argument("-config", "-c", default="config.yaml", help="config file path")
    p.add_argument("-model", "-m", required=True, help="base model checkpoint (.ckpt)")
    p.add_argument("-output", "-o", required=True, help="output prefix: <o>.ckpt, <o>.bank.pt, <o>.json")
    p.add_argument("-speaker", required=True, help="the speaker's name (with -d: its name in the set)")
    p.add_argument("-attr", "-a", help="mel statistics for -wav recordings")
    p.add_argument("-wav", nargs="+", help="the speaker's recordings")
    p.add_argument("-holdout", nargs="+", help="held-out recordings of the speaker (with -wav)")
    p.add_argument("-data_dir", "-d", help="data directory written by preprocess.py (with -set)")
    p.add_argument("-set", help="set name: the speaker's utterances of <data_dir>/<set>.pkl (with -d)")
    p.add_argument("-eval_set", help="held-out set: the speaker's utterances of <data_dir>/<eval_set>.pkl (with -d)")
    p.add_argument("-transcripts", help="directory of <id>.txt transcripts: MCD-DTW on -eval_set (with -d)")
    p.add_argument("-steps", type=int, default=500, help="adaptation steps (not tuned)")
    p.add_argument("-lr", type=float, default=None, help="Adam's rate (default: the config's; not tuned)")
    p.add_argument("-batch_size", type=int, default=None, help="crops per step (default: the config's)")
    p.add_argument("-seed", type=int, default=0, help="seed of the crop order and the noise")
    return p


def check_args(p, args, config=None):
    """Argument errors (p.error): exactly one source, -a with -wav, -holdout with -wav, -set / -eval_set /
    -transcripts with -d, held-out recordings that are adaptation recordings, frame_size 1."""
    if bool(args.wav) == bool(args.data_dir or args.set):
        p.error("give either -wav FILE [FILE ...] or -d DIR -set NAME")
    if args.wav:
        if not args.attr:
            p.error("-wav needs -a attr.pkl to normalise the recordings")
        if args.eval_set or args.transcripts:
            p.error("-eval_set and -transcripts go with -d; with -wav give -holdout FILE ...")
        for f in args.wav + (args.holdout or []):
            if not os.path.isfile(f):
                p.error(f"{f} is not a file")
        if args.holdout:
            from adaptive_voice_conversion_b200.adapt import check_disjoint
            try:
                check_disjoint([os.path.realpath(f) for f in args.wav], [os.path.realpath(f) for f in args.holdout],
                               "recording")
            except ValueError as e:
                p.error(str(e))
    else:
        if not (args.data_dir and args.set):
            p.error("-d and -set go together")
        if args.holdout:
            p.error("-holdout goes with -wav; with -d give -eval_set NAME")
        if args.transcripts and not args.eval_set:
            p.error("-transcripts needs -eval_set (the set MCD-DTW is measured on)")
    if args.steps < 1 or (args.batch_size is not None and args.batch_size < 1):
        p.error("-steps and -batch_size must be >= 1")
    if config is not None and int(config["data_loader"]["frame_size"]) != 1:
        p.error(f"speaker adaptation supports data_loader.frame_size 1 only (got {config['data_loader']['frame_size']})")


def set_clips(p, args, name):
    """{utterance id: mel} of -speaker's utterances in <data_dir>/<name>.pkl."""
    from adaptive_voice_conversion_b200.evaluate import speaker_of
    with open(os.path.join(args.data_dir, f"{name}.pkl"), "rb") as f:
        data = pickle.load(f)
    clips = {u: v for u, v in data.items() if speaker_of(u) == args.speaker}
    if not clips:
        p.error(f"speaker {args.speaker} has no utterance in {name}")
    return data, clips


def wav_clips(args, config, dev, files):
    """{path: attr-normalised mel} of recordings, analysed as speaker_bank.py -wav analyses them."""
    from speaker_bank import wav_mels
    mels, _ = wav_mels(types.SimpleNamespace(attr=args.attr, wav=[[args.speaker] + list(files)]), config, dev)
    return dict(zip(files, (mels[u] for u in sorted(mels))))


def main(argv=None):
    p = parser()
    args = p.parse_args(argv)
    config = load_config(args.config)
    check_args(p, args, config)
    from adaptive_voice_conversion_b200.adapt import adapt, check_disjoint, save
    heldout, mcd = None, None
    if args.data_dir:   # the sets are read and checked before the model is loaded
        _, clips = set_clips(p, args, args.set)
        if args.eval_set:
            eval_data, heldout = set_clips(p, args, args.eval_set)
            try:
                check_disjoint(list(clips), list(heldout))
            except ValueError as e:
                p.error(str(e))
            if args.transcripts:
                from adaptive_voice_conversion_b200.mcd import evaluate_mcd, read_transcripts
                with open(os.path.join(args.data_dir, "attr.pkl"), "rb") as f:
                    attr = pickle.load(f)
                texts = read_transcripts(args.transcripts, eval_data)

                def mcd(m, code):
                    return evaluate_mcd(m, eval_data, attr, texts, seed=args.seed, target_codes={args.speaker: code})
    from adaptive_voice_conversion_b200.model import AE
    from adaptive_voice_conversion_b200.utils import local_device
    dev = local_device()
    model = AE(config).to(dev)
    model.load_state_dict(torch.load(args.model, map_location=dev), strict=True)
    if args.wav:
        clips = wav_clips(args, config, dev, args.wav)
        if args.holdout:
            heldout = wav_clips(args, config, dev, args.holdout)
    res = adapt(model, config, args.speaker, clips, args.steps, lr=args.lr, batch_size=args.batch_size, seed=args.seed,
                heldout=heldout, mcd=mcd)
    res["report"]["settings"]["base_model"] = os.path.abspath(args.model)
    save(res, model, args.output)
    r = res["report"]
    last = r["losses"][-1]
    print(f"adapted {args.speaker}: {len(r['clips']['used'])} clips ({len(r['clips']['skipped'])} too short skipped), "
          f"{args.steps} steps, loss_rec {r['losses'][0]['loss_rec']:.4f} -> {last['loss_rec']:.4f}")
    if r["heldout"] is not None:
        for k in r["heldout"]["before"]:
            b, a = r["heldout"]["before"][k], r["heldout"]["after"][k]
            key = "rec" if k == "rec" else "mcd"
            print(f"held-out {k}: {b.get(key)} -> {a.get(key)} (n={a.get('n')})")
    print(f"-> {args.output}.ckpt, {args.output}.bank.pt, {args.output}.json")
    return res


if __name__ == "__main__":
    main()
