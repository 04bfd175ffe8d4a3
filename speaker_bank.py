"""Build a speaker bank: every usable utterance of each speaker pooled into one speaker code, saved for
inference.py -bank and evaluate.py -spk -bank (adaptive_voice_conversion_b200/speaker_bank.py gives the definitions).

From a prepared set (``<data_dir>/<set>.pkl``, attr-normalised mels; optionally only some speakers):

    python speaker_bank.py -c config.yaml -m model.ckpt -d data/ -set train -o bank.pt [-speakers p225,p226]

From your own recordings, analysed by the GPU vocoder and normalised with -a (repeat -wav for every speaker):

    python speaker_bank.py -c config.yaml -m model.ckpt -a attr.pkl -wav alice a1.wav a2.wav -wav bob b1.wav -o bank.pt

Prints the number of speakers, the utterances pooled and the utterances skipped (shorter than the model accepts).

With -fit_steps the pooled codes are then fitted to the model (adaptive_voice_conversion_b200/fit.py): each speaker's
code is optimised on that speaker's own recordings with every model weight frozen, many speakers per step, and the bank
records the content encoder and decoder it was fitted to.  Held out on another set, with MCD-DTW on its parallel
utterances when -transcripts is given:

    python speaker_bank.py -c config.yaml -m model.ckpt -d data/ -set train -o bank.pt -fit_steps 300 \
        [-fit_lr LR] [-fit_crops 8] [-fit_speakers 16] [-seed 0] [-holdout_set in_test] [-transcripts DIR] \
        [-report out.json]

The defaults of -fit_steps, -fit_lr (the config's rate), -fit_crops and -fit_speakers are not tuned.
data_loader.frame_size 1 only.

With -f0 the bank also records each speaker's pitch profile (speaker_bank.build_pitch_profiles): the mean and std of
log2 F0 over the voiced frames of the speaker's pooled utterances, each copy-synthesised from its denormalised mel by
the GPU Griffin-Lim vocoder (-gl_iters, -gl_momentum, -gl_init; defaults 100, 0, zero, as inference.py) and tracked by
YIN.  The mel statistics are -a, or <data_dir>/attr.pkl for a prepared set.  inference.py -pitch_shift mv needs the
record to match a conversion's pitch to a banked speaker, mix or morph; without -f0 the bank is unchanged:

    python speaker_bank.py -c config.yaml -m model.ckpt -d data/ -set train -o bank.pt -f0 [-gl_iters 100]
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
    p.add_argument("-fit_steps", type=int, default=None, help="fit every code to the model for this many steps")
    p.add_argument("-fit_lr", type=float, default=None, help="Adam's rate of the fit (default: the config's; not tuned)")
    p.add_argument("-fit_crops", type=int, default=8, help="crops per speaker and step (not tuned)")
    p.add_argument("-fit_speakers", type=int, default=16, help="speakers per step (a speed-up only; not tuned)")
    p.add_argument("-seed", type=int, default=0, help="seed of every speaker's crop order")
    p.add_argument("-holdout_set", help="held-out set of the banked speakers: <data_dir>/<holdout_set>.pkl (with -d)")
    p.add_argument("-transcripts", help="directory of <id>.txt transcripts: MCD-DTW on -holdout_set")
    p.add_argument("-report", help="fit report to write (JSON)")
    p.add_argument("-f0", action="store_true", help="also record every speaker's pitch profile (for -pitch_shift mv)")
    p.add_argument("-gl_iters", type=int, default=None, help="Griffin-Lim iterations of -f0's copy-synthesis (100)")
    p.add_argument("-gl_momentum", type=float, default=None, help="fast Griffin-Lim momentum in [0, 1) of -f0's (0)")
    p.add_argument("-gl_init", default=None, choices=["zero", "pghi"], help="Griffin-Lim start phase of -f0's (zero)")
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
    gl = [f"-{k}" for k in ("gl_iters", "gl_momentum", "gl_init") if getattr(args, k) is not None]
    if gl and not args.f0:
        p.error(f"{', '.join(gl)} set(s) the copy-synthesis of -f0")
    if args.gl_iters is not None and args.gl_iters < 0:
        p.error("-gl_iters must be >= 0")
    if args.gl_momentum is not None and not 0.0 <= args.gl_momentum < 1.0:
        p.error("-gl_momentum must lie in [0, 1)")
    if args.f0 and not args.wav and not os.path.isfile(attr_path(args)):
        p.error(f"-f0 needs the mel statistics: {attr_path(args)} does not exist (pass -a)")
    fit_only = [f"-{k}" for k in ("fit_lr", "holdout_set", "transcripts", "report") if getattr(args, k) is not None]
    if args.fit_steps is None:
        if fit_only:
            p.error(f"{', '.join(fit_only)} go(es) with -fit_steps")
        return
    if args.fit_steps < 1 or args.fit_crops < 1 or args.fit_speakers < 1:
        p.error("-fit_steps, -fit_crops and -fit_speakers must be >= 1")
    if args.fit_lr is not None and not args.fit_lr > 0:
        p.error("-fit_lr must be > 0")
    if args.holdout_set and not args.data_dir:
        p.error("-holdout_set goes with -d (a held-out set of the prepared data)")
    if args.transcripts and not args.holdout_set:
        p.error("-transcripts needs -holdout_set (the set MCD-DTW is measured on)")


def attr_path(args):
    """The mel statistics: -a, or <data_dir>/attr.pkl of a prepared set."""
    return args.attr or os.path.join(args.data_dir, "attr.pkl")


def pitch_record(args, bank, mels):
    """build_pitch_profiles of the bank's pooled utterances at the -gl_* settings."""
    from adaptive_voice_conversion_b200.speaker_bank import build_pitch_profiles
    from adaptive_voice_conversion_b200.vocoder import AudioParams
    with open(attr_path(args), "rb") as f:
        attr = pickle.load(f)
    d = AudioParams()
    hp = AudioParams(n_iter=d.n_iter if args.gl_iters is None else args.gl_iters,
                     momentum=d.momentum if args.gl_momentum is None else args.gl_momentum,
                     gl_init=args.gl_init or d.gl_init)
    return build_pitch_profiles(bank, mels, attr, hp)


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


def holdout_mels(args, bank, speaker_of):
    """(the held-out set's pickle, {speaker: {id: mel}} of the bank's speakers in it).  SystemExit when a held-out
    utterance is one the bank pooled (and so would be fitted on)."""
    from adaptive_voice_conversion_b200.adapt import check_disjoint
    with open(os.path.join(args.data_dir, f"{args.holdout_set}.pkl"), "rb") as f:
        data = pickle.load(f)
    try:
        check_disjoint(bank.utterance_ids(), list(data))
    except ValueError as e:
        raise SystemExit(f"speaker_bank.py: {e}")
    held = {}
    for u in sorted(data):
        if speaker_of(u) in bank:
            held.setdefault(speaker_of(u), {})[u] = data[u]
    return data, held


def fit(args, model, bank, mels, speaker_of):
    """fit_bank with the -fit_* settings; held out on -holdout_set (MCD-DTW with -transcripts).  -> (bank, report)"""
    from adaptive_voice_conversion_b200.fit import fit_bank
    held, mcd = None, None
    if args.holdout_set:
        data, held = holdout_mels(args, bank, speaker_of)
        if args.transcripts:
            from adaptive_voice_conversion_b200.mcd import evaluate_mcd, read_transcripts
            with open(os.path.join(args.data_dir, "attr.pkl"), "rb") as f:
                attr = pickle.load(f)
            texts = read_transcripts(args.transcripts, data)

            def mcd(m, codes):
                return evaluate_mcd(m, data, attr, texts, seed=args.seed, target_codes=codes)
    return fit_bank(model, bank, mels, args.fit_steps, lr=args.fit_lr, crops=args.fit_crops,
                    speakers_per_wave=args.fit_speakers, seed=args.seed, heldout=held, mcd=mcd)


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
    if args.f0:
        bank = bank.with_pitch(pitch_record(args, bank, mels))
        unvoiced = [s for s, n in zip(bank.speakers, bank.pitch["voiced"]) if n == 0]
        print(f"pitch profiles: {len(bank) - len(unvoiced)} speakers voiced"
              + (f", no voiced frame for {', '.join(unvoiced)}" if unvoiced else ""))
    if args.fit_steps is None:
        bank.save(args.output)
        print(f"bank: {len(bank)} speakers, {sum(bank.n_utts)} utterances pooled, {bank.n_skipped} skipped -> {args.output}")
        return bank
    bank, report = fit(args, model, bank, mels, speaker_of)
    bank.save(args.output)
    if args.report:
        import json
        with open(args.report, "w") as f:
            json.dump(report, f, indent=1)
    n_fit = len(bank) - len(report["unfitted"])
    print(f"bank: {len(bank)} speakers, {sum(bank.n_utts)} utterances pooled, {bank.n_skipped} skipped; {n_fit} codes "
          f"fitted for {args.fit_steps} steps, {len(report['unfitted'])} unfitted -> {args.output}")
    return bank


if __name__ == "__main__":
    main()
