"""One-shot voice conversion entry point with the reference's flags (inference.py:95-109).

Mels ending in .wav are read and written through the GPU Griffin-Lim vocoder (adaptive_voice_conversion_b200.vocoder),
as the reference does:

    python inference.py -c config.yaml -m model.ckpt -a attr.pkl -s src.wav -t tgt.wav -o out.wav

-gl_iters (default 100) and -gl_momentum (default 0, plain Griffin-Lim) set the synthesis of a .wav output; a
momentum such as 0.99 runs fast Griffin-Lim.  -gl_init pghi starts Griffin-Lim from a phase-gradient (PGHI) estimate
instead of zero phase (the default, -gl_init zero).

Any of the three may instead be a .npy mel ([T, n_mels], already normalised when -attr is omitted):

    python inference.py -c config.yaml -m model.ckpt -s src.npy -t tgt.npy -o out.npy

Few-shot: several -t files of the target speaker condition the decoder on their pooled speaker code
(AE.get_speaker_embeddings with groups); one -t file runs the one-shot path:

    python inference.py -c config.yaml -m model.ckpt -a attr.pkl -s src.wav -t tgt1.wav tgt2.wav tgt3.wav -o out.wav

Many pairs in one call: -pairs FILE names one pair per line, ``source target [output_name]`` (blank lines and lines
starting with # are skipped), and -o is the output directory:

    python inference.py -c config.yaml -m model.ckpt -a attr.pkl -pairs pairs.txt -o out_dir

The target field is one file when it names an existing file (even one whose name contains commas); otherwise it is a
comma-separated reference set, ``a.wav,b.wav,c.wav``, whose every member must be an existing .wav or .npy.  Lines
naming the same set share one speaker code.
output_name defaults to ``<source stem>_to_<target stem>.wav`` (a set: its first file's stem); a name ending in .npy saves the converted mel, any other
name gets a .wav.

Speaker banks (speaker_bank.py): -bank bank.pt -speaker SPEC converts to a banked speaker's code instead of -t
(exactly one of the two), SPEC naming one speaker, ``p225``, or a weighted mix, ``p225:0.7,p226:0.3``
(SpeakerBank.code):

    python inference.py -c config.yaml -m model.ckpt -a attr.pkl -s src.wav -bank bank.pt -speaker p225 -o out.wav

Time-varying morphs: -bank bank.pt -morph SPEC@SECONDS [SPEC@SECONDS ...] converts one source with the decoder
conditioned, frame by frame, on a mix of banked speakers (Inferencer.inference_morph).  Each keyframe names a speaker
or a mix at a time in seconds (frames at the vocoder's sr / hop_length per second); the mix glides linearly from one
keyframe to the next, is held before the first and after the last, and two keyframes at the same time make a hard
cut.  -morph excludes -t, -speaker and -pairs:

    python inference.py -c config.yaml -m model.ckpt -a attr.pkl -s dialogue.wav -bank bank.pt \
        -morph p225@0 p225@4.0 p226@4.3 p226@9 p225:0.5,p226:0.5@12 -o out.wav

With -bank, a -pairs target field ``@SPEC`` is resolved through the bank (a field naming an existing file stays that
file, even one whose name starts with @), and its output name defaults to ``<source stem>_to_<SPEC>.wav`` (``:`` and
``,`` replaced by ``-`` and ``+``).  Without -bank every field is read as above.  The sources and targets are analysed in one batched Vocoder.wav_to_mel call (.npy mels are read
as in the single-pair mode), converted by Inferencer.inference_padded, and the .wav outputs synthesised in one batched
Vocoder.mel_to_wav call (-gl_iters, -gl_momentum, -gl_init).  A missing file, a malformed line or an utterance shorter than the
model accepts is reported with its line number before anything runs on the GPU.

Pitch: -pitch_shift SEMITONES (in [-24, 24], default 0) transposes every .wav output by a formant-preserving shift of
the synthesis (Vocoder.mel_to_signal's ``semitones``), for one conversion, -t sets, -bank -speaker, -morph and -pairs:

    python inference.py -c config.yaml -m model.ckpt -a attr.pkl -s src.wav -t tgt.wav -o out.wav -pitch_shift -5

-pitch_shift match instead shifts each conversion so that its mean log2 F0 meets its -t file's or set's, both tracked
as synthesised (adaptive_voice_conversion_b200/f0.py match_shifts), clamped to [-24, 24] and 0 when either side has no
voiced frame; one line per conversion reports the output, the shift and the voiced frame counts.  It works with -t
and in -pairs with file and set targets; banked speakers and morphs have no mels to match, so -speaker, -morph and
@SPEC lines are refused, as is a shift of a .npy output (a mel is not synthesised):

    python inference.py -c config.yaml -m model.ckpt -a attr.pkl -pairs pairs.txt -o out_dir -pitch_shift match

-pitch_shift mv matches the pitch range as well as the level, frame by frame (f0.mv_shifts): on each voiced frame the
conversion's log2 F0 l becomes mu_t + sigma_t / sigma_c (l - mu_c), (mu_c, sigma_c) the mean and std of the
conversion's voiced log2 F0 and (mu_t, sigma_t) the target's; unvoiced frames take the shift interpolated between
their voiced neighbours, every shift is clamped to [-24, 24], and with too little voicing it falls back to match's
constant shift (mean only) or to 0 (unmatched).  It serves every target: a -t file or set and -pairs file and set
lines (their profile tracked as match does), and banked speakers, mixes (-speaker, @SPEC lines) and -morph (a
profile per frame), whose profiles the bank records when speaker_bank.py -f0 built it.  A bank without them, and a
.npy output, are refused before anything runs; a note is printed when the Griffin-Lim settings differ from those the
bank's profiles were synthesised with:

    python inference.py -c config.yaml -m model.ckpt -a attr.pkl -s src.wav -bank bank.pt -speaker p226 -o out.wav \
        -pitch_shift mv
"""
import os
from argparse import ArgumentParser
from typing import NamedTuple

import numpy as np
import torch

from adaptive_voice_conversion_b200.config import load_config
from adaptive_voice_conversion_b200.inference import Inferencer
from adaptive_voice_conversion_b200.utils import local_device


def is_wav(path):
    return str(path).lower().endswith(".wav")


class BankTarget(NamedTuple):
    """A target the -bank file holds, which needs no input file: a banked speaker or mix, spec (-speaker, a pairs
    file's ``@SPEC``; SpeakerBank.code), or a morph, keyframes (-morph's parsed (SPEC, seconds))."""
    spec: str | None = None
    keyframes: tuple | None = None


def target_files(target):
    """The input files a conversion target needs: a target is a path (one file), a tuple of paths (a reference set:
    their pooled speaker code) or a BankTarget (none)."""
    return () if isinstance(target, BankTarget) else (target,) if isinstance(target, str) else tuple(target)


def target_field(field, bank=False):
    """A pairs file's target field: the path itself when it names an existing file (a name containing commas or
    starting with @ too); with bank, a BankTarget for ``@SPEC``; otherwise a tuple of the comma-separated paths of a
    reference set.  The caller checks that each exists."""
    if os.path.isfile(field):
        return field
    if bank and field.startswith("@"):
        from adaptive_voice_conversion_b200.speaker_bank import parse_spec
        parse_spec(field[1:])
        return BankTarget(field[1:])
    if "," not in field:
        return field
    return tuple(field.split(","))


def read_pairs(path, bank=False):
    """[(line number, source, target, output name)] of a pairs file; ValueError naming the line of a malformed entry
    or a missing input.  target is a path, a tuple of paths for a comma-separated reference set, or (bank) a
    BankTarget for an @SPEC field (target_field)."""
    out = []
    with open(path) as f:
        for n, line in enumerate(f, 1):
            parts = line.split()
            if not parts or parts[0].startswith("#"):
                continue
            err = lambda msg: ValueError(f"{path} line {n}: {msg}")  # noqa: E731
            if len(parts) not in (2, 3):
                raise err(f"expected 'source target [output_name]', got {len(parts)} fields")
            try:
                tgt = target_field(parts[1], bank)
            except ValueError as e:
                raise err(str(e)) from None
            for fp in (parts[0], *target_files(tgt)):
                if not os.path.isfile(fp) or not (is_wav(fp) or fp.lower().endswith(".npy")):
                    raise err(f"{fp} is not an existing .wav or .npy file")
            stem = lambda p: os.path.splitext(os.path.basename(p))[0]  # noqa: E731
            if isinstance(tgt, BankTarget):   # a weight's '.' is not an extension: the default name gets .wav now
                first = tgt.spec.replace(":", "-").replace(",", "+") + ".wav"
            else:
                first = stem(target_files(tgt)[0])
            name = parts[2] if len(parts) == 3 else f"{stem(parts[0])}_to_{first}"
            ext = os.path.splitext(name)[1].lower()
            if os.path.basename(name) != name or ext not in ("", ".wav", ".npy"):
                raise err(f"output_name {name} must be a file name ending in .wav, .npy or nothing")
            out.append((n, parts[0], tgt, name if ext else name + ".wav"))
    if not out:
        raise ValueError(f"{path}: no pairs")
    return out


def check_frames(pairs, src_frames, tgt_frames, minimum):
    """ValueError naming the line of the first pair whose source / target is shorter than (min_src, min_ref).
    tgt_frames[i] lists the frames of the target_files of pairs[i]'s target (a one-file target's may be its count)."""
    for (n, src, tgt, _), ts, tt in zip(pairs, src_frames, tgt_frames):
        if ts < minimum[0]:
            raise ValueError(f"line {n}: source {src} has {ts} frames; the model needs at least {minimum[0]}")
        for t, f in zip(target_files(tgt), [tt] if isinstance(tt, int) else tt):
            if f < minimum[1]:
                raise ValueError(f"line {n}: target {t} has {f} frames; the model needs at least {minimum[1]}")


def convert_pairs(inf, pairs, mels, bank=None):
    """Converted mels of every pair (normalised mels by path in `mels`): the single-target lines through
    Inferencer.inference_padded as one batch, the reference-set lines as another, lines naming the same set sharing
    one list object (embedded once), and the @SPEC lines with their bank codes through Inferencer.inference_with_codes
    as a third."""
    banked = [i for i, (_, _, t, _) in enumerate(pairs) if isinstance(t, BankTarget)]
    single = [i for i, (_, _, t, _) in enumerate(pairs) if isinstance(t, str)]
    multi = [i for i, (_, _, t, _) in enumerate(pairs) if not isinstance(t, (str, BankTarget))]
    decs = [None] * len(pairs)
    if banked:
        codes = torch.stack([bank.code(pairs[i][2].spec) for i in banked])
        for i, d in zip(banked, inf.inference_with_codes([mels[pairs[i][1]] for i in banked], codes)):
            decs[i] = d
    if single:
        for i, d in zip(single, inf.inference_padded([mels[pairs[i][1]] for i in single],
                                                     [mels[pairs[i][2]] for i in single])):
            decs[i] = d
    if multi:
        sets = {}
        for i in multi:
            sets.setdefault(pairs[i][2], [mels[p] for p in pairs[i][2]])
        for i, d in zip(multi, inf.inference_padded([mels[pairs[i][1]] for i in multi], [sets[pairs[i][2]] for i in multi])):
            decs[i] = d
    return decs


def refuse_bank_targets(pairs, path):
    """ValueError naming the first @SPEC line: -pitch_shift match needs the target's mels."""
    for n, _, t, _ in pairs:
        if isinstance(t, BankTarget):
            raise ValueError(f"{path} line {n}: -pitch_shift match needs the target's recordings; a banked speaker "
                             f"(@{t.spec}) has none")


def refuse_unprofiled_bank(path):
    """ValueError when the bank file at `path` has no pitch profiles (read on the host, before any model or GPU work):
    -pitch_shift mv needs them for a banked target."""
    d = torch.load(path, map_location="cpu", weights_only=True)
    if not isinstance(d, dict) or d.get("pitch") is None:
        raise ValueError(f"{path}: the bank has no pitch profiles, which -pitch_shift mv needs for a banked target; "
                         f"rebuild it with speaker_bank.py -f0")


def print_mv(names, info, bank=None, hp=None):
    """One line per conversion of -pitch_shift mv, and a note when hp's Griffin-Lim settings are not those of the
    bank's pitch profiles."""
    if bank is not None and bank.pitch is not None:
        gl = {"n_iter": int(hp.n_iter), "momentum": float(hp.momentum), "init": hp.gl_init}
        if gl != bank.pitch["griffin_lim"]:
            print(f"note: the bank's pitch profiles were synthesised with Griffin-Lim {bank.pitch['griffin_lim']}, "
                  f"these conversions with {gl}")
    for name, d in zip(names, info):
        note = (" (unmatched: no voiced frame)" if d["unmatched"] else " (mean only)" if d["mean_only"] else "")
        print(f"{name}: pitch shift mv mean {d['mean_shift']:+.3f} semitones, voiced frames {d['voiced_conv']} "
              f"conversion, {d['clamped_frames']} clamped{note}")


def print_matches(names, info):
    for name, d in zip(names, info):
        note = " (unmatched: no voiced frame)" if d["unmatched"] else " (clamped)" if d["clamped"] else ""
        print(f"{name}: pitch shift {d['shift']:+.3f} semitones, voiced frames {d['voiced_conv']} conversion / "
              f"{d['voiced_refs']} target{note}")


def run_pairs(args, config):
    """The -pairs mode: every line of the file, refused as a whole before anything runs (see the module docstring)."""
    pairs = read_pairs(args.pairs, bank=bool(args.bank))
    if args.semitones == "match":
        refuse_bank_targets(pairs, args.pairs)
    if args.semitones == "mv" and any(isinstance(t, BankTarget) and is_wav(name) for _, _, t, name in pairs):
        refuse_unprofiled_bank(args.bank)
    os.makedirs(args.output, exist_ok=True)
    run(args, config, pairs)


def run(args, config, jobs):
    """Converts jobs, [(line number or None, source, target, output name)]: the lines of a pairs file, their outputs
    named in the -o directory, or one conversion, its output the -o path.  Every input is read once (the .wav files in
    one Vocoder.wav_to_mel call), normalised on the device, converted, denormalised, pitch-shifted and synthesised
    (every .wav output in one Vocoder.mel_to_wav call); see the module docstring."""
    from adaptive_voice_conversion_b200.mcd import min_frames
    from adaptive_voice_conversion_b200.vocoder import AudioParams, Vocoder, load_wav
    dev = local_device()
    files = sorted({p for _, s, t, _ in jobs for p in (s, *target_files(t))})
    hp = AudioParams(n_iter=args.gl_iters, momentum=args.gl_momentum, gl_init=args.gl_init,
                     pitch_shift=0.0 if isinstance(args.semitones, str) else args.semitones)
    vocoder = None
    if any(is_wav(f) for f in files) or any(is_wav(out) for *_, out in jobs):
        vocoder = Vocoder(n_mels=config["SpeakerEncoder"]["c_in"] // config["data_loader"]["frame_size"], hp=hp)
    wavs = [f for f in files if is_wav(f)]
    raw = {}
    if wavs:
        sigs = [torch.from_numpy(load_wav(f, hp.sr)).to(dev) for f in wavs]
        raw.update((f, m) for f, (m, _) in zip(wavs, vocoder.wav_to_mel(sigs)))
    raw.update((f, torch.from_numpy(np.load(f).astype(np.float32)).to(dev)) for f in files if not is_wav(f))
    if args.pairs:
        check_frames(jobs, [raw[s].shape[0] for _, s, _, _ in jobs],
                     [[raw[p].shape[0] for p in target_files(t)] for _, _, t, _ in jobs], min_frames(config))
    inf = Inferencer(config=config, args=args)
    # the mels of every target are normalised and denormalised here, on the device, so inference_one_utterance must
    # hand back its mels normalised
    attr, inf.attr = inf.attr, None
    bank = load_bank(args.bank, inf.model) if args.bank else None
    for n, _, t, _ in jobs:
        if args.pairs and isinstance(t, BankTarget):
            try:
                bank.code(t.spec)
            except ValueError as e:
                raise ValueError(f"{args.pairs} line {n}: {e}") from None
    mels = raw
    if attr is not None:
        mean = torch.as_tensor(np.asarray(attr["mean"], np.float32)).to(dev)
        std = torch.as_tensor(np.asarray(attr["std"], np.float32)).to(dev)
        mels = {f: (m - mean) / std for f, m in raw.items()}
    fps = hp.sr / hp.hop_length
    _, src, tgt, _ = jobs[0]
    if isinstance(tgt, BankTarget) and tgt.keyframes is not None:
        from adaptive_voice_conversion_b200.speaker_bank import morph_table
        codes, weights = morph_table(bank, tgt.keyframes, mels[src].shape[0], fps)
        decs = inf.inference_morph([mels[src]], [codes], [weights.to(dev)])
    elif not isinstance(tgt, BankTarget) and not args.pairs:
        # one -t file or set: unpadded, since the padded path agrees with it only within rounding
        refs = [mels[p] for p in target_files(tgt)]
        _, dec = inf.inference_one_utterance(mels[src], refs[0] if len(refs) == 1 else refs)
        decs = [torch.from_numpy(dec).to(dev)]
    else:
        decs = convert_pairs(inf, jobs, mels, bank)
    if attr is not None:
        decs = [d * std + mean for d in decs]
    to_wav = [i for i, (*_, out) in enumerate(jobs) if is_wav(out)]
    shifts = None
    if args.semitones == "match" and to_wav:
        from adaptive_voice_conversion_b200.f0 import match_shifts
        shifts, info = match_shifts(vocoder, [decs[i].contiguous() for i in to_wav],
                                    [[raw[p] for p in target_files(jobs[i][2])] for i in to_wav], vocoder.hp)
        print_matches([jobs[i][3] for i in to_wav], info)
    if args.semitones == "mv" and to_wav:
        from adaptive_voice_conversion_b200.f0 import mv_match
        tgts = [jobs[i][2] for i in to_wav]
        profiles = [None if not isinstance(t, BankTarget) else bank.pitch_profile(t.spec) if t.keyframes is None else
                    bank.morph_pitch_profile(t.keyframes, decs[i].shape[0], fps) for i, t in zip(to_wav, tgts)]
        shifts, info = mv_match(vocoder, [decs[i].contiguous() for i in to_wav], vocoder.hp,
                                ref_sets=[[raw[p] for p in target_files(t)] or None for t in tgts], profiles=profiles)
        banked = any(isinstance(t, BankTarget) for t in tgts)
        print_mv([jobs[i][3] for i in to_wav], info, bank if banked else None, vocoder.hp)
    ys = []
    if to_wav:   # a fixed shift is the vocoder's hp.pitch_shift
        ys = vocoder.mel_to_wav([decs[i].contiguous() for i in to_wav], **({} if shifts is None else {"semitones": shifts}))
    out_dir = args.output if args.pairs else ""
    for i, y in zip(to_wav, ys):
        inf.write_wav_to_file(y.cpu().numpy(), os.path.join(out_dir, jobs[i][3]))
    for i, (*_, out) in enumerate(jobs):
        if not is_wav(out):
            np.save(os.path.join(out_dir, out), decs[i].cpu().numpy())


def load_bank(path, model):
    from adaptive_voice_conversion_b200.speaker_bank import SpeakerBank
    return SpeakerBank.load(path, model)


def pitch_shift_arg(p, args):
    """args.semitones: "match", "mv" or the -pitch_shift float; p.error for a value that is not finite or outside
    [-24, 24], match with -speaker or -morph, and a non-zero shift of a single .npy output."""
    from adaptive_voice_conversion_b200.vocoder import PITCH_SHIFT_MAX
    v = str(args.pitch_shift)
    if v == "mv":
        args.semitones = "mv"
    elif v == "match":
        args.semitones = "match"
        if args.speaker is not None or args.morph is not None:
            p.error("-pitch_shift match needs the target's recordings: banked speakers (-speaker, -morph) have none")
    else:
        try:
            args.semitones = float(v)
        except ValueError:
            p.error(f"-pitch_shift must be a number of semitones or 'match' or 'mv' (got {v!r})")
        if not np.isfinite(args.semitones) or abs(args.semitones) > PITCH_SHIFT_MAX:
            p.error(f"-pitch_shift must be finite and in [-{PITCH_SHIFT_MAX:g}, {PITCH_SHIFT_MAX:g}] semitones (got {v})")
    if args.semitones != 0.0 and not args.pairs and not is_wav(args.output):
        p.error("-pitch_shift shifts the synthesis: a .npy output is a mel and is not synthesised")


def check_args(p, args):
    """Argument errors (p.error): -t, or -bank with -speaker, for one conversion; -speaker needs -bank; -morph needs
    -bank, excludes -t, -speaker and -pairs, and its keyframes must parse; -pitch_shift as pitch_shift_arg."""
    pitch_shift_arg(p, args)
    if args.morph is not None:
        if not args.bank:
            p.error("-morph needs -bank")
        if args.target is not None or args.speaker is not None or args.pairs:
            p.error("-morph converts one source with banked speakers: it excludes -t, -speaker and -pairs")
        from adaptive_voice_conversion_b200.speaker_bank import parse_keyframe
        try:
            args.keyframes = [parse_keyframe(k) for k in args.morph]
        except ValueError as e:
            p.error(str(e))
        times = [t for _, t in args.keyframes]
        if any(b < a for a, b in zip(times, times[1:])):
            p.error(f"-morph: keyframe times must not decrease, got {times}")
        return
    if args.speaker is not None and not args.bank:
        p.error("-speaker needs -bank")
    if args.pairs:
        if args.speaker is not None:
            p.error("-speaker converts one source; in a -pairs file name a banked speaker as @SPEC")
        return
    if (args.target is None) == (args.speaker is None):
        p.error("give exactly one of -t FILE [FILE ...] and -bank BANK -speaker SPEC")


def parser():
    p = ArgumentParser()
    p.add_argument("-attr", "-a", help="attr file path")
    p.add_argument("-config", "-c", help="config file path")
    p.add_argument("-model", "-m", help="model path")
    p.add_argument("-source", "-s", help="source .wav or mel .npy")
    p.add_argument("-target", "-t", nargs="+",
                   help="target .wav or mel .npy; several files of the target speaker pool their speaker code")
    p.add_argument("-output", "-o", help="output .wav or mel .npy")
    p.add_argument("-sample_rate", "-sr", default=24000, type=int)
    p.add_argument("-gl_iters", default=100, type=int, help="Griffin-Lim iterations of a .wav output")
    p.add_argument("-gl_momentum", default=0.0, type=float,
                   help="fast Griffin-Lim momentum in [0, 1) of a .wav output (0: plain Griffin-Lim)")
    p.add_argument("-gl_init", default="zero", choices=["zero", "pghi"],
                   help="Griffin-Lim start phase of a .wav output: zero phase, or the PGHI phase-gradient estimate")
    p.add_argument("-pairs", help="file of 'source target [output_name]' lines: convert them all, into the -o directory")
    p.add_argument("-bank", help="speaker bank (speaker_bank.py) for -speaker and the @SPEC fields of -pairs")
    p.add_argument("-speaker", help="banked target: NAME or a weighted mix NAME:W,NAME:W,... (needs -bank)")
    p.add_argument("-morph", nargs="+", metavar="SPEC@SECONDS",
                   help="time-varying target: banked speakers or mixes at keyframe times, interpolated (needs -bank)")
    p.add_argument("-pitch_shift", default="0", metavar="{SEMITONES,match,mv}",
                   help="transpose every .wav output by SEMITONES in [-24, 24] (formant-preserving), 'match' each "
                        "conversion's pitch level to its -t target's, or 'mv': level and range to any target's")
    return p


def main(argv=None):
    p = parser()
    args = p.parse_args(argv)
    check_args(p, args)
    if args.semitones == "mv" and (args.speaker is not None or args.morph is not None):
        try:
            refuse_unprofiled_bank(args.bank)
        except ValueError as e:
            p.error(str(e))
    config = load_config(args.config)
    if args.pairs:
        run_pairs(args, config)
        raise SystemExit(0)
    target = (BankTarget(keyframes=tuple(args.keyframes)) if args.morph is not None else
              BankTarget(args.speaker) if args.speaker is not None else
              args.target[0] if len(args.target) == 1 else tuple(args.target))
    run(args, config, [(None, args.source, target, args.output)])


if __name__ == "__main__":
    main()
