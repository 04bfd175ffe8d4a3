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

Streaming: -stream feeds -s to a StreamingConverter (adaptive_voice_conversion_b200/streaming.py) in -stream_chunk_ms
chunks (default 20 ms) and writes the untrimmed stream it gives back; the target is -t files (their pooled code) or
-bank -speaker SPEC.  With -pairs every line is one stream, all fed in lockstep.  -stream_hop, -stream_lookahead
(mel frames, multiples of 8; defaults 8 and 8), -stream_gl_lookahead (default 3) and -stream_gl_iters (default 8) set
the block schedule and RTISI-LA, and -stream_gl_init pghi starts each RTISI-LA frame from a streamed phase-gradient
(PGHI) estimate instead of the current estimate's phase (-stream_gl_init estimate, the default), one frame later;
-morph (use -stream_morph), a -pitch_shift other than 0 (use -stream_pitch) and the -gl_* options are refused with it:

    python inference.py -c config.yaml -m model.ckpt -a attr.pkl -s src.wav -t tgt.wav -o out.wav -stream

-stream_pitch moves a stream's pitch as it is synthesised (streaming.PitchStage).  SEMITONES (in [-24, 24]) shifts every
block by a fixed amount and adds no latency.  match and mv track the stream's unshifted synthesis causally and move its
running pitch level (match) or level and range (mv) to the target's profile, at the cost of the longer
tracked latency the run prints.  The profile of -t files and sets is tracked from the references synthesised by
RTISI-LA at the stream's settings; a banked target (-speaker, @SPEC lines) uses the bank's pitch record (its references
were synthesised by Griffin-Lim), so a bank without one is refused.  Unlike -pitch_shift match, -stream_pitch match
accepts banked targets: both modes read the same profile.  A target without a voiced frame leaves its stream unshifted:

    python inference.py -c config.yaml -m model.ckpt -a attr.pkl -s src.wav -bank bank.pt -speaker p225 -o out.wav \
        -stream -stream_pitch mv

-stream_morph SPEC@SECONDS [SPEC@SECONDS ...] is -morph's streaming counterpart: it needs -stream and -bank and
excludes -t, -speaker and -pairs.  Keyframe k lies at mel frame floor(seconds sr / hop + 0.5); the stream opens with
the first keyframe's code, and each later keyframe k becomes StreamingConverter.retarget(code_k, at=frame_{k-1},
ramp=frame_k - frame_{k-1}) before the first chunk, so ``A@0 A@4 B@4.3`` glides from A to B over 0.3 s from 4 s, as
-morph does.  A mix keyframe is one anchor, its mixed code (SpeakerBank.code), where -morph mixes the decoder's AdaIN
rows; the two agree up to rounding.  The decoder's windows reach H + LA frames (16, 0.2 s, with the defaults) past
the block they emit, so a block's voice starts to move up to that much before a keyframe's time.  With -stream_pitch
match or mv each keyframe's target profile is the bank's (SpeakerBank.pitch_profile) and the stream's target follows
the same weights; a bank without a pitch record is refused, and when some keyframe has no voiced frame the stream is
left unshifted, which the run prints:

    python inference.py -c config.yaml -m model.ckpt -a attr.pkl -s src.wav -bank bank.pt -o out.wav -stream \
        -stream_morph p225@0 p225@4.0 p226@4.3 -stream_pitch mv
"""
import math
import os
import sys
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


def refuse_unprofiled_bank(path, option="-pitch_shift mv"):
    """ValueError when the bank file at `path` has no pitch profiles (read on the host, before any model or GPU work):
    `option` (-pitch_shift mv, -stream_pitch match or -stream_pitch mv) needs them for a banked target."""
    d = torch.load(path, map_location="cpu", weights_only=True)
    if not isinstance(d, dict) or d.get("pitch") is None:
        raise ValueError(f"{path}: the bank has no pitch profiles, which {option} needs for a banked target; "
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


def parse_keyframes(p, option, given):
    """[(SPEC, seconds)] of -morph's or -stream_morph's keyframes; p.error for one that does not parse or times that
    decrease."""
    from adaptive_voice_conversion_b200.speaker_bank import parse_keyframe
    try:
        keyframes = [parse_keyframe(k) for k in given]
    except ValueError as e:
        p.error(str(e))
    times = [t for _, t in keyframes]
    if any(b < a for a, b in zip(times, times[1:])):
        p.error(f"{option}: keyframe times must not decrease, got {times}")
    return keyframes


def keyframe_frame(seconds, sr, hop):
    """The mel frame of a -stream_morph keyframe time: floor(seconds sr / hop + 0.5)."""
    return int(math.floor(seconds * sr / hop + 0.5))


def check_args(p, args):
    """Argument errors (p.error): -t, or -bank with -speaker, for one conversion; -speaker needs -bank; -morph and
    -stream_morph need -bank, exclude -t, -speaker and -pairs, and their keyframes must parse; -pitch_shift as
    pitch_shift_arg."""
    pitch_shift_arg(p, args)
    if args.stream_morph is not None:
        if not args.bank:
            p.error("-stream_morph needs -bank")
        if args.target is not None or args.speaker is not None or args.pairs:
            p.error("-stream_morph streams one source through banked speakers: it excludes -t, -speaker and -pairs")
        args.keyframes = parse_keyframes(p, "-stream_morph", args.stream_morph)
        return
    if args.morph is not None:
        if not args.bank:
            p.error("-morph needs -bank")
        if args.target is not None or args.speaker is not None or args.pairs:
            p.error("-morph converts one source with banked speakers: it excludes -t, -speaker and -pairs")
        args.keyframes = parse_keyframes(p, "-morph", args.morph)
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
    p.add_argument("-stream", action="store_true",
                   help="convert as a live stream: feed -s in chunks to a StreamingConverter (one stream per -pairs line)")
    p.add_argument("-stream_chunk_ms", default=20.0, type=float, help="-stream: input chunk length in milliseconds")
    p.add_argument("-stream_window", default=None, type=int, help="-stream: frames per converted window (segment_size)")
    p.add_argument("-stream_hop", default=8, type=int, help="-stream: frames emitted per block (multiple of 8)")
    p.add_argument("-stream_lookahead", default=8, type=int, help="-stream: look-ahead frames of a block's window")
    p.add_argument("-stream_gl_lookahead", default=3, type=int, help="-stream: RTISI-LA look-ahead frames (0 .. 7)")
    p.add_argument("-stream_gl_iters", default=8, type=int, help="-stream: RTISI-LA iterations per frame step")
    p.add_argument("-stream_gl_init", default=None, choices=["estimate", "pghi"],
                   help="-stream: RTISI-LA's start phase of each frame: the current estimate's (default) or a streamed "
                        "phase-gradient (PGHI) estimate, one frame later")
    p.add_argument("-stream_pitch", default=None, metavar="{SEMITONES,match,mv}",
                   help="-stream: shift every block by SEMITONES in [-24, 24], or track the stream and 'match' its "
                        "pitch level, or 'mv' its level and range, to the target's profile")
    p.add_argument("-stream_morph", nargs="+", metavar="SPEC@SECONDS",
                   help="-stream: banked speakers or mixes at keyframe times, glided between while streaming (needs "
                        "-bank; excludes -t, -speaker and -pairs).  A mix keyframe is one anchor, its mixed code; "
                        "offline -morph mixes the AdaIN rows instead, and the two agree up to rounding")
    return p


def check_stream_args(p, args, argv):
    """-stream's refusals (p.error): -morph, a pitch shift, any -gl_* option (streams are synthesised by RTISI-LA), a
    .npy output, a chunk length that is not positive and a block schedule streaming.check_params refuses."""
    if args.morph is not None:
        p.error("-morph is not supported with -stream; use -stream_morph SPEC@SECONDS [SPEC@SECONDS ...]")
    if str(args.pitch_shift) not in ("0", "0.0"):
        p.error("-pitch_shift is not supported with -stream; use -stream_pitch {SEMITONES,match,mv}")
    stream_pitch_arg(p, args)
    given = [a.split("=")[0] for a in argv if a.startswith("-gl_")]
    if given:
        p.error(f"{given[0]}: -stream synthesises with RTISI-LA (-stream_gl_lookahead, -stream_gl_iters), not "
                f"Griffin-Lim; -gl_* options are refused")
    if args.stream_chunk_ms <= 0:
        p.error("-stream_chunk_ms must be positive")
    if not args.pairs and not is_wav(args.output):
        p.error("-stream writes the synthesised stream: -o must be a .wav")
    from adaptive_voice_conversion_b200.streaming import check_params
    try:
        check_params(stream_params(args), 128 if args.stream_window is None else args.stream_window)
    except ValueError as e:
        p.error(str(e))


def stream_pitch_arg(p, args):
    """args.stream_pitch becomes None, "match", "mv" or a float in [-24, 24] (p.error otherwise)."""
    from adaptive_voice_conversion_b200.vocoder import PITCH_SHIFT_MAX
    v = args.stream_pitch
    if v is None or v in ("match", "mv"):
        return
    try:
        args.stream_pitch = float(v)
    except ValueError:
        p.error(f"-stream_pitch must be a number of semitones or 'match' or 'mv' (got {v!r})")
    if not np.isfinite(args.stream_pitch) or abs(args.stream_pitch) > PITCH_SHIFT_MAX:
        p.error(f"-stream_pitch must be finite and in [-{PITCH_SHIFT_MAX:g}, {PITCH_SHIFT_MAX:g}] semitones (got {v})")


def stream_params(args):
    from adaptive_voice_conversion_b200.streaming import StreamParams
    return StreamParams(window=args.stream_window, hop=args.stream_hop, lookahead=args.stream_lookahead,
                        gl_lookahead=args.stream_gl_lookahead, gl_iters=args.stream_gl_iters,
                        gl_init=args.stream_gl_init or "estimate")


def run_stream(args, config, jobs):
    """-stream: every job's source fed to a StreamingConverter in -stream_chunk_ms chunks, all jobs in lockstep (one
    update per chunk), and each stream's untrimmed output written.  Targets: -t files or sets (their pooled code,
    Inferencer.embed_speakers of the trimmed, normalised reference mels) or banked speakers (SpeakerBank.code)."""
    from adaptive_voice_conversion_b200.streaming import StreamingConverter
    from adaptive_voice_conversion_b200.vocoder import AudioParams, Vocoder, load_wav
    dev = local_device()
    for n, src, t, name in jobs:
        if not is_wav(src) or not is_wav(name) or not all(is_wav(f) for f in target_files(t)):
            where = f"line {n}: " if n is not None else ""
            raise ValueError(f"{where}-stream converts .wav sources to .wav outputs with .wav targets")
    tracked = args.stream_pitch in ("match", "mv")
    if tracked and any(isinstance(t, BankTarget) for _, _, t, _ in jobs):
        refuse_unprofiled_bank(args.bank, f"-stream_pitch {args.stream_pitch}")
    vocoder = Vocoder(n_mels=config["SpeakerEncoder"]["c_in"] // config["data_loader"]["frame_size"], hp=AudioParams())
    hp = vocoder.hp
    inf = Inferencer(config=config, args=args)
    bank = load_bank(args.bank, inf.model) if args.bank else None
    refs = sorted({f for _, _, t, _ in jobs for f in target_files(t)})
    raw, mel = {}, {}
    if refs:
        raw = dict(zip(refs, (m for m, _ in vocoder.wav_to_mel([torch.from_numpy(load_wav(f, hp.sr)).to(dev)
                                                                   for f in refs]))))
        mel = raw
        if inf.attr is not None:
            mean = torch.as_tensor(np.asarray(inf.attr["mean"], np.float32)).to(dev)
            std = torch.as_tensor(np.asarray(inf.attr["std"], np.float32)).to(dev)
            mel = {f: (m - mean) / std for f, m in raw.items()}
    params = stream_params(args)
    conv = StreamingConverter(inf, vocoder, params)
    profiles = stream_profiles(jobs, raw, bank, vocoder, params) if tracked else None
    sets = {}
    ids = []
    for k, (n, _, t, name) in enumerate(jobs):
        if isinstance(t, BankTarget) and t.keyframes is not None:
            code = bank.code(t.keyframes[0][0]).to(dev)
        elif isinstance(t, BankTarget):
            code = bank.code(t.spec).to(dev)
        else:
            key = target_files(t)
            if key not in sets:
                sets[key] = inf.embed_speakers([[mel[f] for f in key]])[0]
            code = sets[key]
        pitch = args.stream_pitch
        morph = isinstance(t, BankTarget) and t.keyframes is not None
        if tracked:
            pr = profiles[k]
            if morph:   # a profile per keyframe; unmatched when any keyframe has none
                pitch = None if any(x is None for x in pr) else [(args.stream_pitch, *x) for x in pr]
            else:
                pitch = None if pr is None else (args.stream_pitch, pr[0], pr[1])
            head = pr[0] if morph and pitch is not None else pr
            print(f"{name}: -stream_pitch {args.stream_pitch} " + (
                ("unmatched: a keyframe's target has no voiced frame, the stream is left unshifted" if morph else
                 "unmatched: the target has no voiced frame, every shift is 0") if pitch is None else
                f"toward log2 F0 mean {head[0]:.4f}, std {head[1]:.4f}" + (" at the first keyframe" if morph else "")))
        if morph:
            ids.append(open_morph(conv, code, bank, t.keyframes, pitch, hp, dev))
        else:
            ids.append(conv.open(code, pitch))
    srcs = [load_wav(src, hp.sr) for _, src, _, _ in jobs]
    chunk = max(1, int(round(hp.sr * args.stream_chunk_ms / 1000.0)))
    outs = [[] for _ in jobs]
    for k in range(0, max(len(y) for y in srcs), chunk):
        feed = {sid: torch.from_numpy(y[k:k + chunk]) for sid, y in zip(ids, srcs) if k < len(y)}
        for sid, y in conv.push(feed).items():
            outs[ids.index(sid)].append(y)
    for sid, y in conv.update({}, close=ids).items():
        outs[ids.index(sid)].append(y)
    print(f"streamed {len(jobs)} stream(s) in {chunk}-sample chunks; latency {conv.latency_samples} samples "
          f"({conv.latency_samples / hp.sr * 1000:.1f} ms at {hp.sr} Hz), with pitch tracking "
          f"{conv.tracked_latency_samples} samples ({conv.tracked_latency_samples / hp.sr * 1000:.1f} ms)")
    out_dir = args.output if args.pairs else ""
    for (_, _, _, name), ys in zip(jobs, outs):
        inf.write_wav_to_file(torch.cat(ys).cpu().numpy(), os.path.join(out_dir, name))


def open_morph(conv, code, bank, keyframes, pitch, hp, dev):
    """A stream of -stream_morph: opened with code, the first keyframe's, then keyframe k >= 1 becomes a retarget to
    its code at keyframe k - 1's frame over the frames between them (keyframe_frame), before any input.  pitch: None,
    a fixed shift (every anchor's) or one (mode, mu, sigma) profile per keyframe."""
    frames = [keyframe_frame(sec, hp.sr, hp.hop_length) for _, sec in keyframes]
    per = pitch if isinstance(pitch, list) else [pitch] * len(keyframes)
    sid = conv.open(code, per[0])
    for k in range(1, len(keyframes)):
        conv.retarget(sid, bank.code(keyframes[k][0]).to(dev), at=frames[k - 1], ramp=frames[k] - frames[k - 1],
                      pitch=per[k])
    return sid


def stream_profiles(jobs, raw, bank, vocoder, params):
    """The (log2 mean, log2 std) target profile of every job for -stream_pitch match / mv, or None (unmatched).  -t
    files and sets: their denormalised mels (raw) synthesised through RTISI-LA at the converter's settings, tracked by
    the streams' tracker (f0.yin, which gives avc_yin_window's bits, and f0.voicing) and pooled (f0.track_profile).
    Banked targets: SpeakerBank.pitch_profile, with a note that the bank's record was synthesised by Griffin-Lim.
    ValueError naming the file, before any synthesis, for a reference too short for the tracker."""
    from adaptive_voice_conversion_b200.f0 import F0Params, track, track_profile
    from adaptive_voice_conversion_b200.streaming import Rtisi
    hp = vocoder.hp
    refs = sorted({f for _, _, t, _ in jobs if not isinstance(t, BankTarget) for f in target_files(t)})
    need = F0Params().min_samples(hp.sr)
    for f in refs:
        n = hp.hop_length * (int(raw[f].shape[0]) - 1)     # the synthesis of T frames has hop (T - 1) samples
        if n < need:
            raise ValueError(f"{f}: -stream_pitch tracks the pitch of the target's references; after trimming this one "
                             f"synthesises to {n} samples, and the tracker needs at least {need}")
    tracks = {}
    if refs:
        rt = Rtisi(hp, params.gl_lookahead, params.gl_iters, vocoder.device, params.gl_init)
        for f in refs:
            rt.open(f)
        sig = rt.run(dict(zip(refs, vocoder.mel_to_mag([raw[f] for f in refs]))), close=refs)
        tracks = dict(zip(refs, track([sig[f] for f in refs], hp.sr, hp.hop_length)))
    if any(isinstance(t, BankTarget) for _, _, t, _ in jobs):
        print(f"note: the bank's pitch records were tracked from Griffin-Lim copy-syntheses "
              f"({bank.pitch['griffin_lim']}), not RTISI-LA")
    return [([bank.pitch_profile(spec) for spec, _ in t.keyframes] if t.keyframes is not None else
             bank.pitch_profile(t.spec)) if isinstance(t, BankTarget) else
            track_profile([tracks[f] for f in target_files(t)]) for _, _, t, _ in jobs]


def main(argv=None):
    p = parser()
    argv = sys.argv[1:] if argv is None else list(argv)
    args = p.parse_args(argv)
    if args.stream:
        check_stream_args(p, args, argv)
    elif args.stream_pitch is not None:
        p.error("-stream_pitch needs -stream (offline conversions take -pitch_shift)")
    elif args.stream_morph is not None:
        p.error("-stream_morph needs -stream (offline conversions take -morph)")
    elif args.stream_gl_init is not None:
        p.error("-stream_gl_init needs -stream (offline conversions take -gl_init)")
    check_args(p, args)
    try:
        if args.semitones == "mv" and (args.speaker is not None or args.morph is not None):
            refuse_unprofiled_bank(args.bank)
        elif args.stream and args.stream_pitch in ("match", "mv") and (args.speaker is not None
                                                                       or args.stream_morph is not None):
            refuse_unprofiled_bank(args.bank, f"-stream_pitch {args.stream_pitch}")
    except ValueError as e:
        p.error(str(e))
    config = load_config(args.config)
    if args.stream:
        if args.pairs:
            jobs = read_pairs(args.pairs, bank=bool(args.bank))
            os.makedirs(args.output, exist_ok=True)
        else:
            target = (BankTarget(keyframes=tuple(args.keyframes)) if args.stream_morph is not None else
                      BankTarget(args.speaker) if args.speaker is not None else
                      args.target[0] if len(args.target) == 1 else tuple(args.target))
            jobs = [(None, args.source, target, args.output)]
        run_stream(args, config, jobs)
        raise SystemExit(0)
    if args.pairs:
        run_pairs(args, config)
        raise SystemExit(0)
    target = (BankTarget(keyframes=tuple(args.keyframes)) if args.morph is not None else
              BankTarget(args.speaker) if args.speaker is not None else
              args.target[0] if len(args.target) == 1 else tuple(args.target))
    run(args, config, [(None, args.source, target, args.output)])


if __name__ == "__main__":
    main()
