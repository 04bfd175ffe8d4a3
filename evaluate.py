"""Held-out evaluation of a checkpoint: the reconstruction and KL losses of the conversion path on the test sets of a
data directory (adaptive_voice_conversion_b200/evaluate.py gives the definition).

    python evaluate.py -c config.yaml -m model.ckpt -d data/ [-eval_sets in_test,out_test] [-o eval.json]
                       [-mcd -transcripts VCTK-Corpus/txt [-attr data/attr.pkl] [-mcd_dims 24]] [-spk]
                       [-f0 [-gl_iters 100] [-gl_momentum 0] [-gl_init zero] [-pitch_shift match|mv]]
                       [-max_pairs 0] [-seed 0] [-n_refs 1] [-bank bank.pt] [-probe [-probe_set train] [-probe_utts 64]]

The checkpoint is loaded strictly (reference checkpoints too, and the `sn: True` layout).  Each set's losses are
printed; -o writes them with the per-speaker means as JSON.  -mcd also measures conversion itself: the mel-cepstral
distortion after DTW between speaker A's utterance converted to speaker B and B's recording of the same sentence
(adaptive_voice_conversion_b200/mcd.py gives the definition), one more line per set and an "mcd" entry per set in -o.
-spk measures speakers: the verification EER of the speaker embedding, the pooled content code and the pooled input
mel, and the speaker similarity of conversions to the target speaker's other utterances
(adaptive_voice_conversion_b200/speaker_eval.py gives the definitions), two more lines per set and a "spk" entry per
set in -o.
-f0 measures the pitch of conversions as synthesised: every utterance -spk embeds and every conversion of the -spk
pairs (the same pairs, the same -seed, -max_pairs and -n_refs) is denormalised with -attr, synthesised by the project's
Griffin-Lim vocoder untrimmed (-gl_iters, -gl_momentum, -gl_init; defaults 100, 0, zero, as inference.py) and tracked
by YIN on the GPU (adaptive_voice_conversion_b200/f0.py gives the definitions): vuv_agree (voicing agreement with the
source's copy-synthesis), f0_corr (Pearson correlation of log2 F0 over the frames voiced in both), st_target and
st_source (semitones between the conversion's mean log2 F0 and the target's and the source's speaker profile, each
leaving out the pair's own utterances), f0_success = [st_target < st_source] and st_target_source (the unconverted
baseline); one more line per set and an "f0" entry per set in -o.  These are F0 measures of this project's Griffin-Lim
output, not of the original recordings.
-pitch_shift match (with -f0) also shifts each conversion toward its reference(s)' mean log2 F0 (f0.match_shifts),
re-synthesises and re-scores it against the same leave-out profiles: the "f0" entry then holds the shifted scores,
"pitch_shift" (mean and mean absolute shift, unmatched and clamped pairs) and "unshifted", the scores without it.
-pitch_shift mv shifts each conversion frame by frame toward the mean and std of its reference(s)' log2 F0
(f0.mv_shifts) instead; "pitch_shift" then also holds n_mean_only, n_clamped_frames, and sd_target and
sd_target_unshifted, the mean of 12 |log2 std of the conversion's voiced F0 - the references'| with and without it.
-n_refs K (default 1) converts with K references of the target speaker per conversion, their speaker codes pooled
(-mcd and -spk): the first reference is drawn as with one, the K - 1 others from a second generator seeded with
seed + 1; sim_target then skips all K.  With K > 1 each result also reports n_refs and n_few (conversions dropped for
want of K references).
-bank bank.pt (with -spk; speaker_bank.py) also identifies each conversion among the banked speakers by nearest
speaker code: id_target and id_source are the shares of conversions nearest the target's and the source's code,
id_real the share of the set's own utterances nearest their speaker's (the encoder's ceiling), over the n_banked
pairs whose two speakers are banked (n_unbanked the others), with bank_speakers.  A bank that pooled any of the
evaluated utterances is refused; a train bank leaves in_test leak-free and reports out_test's unseen speakers as
unbanked.
-probe trains speaker-classifier probes (a small MLP each) on -probe_set's speaker codes, pooled content codes, content
code frames and pooled mels, up to -probe_utts utterances per speaker drawn with -seed, and reports their accuracy on
each set's utterances of those speakers (adaptive_voice_conversion_b200/speaker_probe.py gives the definitions): one
more line per set and a "probe" entry per set in -o.  The probe set must be disjoint from the evaluated sets.
"""
import json
import os
import pickle
from argparse import ArgumentParser

import torch

from adaptive_voice_conversion_b200.config import load_config
from adaptive_voice_conversion_b200.evaluate import HeldOut
from adaptive_voice_conversion_b200.model import AE
from adaptive_voice_conversion_b200.utils import local_device


def main(argv=None):
    p = ArgumentParser(description="AdaIN-VC held-out evaluation on H100")
    p.add_argument("-config", "-c", default="config.yaml", help="config file path")
    p.add_argument("-model", "-m", required=True, help="model checkpoint (.ckpt)")
    p.add_argument("-data_dir", "-d", required=True, help="data directory written by preprocess.py")
    p.add_argument("-eval_sets", default="in_test,out_test", help="comma-separated set names (<set>.pkl)")
    p.add_argument("-output", "-o", default=None, help="JSON file for the per-set and per-speaker results")
    p.add_argument("-mcd", action="store_true", help="also measure MCD-DTW of conversions on parallel utterances")
    p.add_argument("-transcripts", default=None, help="directory searched for <id>.txt / <id>.normalized.txt (-mcd)")
    p.add_argument("-attr", default=None, help="mel statistics (default <data_dir>/attr.pkl) (-mcd, -f0)")
    p.add_argument("-mcd_dims", type=int, default=24, help="cepstral coefficients c_1..c_D (-mcd)")
    p.add_argument("-spk", action="store_true", help="also measure speaker EERs and the speaker similarity of conversions")
    p.add_argument("-f0", action="store_true", help="also measure the F0 of synthesised conversions (YIN on the GPU)")
    p.add_argument("-gl_iters", default=100, type=int, help="Griffin-Lim iterations of the synthesis (-f0)")
    p.add_argument("-gl_momentum", default=0.0, type=float, help="fast Griffin-Lim momentum in [0, 1) (-f0)")
    p.add_argument("-gl_init", default="zero", choices=["zero", "pghi"], help="Griffin-Lim start phase (-f0)")
    p.add_argument("-pitch_shift", default=None, choices=["match", "mv"],
                   help="also score each conversion shifted to its reference(s)' pitch level (match) or level and "
                        "range (mv) (-f0)")
    p.add_argument("-max_pairs", type=int, default=0,
                   help="keep at most this many triplets (-mcd) and conversion pairs (-spk) per set, 0 = all; "
                        "-f0 scores the -spk pairs")
    p.add_argument("-seed", type=int, default=0, help="seed of the reference choice and the sampling (-mcd, -spk); "
                                                      "-f0 as -spk")
    p.add_argument("-n_refs", type=int, default=1,
                   help="references of the target speaker per conversion, their speaker codes pooled (-mcd, -spk); "
                        "-f0 as -spk")
    p.add_argument("-bank", default=None, help="speaker bank: identify conversions among its speakers (-spk)")
    p.add_argument("-probe", action="store_true",
                   help="also train speaker-classifier probes on the speaker code, the content code and the mel, and "
                        "report their accuracy on each set")
    p.add_argument("-probe_set", default="train", help="set the probes are fitted on (<probe_set>.pkl) (-probe)")
    p.add_argument("-probe_utts", type=int, default=64, help="fit utterances drawn per speaker (-probe)")
    args = p.parse_args(argv)
    eval_sets = [s for s in args.eval_sets.split(",") if s]
    if args.probe:
        if args.probe_set in eval_sets:
            p.error(f"-probe_set {args.probe_set} is also one of -eval_sets; a probe must be scored on other utterances")
        if not os.path.isfile(os.path.join(args.data_dir, f"{args.probe_set}.pkl")):
            p.error(f"-probe needs {os.path.join(args.data_dir, args.probe_set + '.pkl')} (pass -probe_set)")
        if args.probe_utts < 1:
            p.error("-probe_utts must be >= 1")
    if args.mcd and not args.transcripts:
        p.error("-mcd needs -transcripts DIR")
    if args.bank and not args.spk:
        p.error("-bank needs -spk")
    if not 1 <= args.n_refs <= 64:
        p.error("-n_refs must lie in [1, 64]")
    if args.gl_iters < 0:
        p.error("-gl_iters must be >= 0")
    if not 0.0 <= args.gl_momentum < 1.0:
        p.error("-gl_momentum must lie in [0, 1)")
    if args.pitch_shift and not args.f0:
        p.error("-pitch_shift needs -f0")
    attr_path = args.attr or os.path.join(args.data_dir, "attr.pkl")
    if args.f0 and not os.path.isfile(attr_path):
        p.error(f"-f0 needs the mel statistics: {attr_path} does not exist (pass -attr)")
    few = {} if args.n_refs == 1 else {"n_refs": args.n_refs}
    config = load_config(args.config)
    dev = local_device()
    model = AE(config).to(dev)
    model.load_state_dict(torch.load(args.model, map_location=dev), strict=True)
    model.eval()
    held = HeldOut(eval_sets, args.data_dir, config, device=dev)
    res = held.evaluate(model, per_speaker=True)
    for s, r in res.items():
        print(f"{s}: n={r['n']} loss_rec={r['loss_rec']:.6f} loss_kl={r['loss_kl']:.6f} ({len(r['speakers'])} speakers)")
    if args.mcd:
        from adaptive_voice_conversion_b200.mcd import evaluate_mcd, read_transcripts
        with open(attr_path, "rb") as f:
            attr = pickle.load(f)
        for s in res:
            with open(os.path.join(args.data_dir, f"{s}.pkl"), "rb") as f:
                data = pickle.load(f)
            m = evaluate_mcd(model, data, attr, read_transcripts(args.transcripts, data), dims=args.mcd_dims,
                             max_pairs=args.max_pairs, seed=args.seed, device=dev, **few)
            res[s]["mcd"] = m
            means = f" mcd={m['mcd']:.4f} mcd_source={m['mcd_source']:.4f}" if m["n"] else ""
            means += f" n_refs={m['n_refs']} n_few={m['n_few']}" if few else ""
            print(f"{s}: mcd n={m['n']} n_short={m['n_short']}{means} (dims {m['dims']}, "
                  f"{len(m['speakers'])} target speakers)")
    if args.spk:
        from adaptive_voice_conversion_b200.speaker_eval import evaluate_speakers
        banked = {}
        if args.bank:
            from adaptive_voice_conversion_b200.speaker_bank import SpeakerBank
            banked["bank"] = SpeakerBank.load(args.bank, model)
        for s in res:
            with open(os.path.join(args.data_dir, f"{s}.pkl"), "rb") as f:
                data = pickle.load(f)
            r = evaluate_speakers(model, data, seed=args.seed, max_pairs=args.max_pairs, device=dev, **few, **banked)
            res[s]["spk"] = r
            e = r["eer"]
            eers = " ".join(f"{k}=" + ("n/a" if e[k]["eer"] is None else f"{e[k]['eer']:.4f}") for k in ("speaker", "content", "mel"))
            print(f"{s}: spk eer {eers} (n_utts={r['n_utts']} n_short={r['n_short']})")
            c = r["conversion"]
            means = (f" sim_target={c['sim_target']:.4f} sim_source={c['sim_source']:.4f} success={c['success']:.4f} "
                     f"sim_target_source={c['sim_target_source']:.4f}") if c["n"] else ""
            means += f" n_refs={c['n_refs']} n_few={c['n_few']}" if few else ""
            print(f"{s}: spk conversion n={c['n']} n_short={c['n_short']}{means} ({len(c['speakers'])} target speakers)")
            if args.bank:
                ids = " ".join(f"{k}=" + ("n/a" if c[k] is None else f"{c[k]:.4f}") for k in ("id_target", "id_source", "id_real"))
                print(f"{s}: spk bank {ids} n_banked={c['n_banked']} n_unbanked={c['n_unbanked']} "
                      f"({c['bank_speakers']} banked speakers)")
    if args.f0:
        from adaptive_voice_conversion_b200.f0 import evaluate_f0
        from adaptive_voice_conversion_b200.vocoder import AudioParams
        with open(attr_path, "rb") as f:
            attr = pickle.load(f)
        hp = AudioParams(n_iter=args.gl_iters, momentum=args.gl_momentum, gl_init=args.gl_init)
        for s in res:
            with open(os.path.join(args.data_dir, f"{s}.pkl"), "rb") as f:
                data = pickle.load(f)
            r = evaluate_f0(model, data, attr, seed=args.seed, max_pairs=args.max_pairs, device=dev, hp=hp,
                            pitch_shift=args.pitch_shift, **few)
            res[s]["f0"] = r
            means = (f" vuv_agree={r['vuv_agree']:.4f} f0_corr={r['f0_corr']:.4f} st_target={r['st_target']:.4f} "
                     f"st_source={r['st_source']:.4f} f0_success={r['f0_success']:.4f} "
                     f"st_target_source={r['st_target_source']:.4f}") if r["n"] else ""
            means += f" n_refs={r['n_refs']} n_few={r['n_few']}" if few else ""
            print(f"{s}: f0 n={r['n']} n_short={r['n_short']} n_unvoiced={r['n_unvoiced']}{means} "
                  f"({len(r['speakers'])} target speakers)")
            if args.pitch_shift:
                ps = r["pitch_shift"]
                mv = "" if args.pitch_shift == "match" else (
                    f" n_mean_only={ps['n_mean_only']} n_clamped_frames={ps['n_clamped_frames']} sd_target="
                    + ("n/a" if ps["sd_target"] is None else f"{ps['sd_target']:.4f}") + " (unshifted sd_target="
                    + ("n/a" if ps["sd_target_unshifted"] is None else f"{ps['sd_target_unshifted']:.4f}") + ")")
                print(f"{s}: f0 pitch_shift {args.pitch_shift} mean={ps['mean_semitones']:+.4f} "
                      f"mean_abs={ps['mean_abs_semitones']:.4f} n_unmatched={ps['n_unmatched']} "
                      f"n_clamped={ps['n_clamped']}{mv} (unshifted st_target="
                      + ("n/a" if not r["unshifted"]["n"] else f"{r['unshifted']['st_target']:.4f}") + ")")
    if args.probe:
        from adaptive_voice_conversion_b200.speaker_probe import evaluate_probe
        with open(os.path.join(args.data_dir, f"{args.probe_set}.pkl"), "rb") as f:
            fit_data = pickle.load(f)
        sets = {}
        for s in res:
            with open(os.path.join(args.data_dir, f"{s}.pkl"), "rb") as f:
                sets[s] = pickle.load(f)
        probes = evaluate_probe(model, fit_data, sets, seed=args.seed, per_speaker_utts=args.probe_utts, device=dev,
                                fit_name=args.probe_set)
        for s, r in probes.items():
            res[s]["probe"] = r
            accs = " ".join(f"{k}=" + ("n/a" if r[k]["acc"] is None else f"{r[k]['acc']:.4f}")
                            for k in ("speaker", "content", "content_frames", "mel"))
            print(f"{s}: probe {accs} chance={r['chance']:.4f} (n={r['n']} n_unseen={r['n_unseen']} n_short={r['n_short']}, "
                  f"{r['speakers']} speakers, fit on {args.probe_set}: {r['n_fit']} utterances)")
    if args.output:
        with open(args.output, "w") as f:
            json.dump(res, f, indent=1)
    return res


if __name__ == "__main__":
    main()
