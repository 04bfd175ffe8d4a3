"""Build the training data directory from a VCTK 0.80 wav tree (the reference's preprocess_vctk.sh and its three
scripts, without librosa or tensorflow; the signal work runs on the GPU):

    python preprocess.py <wav48_dir> <speaker-info.txt> <out_dir> [--n_out_speakers 20] [--test_prop 0.1]
        [--sample_rate 24000] [--n_utts_attr 5000] [--n_mels 512] [--segment_size 128]
        [--training_samples 10000000] [--testing_samples 10000] [--seed 0] [--stage 0] [--chunk_seconds 1800]

Writes attr.pkl, {train,in_test,out_test}.pkl, train_<seg>.pkl, {train,in_test,out_test}_samples_<seg>.json,
in_test_files.txt, out_test_files.txt and skipped_files.txt: what `DATA_DIR=<out_dir> sh train.sh` and
`inference.py -a <out_dir>/attr.pkl` read.  --stage as in the shell script: 0 = split and features, 1 = reduce,
2 = train index, 3 = test indexes.
"""
from argparse import ArgumentParser

from adaptive_voice_conversion_b200.prepare import run


def parse_args(argv=None):
    p = ArgumentParser(description="VCTK wav tree -> training data directory")
    p.add_argument("wav_dir")
    p.add_argument("speaker_info")
    p.add_argument("out_dir")
    p.add_argument("--n_out_speakers", type=int, default=20)
    p.add_argument("--test_prop", type=float, default=0.1)
    p.add_argument("--sample_rate", type=int, default=24000)
    p.add_argument("--n_utts_attr", type=int, default=5000)
    p.add_argument("--n_mels", type=int, default=512)
    p.add_argument("--segment_size", type=int, default=128)
    p.add_argument("--training_samples", type=int, default=10000000)
    p.add_argument("--testing_samples", type=int, default=10000)
    p.add_argument("--seed", type=int, default=0)
    p.add_argument("--stage", type=int, default=0)
    p.add_argument("--chunk_seconds", type=float, default=1800.0,
                   help="audio per GPU batch, in seconds at --sample_rate (a longer file is a batch of its own)")
    return p.parse_args(argv)


if __name__ == "__main__":
    run(**vars(parse_args()))
