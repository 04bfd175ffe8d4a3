"""Build the training data directory from a LibriTTS tree (the reference's preprocess_libri.sh and its three scripts,
without librosa or tensorflow; the signal work runs on the GPU):

    python preprocess_libri.py <LibriTTS root> <out_dir> [--train_set train-clean-100] [--test_set dev-clean]
        [--test_prop 0.05] [--sample_rate 24000] [--n_utts_attr 5000] [--n_mels 512] [--segment_size 128]
        [--training_samples 10000000] [--testing_samples 10000] [--seed 0] [--stage 0] [--chunk_seconds 1800]

Reads <root>/<train_set>/*/*/*.wav and <root>/<test_set>/*/*/*.wav.  Of the training subset, a seeded shuffle puts
int(files * test_prop) files in dev and the rest in train; test is the whole test subset.  Writes attr.pkl,
{train,dev,test}.pkl, train_<seg>.pkl, {train,dev,test}_samples_<seg>.json, {train,dev,test}_files.txt and
skipped_files.txt: what `DATA_DIR=<out_dir> EVAL_SETS=dev,test sh train.sh` and `inference.py -a <out_dir>/attr.pkl`
read.  --stage as in the shell script: 0 = split and features, 1 = reduce, 2 = train index, 3 = dev and test indexes.
"""
from argparse import ArgumentParser

from adaptive_voice_conversion_b200.prepare import run_libri


def parse_args(argv=None):
    p = ArgumentParser(description="LibriTTS tree -> training data directory")
    p.add_argument("root")
    p.add_argument("out_dir")
    p.add_argument("--train_set", default="train-clean-100")
    p.add_argument("--test_set", default="dev-clean")
    p.add_argument("--test_prop", type=float, default=0.05)
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
    run_libri(**vars(parse_args()))
