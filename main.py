"""Training entry point; accepts the reference's command line (flag names of its main.py:9-22).

    python main.py -c config.yaml -d <data_dir|synthetic> -train_set train_128 \
        -train_index_file train_samples_128.json -store_model_path <path> -t <tag> -iters N

Under ``torchrun --nproc-per-node N`` every rank trains on its own batches with one NCCL
gradient all-reduce per step (data parallel).
"""
import os
from argparse import ArgumentParser

import torch

from adaptive_voice_conversion_b200.config import load_config
from adaptive_voice_conversion_b200.solver import Solver

# (flags, default, type) -- string options first, then integers; the two switches are added below
OPTIONS = [
    (("-config", "-c"), "config.yaml", str),
    (("-data_dir", "-d"), "synthetic", str),
    (("-train_set",), "train", str),
    (("-train_index_file",), "train_samples_64.json", str),
    (("-logdir",), "log/", str),
    (("-store_model_path",), "model", str),
    (("-load_model_path",), "model", str),
    (("-tag", "-t"), "init", str),
    (("-summary_steps",), 100, int),
    (("-save_steps",), 5000, int),
    (("-iters",), 0, int),
]


def parse_args(argv=None):
    parser = ArgumentParser(description="AdaIN-VC training on H100")
    for flags, default, kind in OPTIONS:
        parser.add_argument(*flags, default=default, type=kind)
    for switch in ("--load_model", "--load_opt"):
        parser.add_argument(switch, action="store_true")
    return parser.parse_args(argv)


def main(argv=None):
    args = parse_args(argv)
    if int(os.environ.get("WORLD_SIZE", "1")) > 1:
        torch.cuda.set_device(int(os.environ.get("LOCAL_RANK", "0")))
        torch.distributed.init_process_group("nccl")
    solver = Solver(config=load_config(args.config), args=args)
    if args.iters > 0:
        solver.train(n_iterations=args.iters)


if __name__ == "__main__":
    main()
