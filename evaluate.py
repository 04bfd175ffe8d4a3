"""Held-out evaluation of a checkpoint: the reconstruction and KL losses of the conversion path on the test sets of a
data directory (adaptive_voice_conversion_b200/evaluate.py gives the definition).

    python evaluate.py -c config.yaml -m model.ckpt -d data/ [-eval_sets in_test,out_test] [-o eval.json]

The checkpoint is loaded strictly (reference checkpoints too, and the `sn: True` layout).  Each set's losses are
printed; -o writes them with the per-speaker means as JSON.
"""
import json
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
    args = p.parse_args(argv)
    config = load_config(args.config)
    dev = local_device()
    model = AE(config).to(dev)
    model.load_state_dict(torch.load(args.model, map_location=dev), strict=True)
    model.eval()
    held = HeldOut([s for s in args.eval_sets.split(",") if s], args.data_dir, config, device=dev)
    res = held.evaluate(model, per_speaker=True)
    for s, r in res.items():
        print(f"{s}: n={r['n']} loss_rec={r['loss_rec']:.6f} loss_kl={r['loss_kl']:.6f} ({len(r['speakers'])} speakers)")
    if args.output:
        with open(args.output, "w") as f:
            json.dump(res, f, indent=1)
    return res


if __name__ == "__main__":
    main()
