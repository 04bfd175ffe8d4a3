"""Generated data directories for the held-out evaluation tests (tests/test_gpu_eval.py, tests/_dp_eval_worker.py):
VCTK-like utterance ids (p<speaker>_<utt>), N(0,1) mels, and an index of random crops per set."""
import json
import os
import pickle

import numpy as np

SEG = 128


def make_set(n_mels, n_entries, seed, n_speakers=4, utts_per_speaker=5, seg=SEG):
    rng = np.random.default_rng(seed)
    data = {}
    for s in range(n_speakers):
        for u in range(utts_per_speaker):
            data[f"p{300 + 10 * seed + s}_{u:03d}"] = rng.standard_normal((int(rng.integers(seg + 1, 400)), n_mels)).astype(np.float32)
    utts = list(data)
    index = []
    for _ in range(n_entries):
        utt = utts[int(rng.integers(len(utts)))]
        index.append([utt, int(rng.integers(0, len(data[utt]) - seg + 1))])
    return data, index


def write_data_dir(root, n_mels, sets, seed=0, seg=SEG):
    """<root>/<name>.pkl and <name>_samples_<seg>.json for every {name: n_entries} of `sets`; returns root."""
    os.makedirs(root, exist_ok=True)
    for k, (name, n) in enumerate(sets.items()):
        data, index = make_set(n_mels, n, seed + k, seg=seg)
        with open(os.path.join(root, f"{name}.pkl"), "wb") as f:
            pickle.dump(data, f)
        with open(os.path.join(root, f"{name}_samples_{seg}.json"), "w") as f:
            json.dump(index, f)
    return str(root)
