"""GPU: preprocess_libri.py end to end on a seeded synthetic LibriTTS-shaped tree (train-clean-100 and dev-clean,
several speakers and chapters, transcripts beside the wavs, one silent file): its files, the processing order the
pickles and attr.pkl carry, its mels against the single-file vocoder path, its reproducibility across runs and chunk
sizes, and training, held-out evaluation and one-shot conversion from its output."""
import json
import os
import subprocess
import sys
import types

import numpy as np
import pytest
import torch
from scipy.io import wavfile

from adaptive_voice_conversion_b200 import prepare as P
from adaptive_voice_conversion_b200 import vocoder as V
from conftest import ROOT
from test_gpu_prepare import bits, load, to_s16, utterance

pytestmark = pytest.mark.gpu

SR = 24000
N_MELS = 80
# {subset: {speaker: {chapter: utterances}}}; 103 and 1034 sort differently as paths and as basenames
TREE = {"train-clean-100": {"103": {"1240": 4, "1241": 3}, "1034": {"121": 4}, "19": {"198": 3}, "26": {"495": 4}},
        "dev-clean": {"84": {"121123": 3, "121550": 2}, "174": {"50561": 3}}}
SILENT = os.path.join("train-clean-100", "19", "198", "19_198_000099_000000.wav")
OPTS = dict(test_prop=0.2, n_utts_attr=6, n_mels=N_MELS, segment_size=128, training_samples=300, testing_samples=40,
            seed=5)
FILES = ["attr.pkl", "train.pkl", "dev.pkl", "test.pkl", "train_128.pkl", "train_samples_128.json",
         "dev_samples_128.json", "test_samples_128.json", "train_files.txt", "dev_files.txt", "test_files.txt",
         "skipped_files.txt"]


def write_tree(root):
    rng = np.random.default_rng(2025)
    for subset, speakers in TREE.items():
        for spk, chapters in speakers.items():
            for ch, n in chapters.items():
                d = os.path.join(root, subset, spk, ch)
                os.makedirs(d)
                for i in range(n):
                    stem = os.path.join(d, f"{spk}_{ch}_{i:06d}_{i + 1:06d}")
                    wavfile.write(stem + ".wav", SR, to_s16(utterance(rng, SR, rng.uniform(2.0, 3.5))))
                    for ext in (".normalized.txt", ".original.txt"):
                        with open(stem + ext, "w") as f:
                            f.write("Some words.\n")
    wavfile.write(os.path.join(root, SILENT), SR, np.zeros(2 * SR, np.int16))
    # a wav outside speaker / chapter / file: not listed
    wavfile.write(os.path.join(root, "dev-clean", "84", "stray.wav"), SR, to_s16(utterance(rng, SR, 2.0)))


@pytest.fixture(scope="module")
def tree(tmp_path_factory):
    root = tmp_path_factory.mktemp("libri")
    libri = str(root / "LibriTTS")
    write_tree(libri)
    out = str(root / "cli")
    cmd = [sys.executable, os.path.join(ROOT, "preprocess_libri.py"), libri, out]
    for k, v in OPTS.items():
        cmd += [f"--{k}", str(v)]
    r = subprocess.run(cmd, capture_output=True, text=True, cwd=str(root))
    assert r.returncode == 0, r.stdout + r.stderr
    print(r.stdout)
    train = P.read_libri_paths(libri, "train-clean-100")
    sets = dict(zip(P.LIBRI_SETS, P.split_libri(train, P.read_libri_paths(libri, "dev-clean"), 0.2, OPTS["seed"])))
    return types.SimpleNamespace(root=root, libri=libri, out=out, stdout=r.stdout, sets=sets)


def usable(paths):
    return [os.path.basename(p) for p in paths if not p.endswith(SILENT)]


def test_preprocess_libri_writes_the_reference_files(tree):
    assert sorted(os.listdir(tree.out)) == sorted(FILES)
    skipped = open(os.path.join(tree.out, "skipped_files.txt")).read().splitlines()
    assert len(skipped) == 1 and skipped[0].split("\t")[0].endswith(SILENT) and "silent" in skipped[0].split("\t")[1]
    assert "1 files skipped" in tree.stdout
    assert len(tree.sets["train"]) + len(tree.sets["dev"]) == 19 and len(tree.sets["dev"]) == 3
    assert len(tree.sets["test"]) == 8
    for name in P.LIBRI_SETS:
        # the reference writes the basenames of the sorted paths, skipped files included
        names = open(os.path.join(tree.out, f"{name}_files.txt")).read().splitlines()
        assert names == [os.path.basename(p) for p in sorted(tree.sets[name])], name
        data = load(os.path.join(tree.out, f"{name}.pkl"))
        # key order = processing order: shuffled for train and dev, sorted for test
        assert list(data) == usable(tree.sets[name]), name
        assert all(v.dtype == np.float32 and v.ndim == 2 and v.shape[1] == N_MELS for v in data.values())
        index = json.load(open(os.path.join(tree.out, f"{name}_samples_128.json")))
        assert len(index) == (300 if name == "train" else 40)
        assert index == [list(e) for e in P.sample_segments(data, len(index), 128, OPTS["seed"])]
    assert list(load(os.path.join(tree.out, "test.pkl"))) == sorted(usable(tree.sets["test"]))
    shuffled = usable(tree.sets["train"])
    assert shuffled != sorted(shuffled)
    train = load(os.path.join(tree.out, "train.pkl"))
    reduced = load(os.path.join(tree.out, "train_128.pkl"))
    assert list(reduced) == [k for k, v in train.items() if v.shape[0] > 128]


def test_attr_covers_the_first_training_utterances_in_shuffled_order(tree):
    attr = load(os.path.join(tree.out, "attr.pkl"))
    voc = V.Vocoder(n_mels=N_MELS)
    prep = P.Preparer(N_MELS, SR)
    n = OPTS["n_utts_attr"]

    def stats(paths):
        raws = [voc.get_spectrograms(p)[0] for p in paths[:n]]
        mom = torch.empty(n, N_MELS, 2, dtype=torch.float64, device="cuda")
        counts = [r.shape[0] for r in raws]
        prep.moments(torch.from_numpy(np.concatenate(raws)).cuda(), counts, mom, 0)
        return prep.merge(mom, counts)[:2]

    train = [p for p in tree.sets["train"] if not p.endswith(SILENT)]
    assert len(train) > n and set(train[:n]) != set(sorted(train)[:n])   # the seed makes the two prefixes differ
    mean, std = stats(train)
    assert np.array_equal(bits(attr["mean"]), bits(mean)) and np.array_equal(bits(attr["std"]), bits(std))
    smean, sstd = stats(sorted(train))
    assert not np.array_equal(bits(attr["mean"]), bits(smean)) and not np.array_equal(bits(attr["std"]), bits(sstd))


def test_mels_equal_the_single_file_path(tree):
    attr = load(os.path.join(tree.out, "attr.pkl"))
    mean, std = attr["mean"], attr["std"]
    voc = V.Vocoder(n_mels=N_MELS)
    n = 0
    for name in P.LIBRI_SETS:
        data = load(os.path.join(tree.out, f"{name}.pkl"))
        for p in tree.sets[name]:
            if p.endswith(SILENT):
                continue
            ref = (voc.get_spectrograms(p)[0] - mean) / std
            assert np.array_equal(bits(data[os.path.basename(p)]), bits(ref)), p
            n += 1
    assert n == 26


def test_output_is_reproducible_across_runs_and_chunk_sizes(tree):
    outs = []
    for tag, chunk in (("same", 1800.0), ("per_file", 0.001)):
        out = str(tree.root / f"run_{tag}")
        P.run_libri(tree.libri, out, chunk_seconds=chunk, log=lambda *a: None, **OPTS)
        outs.append(out)
    for f in FILES:
        ref = open(os.path.join(tree.out, f), "rb").read()
        for out in outs:
            assert open(os.path.join(out, f), "rb").read() == ref, (out, f)


def test_training_evaluation_and_conversion_from_the_prepared_directory(tree, tmp_path):
    from adaptive_voice_conversion_b200 import data_utils as D
    from adaptive_voice_conversion_b200.config import default_config
    from adaptive_voice_conversion_b200.solver import Solver
    cfg = default_config(N_MELS)
    cfg["data_loader"]["batch_size"] = 16
    store = str(tmp_path / "m")
    args = types.SimpleNamespace(data_dir=tree.out, train_set="train_128", train_index_file="train_samples_128.json",
                                 logdir=str(tmp_path / "log"), load_model=False, load_opt=False, store_model_path=store,
                                 load_model_path=store, summary_steps=1, save_steps=1000, tag="t", iters=0)
    torch.manual_seed(0)
    s = Solver(cfg, args)
    assert isinstance(s.train_loader, D.DeviceSegments)
    s.train(4)
    meta, _ = s.logger.last["t/ae_train"]
    assert all(np.isfinite(v) for v in meta.values()), meta
    del s

    ev = str(tmp_path / "eval.json")
    r = subprocess.run([sys.executable, os.path.join(ROOT, "evaluate.py"), "-c", f"{store}.config.yaml", "-m",
                        f"{store}.ckpt", "-d", tree.out, "-eval_sets", "dev,test", "-o", ev],
                       capture_output=True, text=True, cwd=str(tmp_path))
    assert r.returncode == 0, r.stdout + r.stderr
    res = json.load(open(ev))
    assert list(res) == ["dev", "test"]
    for name in ("dev", "test"):
        # the speaker directory of each file of the set
        speakers = {p.split(os.sep)[-3] for p in tree.sets[name] if not p.endswith(SILENT)}
        assert set(res[name]["speakers"]) == speakers, name
        assert np.isfinite(res[name]["loss_rec"]) and np.isfinite(res[name]["loss_kl"]) and res[name]["n"] == 40
    assert set(res["test"]["speakers"]) == {"84", "174"}

    src = [p for p in tree.sets["test"] if p.split(os.sep)[-3] == "84"][0]
    tgt = [p for p in tree.sets["train"] if not p.endswith(SILENT)][0]
    out = str(tmp_path / "out.wav")
    r = subprocess.run([sys.executable, os.path.join(ROOT, "inference.py"), "-c", f"{store}.config.yaml", "-m",
                        f"{store}.ckpt", "-a", os.path.join(tree.out, "attr.pkl"), "-s", src, "-t", tgt, "-o", out],
                       capture_output=True, text=True, cwd=str(tmp_path))
    assert r.returncode == 0, r.stdout + r.stderr
    rate, wav = wavfile.read(out)
    assert rate == SR and wav.size > 0 and np.isfinite(wav).all()
