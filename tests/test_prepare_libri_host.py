"""CPU: the host half of LibriTTS preparation (prepare.py's listing, split and checks, preprocess_libri.py's options)
against restatements of the reference's preprocess/make_datasets_libri.py and libri.config."""
import glob
import os
import random

import pytest

import preprocess_libri
from adaptive_voice_conversion_b200 import evaluate as E
from adaptive_voice_conversion_b200 import prepare as P


def touch(path):
    os.makedirs(os.path.dirname(path), exist_ok=True)
    open(path, "wb").close()


def write_subset(root, subset, speakers):
    """speakers: {speaker: {chapter: n_utterances}}; each wav gets its two transcripts beside it, as in LibriTTS."""
    for spk, chapters in speakers.items():
        for ch, n in chapters.items():
            for i in range(n):
                stem = os.path.join(root, subset, spk, ch, f"{spk}_{ch}_{i:06d}_{i + 1:06d}")
                for ext in (".wav", ".normalized.txt", ".original.txt"):
                    touch(stem + ext)


def reference_split(root, train_set, test_set, dev_proportion, seed):
    """make_datasets_libri.py:47-52 as written (read_paths :23-25), on the module-level random after random.seed(seed)."""
    def read_paths(root_dir, dset):
        return sorted(glob.glob(os.path.join(root_dir, f'{dset}/*/*/*.wav')))

    random.seed(seed)
    paths = read_paths(root, train_set)
    random.shuffle(paths)
    dev_data_size = int(len(paths) * dev_proportion)
    train_paths = paths[:-dev_data_size]
    dev_paths = paths[-dev_data_size:]
    test_paths = read_paths(root, test_set)
    return train_paths, dev_paths, test_paths


def split(root, train_set, test_set, test_prop, seed):
    return P.split_libri(P.read_libri_paths(root, train_set), P.read_libri_paths(root, test_set), test_prop, seed)


@pytest.mark.parametrize("seed", [0, 1, 7, 1234])
@pytest.mark.parametrize("sizes", [(3, 4, 5), (1, 9, 2), (12, 7, 30)])
def test_split_equals_the_reference_algorithm(tmp_path, seed, sizes):
    root = str(tmp_path)
    a, b, c = sizes
    write_subset(root, "train-clean-100", {"103": {"1241": a, "1240": b}, "1034": {"121": c}, "19": {"198": a + b}})
    write_subset(root, "dev-clean", {"84": {"121123": b}, "174": {"50561": c}})
    for prop in (0.05, 0.1, 0.3):
        if int((2 * (a + b) + c) * prop) == 0:
            continue
        got = split(root, "train-clean-100", "dev-clean", prop, seed)
        assert got == reference_split(root, "train-clean-100", "dev-clean", prop, seed), (seed, sizes, prop)
        train, dev, test = got
        assert sorted(train + dev) == P.read_libri_paths(root, "train-clean-100")
        assert test == sorted(test) and len(test) == b + c          # sorted, not shuffled
        assert len(dev) == int(len(train + dev) * prop)


def test_listing_takes_only_wavs_three_levels_down(tmp_path):
    root = str(tmp_path)
    write_subset(root, "train-clean-100", {"103": {"1241": 2}, "19": {"198": 1}})
    decoys = ["train-clean-100/stray.wav", "train-clean-100/103/stray.wav", "train-clean-100/103/1241/x/deep.wav",
              "train-clean-100/103/1241/103_1241_000009_000000.flac", "other-subset/5/6/5_6_000000_000000.wav",
              "train-clean-100/103/1241/103_1241_000001_000002.wav.bak"]
    for d in decoys:
        touch(os.path.join(root, d))
    got = P.read_libri_paths(root, "train-clean-100")
    rel = [os.path.relpath(p, root) for p in got]
    assert rel == ["train-clean-100/103/1241/103_1241_000000_000001.wav",
                   "train-clean-100/103/1241/103_1241_000001_000002.wav",
                   "train-clean-100/19/198/19_198_000000_000001.wav"]


def test_no_dev_file_raises():
    paths = [f"/r/t/1/1/1_1_0_{i}.wav" for i in range(19)]
    with pytest.raises(ValueError, match="no dev file"):
        P.split_libri(paths, paths, 0.05, 0)            # int(19 * 0.05) == 0: the reference's train would be empty
    with pytest.raises(ValueError, match="no dev file"):
        P.split_libri([], paths, 0.5, 0)
    assert len(P.split_libri(paths + ["/r/t/1/1/1_1_0_x.wav"], paths, 0.05, 0)[1]) == 1


def test_duplicate_basename_raises():
    P.check_basenames("train", ["/r/a/1/1/1_1_0_0.wav", "/r/a/1/1/1_1_0_1.wav"])
    with pytest.raises(ValueError, match="two files named 1_1_0_0.wav"):
        P.check_basenames("test", ["/r/a/1/1/1_1_0_0.wav", "/r/a/1/2/1_1_0_1.wav", "/r/a/2/9/1_1_0_0.wav"])


def test_run_libri_rejects_bad_input_before_any_device_work(tmp_path, monkeypatch):
    def no_device(*a, **k):
        raise AssertionError("the Preparer was constructed")

    monkeypatch.setattr(P, "Preparer", no_device)
    root, out = str(tmp_path / "libri"), str(tmp_path / "out")
    write_subset(root, "train-clean-100", {"103": {"1241": 10}})
    write_subset(root, "dev-clean", {"84": {"121": 2}})
    with pytest.raises(ValueError, match="no dev file"):
        P.run_libri(root, out, test_prop=0.05, log=lambda *a: None)
    with pytest.raises(ValueError, match="dev-other"):
        P.run_libri(root, out, test_set="dev-other", test_prop=0.5, log=lambda *a: None)
    touch(os.path.join(root, "dev-clean", "84", "999", "84_121_000000_000001.wav"))   # same name, other chapter
    with pytest.raises(ValueError, match="test set holds two files named 84_121_000000_000001.wav"):
        P.run_libri(root, out, test_prop=0.5, log=lambda *a: None)
    with pytest.raises(ValueError, match="n_utts_attr"):
        P.run_libri(root, out, test_prop=0.5, n_utts_attr=0, log=lambda *a: None)


def test_cli_defaults_are_libri_config():
    a = preprocess_libri.parse_args(["/data/LibriTTS", "/data/out"])
    # libri.config, then the options shared with preprocess.py
    assert vars(a) == dict(root="/data/LibriTTS", out_dir="/data/out", train_set="train-clean-100",
                           test_set="dev-clean", test_prop=0.05, n_utts_attr=5000, training_samples=10000000,
                           testing_samples=10000, segment_size=128, n_mels=512, sample_rate=24000, seed=0, stage=0,
                           chunk_seconds=1800.0)


def test_speaker_of_a_libritts_utterance():
    assert E.speaker_of("103_1241_000000_000001.wav") == "103"
    assert E.speaker_of("1034_121_000000_000001") == "1034"
