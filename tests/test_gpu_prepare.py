"""GPU: corpus preparation.  avc_resample_poly against float64 scipy.signal.resample_poly on the same PCM, the corpus
statistics against float64 numpy, and preprocess.py end to end on a seeded synthetic VCTK-shaped tree: its files, its
mels against the single-file vocoder path and the float64 oracle, its reproducibility across runs and chunk sizes, and
training and one-shot conversion from its output."""
import json
import os
import pickle
import subprocess
import sys
import types

import numpy as np
import pytest
import torch
from scipy.io import wavfile
from scipy.signal import resample_poly

import oracle.audio_oracle as ao
from adaptive_voice_conversion_b200 import _lib as L
from adaptive_voice_conversion_b200 import prepare as P
from adaptive_voice_conversion_b200 import vocoder as V
from conftest import ROOT

pytestmark = pytest.mark.gpu

SR = 24000
N_MELS = 80
RATES = [8000, 11025, 16000, 22050, 24000, 32000, 44100, 48000, 88200, 96000]


def stream():
    return torch.cuda.current_stream().cuda_stream


def bits(t):
    return np.ascontiguousarray(t).view(np.uint32)


# ------------------------------------------------------------------ resampler
def scaled_mono(data):
    y = V.scale_pcm(data)
    return y.mean(axis=1) if y.ndim == 2 else y


def pcm_case(rng, n, fmt, ch):
    if fmt == "s16":
        a = rng.integers(-32768, 32768, (n, ch) if ch > 1 else n).astype(np.int16)
    else:
        a = (0.5 * rng.standard_normal((n, ch) if ch > 1 else n)).astype(np.float32)
    return a


def test_resampler_matches_resample_poly_and_is_batch_invariant():
    prep = P.Preparer(N_MELS, SR)
    rng = np.random.default_rng(0)
    items = []
    for rate in RATES:
        up, down = P.rate_pair(rate, SR)
        half = 10 * max(up, down)
        for fmt in ("s16", "f32"):
            for ch in (1, 2):
                for n in sorted({5, max(1, half - 1), half + 1, 4801, 30011}):
                    items.append((rate, pcm_case(rng, n, fmt, ch)))
    got = [y.cpu().numpy() for y in prep.resample(items)]
    worst = (0.0, None)
    for (rate, a), y in zip(items, got):
        up, down = P.rate_pair(rate, SR)
        x = scaled_mono(a)
        ref = x if (up, down) == (1, 1) else resample_poly(x, up, down)
        assert y.dtype == np.float32 and y.shape == ref.shape, (rate, a.shape, y.shape, ref.shape)
        if (up, down) == (1, 1):
            r32 = ref.astype(np.float32)
            if a.dtype == np.int16 or a.ndim == 1:
                assert np.array_equal(y, r32), (rate, a.dtype, a.shape)   # conversion and a mono copy are exact
            else:
                assert (np.abs(y - r32) <= np.spacing(np.abs(r32))).all(), (rate, a.dtype, a.shape)
            continue
        err = float(np.abs(y - ref).max() / np.abs(x).max())
        if err > worst[0]:
            worst = (err, (rate, str(a.dtype), a.shape))
        assert err <= 5e-6, (rate, a.dtype, a.shape, err)
    print(f"resampler: worst max |error| / input peak {worst[0]:.2e} at {worst[1]}")
    # alone, each utterance gets the bits it gets in the batch
    for i in range(0, len(items), 7):
        alone = prep.resample([items[i]])[0].cpu().numpy()
        assert np.array_equal(bits(alone), bits(got[i])), items[i][0]


def test_resampler_rejects_invalid_arguments_and_tables_past_its_limits():
    lib = L.load()
    prep = P.Preparer(N_MELS, SR)
    half, n_taps, taps = prep.taps(1, 2)
    segs = torch.zeros(32, dtype=torch.uint8, device="cuda")
    pcm = torch.zeros(64, dtype=torch.int16, device="cuda")
    out = torch.zeros(64, device="cuda")
    good = dict(format=L.PCM_S16, up=1, down=2, half_len=half, n_taps=n_taps, n_seg=1, n_tiles=0, segs=segs.data_ptr(),
                pcm=pcm.data_ptr(), taps=taps.data_ptr(), out=out.data_ptr())
    assert lib.avc_resample_poly(L.ResampleDesc(**good), stream()) == L.OK
    invalid = [({"segs": None}, "null pointer"), ({"pcm": None}, "null pointer"), ({"out": None}, "null pointer"),
               ({"n_seg": 0}, "empty table"), ({"n_tiles": -1}, "empty table"), ({"format": 7}, "unknown format"),
               ({"up": 0}, "must be >= 1"), ({"down": -2}, "must be >= 1"), ({"taps": None}, "null tap table"),
               ({"half_len": half + 1}, "tap table"), ({"n_taps": n_taps - 1}, "tap table")]
    unsupported = [({"up": 5, "down": 64, "half_len": 640, "n_taps": 257}, "taps per phase"),
                   ({"up": 331, "down": 1638, "half_len": 16380, "n_taps": 99}, "taps per phase")]
    n0 = L.launch_count()
    for cases, code in ((invalid, L.ERR_INVALID), (unsupported, L.ERR_UNSUPPORTED)):
        for patch, msg in cases:
            assert lib.avc_resample_poly(L.ResampleDesc(**{**good, **patch}), stream()) == code, patch
            assert msg in L.last_error(), (patch, L.last_error())
    assert lib.avc_resample_poly(None, stream()) == L.ERR_INVALID and "null descriptor" in L.last_error()
    assert L.launch_count() == n0


# ------------------------------------------------------------------ corpus statistics
def ragged_mels(seed, n_utt=9):
    rng = np.random.default_rng(seed)
    return [(0.3 + 0.4 * rng.random((int(rng.integers(1, 700)), N_MELS))).astype(np.float32) for _ in range(n_utt)]


def moments_of(prep, chunks):
    """(mean, std, mean64, std64) over the utterances fed in the given chunks, and the raw moments buffer."""
    counts = [m.shape[0] for c in chunks for m in c]
    mom = torch.full((len(counts), N_MELS, 2), float("nan"), dtype=torch.float64, device="cuda")
    first = 0
    for c in chunks:
        M = torch.from_numpy(np.concatenate(c)).cuda()
        prep.moments(M, [m.shape[0] for m in c], mom, first)
        first += len(c)
    return prep.merge(mom, counts), mom.cpu().numpy()


def test_moments_match_numpy_and_do_not_depend_on_chunking():
    prep = P.Preparer(N_MELS, SR)
    mels = ragged_mels(1)
    (mean, std, mean64, std64), mom = moments_of(prep, [mels])
    cat = np.concatenate(mels).astype(np.float64)
    rmean, rstd = cat.mean(axis=0), cat.std(axis=0)
    assert mean.dtype == np.float32 and std.dtype == np.float32 and mean.shape == (N_MELS,)
    for got, ref in ((mean, rmean), (std, rstd)):
        r32 = ref.astype(np.float32)
        assert (np.abs(got - r32) <= np.spacing(r32)).all(), np.abs(got - r32).max()
    assert np.abs(mean64 - rmean).max() <= 1e-12 and np.abs(std64 - rstd).max() <= 1e-12
    for u, m in enumerate(mels):
        a = m.astype(np.float64)
        assert np.allclose(mom[u, :, 0], a.mean(axis=0), rtol=0, atol=1e-13)
        assert np.allclose(mom[u, :, 1], ((a - a.mean(axis=0)) ** 2).sum(axis=0), rtol=1e-12, atol=1e-12)
    (m2, s2, m2_64, s2_64), mom2 = moments_of(prep, [[m] for m in mels])
    (m3, s3, _, _), _ = moments_of(prep, [mels[:4], mels[4:]])
    assert np.array_equal(mom.view(np.uint64), mom2.view(np.uint64))
    for a, b in ((mean, m2), (std, s2), (mean, m3), (std, s3)):
        assert np.array_equal(bits(a), bits(b))
    assert np.array_equal(mean64.view(np.uint64), m2_64.view(np.uint64))


def test_moments_reject_invalid_arguments():
    lib = L.load()
    segs = torch.zeros(24, dtype=torch.uint8, device="cuda")
    mels = torch.zeros(N_MELS, device="cuda")
    mom = torch.zeros(N_MELS * 2, dtype=torch.float64, device="cuda")
    good = dict(n_mels=N_MELS, n_seg=1, first=0, segs=segs.data_ptr(), mels=mels.data_ptr(), moments=mom.data_ptr())
    n0 = L.launch_count()
    for patch, msg in [({"segs": None}, "null pointer"), ({"mels": None}, "null pointer"), ({"moments": None}, "null pointer"),
                       ({"n_seg": 0}, "bad shape"), ({"n_mels": 0}, "bad shape"), ({"first": -1}, "bad shape")]:
        assert lib.avc_mel_moments(L.MomentsDesc(**{**good, **patch}), stream()) == L.ERR_INVALID, patch
        assert msg in L.last_error(), (patch, L.last_error())
    assert lib.avc_mel_moments(None, stream()) == L.ERR_INVALID and "null descriptor" in L.last_error()
    cnt = torch.ones(1, dtype=torch.int32, device="cuda")
    o32, o64 = torch.zeros(N_MELS, device="cuda"), torch.zeros(N_MELS, dtype=torch.float64, device="cuda")
    args = [mom.data_ptr(), cnt.data_ptr(), 1, N_MELS, o32.data_ptr(), o32.data_ptr(), o64.data_ptr(), o64.data_ptr()]
    for i, v, msg in [(0, None, "null pointer"), (1, None, "null pointer"), (4, None, "null pointer"),
                      (7, None, "null pointer"), (2, 0, "bad shape"), (3, 0, "bad shape")]:
        a = list(args)
        a[i] = v
        assert lib.avc_mel_moments_merge(*a, stream()) == L.ERR_INVALID, i
        assert msg in L.last_error(), (i, L.last_error())
    assert L.launch_count() == n0


# ------------------------------------------------------------------ the whole pipeline on a synthetic tree
def utterance(rng, sr, seconds, silence=(0.3, 0.4)):
    n = int(sr * seconds)
    t = np.arange(n) / sr
    f0 = rng.uniform(110, 220) * (1 + 0.03 * np.sin(2 * np.pi * rng.uniform(4, 6) * t))
    ph = 2 * np.pi * np.cumsum(f0) / sr
    y = sum(rng.uniform(0.05, 0.25) / k * np.sin(k * ph + rng.uniform(0, 6.3)) for k in range(1, 7))
    a, b = n // 3, n // 3 + n // 8
    y[a:b] += 0.1 * rng.standard_normal(b - a)
    y += 0.01 * rng.standard_normal(n)   # a noise floor: no mel bin is constant over a segment, as in recorded speech
    return np.concatenate([np.zeros(int(silence[0] * sr)), y, np.zeros(int(silence[1] * sr))])


def to_s16(y):
    return np.round(np.clip(y, -1, 1 - 2 ** -15) * 32768).astype(np.int16)


SPEAKERS = ["225", "226", "227", "228", "229", "230"]
SPECIAL = {"p225_901.wav": 44100, "p226_902.wav": 24000, "p227_903.wav": 0}   # 0: all silent, 48 kHz


def write_tree(root):
    rng = np.random.default_rng(2024)
    wav = os.path.join(root, "wav48")
    for spk in SPEAKERS:
        os.makedirs(os.path.join(wav, f"p{spk}"))
        for i in range(4):
            y = utterance(rng, 48000, rng.uniform(2.0, 4.0))
            wavfile.write(os.path.join(wav, f"p{spk}", f"p{spk}_{i + 1:03d}.wav"), 48000, to_s16(y))
    for name, rate in SPECIAL.items():
        path = os.path.join(wav, f"p{name[1:4]}", name)
        if rate == 44100:
            y = utterance(rng, rate, 2.5)
            wavfile.write(path, rate, to_s16(np.stack([y, 0.5 * y], axis=1)))
        elif rate == 24000:
            wavfile.write(path, rate, to_s16(utterance(rng, rate, 3.0)))
        else:
            wavfile.write(path, 48000, np.zeros(96000, np.int16))
    info = os.path.join(root, "speaker-info.txt")
    with open(info, "w") as f:
        f.write("ID  AGE  GENDER  ACCENTS  REGION\n")
        f.writelines(f"{s}  23  F  English  Somewhere\n" for s in SPEAKERS)
    return wav, info


OPTS = dict(n_out_speakers=2, test_prop=0.25, n_utts_attr=10, n_mels=N_MELS, segment_size=128, training_samples=300,
            testing_samples=40, seed=3)
FILES = ["attr.pkl", "train.pkl", "in_test.pkl", "out_test.pkl", "train_128.pkl", "train_samples_128.json",
         "in_test_samples_128.json", "out_test_samples_128.json", "in_test_files.txt", "out_test_files.txt",
         "skipped_files.txt"]


@pytest.fixture(scope="module")
def tree(tmp_path_factory):
    root = tmp_path_factory.mktemp("vctk")
    wav, info = write_tree(str(root))
    out = str(root / "cli")
    cmd = [sys.executable, os.path.join(ROOT, "preprocess.py"), wav, info, out]
    for k, v in OPTS.items():
        cmd += [f"--{k}", str(v)]
    r = subprocess.run(cmd, capture_output=True, text=True, cwd=str(root))
    assert r.returncode == 0, r.stdout + r.stderr
    print(r.stdout)
    return types.SimpleNamespace(root=root, wav=wav, info=info, out=out, stdout=r.stdout)


def load(path):
    with open(path, "rb") as f:
        return pickle.load(f)


def test_preprocess_writes_the_reference_files(tree):
    assert sorted(os.listdir(tree.out)) == sorted(FILES)
    attr = load(os.path.join(tree.out, "attr.pkl"))
    assert set(attr) == {"mean", "std"}
    assert all(v.dtype == np.float32 and v.shape == (N_MELS,) for v in attr.values())
    skipped = open(os.path.join(tree.out, "skipped_files.txt")).read().splitlines()
    assert len(skipped) == 1 and skipped[0].split("\t")[0].endswith("p227_903.wav") and "silent" in skipped[0]
    assert "1 files skipped" in tree.stdout
    s2f = P.read_filenames(tree.wav)
    sets = dict(zip(P.SETS, P.split_files(P.read_speaker_info(tree.info), s2f, 2, 0.25, 3)))
    for name in ("in_test", "out_test"):
        assert open(os.path.join(tree.out, f"{name}_files.txt")).read().splitlines() == sets[name]
    for name in P.SETS:
        data = load(os.path.join(tree.out, f"{name}.pkl"))
        expect = [os.path.basename(p) for p in sorted(sets[name]) if not p.endswith("p227_903.wav")]
        assert list(data) == expect, name
        assert all(v.dtype == np.float32 and v.ndim == 2 and v.shape[1] == N_MELS for v in data.values())
        index = json.load(open(os.path.join(tree.out, f"{name}_samples_128.json")))
        assert len(index) == (300 if name == "train" else 40)
        assert all(data[u].shape[0] > 128 and 0 <= t <= data[u].shape[0] - 128 for u, t in index)
        assert index == [list(e) for e in P.sample_segments(data, len(index), 128, 3)]
    train = load(os.path.join(tree.out, "train.pkl"))
    reduced = load(os.path.join(tree.out, "train_128.pkl"))
    assert list(reduced) == [k for k, v in train.items() if v.shape[0] > 128] and len(reduced) >= len(train) - 1


def test_mels_equal_the_single_file_paths_and_track_the_oracle(tree):
    attr = load(os.path.join(tree.out, "attr.pkl"))
    mean, std = attr["mean"], attr["std"]
    data = {}
    for name in P.SETS:
        data.update(load(os.path.join(tree.out, f"{name}.pkl")))
    voc = V.Vocoder(n_mels=N_MELS)
    prep = P.Preparer(N_MELS, SR)
    p24 = os.path.join(tree.wav, "p226", "p226_902.wav")
    assert np.array_equal(bits(data["p226_902.wav"]), bits((voc.get_spectrograms(p24)[0] - mean) / std))
    fb = ao.mel_filterbank(SR, 2048, N_MELS)
    worst = 0.0
    for spk in SPEAKERS:
        for i in range(4):
            name = f"p{spk}_{i + 1:03d}.wav"
            rate, pcm = V.read_pcm(os.path.join(tree.wav, f"p{spk}", name))
            y = prep.resample([(rate, pcm)])[0]
            raw = voc.wav_to_mel([y])[0][0].cpu().numpy()
            assert np.array_equal(bits(data[name]), bits((raw - mean) / std)), name
            x = resample_poly(pcm / 32768.0, 1, 2)
            rlin = np.abs(ao.stft(ao.preemphasis(ao.trim(x, 15)))) @ fb.T
            assert raw.shape == rlin.shape, (name, raw.shape, rlin.shape)
            loud = rlin >= 1e-3 * np.maximum(rlin.max(axis=1, keepdims=True), 1e-5)
            err = float(np.abs(raw - ao.normalize_db(rlin))[loud].max())
            worst = max(worst, err)
            assert err < 1e-5, (name, err)
    print(f"pipeline mels vs float64 oracle within 60 dB of the frame peak: worst {worst:.2e}")


def test_output_is_reproducible_across_runs_and_chunk_sizes(tree):
    outs = []
    for tag, chunk in (("same", 1800.0), ("per_file", 0.001)):
        out = str(tree.root / f"run_{tag}")
        P.run(tree.wav, tree.info, out, chunk_seconds=chunk, log=lambda *a: None, **OPTS)
        outs.append(out)
    for f in FILES:
        ref = open(os.path.join(tree.out, f), "rb").read()
        for out in outs:
            assert open(os.path.join(out, f), "rb").read() == ref, (out, f)


def test_training_and_conversion_from_the_prepared_directory(tree, tmp_path):
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
    src = os.path.join(tree.wav, "p226", "p226_902.wav")
    tgt = os.path.join(tree.wav, "p228", "p228_001.wav")
    out = str(tmp_path / "out.wav")
    r = subprocess.run([sys.executable, os.path.join(ROOT, "inference.py"), "-c", f"{store}.config.yaml", "-m",
                        f"{store}.ckpt", "-a", os.path.join(tree.out, "attr.pkl"), "-s", src, "-t", tgt, "-o", out],
                       capture_output=True, text=True, cwd=str(tmp_path))
    assert r.returncode == 0, r.stdout + r.stderr
    rate, wav = wavfile.read(out)
    assert rate == SR and wav.size > 0 and np.isfinite(wav).all()
