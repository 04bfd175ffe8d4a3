"""CPU: the host half of corpus preparation (prepare.py) against restatements of the reference's scripts
(preprocess/make_datasets_vctk.py, reduce_dataset.py, sample_single_segments.py), the resampler's tap table and index
arithmetic against scipy.signal.resample_poly, the chunk planner, the struct layouts and the kernels' resources."""
import ctypes
import os
import random
import re
import subprocess
import tempfile
from collections import defaultdict

import numpy as np
import pytest
from scipy.signal import firwin, resample_poly

from adaptive_voice_conversion_b200 import _lib as L
from adaptive_voice_conversion_b200 import prepare as P
from conftest import ROOT

# the file rates a user meets, each to every target rate --sample_rate is meant for
RATES = [8000, 11025, 12000, 16000, 22050, 24000, 32000, 44100, 48000, 88200, 96000, 176400, 192000]
TARGETS = [16000, 22050, 24000, 44100, 48000]


def write_tree(root, speakers):
    for spk, n in speakers.items():
        d = os.path.join(root, f"p{spk}")
        os.makedirs(d, exist_ok=True)
        for i in range(n):
            open(os.path.join(d, f"p{spk}_{i + 1:03d}.wav"), "wb").close()


def test_speaker_info_skips_the_header(tmp_path):
    p = tmp_path / "speaker-info.txt"
    p.write_text("ID  AGE  GENDER  ACCENTS  REGION\n225  23  F    English    Southern  England\n226  22  M  English\n")
    assert P.read_speaker_info(str(p)) == ["225", "226"]


def test_file_listing_groups_by_speaker_in_sorted_order(tmp_path):
    write_tree(str(tmp_path), {"226": 3, "225": 2})
    got = P.read_filenames(str(tmp_path))
    assert sorted(got) == ["225", "226"]
    assert [os.path.basename(p) for p in got["226"]] == ["p226_001.wav", "p226_002.wav", "p226_003.wav"]
    assert got["999"] == []          # a speaker of speaker-info without files


def test_file_listing_names_a_file_that_does_not_match(tmp_path):
    write_tree(str(tmp_path), {"225": 2})
    bad = tmp_path / "p225" / "readme.txt"
    bad.write_text("x")
    with pytest.raises(ValueError, match=re.escape(str(bad))):
        P.read_filenames(str(tmp_path))


def reference_split(speaker_ids, speaker2filenames, test_speakers, test_proportion, seed):
    """make_datasets_vctk.py:49-76 as written, on the module-level random after random.seed(seed)."""
    random.seed(seed)
    speaker_ids = list(speaker_ids)
    speaker2filenames = defaultdict(lambda: [], {k: list(v) for k, v in speaker2filenames.items()})
    random.shuffle(speaker_ids)
    train_speaker_ids = speaker_ids[:-test_speakers]
    test_speaker_ids = speaker_ids[-test_speakers:]
    train_path_list, in_test_path_list, out_test_path_list = [], [], []
    for speaker in train_speaker_ids:
        path_list = speaker2filenames[speaker]
        random.shuffle(path_list)
        test_data_size = int(len(path_list) * test_proportion)
        train_path_list += path_list[:-test_data_size]
        in_test_path_list += path_list[-test_data_size:]
    for speaker in test_speaker_ids:
        out_test_path_list += speaker2filenames[speaker]
    return train_path_list, in_test_path_list, out_test_path_list


@pytest.mark.parametrize("seed", [0, 1, 7, 1234])
def test_split_equals_the_reference_algorithm(tmp_path, seed):
    # speaker 230 has 5 files: int(5 * 0.1) == 0 sends all of them to in_test, as the reference does
    counts = {"225": 31, "226": 12, "227": 20, "228": 40, "229": 17, "230": 5, "231": 25, "232": 11}
    write_tree(str(tmp_path), counts)
    s2f = P.read_filenames(str(tmp_path))
    ids = list(counts) + ["240"]     # 240: listed in speaker-info, no files
    got = P.split_files(ids, s2f, 3, 0.1, seed)
    assert got == reference_split(ids, s2f, 3, 0.1, seed)
    train, in_test, out_test = got
    assert sorted(train + in_test + out_test) == sorted(p for v in s2f.values() for p in v)


def test_split_sends_every_file_of_a_small_speaker_to_in_test(tmp_path):
    write_tree(str(tmp_path), {"225": 5, "226": 5})
    s2f = P.read_filenames(str(tmp_path))
    for seed in range(5):
        train, in_test, out_test = P.split_files(["225", "226"], s2f, 1, 0.1, seed)
        assert train == [] and len(in_test) == 5 and len(out_test) == 5


def reference_samples(data, n_samples, segment_size, seed):
    """sample_single_segments.py:16-30 after random.seed(seed)."""
    random.seed(seed)
    samples = []
    utt_list = sorted(list(filter(lambda u: len(data[u]) > segment_size, [key for key in data])))
    for utt_ind in random.choices(range(len(utt_list)), k=n_samples):
        utt_id = utt_list[utt_ind]
        samples.append((utt_id, random.randint(0, len(data[utt_id]) - segment_size)))
    return samples


def toy_data(seed, n=40):
    rng = np.random.default_rng(seed)
    return {f"p{225 + i % 7}_{i:03d}.wav": np.zeros((int(rng.integers(60, 400)), 4), np.float32) for i in range(n)}


@pytest.mark.parametrize("seed", [0, 3, 99])
def test_index_sampling_equals_the_reference_algorithm(seed):
    data = toy_data(seed)
    assert P.sample_segments(data, 500, 128, seed) == reference_samples(data, 500, 128, seed)


def test_reduce_keeps_exactly_the_utterances_longer_than_the_segment():
    data = {"a": np.zeros((128, 2)), "b": np.zeros((129, 2)), "c": np.zeros((127, 2)), "d": np.zeros((400, 2))}
    assert list(P.reduce_set(data, 128)) == ["b", "d"]


def test_index_sampling_of_a_set_without_long_utterances_raises():
    with pytest.raises(ValueError, match="segment_size"):
        P.sample_segments({"a": np.zeros((128, 2))}, 10, 128, 0)


# ------------------------------------------------------------------ resampler
def pairs():
    return sorted({P.rate_pair(r, sr) for r in RATES for sr in TARGETS} - {(1, 1)})


def test_supported_rates_fit_the_kernel_limits():
    for up, down in pairs():
        half, tab = P.resample_taps(up, down)
        assert tab.shape[1] <= L.RESAMPLE_MAX_PHASE_TAPS and tab.size <= L.RESAMPLE_MAX_TAPS, (up, down, tab.shape)
        assert P.resample_supported(up, down)
    assert max(P.resample_taps(*p)[1].size for p in pairs()) == 25725          # 192 kHz -> 22.05 kHz
    assert max(P.resample_taps(*p)[1].shape[1] for p in pairs()) == 241        # 192 kHz -> 16 kHz


# (up, down) whose tap table is exactly at a limit, and one past it
LIMIT_PAIRS = {(4, 51): (256, 1024), (128, 1633): (256, 32768), (5, 64): (257, 1285), (331, 1638): (99, 32769)}


@pytest.mark.parametrize("up, down", sorted(LIMIT_PAIRS))
def test_limit_pairs_have_the_tables_they_are_meant_to(up, down):
    half, tab = P.resample_taps(up, down)
    assert tab.shape[1::-1] == LIMIT_PAIRS[(up, down)][:1] + (up,) and tab.size == LIMIT_PAIRS[(up, down)][1]
    fits = tab.shape[1] <= L.RESAMPLE_MAX_PHASE_TAPS and tab.size <= L.RESAMPLE_MAX_TAPS
    assert P.resample_supported(up, down) == fits == ((up, down) in ((4, 51), (128, 1633)))


def test_a_refused_rate_stops_the_run_before_any_set_is_analysed(tmp_path):
    """44 056 Hz to 16 kHz is up 2000 / down 5507: 56 taps per phase, 112 000 in all.  The file is in out_test, the
    last set processed; the run must name it before it analyses the training set."""
    from scipy.io import wavfile
    wav = tmp_path / "wav"
    for spk in ("225", "226", "227"):
        os.makedirs(wav / f"p{spk}")
        for i in range(3):
            wavfile.write(str(wav / f"p{spk}" / f"p{spk}_{i + 1:03d}.wav"), 48000, np.zeros(4800, np.int16))
    info = tmp_path / "speaker-info.txt"
    info.write_text("ID  AGE\n225  23\n226  22\n227  21\n")
    out = tmp_path / "out"
    train, _, out_test = P.split_files(["225", "226", "227"], P.read_filenames(str(wav)), 1, 0.34, 0)
    bad = sorted(out_test)[-1]
    wavfile.write(bad, 44056, np.zeros(4800, np.int16))
    with pytest.raises(ValueError, match=re.escape(bad) + ".*44056 Hz.*--sample_rate 16000"):
        P.run(str(wav), str(info), str(out), n_out_speakers=1, test_prop=0.34, sample_rate=16000, log=lambda *a: None)
    assert not [f for f in os.listdir(out) if f.endswith(".pkl")]
    assert not P.resample_supported(*P.rate_pair(44056, 16000))


@pytest.mark.parametrize("up, down", pairs())
def test_tap_table_is_the_firwin_filter_in_polyphase_order(up, down):
    half, tab = P.resample_taps(up, down)
    mx = max(up, down)
    h = firwin(2 * 10 * mx + 1, 1.0 / mx, window=("kaiser", 5.0)) * up
    assert half == 10 * mx and tab.shape == (up, -(-h.size // up))
    for r in range(up):
        n = len(h[r::up])
        assert np.array_equal(tab[r, :n], h[r::up]) and not tab[r, n:].any()


def kernel_restatement(x, up, down):
    """csrc/prep.cu resample_poly_kernel in float64: tiles of RESAMPLE_TILE outputs, a zero-padded window per tile,
    per output the phase r and newest sample k, and the dot product over i < cnt."""
    half, tab = P.resample_taps(up, down)
    n_taps = tab.shape[1]
    n_out = P.n_resampled(len(x), up, down)
    y = np.zeros(n_out)
    for m0 in range(0, n_out, L.RESAMPLE_TILE):
        m1 = min(n_out, m0 + L.RESAMPLE_TILE)
        kw0 = (m0 * down + half) // up - (n_taps - 1)
        nw = ((m1 - 1) * down + half) // up - kw0 + 1
        assert nw <= (L.RESAMPLE_TILE - 1) * down // up + n_taps + 1
        k = np.arange(kw0, kw0 + nw)
        win = np.where((k >= 0) & (k < len(x)), x[np.clip(k, 0, max(len(x) - 1, 0))] if len(x) else 0.0, 0.0)
        for m in range(m0, m1):
            p = m * down + half
            r, kk = p % up, p // up - kw0
            cnt = (2 * half - r) // up + 1
            assert cnt <= n_taps and kk - (cnt - 1) >= 0 and kk < nw
            y[m] = np.dot(win[kk - np.arange(cnt)], tab[r, :cnt])
    return y


@pytest.mark.parametrize("up, down", pairs())
def test_kernel_index_arithmetic_equals_resample_poly(up, down):
    half = 10 * max(up, down)
    rng = np.random.default_rng(up * 1000 + down)
    for n in sorted({1, 5, half - 1, half + 1, 4801}):
        x = rng.standard_normal(n)
        ref = resample_poly(x, up, down)
        got = kernel_restatement(x, up, down)
        assert got.shape == ref.shape, (n, got.shape, ref.shape)
        assert np.abs(got - ref).max() <= 1e-12, (up, down, n, np.abs(got - ref).max())


def test_chunk_planner_keeps_files_whole_and_within_budget():
    rng = np.random.default_rng(0)
    lengths = [int(v) for v in rng.integers(1, 5000, 300)] + [20000] + [int(v) for v in rng.integers(1, 5000, 50)]
    for budget in (1, 4999, 10000, 123456, 10 ** 9):
        chunks = P.plan_chunks(lengths, budget)
        assert [i for c in chunks for i in c] == list(range(len(lengths)))   # every file once, in order, never split
        for c in chunks:
            total = sum(lengths[i] for i in c)
            assert total <= budget or len(c) == 1, (budget, c)
        for a, b in zip(chunks, chunks[1:]):   # greedy: the next file would not have fit
            assert sum(lengths[i] for i in a) + lengths[b[0]] > budget


def test_chunk_planner_never_reaches_two_to_the_31():
    big = 2 ** 30
    chunks = P.plan_chunks([big, big, big, 5], 10 ** 12)
    assert all(sum([big, big, big, 5][i] for i in c) < 2 ** 31 for c in chunks)
    assert chunks == [[0], [1], [2, 3]]
    with pytest.raises(ValueError, match="ragged batch"):
        P.plan_chunks([2 ** 31], 10 ** 12)


# ------------------------------------------------------------------ ABI and resources
def test_prep_struct_layouts_match_gcc():
    prog = ('#include <stdio.h>\n#include "avc_b200.h"\nint main(){printf("%zu %zu %zu %d %d %d\\n", '
            'sizeof(avc_resample_seg), sizeof(avc_resample_desc), sizeof(avc_moments_desc), AVC_RESAMPLE_TILE, '
            'AVC_RESAMPLE_MAX_TAPS, AVC_RESAMPLE_MAX_PHASE_TAPS);return 0;}\n')
    with tempfile.TemporaryDirectory() as td:
        c = os.path.join(td, "s.c")
        open(c, "w").write(prog)
        exe = os.path.join(td, "s")
        subprocess.check_call(["gcc", "-I", os.path.join(ROOT, "include"), c, "-o", exe])
        got = [int(v) for v in subprocess.check_output([exe]).split()]
    assert got == [ctypes.sizeof(L.ResampleSeg), ctypes.sizeof(L.ResampleDesc), ctypes.sizeof(L.MomentsDesc),
                   L.RESAMPLE_TILE, L.RESAMPLE_MAX_TAPS, L.RESAMPLE_MAX_PHASE_TAPS]


def test_prep_kernels_have_no_stack_or_local_memory():
    L.load()
    out = subprocess.run(["cuobjdump", "-res-usage", L.LIB_PATH], capture_output=True, text=True).stdout
    res, fn = {}, None
    for line in out.splitlines():
        m = re.match(r"\s*Function (\S+):", line)
        if m:
            fn = m.group(1)
        elif fn and "REG:" in line and any(k in fn for k in ("resample_poly_kernel", "mel_moments_kernel",
                                                               "moments_merge_kernel")):
            res[fn] = {k: int(v) for k, v in re.findall(r"(\w+):(\d+)", line)}
    assert len(res) == 4, sorted(res)   # S16 and F32 resamplers, moments, merge
    for fn, r in res.items():
        assert r["STACK"] == 0 and r["LOCAL"] == 0, (fn, r)


def test_normalise_is_the_reference_expression_in_place():
    rng = np.random.default_rng(4)
    data = {f"u{i}": rng.random((50 + i, 8)).astype(np.float32) for i in range(3)}
    mean, std = rng.random(8).astype(np.float32), (0.5 + rng.random(8)).astype(np.float32)
    ref = {k: (v - mean) / std for k, v in data.items()}
    out = P.normalise(data, mean, std)
    assert out is data and list(out) == list(ref)
    assert all(v.dtype == np.float32 and np.array_equal(v.view(np.uint32), ref[k].view(np.uint32)) for k, v in out.items())
