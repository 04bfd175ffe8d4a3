"""CPU: the batch schedule of the device-resident corpus (seeded per-rank epoch orders, short last batch, resume),
the corpus validation, the device-path selection rule, and the avc_gather_desc layout."""
import ctypes
import os
import subprocess
import tempfile

import numpy as np
import pytest
import torch

from conftest import ROOT
from adaptive_voice_conversion_b200 import data_utils as D


# ----------------------------------------------------------------------------- order
def test_epoch_order_is_a_permutation():
    for rank, epoch in [(0, 0), (0, 7), (3, 1)]:
        o = D.epoch_order(1000, rank, epoch)
        assert o.dtype == torch.int64
        assert torch.equal(torch.sort(o).values, torch.arange(1000))


def test_orders_differ_across_ranks_and_epochs_and_repeat_for_the_same_pair():
    orders = {(r, e): D.epoch_order(500, r, e) for r in range(3) for e in range(3)}
    keys = list(orders)
    for i, a in enumerate(keys):
        for b in keys[i + 1:]:
            assert not torch.equal(orders[a], orders[b]), (a, b)
    assert torch.equal(D.epoch_order(500, 1, 2), orders[(1, 2)])
    assert len({D.order_seed(r, e) for r in range(8) for e in range(1000)}) == 8000


def test_epoch_order_is_the_documented_randperm():
    g = torch.Generator().manual_seed(D.order_seed(2, 5))
    assert torch.equal(D.epoch_order(300, 2, 5), torch.randperm(300, generator=g))


def test_no_shuffle_is_the_index_order():
    s = D.SegmentSampler(10, 4, rank=3, shuffle=False)
    assert [b.tolist() for b in (next(s) for _ in range(4))] == [[0, 1, 2, 3], [4, 5, 6, 7], [8, 9], [0, 1, 2, 3]]


def test_batch_sizes_across_epoch_boundaries():
    s = D.SegmentSampler(1000, 96)
    assert s.batches_per_epoch == 11
    sizes = [len(next(s)) for _ in range(25)]
    assert sizes == [96] * 10 + [40] + [96] * 10 + [40] + [96] * 3
    assert [s.locate(k) for k in (0, 10, 11, 22)] == [(0, 0, 96), (0, 960, 40), (1, 0, 96), (2, 0, 96)]
    # each epoch visits every entry exactly once
    s.seek(0)
    for epoch in range(2):
        seen = torch.cat([next(s) for _ in range(s.batches_per_epoch)])
        assert torch.equal(seen, D.epoch_order(1000, 0, epoch))
    exact = D.SegmentSampler(960, 96)
    assert exact.batches_per_epoch == 10 and all(len(next(exact)) == 96 for _ in range(30))


def test_seek_equals_stepping():
    for k in (0, 1, 10, 11, 12, 57):
        a, b = D.SegmentSampler(1000, 96, rank=1), D.SegmentSampler(1000, 96, rank=1)
        for _ in range(k):
            next(a)
        b.seek(k)
        assert a.position == b.position == k
        assert torch.equal(next(a), next(b))
    with pytest.raises(ValueError):
        D.SegmentSampler(10, 4).seek(-1)


def test_resumed_sequence_equals_uninterrupted():
    k, m = 17, 20
    full = D.SegmentSampler(1000, 96, rank=1)
    ref = [next(full) for _ in range(k + m)]
    first = D.SegmentSampler(1000, 96, rank=1)
    got = [next(first) for _ in range(k)]
    resumed = D.SegmentSampler(1000, 96, rank=1)     # a fresh process: nothing carried over but the position
    resumed.seek(k)
    got += [next(resumed) for _ in range(m)]
    assert all(torch.equal(a, b) for a, b in zip(ref, got)) and len(got) == len(ref)


# ----------------------------------------------------------------------------- validation
def _corpus(n_mels=8, lens=(20, 30, 25), dtype=np.float32):
    rng = np.random.default_rng(0)
    data = {f"p{i}": rng.standard_normal((T, n_mels)).astype(dtype) for i, T in enumerate(lens)}
    index = [[f"p{i}", t] for i, T in enumerate(lens) for t in range(0, T - 8 + 1, 3)]
    return data, index


def test_validation_accepts_a_good_corpus_and_computes_starts():
    data, index = _corpus()
    starts, n_mels, total = D.validate_corpus(data, index, 8, 1, 8)
    assert (n_mels, total) == (8, 75)
    off = {"p0": 0, "p1": 20, "p2": 50}
    assert starts.tolist() == [off[u] + t for u, t in index]
    data64, _ = _corpus(dtype=np.float64)
    assert D.validate_corpus(data64, index, 8, 1, 8)[1] == 8
    assert D.validate_corpus(data, index, 8, 2, 16)[1] == 8


@pytest.mark.parametrize("case, match", [
    ("missing_utterance", "index entry 2 .*'nobody' is not in the pickle"),
    ("t_negative", "index entry 1 .*t=-1"),
    ("t_past_end", "index entry 3 .*t=13 does not fit in the 20 frames of 'p0'"),
    ("ragged_n_mels", "utterance 'p1': 12 mels, but the first utterance has 8"),
    ("not_2d", "utterance 'p2': expected a 2-D"),
    ("c_in_mismatch", "n_mels 8 x frame_size 1 != c_in 80"),
    ("empty_index", "the index is empty"),
    ("empty_pickle", "no utterance"),
    ("seg_not_multiple_of_frame", "not a positive multiple of frame_size 3"),
    ("bad_entry", "index entry 0 .*expected \\(utt_id, t\\)"),
])
def test_validation_errors(case, match):
    data, index = _corpus()
    seg, frame, c_in = 8, 1, 8
    if case == "missing_utterance":
        index[2] = ["nobody", 0]
    elif case == "t_negative":
        index[1] = ["p0", -1]
    elif case == "t_past_end":
        index[3] = ["p0", 13]
    elif case == "ragged_n_mels":
        data["p1"] = np.zeros((30, 12), np.float32)
    elif case == "not_2d":
        data["p2"] = np.zeros((25, 8, 1), np.float32)
    elif case == "c_in_mismatch":
        c_in = 80
    elif case == "empty_index":
        index = []
    elif case == "empty_pickle":
        data = {}
    elif case == "seg_not_multiple_of_frame":
        frame, c_in = 3, 24
    elif case == "bad_entry":
        index[0] = ["p0"]
    with pytest.raises(ValueError, match=match):
        D.validate_corpus(data, index, seg, frame, c_in)


def test_t_at_the_last_crop_is_valid():
    data, _ = _corpus()
    starts, _, _ = D.validate_corpus(data, [["p0", 12], ["p2", 17], ["p0", 0]], 8, 1, 8)
    assert starts.tolist() == [12, 67, 0]


# ----------------------------------------------------------------------------- selection rule
def test_selection_rule_is_half_of_total_memory():
    assert D.corpus_device_bytes(1000, 80, 10) == 4 * 1000 * 80 + 12 * 10
    total = 80 * 10 ** 9
    # VCTK-sized at 512 mels (~16M frames, 10M entries): 33 GB + 120 MB <= 40 GB
    assert D.device_corpus_fits(16_000_000, 512, 10_000_000, total)
    assert not D.device_corpus_fits(20_000_000, 512, 10_000_000, total)
    n = D.corpus_device_bytes(1000, 80, 10)
    assert D.device_corpus_fits(1000, 80, 10, 2 * n) and D.device_corpus_fits(1000, 80, 10, 2 * n + 1)
    assert not D.device_corpus_fits(1000, 80, 10, 2 * n - 1)
    assert not D.device_corpus_fits(1000, 42, 10, total)     # rows the 16-byte gather cannot read


# ----------------------------------------------------------------------------- C ABI
def test_gather_desc_layout_matches_header():
    from adaptive_voice_conversion_b200 import _lib as L
    prog = ('#include <stdio.h>\n#include <stddef.h>\n#include "avc_b200.h"\nint main(){printf("%zu %zu %zu\\n", '
            'sizeof(avc_gather_desc), offsetof(avc_gather_desc, first), offsetof(avc_gather_desc, n_mels));return 0;}\n')
    with tempfile.TemporaryDirectory() as td:
        c = os.path.join(td, "s.c")
        with open(c, "w") as f:
            f.write(prog)
        exe = os.path.join(td, "s")
        subprocess.check_call(["gcc", "-I", os.path.join(ROOT, "include"), c, "-o", exe])
        sizes = [int(v) for v in subprocess.check_output([exe]).split()]
    assert sizes == [ctypes.sizeof(L.GatherDesc), L.GatherDesc.first.offset, L.GatherDesc.n_mels.offset]
