"""The training data of Solver.  ``PickleDataset`` / ``get_data_loader`` read the reference's
pickle + index-json formats (data_utils.py:43-57, 10-28) with the stock DataLoader;
``DeviceSegments`` keeps the same corpus in HBM and cuts every batch on the GPU
(``avc_segment_gather``, csrc/corpus.cu), in the seeded order ``SegmentSampler`` defines; and
``SyntheticSegments`` provides the N(0,1) segments BASELINE.json benchmarks on.
"""
from __future__ import annotations

import json
import pickle

import numpy as np
import torch
from torch.utils.data import DataLoader, Dataset

from . import _lib as L
from .engine import decoder_length
from .utils import local_device


def load_corpus(pickle_path, sample_index_path):
    """({utt_id: [T, n_mels] array}, [(utt_id, t), ...]) as the reference's preprocessing writes them."""
    with open(pickle_path, "rb") as f:
        data = pickle.load(f)
    with open(sample_index_path) as f:
        indexes = json.load(f)
    return data, indexes


class PickleDataset(Dataset):
    """(utt_id, t) index over a dict of [T, n_mels] arrays -> [segment_size, n_mels] crops."""

    def __init__(self, pickle_path, sample_index_path, segment_size):
        self.data, self.indexes = load_corpus(pickle_path, sample_index_path)
        self.segment_size = segment_size

    @classmethod
    def from_loaded(cls, data, indexes, segment_size):
        """The same dataset over a pickle and an index already in memory."""
        self = cls.__new__(cls)
        self.data, self.indexes, self.segment_size = data, indexes, segment_size
        return self

    def __len__(self):
        return len(self.indexes)

    def __getitem__(self, i):
        utt, t = self.indexes[i]
        return self.data[utt][t:t + self.segment_size]


class CollateFn:
    """[B, T, n_mels] crops -> [B, n_mels*frame_size, T/frame_size] (data_utils.py:10-22)."""

    def __init__(self, frame_size):
        self.frame_size = frame_size

    def __call__(self, items):
        t = torch.from_numpy(np.asarray(items, dtype=np.float32))
        b, n, m = t.shape
        return t.reshape(b, n // self.frame_size, self.frame_size * m).transpose(1, 2).contiguous()


def get_data_loader(dataset, batch_size, frame_size, shuffle=True, num_workers=4, drop_last=False):
    return DataLoader(dataset, batch_size=batch_size, shuffle=shuffle, num_workers=num_workers,
                      collate_fn=CollateFn(frame_size), pin_memory=True, drop_last=drop_last)


# ----------------------------------------------------------------------------- device-resident corpus
_M64 = (1 << 64) - 1


def order_seed(rank: int, epoch: int) -> int:
    """Seed of the shuffle of (rank, epoch): splitmix64's finaliser applied to rank * 2**32 + epoch.  The finaliser
    is a bijection of 64-bit words, so distinct (rank, epoch) pairs (both below 2**32) get distinct seeds."""
    z = ((rank << 32) + epoch + 0x9E3779B97F4A7C15) & _M64
    z = ((z ^ (z >> 30)) * 0xBF58476D1CE4E5B9) & _M64
    z = ((z ^ (z >> 27)) * 0x94D049BB133111EB) & _M64
    return z ^ (z >> 31)


def epoch_order(n: int, rank: int, epoch: int, shuffle: bool = True, seed: int = 0) -> torch.Tensor:
    """The order in which rank `rank` visits the n index entries in epoch `epoch` (int64, on the host): a pure
    function of (rank, epoch, seed), so a resumed run draws the same orders again; the index order when not shuffling.
    seed 0 is the training run's order; another seed (speaker adaptation's -seed) XORs seed * 0x9E3779B97F4A7C15
    (mod 2^64, distinct for distinct seeds below 2^64) into the shuffle's generator seed."""
    if not shuffle:
        return torch.arange(n, dtype=torch.int64)
    s = order_seed(rank, epoch) ^ ((seed * 0x9E3779B97F4A7C15) & _M64)
    return torch.randperm(n, generator=torch.Generator().manual_seed(s))


class SegmentSampler:
    """The batch schedule of a run over n index entries: batch k of the run is batch k mod ceil(n/B) of epoch
    k div ceil(n/B).  Every entry is visited once per epoch, in ``epoch_order``; the last batch of an epoch is short
    when B does not divide n (the loader's drop_last=False).  Iterating yields the entries of each batch.

    drop_last=True (speaker adaptation): every batch has exactly B entries; an epoch is its order's first
    floor(n/B) * B entries, the rest of that epoch's order is not visited (B <= n is required)."""

    def __init__(self, n: int, batch_size: int, rank: int = 0, shuffle: bool = True, seed: int = 0,
                 drop_last: bool = False):
        if n < 1 or batch_size < 1:
            raise ValueError(f"SegmentSampler: need n >= 1 and batch_size >= 1 (got n={n}, batch_size={batch_size})")
        if drop_last and batch_size > n:
            raise ValueError(f"SegmentSampler: drop_last needs batch_size <= n (got n={n}, batch_size={batch_size})")
        self.n, self.batch_size, self.rank, self.shuffle, self.seed = n, batch_size, rank, shuffle, seed
        self.batches_per_epoch = n // batch_size if drop_last else -(-n // batch_size)
        self.position = 0          # batches handed out so far
        self._cached = (None, None)

    def seek(self, k: int):
        """Position the schedule at batch k of the run (k batches done)."""
        if k < 0:
            raise ValueError(f"SegmentSampler.seek: negative position {k}")
        self.position = int(k)

    def locate(self, k: int):
        """(epoch, first position in that epoch's order, entries) of batch k of the run."""
        epoch, j = divmod(k, self.batches_per_epoch)
        first = j * self.batch_size
        return epoch, first, min(self.batch_size, self.n - first)

    def order(self, epoch: int) -> torch.Tensor:
        if self._cached[0] != epoch:
            self._cached = (epoch, epoch_order(self.n, self.rank, epoch, self.shuffle, self.seed))
        return self._cached[1]

    def step(self):
        """locate() of the current position, then advance by one batch."""
        loc = self.locate(self.position)
        self.position += 1
        return loc

    def __iter__(self):
        return self

    def __next__(self) -> torch.Tensor:
        epoch, first, count = self.step()
        return self.order(epoch)[first:first + count]


def corpus_device_bytes(total_frames: int, n_mels: int, n_entries: int) -> int:
    """HBM DeviceSegments holds: the fp32 frames, the int64 start table and one int32 epoch order."""
    return 4 * total_frames * n_mels + 8 * n_entries + 4 * n_entries


def device_corpus_fits(total_frames: int, n_mels: int, n_entries: int, total_memory: int) -> bool:
    """Whether Solver trains from the device-resident corpus: its frames, starts and one epoch order take at most
    half of the device's total memory (the training step itself needs a few GB at the shipped config: DESIGN.md
    section 4), and the gather kernel supports n_mels (a multiple of 4).  Total, not free, memory: the same choice on
    every run."""
    return n_mels % 4 == 0 and corpus_device_bytes(total_frames, n_mels, n_entries) <= total_memory // 2


def check_segment_size(config: dict):
    """Raise ValueError unless the decoder reproduces a segment of the config's segment_size (engine.decoder_length):
    the reconstruction loss compares the decoder's output with its input frame by frame."""
    dl = config["data_loader"]
    seg, frame = int(dl["segment_size"]), int(dl["frame_size"])
    if frame < 1 or seg < 1 or seg % frame != 0:
        raise ValueError(f"segment_size {seg} is not a positive multiple of frame_size {frame}")
    T = seg // frame
    T_dec = decoder_length(config, T)
    if T_dec != T:
        raise ValueError(f"segment_size {seg}: a segment of {T} frames decodes to {T_dec} frames; the decoder reproduces "
                         "only lengths its subsampling and upsampling map onto themselves")


def validate_corpus(data, indexes, segment_size: int, frame_size: int, c_in: int):
    """Check a pickle {utt_id: [T, n_mels]} and an index [(utt_id, t), ...] against the model: every array is 2-D with
    the same n_mels, n_mels * frame_size == c_in, segment_size % frame_size == 0, and every index entry names an
    utterance of the pickle with 0 <= t and t + segment_size <= T.  Raises ValueError naming the first offending
    utterance or entry.  Returns (starts, n_mels, total_frames): starts[i] = the absolute first frame of entry i in
    the utterances laid end to end in the pickle's order."""
    if frame_size < 1 or segment_size < 1 or segment_size % frame_size != 0:
        raise ValueError(f"segment_size {segment_size} is not a positive multiple of frame_size {frame_size}")
    offsets, n_mels, total = {}, None, 0
    for utt, a in data.items():
        shape = np.shape(a)
        if len(shape) != 2:
            raise ValueError(f"utterance {utt!r}: expected a 2-D [T, n_mels] array, got shape {shape}")
        if n_mels is None:
            n_mels = shape[1]
        elif shape[1] != n_mels:
            raise ValueError(f"utterance {utt!r}: {shape[1]} mels, but the first utterance has {n_mels}")
        offsets[utt] = (total, shape[0])
        total += shape[0]
    if n_mels is None:
        raise ValueError("the pickle holds no utterance")
    if n_mels * frame_size != c_in:
        raise ValueError(f"n_mels {n_mels} x frame_size {frame_size} != c_in {c_in} of the model")
    if len(indexes) == 0:
        raise ValueError("the index is empty")
    starts = np.empty(len(indexes), dtype=np.int64)
    for i, entry in enumerate(indexes):
        try:
            utt, t = entry
        except (TypeError, ValueError):
            raise ValueError(f"index entry {i} {entry!r}: expected (utt_id, t)") from None
        if utt not in offsets:
            raise ValueError(f"index entry {i} {entry!r}: utterance {utt!r} is not in the pickle")
        off, T = offsets[utt]
        if not isinstance(t, (int, np.integer)) or isinstance(t, bool) or t < 0 or t + segment_size > T:
            raise ValueError(f"index entry {i} {entry!r}: a crop of {segment_size} frames at t={t!r} does not fit in the "
                             f"{T} frames of {utt!r}")
        starts[i] = off + t
    return starts, n_mels, total


class DeviceSegments:
    """Endless iterator of device batches [B, c_in, segment_size/frame_size] cut from a corpus kept in HBM.

    The pickle's frames (rounded to float32 as CollateFn rounds them), the start frame of every index entry and the
    current epoch order live on the device; the host copy of the frames is not kept.  Each ``next()`` enqueues one
    ``avc_segment_gather`` on the current stream into a fresh tensor from the caching allocator, so a consumer on the
    same stream sees the batch in stream order.  The batches are those of ``DataLoader(PickleDataset, batch_size,
    collate_fn=CollateFn(frame_size), drop_last=False)`` with ``SegmentSampler``'s order, bit for bit; ``seek(k)``
    positions the iterator at batch k of the run (a resumed run continues the uninterrupted run's sequence)."""

    _UPLOAD_FLOATS = 1 << 26    # host staging per host-to-device copy while loading (256 MB)

    def __init__(self, data, indexes, segment_size, frame_size, batch_size, c_in, rank=0, shuffle=True, device=None,
                 seed=0, drop_last=False):
        starts, n_mels, total = validate_corpus(data, indexes, segment_size, frame_size, c_in)
        if n_mels % 4 != 0:
            raise ValueError(f"n_mels {n_mels} is not a multiple of 4: the device corpus needs 16-byte rows")
        self.lib = L.load()
        self.dev = torch.device(device) if device is not None else local_device()
        self.n_mels, self.frame_size, self.segment_size, self.c_in = n_mels, frame_size, segment_size, c_in
        self.T = segment_size // frame_size
        self.sampler = SegmentSampler(len(indexes), batch_size, rank, shuffle, seed, drop_last)
        self.corpus = torch.empty((total, n_mels), dtype=torch.float32, device=self.dev)
        row, rows, chunk = 0, 0, []
        for i, a in enumerate(data.values()):
            chunk.append(np.asarray(a, dtype=np.float32))
            rows += chunk[-1].shape[0]
            if rows * n_mels >= self._UPLOAD_FLOATS or i == len(data) - 1:
                if rows:
                    self.corpus[row:row + rows].copy_(torch.from_numpy(np.concatenate(chunk)))
                row, rows, chunk = row + rows, 0, []
        self.starts = torch.from_numpy(starts).to(self.dev)
        self._epoch, self._order = None, None

    def seek(self, k: int):
        self.sampler.seek(k)

    def __iter__(self):
        return self

    def gather(self, first: int, count: int) -> torch.Tensor:
        """Entries order[first : first + count] of the loaded epoch order as one batch, enqueued on the current stream."""
        if self._order is None or first < 0 or count < 1 or first + count > self.sampler.n:
            raise ValueError(f"DeviceSegments.gather: entries [{first}, {first + count}) of an order of {self.sampler.n}"
                             f"{'' if self._order is not None else ' that is not loaded yet'}")
        x = torch.empty((count, self.c_in, self.T), dtype=torch.float32, device=self.dev)
        stream = torch.cuda.current_stream(self.dev)
        self._order.record_stream(stream)
        d = L.GatherDesc(corpus=self.corpus.data_ptr(), starts=self.starts.data_ptr(), order=self._order.data_ptr(),
                         x=x.data_ptr(), first=first, batch=count, seg=self.segment_size, frame=self.frame_size,
                         n_mels=self.n_mels)
        L.check(self.lib.avc_segment_gather(d, stream.cuda_stream), "avc_segment_gather")
        return x

    def load_epoch(self, epoch: int):
        """Make `epoch`'s order the one gather() reads: drawn on the host and uploaded (int32, 4 bytes per entry) once
        per epoch."""
        if epoch != self._epoch:
            host = self.sampler.order(epoch).to(torch.int32).pin_memory()
            self._order = host.to(self.dev, non_blocking=True)
            self._epoch = epoch

    def __next__(self) -> torch.Tensor:
        epoch, first, count = self.sampler.step()
        self.load_epoch(epoch)
        return self.gather(first, count)


class SyntheticSegments:
    """Endless iterator of pinned N(0,1) batches [B, n_mels, T] (training data is per-mel
    z-normalised, so N(0,1) is representative; SURVEY.md section 8d)."""

    def __init__(self, batch_size, n_mels, segment_size, seed=1, n_distinct=4):
        g = torch.Generator().manual_seed(seed)
        self.batches = [torch.randn((batch_size, n_mels, segment_size), generator=g) for _ in range(n_distinct)]
        if torch.cuda.is_available():
            self.batches = [b.pin_memory() for b in self.batches]
        self.i = 0

    def __iter__(self):
        return self

    def __next__(self):
        b = self.batches[self.i % len(self.batches)]
        self.i += 1
        return b
