"""Training corpus preparation from a VCTK 0.80 or a LibriTTS wav tree: the reference's preprocess_vctk.sh
(make_datasets_vctk.py, reduce_dataset.py, sample_single_segments.py) and preprocess_libri.sh (make_datasets_libri.py
and the same two scripts) without librosa or tensorflow, with the signal work on the GPU.

The split, the file order, the output formats and the index sampling are the reference's.  Its one unseeded source of
randomness, the module-level ``random``, is a ``random.Random(seed)`` here, used in the reference's call order: the
split is exactly what the reference produces after ``random.seed(seed)``.  The features differ from the reference's in
one respect only: files not at ``sample_rate`` are resampled with scipy.signal.resample_poly's filter (on the GPU,
csrc/prep.cu), where librosa used resampy.

Each set is processed in the reference's order for its corpus: VCTK sets in sorted path order; LibriTTS's train and
dev sets in their shuffled split order and its test set sorted.  The pickles' key order is that order, and attr.pkl
covers the first ``n_utts_attr`` training utterances in it.  Processing runs in chunks of at most ``chunk_seconds`` of
output audio.  Per chunk: the
files' PCM is decoded on the host as stored, packed into one pinned buffer and copied to the device once; one
``avc_resample_poly`` launch per (rate pair, sample format); the silence trim's frame powers find the files too short
for the STFT; ``Vocoder.wav_to_mel`` analyses the untrimmed signals of the others (it trims them itself); the mels are
copied back.  For the first ``n_utts_attr`` training utterances ``avc_mel_moments`` also writes their float64 (mean,
M2) while the mels are resident; ``avc_mel_moments_merge`` combines them into attr.pkl's mean and std.  Every kernel
gives an utterance the same bits in any chunk, so the output files do not depend on the chunk size.
"""
from __future__ import annotations

import contextlib
import ctypes as C
import glob
import json
import os
import pickle
import random
import re
from collections import defaultdict
from math import gcd

import numpy as np
import torch

from . import _lib as L
from . import vocoder as V

SETS = ("train", "in_test", "out_test")
LIBRI_SETS = ("train", "dev", "test")
RAGGED_MAX = 2 ** 31 - 1     # vocoder._Ragged: samples and frames of one ragged batch
_NAME = re.compile(r"p(\d+)_(\d+)\.wav")
SILENCE_POWER = 1e-10      # librosa's amin of the trim's power_to_db: -100 dB


# ------------------------------------------------------------------ file list and split (make_datasets_vctk.py)
def read_speaker_info(path):
    """Speaker ids: the first column of every line after the header."""
    ids = []
    with open(path) as f:
        for i, line in enumerate(f):
            if i == 0:
                continue
            ids.append(line.strip().split()[0])
    return ids


def read_filenames(root):
    """{speaker id: [paths]} of <root>/*/* in sorted order; every file name must start as p<speaker>_<utt>.wav."""
    speaker2filenames = defaultdict(list)
    for path in sorted(glob.glob(os.path.join(root, "*/*"))):
        m = _NAME.match(path.strip().split("/")[-1])
        if m is None:
            raise ValueError(f"{path}: the file name does not match p<speaker>_<utterance>.wav")
        speaker2filenames[m.group(1)].append(path)
    return speaker2filenames


def split_files(speaker_ids, speaker2filenames, n_out_speakers, test_prop, seed):
    """(train, in_test, out_test) path lists.  The last n_out_speakers of the shuffled speakers are the out-of-domain
    test speakers; each other speaker's files are shuffled and int(len * test_prop) of them go to in_test.  As in the
    reference, a speaker with int(len * test_prop) == 0 puts every file in in_test (path_list[:-0] is empty)."""
    rng = random.Random(seed)
    ids = list(speaker_ids)
    rng.shuffle(ids)
    train, in_test, out_test = [], [], []
    for speaker in ids[:-n_out_speakers]:
        paths = list(speaker2filenames.get(speaker, []))
        rng.shuffle(paths)
        n = int(len(paths) * test_prop)
        train += paths[:-n]
        in_test += paths[-n:]
    for speaker in ids[-n_out_speakers:]:
        out_test += speaker2filenames.get(speaker, [])
    return train, in_test, out_test


# ------------------------------------------------------------------ file list and split (make_datasets_libri.py)
def read_libri_paths(root, subset):
    """Sorted <root>/<subset>/*/*/*.wav: speaker / chapter / file, exactly three levels down.  The transcripts beside
    the wavs, and wavs at any other depth, are not listed."""
    return sorted(glob.glob(os.path.join(root, subset, "*/*/*.wav")))


def split_libri(train_paths, test_paths, test_prop, seed):
    """(train, dev, test) path lists in processing order.  The training subset's listing is shuffled once and its last
    int(len * test_prop) paths are dev; test is the test subset's listing as given (sorted).  Where the reference
    would go on with an empty train set (int(len * test_prop) == 0 makes paths[:-0] empty) this raises ValueError."""
    paths = list(train_paths)
    random.Random(seed).shuffle(paths)
    n = int(len(paths) * test_prop)
    if n == 0:
        raise ValueError(f"test_prop = {test_prop} of {len(paths)} training files gives no dev file, and the "
                         "reference's split would leave the training set empty")
    return paths[:-n], paths[-n:], list(test_paths)


def check_basenames(name, paths):
    """A set's pickle is keyed by file name, so two files of one set with the same name would silently keep one."""
    seen = {}
    for p in paths:
        b = os.path.basename(p)
        if b in seen:
            raise ValueError(f"the {name} set holds two files named {b}: {seen[b]} and {p}")
        seen[b] = p


# ------------------------------------------------------------------ reduce and index sampling
def reduce_set(data, segment_size):
    """reduce_dataset.py: the utterances longer than segment_size frames."""
    return {k: v for k, v in data.items() if v.shape[0] > segment_size}


def sample_segments(data, n_samples, segment_size, seed):
    """sample_single_segments.py on a fresh random.Random(seed): [(utt_id, t)] over the sorted utterances longer than
    segment_size frames."""
    utts = sorted(u for u in data if len(data[u]) > segment_size)
    if not utts:
        raise ValueError(f"no utterance is longer than segment_size = {segment_size} frames")
    rng = random.Random(seed)
    picks = rng.choices(range(len(utts)), k=n_samples)
    return [(utts[i], rng.randint(0, len(data[utts[i]]) - segment_size)) for i in picks]


# ------------------------------------------------------------------ resampling
def rate_pair(rate, sr):
    g = gcd(int(rate), int(sr))
    return int(sr) // g, int(rate) // g


def resample_taps(up, down):
    """(half_len, [up][n_taps] float64): resample_poly's filter firwin(2 half_len + 1, 1/max, ('kaiser', 5)) * up in
    polyphase order, table[r][i] = h[r + i up], zero past h's end."""
    from scipy.signal import firwin
    mx = max(up, down)
    half = 10 * mx
    h = firwin(2 * half + 1, 1.0 / mx, window=("kaiser", 5.0)) * up
    n_taps = -(-(2 * half + 1) // up)
    padded = np.zeros(up * n_taps)
    padded[:h.size] = h
    return half, np.ascontiguousarray(padded.reshape(n_taps, up).T)


def resample_supported(up, down):
    """Whether avc_resample_poly takes the pair: up = down = 1, or a tap table within RESAMPLE_MAX_PHASE_TAPS taps per
    phase and RESAMPLE_MAX_TAPS in all (resample_taps' shape, without designing the filter)."""
    if (up, down) == (1, 1):
        return True
    n_taps = -(-(20 * max(up, down) + 1) // up)
    return n_taps <= L.RESAMPLE_MAX_PHASE_TAPS and up * n_taps <= L.RESAMPLE_MAX_TAPS


def check_rates(sets, sample_rate):
    """Reads every header of every set ({name: paths}) and raises ValueError naming the first file whose rate the
    resampler cannot take to sample_rate, so that a run stops before it analyses or writes any set."""
    for paths in sets.values():
        for p in paths:
            rate = int(_header(p)[0])
            if not resample_supported(*rate_pair(rate, sample_rate)):
                up, down = rate_pair(rate, sample_rate)
                raise ValueError(f"{p}: a file at {rate} Hz cannot be resampled to --sample_rate {sample_rate} (up {up} / "
                                 f"down {down} needs more than {L.RESAMPLE_MAX_PHASE_TAPS} taps per phase or "
                                 f"{L.RESAMPLE_MAX_TAPS} in all)")


def n_resampled(n, up, down):
    return -(-n * up // down)


def plan_chunks(lengths, budget):
    """Consecutive runs of file indices whose lengths sum to at most `budget` (capped below 2^31); a file longer than
    the budget is a chunk of its own."""
    budget = min(int(budget), RAGGED_MAX)
    chunks, cur, total = [], [], 0
    for i, n in enumerate(lengths):
        if n > RAGGED_MAX:
            raise ValueError(f"file {i} gives {n} samples: more than a ragged batch holds ({RAGGED_MAX})")
        if cur and total + n > budget:
            chunks.append(cur)
            cur, total = [], 0
        cur.append(i)
        total += n
    if cur:
        chunks.append(cur)
    return chunks


_RSEG = np.dtype([("in_off", "<i8"), ("out_off", "<i8"), ("n_in", "<i4"), ("n_out", "<i4"), ("channels", "<i4"),
                  ("tile0", "<i4")])
assert _RSEG.itemsize == C.sizeof(L.ResampleSeg)


class _NoTimer:
    @contextlib.contextmanager
    def host(self, name):
        yield

    @contextlib.contextmanager
    def device(self, name):
        yield


class Preparer:
    """The device half of the pipeline: resampling, analysis and corpus statistics on one GPU."""

    def __init__(self, n_mels=512, sample_rate=24000, device=None, timer=None):
        self.voc = V.Vocoder(n_mels=n_mels, hp=V.AudioParams(sr=int(sample_rate)), device=device)
        self.hp, self.device = self.voc.hp, self.voc.device
        self.timer = timer or _NoTimer()
        self._taps = {}

    def taps(self, up, down):
        if (up, down) not in self._taps:
            half, tab = resample_taps(up, down)
            self._taps[(up, down)] = (half, tab.shape[1], torch.from_numpy(tab.astype(np.float32)).to(self.device))
        return self._taps[(up, down)]

    def resample(self, items):
        """[(rate, PCM as read_pcm returns it)] -> mono float32 device signals at hp.sr, views of one buffer.  int16 PCM
        travels as is; any other format is scaled to float32 on the host (vocoder.scale_pcm)."""
        sr, dev = self.hp.sr, self.device
        arrs, meta, nbytes = [], [], 0
        for rate, data in items:
            a = np.ascontiguousarray(data if data.dtype == np.int16 else V.scale_pcm(data).astype(np.float32))
            fmt = L.PCM_S16 if a.dtype == np.int16 else L.PCM_F32
            up, down = rate_pair(rate, sr)
            ch = 1 if a.ndim == 1 else a.shape[1]
            meta.append((nbytes // a.itemsize, fmt, up, down, a.shape[0], ch))
            arrs.append((nbytes, a))
            nbytes += -(-a.nbytes // 16) * 16
        with self.timer.host("pack"):
            pinned = torch.empty(max(nbytes, 16), dtype=torch.uint8, pin_memory=True)
            host = pinned.numpy()
            for off, a in arrs:
                host[off:off + a.nbytes] = a.reshape(-1).view(np.uint8)
        with self.timer.device("h2d"):
            pcm = pinned.to(dev, non_blocking=True)
        n_out = [n_resampled(m[4], m[2], m[3]) for m in meta]
        out_offs = np.concatenate([[0], np.cumsum(n_out)]).astype(np.int64)
        out = torch.empty(int(out_offs[-1]), device=dev)
        groups = defaultdict(list)
        for i, m in enumerate(meta):
            groups[m[1:4]].append(i)
        with self.timer.device("resample"):
            for (fmt, up, down), idx in sorted(groups.items()):
                tab = np.zeros(len(idx), _RSEG)
                tab["in_off"] = [meta[i][0] for i in idx]
                tab["out_off"] = out_offs[idx]
                tab["n_in"] = [meta[i][4] for i in idx]
                tab["n_out"] = [n_out[i] for i in idx]
                tab["channels"] = [meta[i][5] for i in idx]
                tiles = -(-tab["n_out"].astype(np.int64) // L.RESAMPLE_TILE)
                tab["tile0"] = np.concatenate([[0], np.cumsum(tiles)[:-1]])
                segs = torch.from_numpy(tab.view(np.uint8)).to(dev)
                half, n_taps, taps = self.taps(up, down) if (up, down) != (1, 1) else (0, 0, None)
                d = L.ResampleDesc(format=fmt, up=up, down=down, half_len=half, n_taps=n_taps, n_seg=len(idx),
                                   n_tiles=int(tiles.sum()), segs=segs.data_ptr(), pcm=pcm.data_ptr(),
                                   taps=None if taps is None else taps.data_ptr(), out=out.data_ptr())
                L.check(L.load().avc_resample_poly(C.byref(d), V._stream(dev)), "avc_resample_poly")
        return list(torch.split(out, n_out))

    def usable(self, ys):
        """Per signal: None, or why it is skipped: its trimmed signal is too short for the STFT, or it is silent.  The
        trim measures loudness against the signal's own peak, so it keeps the whole of a silent signal; its mel would be
        the dB floor in every bin, which carries nothing to learn and only shifts the corpus statistics."""
        hp = self.hp
        why = [None] * len(ys)
        live = []
        for i, y in enumerate(ys):
            if y.numel() < V.TRIM_FRAME // 2 + 1:
                why[i] = f"{y.numel()} samples at {hp.sr} Hz: shorter than one trim frame ({V.TRIM_FRAME // 2 + 1})"
            else:
                live.append(i)
        if live:
            with self.timer.device("skip_check"):
                powers = V.frame_power([ys[i] for i in live])
                host = torch.cat(powers).cpu().numpy()
            f0 = 0
            for i, p in zip(live, powers):
                power = host[f0:f0 + p.numel()]
                f0 += p.numel()
                s, e = V.trim_bounds(power, ys[i].numel(), hp.top_db)
                if power.max() <= SILENCE_POWER:
                    why[i] = f"silent: no trim frame has a mean power above {SILENCE_POWER:g}"
                elif e - s < hp.min_samples:
                    why[i] = f"{e - s} samples after trimming: the STFT needs at least {hp.min_samples}"
        return why

    def mels(self, ys):
        """Raw (unnormalised) mels of untrimmed signals: (device [frames][n_mels], frame counts)."""
        with self.timer.device("analysis"):
            out = self.voc.wav_to_mel(ys)
            M = torch.cat([mel for mel, _ in out])
        return M, [int(mel.shape[0]) for mel, _ in out]

    def moments(self, M, counts, moments, first):
        """avc_mel_moments of the first len(counts) utterances of M into moments[first ...]."""
        r = V._Ragged([0] * len(counts), counts, self.device)
        d = L.MomentsDesc(n_mels=self.hp.n_mels, n_seg=len(counts), first=int(first), segs=r.table.data_ptr(),
                          mels=M.data_ptr(), moments=moments.data_ptr())
        with self.timer.device("moments"):
            L.check(L.load().avc_mel_moments(C.byref(d), V._stream(self.device)), "avc_mel_moments")

    def merge(self, moments, counts):
        """(mean, std) float32 numpy and (mean, std) float64 numpy over the utterances of `moments`."""
        dev, n_mels = self.device, self.hp.n_mels
        cnt = torch.tensor(counts, dtype=torch.int32, device=dev)
        f32 = torch.empty(2, n_mels, device=dev)
        f64 = torch.empty(2, n_mels, dtype=torch.float64, device=dev)
        L.check(L.load().avc_mel_moments_merge(moments.data_ptr(), cnt.data_ptr(), len(counts), n_mels, f32[0].data_ptr(),
                                               f32[1].data_ptr(), f64[0].data_ptr(), f64[1].data_ptr(),
                                               V._stream(dev)), "avc_mel_moments_merge")
        f32, f64 = f32.cpu().numpy(), f64.cpu().numpy()
        return f32[0], f32[1], f64[0], f64[1]

    def process(self, paths, chunk_samples, n_attr=0):
        """Raw mels of `paths` in order: ({basename: float32 [T, n_mels]}, [(path, reason)] skipped, attr or None).
        attr = (mean, std, mean64, std64) over the first n_attr analysed utterances when n_attr > 0."""
        lengths = []
        with self.timer.host("headers"):
            for p in paths:
                rate, data = _header(p)
                lengths.append(n_resampled(data.shape[0], *rate_pair(rate, self.hp.sr)))
        data, skipped, counts = {}, [], []
        moments = (torch.empty(min(n_attr, len(paths)), self.hp.n_mels, 2, dtype=torch.float64, device=self.device)
                   if n_attr > 0 and paths else None)
        for chunk in plan_chunks(lengths, chunk_samples):
            with self.timer.host("decode"):
                items = [V.read_pcm(paths[i]) for i in chunk]
            ys = self.resample(items)
            why = self.usable(ys)
            kept = [i for i, w in enumerate(why) if w is None]
            skipped += [(paths[chunk[i]], w) for i, w in enumerate(why) if w is not None]
            if not kept:
                continue
            M, frames = self.mels([ys[i] for i in kept])
            k = min(len(kept), n_attr - len(counts)) if moments is not None else 0
            if k > 0:
                self.moments(M, frames[:k], moments, len(counts))
                counts += frames[:k]
            with self.timer.device("d2h"):
                host = M.cpu().numpy()
            f0 = 0
            for i, n in zip(kept, frames):
                data[os.path.basename(paths[chunk[i]])] = host[f0:f0 + n]
                f0 += n
        attr = self.merge(moments, counts) if counts else None
        return data, skipped, attr


def _header(path):
    """(rate, samples) without reading the samples where the format allows it."""
    from scipy.io import wavfile
    try:
        return wavfile.read(path, mmap=True)
    except ValueError:
        return wavfile.read(path)


def normalise(data, mean, std):
    """The reference's (val - mean) / std in float32, per utterance, replacing each entry in place (as the reference
    does), so that the raw and the normalised set are never both resident."""
    for k in data:
        data[k] = (data[k] - mean) / std
    return data


def _dump(obj, path):
    with open(path, "wb") as f:
        pickle.dump(obj, f)


def _load(path):
    with open(path, "rb") as f:
        return pickle.load(f)


def _features(sets, out_dir, cache, n_mels, sample_rate, n_utts_attr, chunk_seconds, device, timer, log):
    """Stage 0's features: each set of `sets` ({name: paths in processing order}, "train" first) analysed in that
    order; attr.pkl over the first n_utts_attr analysed training utterances; every set normalised by it and pickled
    (and kept in `cache`); the skipped files in skipped_files.txt.  Every file's rate is checked first (check_rates):
    the sets run one after another, and a file the resampler refuses would otherwise end the run only when its set's
    turn comes, after the training set has been processed."""
    with timer.host("headers"):
        check_rates(sets, sample_rate)
    prep = Preparer(n_mels, sample_rate, device, timer)
    chunk = max(1, int(chunk_seconds * sample_rate))
    skipped, mean = [], None
    for name, paths in sets.items():
        log(f"processing {name} set, {len(paths)} files")
        raw, skip, attr = prep.process(paths, chunk, n_utts_attr if name == "train" else 0)
        skipped += skip
        if name == "train":
            if attr is None:
                raise ValueError("no training utterance could be analysed: attr.pkl cannot be computed")
            mean, std = attr[0], attr[1]
            with timer.host("pickle"):
                _dump({"mean": mean, "std": std}, os.path.join(out_dir, "attr.pkl"))
        with timer.host("pickle"):
            cache[name] = normalise(raw, mean, std)
            del raw
            _dump(cache[name], os.path.join(out_dir, f"{name}.pkl"))
    with open(os.path.join(out_dir, "skipped_files.txt"), "w") as f:
        f.writelines(f"{p}\t{why}\n" for p, why in skipped)
    log(f"{len(skipped)} files skipped (listed in skipped_files.txt)")


def _reduce_and_index(out_dir, cache, test_sets, segment_size, training_samples, testing_samples, seed, stage, timer):
    """Stages 1-3: train_<seg>.pkl, train_samples_<seg>.json and <set>_samples_<seg>.json for each of `test_sets`,
    from the sets in `cache` or, when stage 0 did not run, from their pickles."""
    def load_set(name):
        if name not in cache:
            cache[name] = _load(os.path.join(out_dir, f"{name}.pkl"))
        return cache[name]

    with timer.host("reduce_and_index"):
        if stage <= 1:
            _dump(reduce_set(load_set("train"), segment_size), os.path.join(out_dir, f"train_{segment_size}.pkl"))
        if stage <= 2:
            with open(os.path.join(out_dir, f"train_samples_{segment_size}.json"), "w") as f:
                json.dump(sample_segments(load_set("train"), training_samples, segment_size, seed), f)
        if stage <= 3:
            for name in test_sets:
                with open(os.path.join(out_dir, f"{name}_samples_{segment_size}.json"), "w") as f:
                    json.dump(sample_segments(load_set(name), testing_samples, segment_size, seed), f)


# ------------------------------------------------------------------ the whole preprocess_vctk.sh
def run(wav_dir, speaker_info, out_dir, n_out_speakers=20, test_prop=0.1, sample_rate=24000, n_utts_attr=5000,
        n_mels=512, segment_size=128, training_samples=10000000, testing_samples=10000, seed=0, stage=0,
        chunk_seconds=1800.0, device=None, timer=None, log=print):
    """Stages as preprocess_vctk.sh: 0 = split and features, 1 = reduce, 2 = train index, 3 = test indexes."""
    os.makedirs(out_dir, exist_ok=True)
    timer = timer or _NoTimer()
    cache = {}
    if stage <= 0:
        if n_utts_attr < 1:
            raise ValueError("n_utts_attr must be >= 1")
        sets = dict(zip(SETS, split_files(read_speaker_info(speaker_info), read_filenames(wav_dir), n_out_speakers,
                                          test_prop, seed)))
        for name in ("in_test", "out_test"):
            with open(os.path.join(out_dir, f"{name}_files.txt"), "w") as f:
                f.writelines(f"{p}\n" for p in sets[name])
        _features({name: sorted(sets[name]) for name in SETS}, out_dir, cache, n_mels, sample_rate, n_utts_attr,
                  chunk_seconds, device, timer, log)
    _reduce_and_index(out_dir, cache, ("in_test", "out_test"), segment_size, training_samples, testing_samples, seed,
                      stage, timer)


# ------------------------------------------------------------------ the whole preprocess_libri.sh
def run_libri(root, out_dir, train_set="train-clean-100", test_set="dev-clean", test_prop=0.05, sample_rate=24000,
              n_utts_attr=5000, n_mels=512, segment_size=128, training_samples=10000000, testing_samples=10000, seed=0,
              stage=0, chunk_seconds=1800.0, device=None, timer=None, log=print):
    """Stages as preprocess_libri.sh: 0 = split and features, 1 = reduce, 2 = train index, 3 = dev and test indexes.

    train and dev are processed in their shuffled split order, test in sorted order, so attr.pkl covers the first
    n_utts_attr analysed utterances of the *shuffled* training list (VCTK's covers its sorted list).  The file lists
    hold the sorted basenames of each set."""
    os.makedirs(out_dir, exist_ok=True)
    timer = timer or _NoTimer()
    cache = {}
    if stage <= 0:
        if n_utts_attr < 1:
            raise ValueError("n_utts_attr must be >= 1")
        listings = {s: read_libri_paths(root, s) for s in (train_set, test_set)}
        for s, paths in listings.items():
            if not paths:
                raise ValueError(f"no {os.path.join(root, s, '*/*/*.wav')} files")
        sets = dict(zip(LIBRI_SETS, split_libri(listings[train_set], listings[test_set], test_prop, seed)))
        for name, paths in sets.items():
            check_basenames(name, paths)
        log(f"{len(sets['train'])} training data, {len(sets['dev'])} dev data, {len(sets['test'])} test data")
        for name, paths in sets.items():
            with open(os.path.join(out_dir, f"{name}_files.txt"), "w") as f:
                f.writelines(f"{os.path.basename(p)}\n" for p in sorted(paths))
        _features(sets, out_dir, cache, n_mels, sample_rate, n_utts_attr, chunk_seconds, device, timer, log)
    _reduce_and_index(out_dir, cache, ("dev", "test"), segment_size, training_samples, testing_samples, seed, stage,
                      timer)
