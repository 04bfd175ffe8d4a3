"""GPU: the device-resident corpus.  avc_segment_gather against the stock host path (CollateFn over PickleDataset
items) bit for bit, its argument checks, DeviceSegments against a DataLoader over the same order across epochs and
ranks, and Solver on a real data directory (device path, resume, and the DataLoader path when the corpus does not fit)."""
import json
import pickle
import types

import numpy as np
import pytest
import torch
from torch.utils.data import DataLoader

from adaptive_voice_conversion_b200 import _lib as L
from adaptive_voice_conversion_b200 import data_utils as D

pytestmark = pytest.mark.gpu

SEG = 128
GUARD = 256


def make_corpus(n_mels, n_utt, seed, dtype=np.float32, stride=7, seg=SEG):
    """VCTK-like: utterances of 129-600 frames; the index holds every `stride`-th crop plus each utterance's last one."""
    rng = np.random.default_rng(seed)
    data = {f"p{seed}_{i:03d}": rng.standard_normal((int(rng.integers(129, 601)), n_mels)).astype(dtype) for i in range(n_utt)}
    index = []
    for utt, a in data.items():
        index += [[utt, t] for t in range(0, len(a) - seg + 1, stride)] + [[utt, len(a) - seg]]
    return data, index


def collate_ref(data, index, order, frame, seg=SEG):
    ds = D.PickleDataset.from_loaded(data, index, seg)
    return D.CollateFn(frame)([ds[i] for i in order])


def bits_equal(a, b):
    return a.shape == b.shape and torch.equal(a.contiguous().view(torch.int32), b.contiguous().view(torch.int32))


def gather(corpus, starts, order, first, batch, n_mels, frame, seg=SEG, x=None):
    T, C = seg // frame, frame * n_mels
    buf = torch.full((batch * C * T + 2 * GUARD,), float("nan"), device="cuda")
    x = buf[GUARD:GUARD + batch * C * T] if x is None else x
    d = L.GatherDesc(corpus=corpus.data_ptr(), starts=starts.data_ptr(), order=order.data_ptr(), x=x.data_ptr(), first=first,
                     batch=batch, seg=seg, frame=frame, n_mels=n_mels)
    rc = L.load().avc_segment_gather(d, torch.cuda.current_stream().cuda_stream)
    return rc, buf


def upload(data, index, frame, c_in):
    starts, n_mels, _ = D.validate_corpus(data, index, SEG, frame, c_in)
    corpus = torch.from_numpy(np.concatenate([np.asarray(a, dtype=np.float32) for a in data.values()])).cuda()
    return corpus, torch.from_numpy(starts).cuda()


@pytest.mark.parametrize("n_mels, frame", [(80, 1), (512, 1), (40, 2)])
@pytest.mark.parametrize("B", [1, 128, 256])
def test_gather_matches_collate(n_mels, frame, B):
    data, index = make_corpus(n_mels, 12, seed=n_mels + frame)
    corpus, starts = upload(data, index, frame, n_mels * frame)
    n = len(index)
    assert n >= B + 3
    # the batch sits at position 3 of the order; it starts with the corpus's first crop (frame 0 of the first
    # utterance) and, for B > 1, ends with its last one (ending at the corpus's last frame)
    rest = [i for i in torch.randperm(n, generator=torch.Generator().manual_seed(B)).tolist() if i not in (0, n - 1)]
    batch = [0] if B == 1 else [0] + rest[3:3 + B - 2] + [n - 1]
    order = rest[:3] + batch + rest[3 + max(B - 2, 0):]
    rc, buf = gather(corpus, starts, torch.tensor(order, dtype=torch.int32, device="cuda"), 3, B, n_mels, frame)
    assert rc == L.OK, L.last_error()
    C, T = n_mels * frame, SEG // frame
    x = buf[GUARD:GUARD + B * C * T].view(B, C, T).cpu()
    assert bits_equal(x, collate_ref(data, index, order[3:3 + B], frame))
    assert torch.isnan(buf[:GUARD]).all() and torch.isnan(buf[-GUARD:]).all()
    if B > 1:   # the crops at both ends of the corpus
        assert bits_equal(x[0], torch.from_numpy(data[index[0][0]][:SEG]).reshape(T, C).t())
        last = data[index[-1][0]]
        assert bits_equal(x[-1], torch.from_numpy(last[len(last) - SEG:]).reshape(T, C).t())


def test_gather_float64_pickle_rounds_like_collate():
    data, index = make_corpus(80, 6, seed=3, dtype=np.float64)
    corpus, starts = upload(data, index, 1, 80)
    order = list(range(len(index)))[::-1]
    rc, buf = gather(corpus, starts, torch.tensor(order, dtype=torch.int32, device="cuda"), 0, 64, 80, 1)
    assert rc == L.OK, L.last_error()
    x = buf[GUARD:GUARD + 64 * 80 * SEG].view(64, 80, SEG).cpu()
    assert bits_equal(x, collate_ref(data, index, order[:64], 1))


def test_gather_rejects_invalid_arguments():
    lib = L.load()
    data, index = make_corpus(80, 2, seed=5)
    corpus, starts = upload(data, index, 1, 80)
    order = torch.arange(len(index), dtype=torch.int32, device="cuda")
    x = torch.full((4 * 80 * SEG,), float("nan"), device="cuda")
    good = dict(corpus=corpus.data_ptr(), starts=starts.data_ptr(), order=order.data_ptr(), x=x.data_ptr(), first=0, batch=4,
                seg=SEG, frame=1, n_mels=80)
    st = torch.cuda.current_stream().cuda_stream
    assert lib.avc_segment_gather(L.GatherDesc(**good), st) == L.OK
    torch.cuda.synchronize()
    cases = [({"corpus": None}, "null pointer"), ({"starts": None}, "null pointer"), ({"order": None}, "null pointer"),
             ({"x": None}, "null pointer"), ({"n_mels": 82}, "multiple of 4"), ({"n_mels": 0}, "multiple of 4"),
             ({"seg": 127, "frame": 2}, "multiple of frame"), ({"frame": 0}, "multiple of frame"),
             ({"batch": 0}, "batch must be >= 1"), ({"batch": -3}, "batch must be >= 1"), ({"first": -1}, "first")]
    n0 = L.launch_count()
    for patch, msg in cases:
        rc = lib.avc_segment_gather(L.GatherDesc(**{**good, **patch}), st)
        assert rc == L.ERR_INVALID, patch
        assert msg in L.last_error(), (patch, L.last_error())
    assert lib.avc_segment_gather(None, st) == L.ERR_INVALID and "null descriptor" in L.last_error()
    assert L.launch_count() == n0


@pytest.mark.parametrize("rank", [0, 1])
def test_device_segments_match_dataloader_over_epochs(rank):
    """1000 entries, B = 96: 10 full batches and one of 40 per epoch; a full epoch plus 5 batches of the next."""
    data, index = make_corpus(80, 40, seed=11, stride=5)
    index = index[:1000]
    assert len(index) == 1000
    ds = D.DeviceSegments(data, index, SEG, 1, 96, 80, rank=rank, shuffle=True, device="cuda")
    assert ds.sampler.batches_per_epoch == 11
    with pytest.raises(ValueError, match="not loaded yet"):
        ds.gather(0, 96)
    pds = D.PickleDataset.from_loaded(data, index, SEG)
    ref = []
    for epoch in range(2):
        order = D.epoch_order(1000, rank, epoch).tolist()
        ref += list(DataLoader(pds, sampler=order, batch_size=96, collate_fn=D.CollateFn(1), num_workers=0))
    got = [next(ds) for _ in range(16)]
    with pytest.raises(ValueError, match="entries \\[960, 1056\\) of an order of 1000"):
        ds.gather(960, 96)
    assert [len(b) for b in got] == [96] * 10 + [40] + [96] * 5
    for k, (a, b) in enumerate(zip(got, ref[:16])):
        assert a.is_cuda and bits_equal(a.cpu(), b), k
    other = D.epoch_order(1000, 1 - rank, 0).tolist()
    assert not bits_equal(got[0].cpu(), D.CollateFn(1)([pds[i] for i in other[:96]]))


# ----------------------------------------------------------------------------- Solver on a data directory
N_ENTRIES, B_SOLVER = 100, 16     # 7 batches per epoch: 6 x 16 and a short one of 4


def write_data_dir(tmp_path):
    data, index = make_corpus(80, 20, seed=21, stride=9)
    index = index[:N_ENTRIES]
    assert len(index) == N_ENTRIES
    d = tmp_path / "data"
    d.mkdir()
    with open(d / "train.pkl", "wb") as f:
        pickle.dump(data, f)
    with open(d / "train_samples_128.json", "w") as f:
        json.dump(index, f)
    return str(d), data, index


def solver_args(tmp_path, data_dir, name, load=None):
    return types.SimpleNamespace(data_dir=data_dir, train_set="train", train_index_file="train_samples_128.json",
                                 logdir=str(tmp_path / "log"), load_model=load is not None, load_opt=False,
                                 store_model_path=str(tmp_path / name), load_model_path=str(tmp_path / (load or name)),
                                 summary_steps=1, save_steps=1000, tag="t", iters=0)


def small_config():
    from adaptive_voice_conversion_b200.config import default_config
    cfg = default_config(80)
    cfg["data_loader"]["batch_size"] = B_SOLVER
    return cfg


def recording_solver(cfg, args):
    from adaptive_voice_conversion_b200.solver import Solver
    torch.manual_seed(0)
    s = Solver(cfg, args)
    s.seen = []
    step = s.trainer.step

    def wrapped(x, lambda_kl, **kw):
        s.seen.append(x.detach().cpu().clone())
        return step(x, lambda_kl, **kw)
    s.trainer.step = wrapped
    return s


def mirror(data, index, k0, n):
    s = D.SegmentSampler(len(index), B_SOLVER, rank=0, shuffle=True)
    s.seek(k0)
    pds = D.PickleDataset.from_loaded(data, index, SEG)
    return [D.CollateFn(1)([pds[int(i)] for i in next(s)]) for _ in range(n)]


def assert_finite_losses(s):
    meta, _ = s.logger.last["t/ae_train"]
    assert all(np.isfinite(v) for v in meta.values()), meta


def test_solver_trains_from_the_device_corpus_and_resumes(tmp_path):
    data_dir, data, index = write_data_dir(tmp_path)
    cfg = small_config()
    k, m = 9, 8
    full = recording_solver(cfg, solver_args(tmp_path, data_dir, "full"))
    assert isinstance(full.train_loader, D.DeviceSegments) and full.train_dataset is None
    full.train(k + m)    # 17 steps: graph capture at step 3, eager short batches at steps 7 and 14, replay in between
    assert full.trainer._graphs is not None
    ref = mirror(data, index, 0, k + m)
    assert [len(x) for x in full.seen] == [16] * 6 + [4] + [16] * 6 + [4] + [16] * 3
    assert all(bits_equal(a, b) for a, b in zip(full.seen, ref)) and len(full.seen) == k + m
    assert_finite_losses(full)
    del full

    first = recording_solver(cfg, solver_args(tmp_path, data_dir, "part"))
    first.train(k)       # saves part.ckpt / .opt / .iter at its last step
    seen = first.seen
    del first
    resumed = recording_solver(cfg, solver_args(tmp_path, data_dir, "part2", load="part"))
    assert resumed.iteration == k and resumed.train_loader.sampler.position == k
    resumed.train(m)
    seen += resumed.seen
    assert len(seen) == k + m and all(bits_equal(a, b) for a, b in zip(seen, ref))
    assert_finite_losses(resumed)


def test_solver_falls_back_to_the_dataloader_when_the_corpus_does_not_fit(tmp_path, monkeypatch):
    from adaptive_voice_conversion_b200 import solver as S
    data_dir, _, _ = write_data_dir(tmp_path)
    monkeypatch.setattr(S, "_device_total_memory", lambda dev: 1 << 20)
    s = recording_solver(small_config(), solver_args(tmp_path, data_dir, "dl"))
    assert isinstance(s.train_loader, DataLoader) and isinstance(s.train_dataset, D.PickleDataset)
    s.train(4)
    assert len(s.seen) == 4 and all(x.shape == (16, 80, SEG) for x in s.seen)
    assert_finite_losses(s)
