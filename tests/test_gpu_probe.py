"""GPU: the speaker probes.  Every kernel of csrc/probe.cu against the float64 restatement (tests/_probe_ref.py) on the
device's own inputs (ranks and counts exactly, float64 within 1e-12), three training steps against the restatement,
determinism, two sanity cases on synthetic data, and evaluate_probe / evaluate.py -probe end to end at c_in 80 and
512."""
import json
import os
import pickle
import sys

import numpy as np
import pytest
import torch

import _probe_ref as R
from adaptive_voice_conversion_b200 import _lib as L
from adaptive_voice_conversion_b200 import speaker_probe as P
from adaptive_voice_conversion_b200.config import default_config
from adaptive_voice_conversion_b200.inference import padded_batch, padded_batches
from adaptive_voice_conversion_b200.speaker_eval import representations

pytestmark = pytest.mark.gpu

SENTINEL = -7777.0


def bits_equal(a, b):
    a, b = np.ascontiguousarray(a), np.ascontiguousarray(b)
    return a.shape == b.shape and a.dtype == b.dtype and a.tobytes() == b.tobytes()


def close64(got, ref, rel=1e-12):
    got, ref = np.asarray(got, np.float64), np.asarray(ref, np.float64)
    return float(np.abs(got - ref).max()) <= rel * max(float(np.abs(ref).max()), 1e-300)


# ----------------------------------------------------------------------------- kernels
@pytest.mark.parametrize("C", [128, 512])
def test_frames_are_the_valid_frames(C):
    T = 97
    lens = [97, 1, 50, 33, 96]                     # 97: the padded extent itself
    g = torch.Generator().manual_seed(C)
    x = torch.randn((len(lens), C, T), generator=g)
    off = [0]
    for n in lens:
        off.append(off[-1] + n + 2)                # gaps of two rows stay untouched
    out = torch.full((off[-1] + 2, C), SENTINEL, device="cuda")
    P.frame_rows(x.cuda(), torch.tensor(lens, dtype=torch.int32, device="cuda"),
                 torch.tensor(off[:-1], dtype=torch.int64, device="cuda"), out)
    got = out.cpu().numpy()
    for b, n in enumerate(lens):
        assert bits_equal(got[off[b]:off[b] + n], x[b, :, :n].numpy().T.copy()), b
        assert (got[off[b] + n:off[b] + n + 2] == SENTINEL).all()


@pytest.mark.parametrize("D", [128, 256, 1024])
@pytest.mark.parametrize("N", [1, 1001, 4097])
def test_moments_and_standardize(D, N):
    rng = np.random.default_rng(D + N)
    x = (rng.standard_normal((N, D)) * rng.uniform(0.01, 100, D) + rng.uniform(-50, 50, D)).astype(np.float32)
    x[:, 3] = 1.25                                  # a constant dimension: std 1
    xd = torch.from_numpy(x).cuda()
    mean, std = P.moments(xd)
    rm, rs = R.moments64(x)
    assert close64(mean.cpu().numpy(), rm) and close64(std.cpu().numpy(), rs) and float(std[3]) == 1.0
    m64, s64 = mean.cpu().numpy(), std.cpu().numpy()
    assert bits_equal(P.standardize(xd, mean, std).cpu().numpy(), R.standardize64(x, m64, s64))
    idx = rng.permutation(N)[: max(1, N // 2)]
    got = P.standardize(xd, mean, std, torch.from_numpy(idx).cuda()).cpu().numpy()
    assert bits_equal(got, R.standardize64(x[idx], m64, s64))


def logits_with_ties(R_, S, seed):
    rng = np.random.default_rng(seed)
    z = (rng.standard_normal((R_, S)) * 3).astype(np.float32)
    y = rng.integers(0, S, R_).astype(np.int32)
    for r in range(0, R_, 7):                       # the true class tied with others, below and above its index
        z[r, rng.integers(0, S, min(S, 3))] = z[r, y[r]]
    return z, y


@pytest.mark.parametrize("S", [2, 3, 257, L.PROBE_MAX_CLASSES])
def test_xent_is_the_restatement(S):
    R_ = 1003 if S < 1000 else 97
    z, y = logits_with_ties(R_, S, S)
    y[5] = S                                        # an invalid label
    zd, yd = torch.from_numpy(z).cuda(), torch.from_numpy(y).cuda()
    d = torch.full((R_, S), SENTINEL, device="cuda")
    tot = torch.zeros(1, dtype=torch.float64, device="cuda")
    scratch = torch.empty(L.PROBE_SUM_SCRATCH, dtype=torch.float64, device="cuda")
    loss, rank = P.xent(zd, yd, 0.25, dlogits=d, loss_sum=tot, scratch=scratch)
    loss, rank, d = loss.cpu().numpy(), rank.cpu().numpy(), d.cpu().numpy()
    ok = np.arange(R_) != 5
    rl, rd, rr = R.xent64(z[ok], y[ok], 0.25)
    assert np.array_equal(rank[ok], rr) and rank[5] == -1
    assert np.isnan(loss[5]) and (d[5] == 0).all() and np.isnan(float(tot))
    assert close64(loss[ok], rl)
    assert np.abs(d[ok] - rd).max() <= 2.0 ** -23 * np.abs(rd).max()
    y[5] = 0
    loss2, _ = P.xent(zd, torch.from_numpy(y).cuda(), loss_sum=tot, scratch=scratch)
    assert close64(float(tot), R.xent64(z, y)[0].sum()) and close64(float(tot), loss2.cpu().numpy().sum())


@pytest.mark.parametrize("S", [2, 3, 257, L.PROBE_MAX_CLASSES])
def test_vote_is_the_restatement(S):
    rng = np.random.default_rng(S + 1)
    sizes = [1, 5, 38, 1, 70, 3]
    off = np.concatenate([[0], np.cumsum(sizes)]).astype(np.int64)
    z, _ = logits_with_ties(int(off[-1]), S, S + 2)
    y = rng.integers(0, S, len(sizes)).astype(np.int32)
    z[off[2]:off[3], (y[2] + 1) % S] = z[off[2]:off[3], y[2]]     # a class tied with the truth in every frame
    scores, rank = P.vote(torch.from_numpy(z).cuda(), torch.from_numpy(off).cuda(), torch.from_numpy(y).cuda())
    rs, rr = R.vote64(z, off, y)
    assert close64(scores.cpu().numpy(), rs)
    assert np.array_equal(rank.cpu().numpy(), rr)
    assert rr[2] == R.rank_of(rs[2], y[2])


def test_wrappers_reject_bad_rows_before_a_launch():
    n0 = L.launch_count()
    with pytest.raises(ValueError, match="CUDA"):
        P.fit_probe(torch.zeros(4, 3), [0, 1, 0, 1])
    with pytest.raises(ValueError, match="finite"):
        P.fit_probe(torch.full((4, 3), float("nan"), device="cuda"), [0, 1, 0, 1])
    with pytest.raises(ValueError, match="classes"):
        P.fit_probe(torch.zeros(4, 3, device="cuda"), [0, 1, 0, 4097])
    assert L.launch_count() == n0


# ----------------------------------------------------------------------------- training
def clusters(n_per, S, D, sep, seed, shuffle_labels=False):
    rng = np.random.default_rng(seed)
    centres = rng.standard_normal((S, D)) * sep
    y = np.repeat(np.arange(S), n_per)
    x = (centres[y] + rng.standard_normal((len(y), D))).astype(np.float32)
    if shuffle_labels:
        y = rng.integers(0, S, len(y))
    return x, y


def test_three_steps_match_the_restatement():
    x, y = clusters(96, 8, 128, 0.3, 0)             # 768 rows: three batches of 256 in one epoch
    xd = torch.from_numpy(x).cuda()
    params = P.ProbeParams(utt_epochs=1)
    probe = P.fit_probe(xd, y, params, seed=3)
    xs = P.standardize(xd, probe.mean, probe.std).cpu().numpy().astype(np.float64)
    order = P.epoch_order(len(x), 3, 0).numpy()
    init = [t.numpy().astype(np.float64) for t in P.unflatten(P.init_params(128, 8, params, 3), 128, 256, 8)]
    ref = R.train64(init, xs, y, [order[k * 256:(k + 1) * 256] for k in range(3)])
    got = [t.cpu().numpy().astype(np.float64) for t in probe.views()]
    diff = np.sqrt(sum(((g - r) ** 2).sum() for g, r in zip(got, ref)))
    norm = np.sqrt(sum((r ** 2).sum() for r in ref))
    moved = np.sqrt(sum(((i - r) ** 2).sum() for i, r in zip(init, ref)))
    assert diff <= 1e-4 * norm and moved > 100 * diff, (diff, norm, moved)
    loss0 = np.mean([R.loss64(R.train64(init, xs, y, [order[j * 256:(j + 1) * 256] for j in range(k)]),
                              xs[order[k * 256:(k + 1) * 256]], y[order[k * 256:(k + 1) * 256]]) for k in range(3)])
    assert abs(probe.losses[0] - loss0) <= 1e-4 * loss0


def test_same_seed_same_bits():
    x, y = clusters(50, 5, 64, 0.5, 1)
    xd = torch.from_numpy(x).cuda()
    a = P.fit_probe(xd, y, seed=7)
    b = P.fit_probe(xd, y, seed=7)
    assert torch.equal(a.flat, b.flat) and a.losses == b.losses and len(a.losses) == 50
    c = P.fit_probe(xd, y, seed=8)
    assert not torch.equal(a.flat, c.flat)
    fa = P.fit_probe(xd, y, seed=7, frames=True)
    fb = P.fit_probe(xd, y, seed=7, frames=True)
    assert torch.equal(fa.flat, fb.flat) and len(fa.losses) == 10


def test_separated_clusters_are_learned():
    x, y = clusters(150, 8, 32, 3.0, 2)
    train = np.arange(len(y)) % 3 != 0
    probe = P.fit_probe(torch.from_numpy(x[train]).cuda(), y[train], seed=0)
    rank = P.score_probe(probe, torch.from_numpy(x[~train]).cuda(), y[~train])["rank"]
    assert (rank == 0).all()
    assert probe.losses[-1] < probe.losses[0]


def test_random_labels_score_chance():
    x, y = clusters(500, 4, 32, 0.0, 3, shuffle_labels=True)
    probe = P.fit_probe(torch.from_numpy(x[:1000]).cuda(), y[:1000], seed=0)
    n = 1000
    acc = float((P.score_probe(probe, torch.from_numpy(x[1000:]).cuda(), y[1000:])["rank"] == 0).mean())
    bound = 3.2905 * np.sqrt(0.25 * 0.75 / n)       # two-sided 99.9 % normal bound of Binomial(n, 1/4) / n
    assert abs(acc - 0.25) <= bound, acc


# ----------------------------------------------------------------------------- end to end
def make_sets(n_mels, seed):
    """train: 4 speakers x 8 utterances (some short); in_test: 3 more of each plus a short one; out_test: 2 unseen
    speakers."""
    rng = np.random.default_rng(seed)

    def mel(T, s):
        return (rng.standard_normal((T, n_mels)) + 0.5 * s).astype(np.float32)
    train = {f"p{300 + s}_{k:03d}.wav": mel(int(rng.choice([10, 40, 129, 200, 333])), s) for s in range(4) for k in range(8)}
    in_test = {f"p{300 + s}_{100 + k:03d}.wav": mel(int(rng.integers(129, 300)), s) for s in range(4) for k in range(3)}
    in_test["p300_199.wav"] = mel(12, 0)
    out_test = {f"p{500 + s}_{k:03d}.wav": mel(int(rng.integers(129, 300)), s) for s in range(2) for k in range(3)}
    return train, in_test, out_test


def make_model(c_in):
    from adaptive_voice_conversion_b200.model import AE
    torch.manual_seed(c_in)
    return AE(default_config(c_in)).cuda()


@pytest.mark.parametrize("c_in", [80, 512])
def test_evaluate_probe_end_to_end(c_in):
    train, in_test, out_test = make_sets(c_in, c_in)
    model = make_model(c_in)
    model.train()
    small = P.ProbeParams(utt_epochs=5, frame_epochs=2)
    res = P.evaluate_probe(model, train, {"in_test": in_test, "out_test": out_test}, seed=1, per_speaker_utts=5,
                           params=small, fit_name="train")
    assert model.training
    fit_utts = P.probe_utterances({u: len(v) for u, v in train.items()}, 17, 5, 1)
    a, b = res["in_test"], res["out_test"]
    assert a["n"] == 12 and a["n_unseen"] == 0 and a["n_short"] == 1 and a["speakers"] == 4 and a["chance"] == 0.25
    assert a["n_fit"] == len(fit_utts) and a["majority"] == 0.25
    assert b["n"] == 0 and b["n_unseen"] == 6 and b["majority"] is None
    for k in P.REPRESENTATIONS:
        assert 0.0 <= a[k]["acc"] <= a[k]["top5"] <= 1.0 and 0.0 <= a[k]["fit_acc"] <= 1.0
        assert sorted(a[k]["per_speaker"]) == ["p300", "p301", "p302", "p303"]
        assert b[k]["acc"] is None and b[k]["fit_acc"] == a[k]["fit_acc"]
    assert 0.0 <= a["content_frames"]["frame_acc"] <= 1.0
    assert json.dumps(P.evaluate_probe(model, train, {"in_test": in_test, "out_test": out_test}, seed=1,
                                       per_speaker_utts=5, params=small, fit_name="train")) == json.dumps(res)

    # the features: representations() bit for bit, the frame rows get_content_means' valid frames
    model.eval()
    mels = [torch.from_numpy(train[u]).cuda() for u in fit_utts]
    feats = P.features(model, mels)
    reps = representations(model, mels)
    for k in ("speaker", "content", "mel"):
        assert torch.equal(feats[k], reps[k]), k
    lens = [int(m.shape[0]) for m in mels]
    rows = feats["content_frames"].cpu().numpy()
    off = feats["offsets"]
    with torch.no_grad():
        for idx, T, _, _ in padded_batches(lens, lens):
            x, lx = padded_batch([m.t() for m in mels], idx, T, "cuda")
            mu, lat = model.get_content_means(x, lengths=lx)
            for j, i in enumerate(idx):
                n = int(lat[j])
                assert off[i + 1] - off[i] == n == -(-lens[i] // 8)
                assert bits_equal(rows[off[i]:off[i + 1]], mu[j, :, :n].cpu().numpy().T.copy()), i


def test_cli_probe_leaves_spk_unchanged(tmp_path):
    import yaml
    from conftest import ROOT
    cfg = default_config(80)
    (tmp_path / "config.yaml").write_text(yaml.safe_dump(cfg))
    torch.save(make_model(80).state_dict(), tmp_path / "model.ckpt")
    train, in_test, out_test = make_sets(80, 5)
    for name, d in (("train", train), ("in_test", in_test), ("out_test", out_test)):
        with open(tmp_path / f"{name}.pkl", "wb") as f:
            pickle.dump(d, f)
        with open(tmp_path / f"{name}_samples_128.json", "w") as f:
            json.dump([[u, 0] for u in sorted(d) if len(d[u]) >= 128][:4], f)
    if ROOT not in sys.path:
        sys.path.insert(0, ROOT)
    import evaluate as cli
    base = ["-c", str(tmp_path / "config.yaml"), "-m", str(tmp_path / "model.ckpt"), "-d", str(tmp_path), "-spk",
            "-seed", "2"]
    cli.main(base + ["-o", str(tmp_path / "plain.json")])
    cli.main(base + ["-probe", "-probe_utts", "4", "-o", str(tmp_path / "probe.json")])
    plain, probe = (json.loads((tmp_path / n).read_text()) for n in ("plain.json", "probe.json"))
    entries = {s: probe[s].pop("probe") for s in ("in_test", "out_test")}
    assert json.dumps(probe, indent=1) == (tmp_path / "plain.json").read_text()
    assert entries["in_test"]["n"] == 12 and entries["out_test"]["n_unseen"] == 6
    assert entries["in_test"]["n_fit"] == len(P.probe_utterances({u: len(v) for u, v in train.items()}, 17, 4, 2))
