"""GPU: the speaker measures.  avc_time_stats_varlen bit for bit against the float64 restatement (NaN in the padding,
sentinels around the output, lengths 1 to 4097); avc_spk_eer's scores, counts, EER and threshold bit for bit against
the restatement on the device's own vectors (N from 2 to a few thousand, duplicated and zero vectors), and at the
32 768-vector limit the counts, a permuted set and a second launch; avc_spk_group_mean bit for bit; and
evaluate_speakers end to end (c_in 80 and 512, fp32 and TF32, sn once): the padded representations against unpadded
calls, every number against the restatement, two runs against each other, and a set whose speakers each repeat one mel
(a mel EER of exactly 0)."""
import json

import numpy as np
import pytest
import torch

import _spk_ref as R
from adaptive_voice_conversion_b200 import _lib as L
from adaptive_voice_conversion_b200 import speaker_eval as S
from adaptive_voice_conversion_b200.config import default_config
from adaptive_voice_conversion_b200.evaluate import speaker_of

pytestmark = pytest.mark.gpu

SENTINEL = -7777.0
C_RESULT = 48                        # sizeof(avc_eer_result)
TOL = {"fp32": 2e-5, "tf32": 4e-3}   # a padded sample against its unpadded call (tests/test_gpu_padded_inference.py)


def bits_equal(a, b):
    a, b = np.ascontiguousarray(a), np.ascontiguousarray(b)
    return a.shape == b.shape and a.dtype == b.dtype and a.tobytes() == b.tobytes()


def relerr(a, b):
    a, b = a.detach().float().cpu(), b.detach().float().cpu()
    return float((a - b).abs().max() / (b.abs().max() + 1e-12))


# ----------------------------------------------------------------------------- pooling
@pytest.mark.parametrize("C", [80, 128, 512])
def test_time_stats_bit_for_bit_with_nan_padding_and_sentinels(C):
    lens = [1, 2, 3, 4, 17, 100, 1023, 4097]
    T = 4097
    g = torch.Generator().manual_seed(C)
    x = torch.randn((len(lens), C, T), generator=g) * 3 + 0.5
    for b, n in enumerate(lens):
        x[b, :, n:] = float("nan")
    xd = x.cuda()
    buf = torch.full((len(lens) * 2 * C + 64,), SENTINEL, device="cuda")
    lx = torch.tensor(lens, dtype=torch.int32, device="cuda")
    L.check(L.load().avc_time_stats_varlen(xd.data_ptr(), buf[32:].data_ptr(), len(lens), C, T, lx.data_ptr(),
                                           torch.cuda.current_stream().cuda_stream), "avc_time_stats_varlen")
    got = buf.cpu().numpy()
    assert (got[:32] == SENTINEL).all() and (got[32 + len(lens) * 2 * C:] == SENTINEL).all()
    got = got[32:32 + len(lens) * 2 * C].reshape(len(lens), 2 * C)
    for b, n in enumerate(lens):
        assert bits_equal(got[b], R.pool64(x[b].numpy(), n)), (b, n)
    assert bits_equal(S.time_stats(xd, lens).cpu().numpy(), got)
    with pytest.raises(ValueError, match="lengths"):
        S.time_stats(xd, [0] + lens[1:])
    with pytest.raises(ValueError, match="lengths"):
        S.time_stats(xd, lens[:-1] + [T + 1])


# ----------------------------------------------------------------------------- scores and the EER
def vector_set(n, d, n_spk, seed, dup=0, zeros=0):
    """[n, d] float32 vectors with a speaker offset each (so the EER is neither 0 nor 0.5), `dup` rows copied from
    others (ties) and `zeros` zero rows; labels [n]."""
    rng = np.random.default_rng(seed)
    labels = rng.integers(0, n_spk, n).astype(np.int32)
    centres = rng.standard_normal((n_spk, d)) * 0.7 * d ** -0.25     # a target cosine of about 0.5 / sqrt(d)
    V = (centres[labels] + rng.standard_normal((n, d))).astype(np.float32)
    for k in range(dup):
        i, j = rng.integers(0, n, 2)
        V[i], labels[i] = V[j], labels[j] if k % 2 else labels[i]
    V[rng.choice(n, zeros, replace=False)] = 0.0
    return V, labels


def check_eer(V, labels):
    Vd = torch.from_numpy(V).cuda()
    ws = S.eer_workspace(len(V), "cuda")
    got = S.eer(Vd, labels, ws)
    S_ = R.scores64(V)
    dev = S.trial_scores(ws, len(V))
    iu = np.triu_indices(len(V), 1)
    assert bits_equal(dev[iu], S_[iu])
    assert bits_equal(S_[iu], S_.T[iu])
    ref = R.eer64(*R.trials(S_, labels))
    assert got == ref, (got, ref)
    return got


@pytest.mark.parametrize("n,d", [(2, 128), (3, 128), (64, 128), (65, 256), (300, 128), (2000, 128), (700, 256),
                                 (257, 1024), (40, 2048)])
def test_eer_is_the_restatement_bit_for_bit(n, d):
    V, labels = vector_set(n, d, max(2, n // 20), n + d, dup=n // 10, zeros=min(2, n - 1))
    r = check_eer(V, labels)
    if n >= 64:
        assert r["eer"] is not None and 0.0 < r["eer"] < 0.5


def test_eer_ties_and_nulls():
    # every vector one of three: a few distinct scores, heavy ties
    rng = np.random.default_rng(5)
    base = rng.standard_normal((3, 16)).astype(np.float32)
    pick = rng.integers(0, 3, 150)
    V = base[pick]
    labels = (pick + (rng.random(150) < 0.3)).astype(np.int32) % 3
    check_eer(V, labels)
    check_eer(np.zeros((30, 8), np.float32), np.arange(30) % 4)          # all scores 0
    one = check_eer(V[:20], np.zeros(20, np.int32))                        # one speaker
    assert one["eer"] is None and one["n_nontarget"] == 0 and one["n_target"] == 190
    two = check_eer(V[:2], np.array([0, 1], np.int32))                     # two utterances
    assert two["eer"] is None and two["n_target"] == 0 and two["n_nontarget"] == 1
    single = S.eer(torch.from_numpy(V[:1]).cuda(), [0])
    assert single["n_target"] == single["n_nontarget"] == 0 and single["eer"] is None


def test_eer_at_the_size_limit():
    n = L.SPK_MAX_N
    V, labels = vector_set(n, 128, 400, 9)
    Vd = torch.from_numpy(V).cuda()
    res = torch.empty(2, C_RESULT, dtype=torch.uint8, device="cuda")
    ws = S.eer_workspace(n, "cuda")
    lab = torch.from_numpy(labels).cuda()
    for k in range(2):
        L.check(L.load().avc_spk_eer(Vd.data_ptr(), lab.data_ptr(), n, 128, ws.data_ptr(), ws.numel(), res[k].data_ptr(),
                                     torch.cuda.current_stream().cuda_stream), "avc_spk_eer")
    assert torch.equal(res[0], res[1])
    got = S.eer(Vd, labels, ws)
    counts = np.bincount(labels).astype(np.int64)
    assert got["n_target"] + got["n_nontarget"] == n * (n - 1) // 2
    assert got["n_target"] == int((counts * (counts - 1) // 2).sum())
    assert 0.0 < got["eer"] < 0.5
    perm = np.random.default_rng(1).permutation(n)
    again = S.eer(torch.from_numpy(V[perm]).cuda(), labels[perm], ws)
    assert again == got
    del ws
    with pytest.raises(ValueError, match="vectors"):
        S.eer(torch.zeros(n + 1, 4, device="cuda"), np.zeros(n + 1, np.int32))


def test_permuted_set_gives_the_same_bits():
    V, labels = vector_set(500, 128, 20, 3, dup=30, zeros=2)
    a = S.eer(torch.from_numpy(V).cuda(), labels)
    perm = np.random.default_rng(2).permutation(500)
    b = S.eer(torch.from_numpy(V[perm]).cuda(), labels[perm])
    assert a == b


def test_group_means_are_the_restatement_bit_for_bit():
    V, labels = vector_set(300, 128, 7, 11, dup=10, zeros=1)
    rng = np.random.default_rng(4)
    Q = np.concatenate([rng.standard_normal((20, 128)).astype(np.float32), V[:5], np.zeros((1, 128), np.float32)])
    ql = rng.integers(0, 8, len(Q)).astype(np.int32)                     # label 7: no member -> NaN
    qe = rng.integers(-1, 300, len(Q)).astype(np.int32)
    qe[:5] = [int(np.nonzero(labels == ql[k])[0][0]) if (labels == ql[k]).any() else -1 for k in range(5)]
    got = S.group_means(torch.from_numpy(Q).cuda(), ql, qe, torch.from_numpy(V).cuda(), labels).cpu().numpy()
    ref = np.array([R.group_mean64(Q[m], ql[m], qe[m], V, labels) for m in range(len(Q))])
    assert bits_equal(got, ref)
    assert np.isnan(got[ql == 7]).all() and (ql == 7).any()


# ----------------------------------------------------------------------------- end to end
def make_set(n_mels, seed, repeat=False):
    """6 speakers with 2 to 6 utterances of 10 to 300 frames (some too short to be embedded), one speaker with a single
    utterance.  repeat: every utterance of a speaker is that speaker's first mel."""
    rng = np.random.default_rng(seed)
    data = {}
    for s in range(6):
        first = None
        for k in range(int(rng.integers(2, 7))):
            T = int(rng.choice([10, 17, 18, 40, 101, 300]))
            m = (rng.standard_normal((T, n_mels)) + 0.3 * s).astype(np.float32)
            if repeat:
                first = m if first is None else first
                m = first
            data[f"p{300 + s}_{k:03d}.wav"] = m
    data["p399_001.wav"] = rng.standard_normal((50, n_mels)).astype(np.float32)
    return data


def make_model(c_in, sn, monkeypatch, precision):
    from adaptive_voice_conversion_b200.model import AE
    monkeypatch.setenv("AVC_PRECISION", precision)
    cfg = default_config(c_in)
    cfg["Decoder"]["sn"] = sn
    torch.manual_seed(c_in + sn)
    return AE(cfg).cuda()


@pytest.mark.parametrize("c_in,sn,precision", [(80, False, "fp32"), (80, False, "tf32"), (512, False, "fp32"),
                                               (512, False, "tf32"), (80, True, "tf32")])
def test_evaluate_speakers_end_to_end(monkeypatch, c_in, sn, precision):
    from adaptive_voice_conversion_b200.model import _ContentFn
    data = make_set(c_in, c_in + sn)
    model = make_model(c_in, sn, monkeypatch, precision)
    model.train()
    res = S.evaluate_speakers(model, data, per_pair=True)
    assert model.training
    utts = [u for u in sorted(data) if len(data[u]) >= 17]
    assert res["n_utts"] == len(utts) and res["n_short"] == len(data) - len(utts) > 0

    model.eval()
    mels = [torch.from_numpy(data[u]).cuda() for u in utts]
    reps = S.representations(model, mels)
    speakers = sorted({speaker_of(u) for u in utts})
    labels = np.array([speakers.index(speaker_of(u)) for u in utts], np.int32)
    # the padded representations against unpadded calls
    tol = TOL[precision]
    with torch.no_grad():
        for i, m in enumerate(mels):
            x = m.t().contiguous()[None]
            assert relerr(reps["speaker"][i], model.get_speaker_embeddings(x)[0]) < tol, utts[i]
            mu, _ = _ContentFn.apply(model, x, *model._params("content_encoder."))
            lat = -(-m.shape[0] // 8)
            assert relerr(reps["content"][i], S.time_stats(mu[:, :, :lat].contiguous(), [lat])[0]) < tol, utts[i]
            assert bits_equal(reps["mel"][i].cpu().numpy(), R.pool64(data[utts[i]].T, m.shape[0]))
    # every number is the restatement on the device's vectors
    for k in S.REPRESENTATIONS:
        V = reps[k].cpu().numpy()
        assert res["eer"][k] == R.eer64(*R.trials(R.scores64(V), labels)), k
    lengths = {u: len(v) for u, v in data.items()}
    pairs, n_short = S.conversion_pairs(list(data), lengths, 0, 0, 17, 9, 17)
    conv = res["conversion"]
    assert conv["n"] == len(pairs) > 10 and conv["n_short"] == n_short
    assert [p[:2] for p in conv["pairs"]] == [list(p) for p in pairs]
    dev = {u: torch.from_numpy(v).cuda() for u, v in data.items()}
    y = S.converted_embeddings(model, [dev[u] for u, _ in pairs], [dev[r] for _, r in pairs]).cpu().numpy()
    E = reps["speaker"].cpu().numpy()
    idx = {u: i for i, u in enumerate(utts)}
    rows = []
    for (u, r), yv in zip(pairs, y):
        st = R.group_mean64(yv, speakers.index(speaker_of(r)), idx.get(r, -1), E, labels)
        ss = R.group_mean64(yv, speakers.index(speaker_of(u)), idx[u], E, labels)
        sts = R.group_mean64(E[idx[u]], speakers.index(speaker_of(r)), idx.get(r, -1), E, labels)
        rows.append([st, ss, float(st > ss), sts])
    assert [p[2:] for p in conv["pairs"]] == [[a, b, bool(c), d] for a, b, c, d in rows]
    tot = np.zeros(4)
    for row in rows:
        tot = tot + np.array(row)
    assert [conv[k] for k in ("sim_target", "sim_source", "success", "sim_target_source")] == list(tot / len(rows))
    assert sum(v["n"] for v in conv["speakers"].values()) == len(pairs)
    # two runs, the same JSON
    assert json.dumps(S.evaluate_speakers(model, data, per_pair=True)) == json.dumps(res)
    capped = S.evaluate_speakers(model, data, max_pairs=4, seed=3)
    assert capped["conversion"]["n"] == 4 and "pairs" not in capped["conversion"]


def test_repeated_mels_give_a_mel_eer_of_zero(monkeypatch):
    data = make_set(80, 5, repeat=True)
    model = make_model(80, False, monkeypatch, "tf32")
    res = S.evaluate_speakers(model, data)
    assert res["eer"]["mel"]["eer"] == 0.0 and res["eer"]["mel"]["frr"] == 0.0 and res["eer"]["mel"]["far"] == 0.0
    assert res["eer"]["mel"]["n_target"] > 0
