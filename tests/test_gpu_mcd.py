"""GPU: the MCD-DTW evaluation.  avc_mel_cepstrum against float64 (clip included); avc_dtw bit for bit against the
float64 restatement on the device's cepstra, up to the 4096-frame limit; every pair's bits alone and in a shuffled
batch; the self and doubled-copy identities; the shortest inputs AE.inference accepts; and evaluate_mcd end to end:
its conversions against Inferencer.inference_ragged bit for bit, its numbers against the restatement exactly, and
two runs against each other."""
import json

import numpy as np
import pytest
import torch

from _mcd_ref import MCD_SCALE, cepstrum64, dtw64
from adaptive_voice_conversion_b200 import _lib as L
from adaptive_voice_conversion_b200 import mcd as M
from adaptive_voice_conversion_b200.config import default_config

pytestmark = pytest.mark.gpu


def bits_equal(a, b):
    return a.shape == b.shape and a.dtype == b.dtype and torch.equal(a.contiguous().view(torch.uint8), b.contiguous().view(torch.uint8))


def make_attr(n_mels, seed):
    rng = np.random.default_rng(seed)
    return {"mean": rng.uniform(0.3, 0.7, n_mels).astype(np.float32), "std": rng.uniform(0.1, 0.3, n_mels).astype(np.float32)}


def random_mels(lengths, n_mels, seed):
    g = torch.Generator().manual_seed(seed)
    # N(0, 2) frames: with the attr above a good share of the denormalised values lies outside [0, 1]
    return [(2.0 * torch.randn((T, n_mels), generator=g)).cuda() for T in lengths]


# ----------------------------------------------------------------------------- the cepstrum
@pytest.mark.parametrize("n_mels", [80, 512])
@pytest.mark.parametrize("dims", [1, 13, 24, 64])
def test_cepstrum_matches_float64(n_mels, dims):
    attr = make_attr(n_mels, n_mels + dims)
    mels = random_mels([1, 7, 300, 64], n_mels, dims)
    raw = torch.cat(mels).cpu().numpy() * attr["std"] + attr["mean"]
    assert (raw < 0).mean() > 0.05 and (raw > 1).mean() > 0.05
    got = M.mel_cepstrum(mels, attr, dims=dims)
    for m, c in zip(mels, got):
        assert c.shape == (m.shape[0], dims) and c.dtype == torch.float32
        ref = cepstrum64(m.cpu().numpy(), attr["mean"], attr["std"], dims)
        err = np.abs(c.cpu().numpy().astype(np.float64) - ref).max(axis=1) / np.abs(ref).max(axis=1)
        assert err.max() < 1e-5, err.max()
    # a row gets the same bits in any batch
    alone = M.mel_cepstrum([mels[2][5:6]], attr, dims=dims)[0]
    assert bits_equal(alone, got[2][5:6])


# ----------------------------------------------------------------------------- the DTW
LENGTHS = [1, 2, 17, 128, 333, 1000, 2500]


def cepstra(lengths, dims, seed, n_mels=80):
    return M.mel_cepstrum(random_mels(lengths, n_mels, seed), make_attr(n_mels, seed), dims=dims)


@pytest.mark.parametrize("dims", [24, 64])
def test_dtw_is_the_float64_restatement_bit_for_bit(dims):
    xs = cepstra(LENGTHS, dims, 1)
    ys = cepstra(LENGTHS, dims, 2)
    px = [xs[a] for a in range(len(LENGTHS)) for b in range(len(LENGTHS))]
    py = [ys[b] for a in range(len(LENGTHS)) for b in range(len(LENGTHS))]
    got = M.dtw(px, py).cpu().numpy()
    for k, (x, y) in enumerate(zip(px, py)):
        S, Ln = dtw64(x.cpu().numpy(), y.cpu().numpy())
        assert got[k, 0] == S and got[k, 1] == Ln, (x.shape[0], y.shape[0], got[k], S, Ln)


def test_dtw_at_the_4096_frame_limit():
    xs = cepstra([4096, 4100], 24, 3)
    got = M.dtw([xs[0], xs[1]], [xs[1], xs[0]]).cpu().numpy()
    for k, (x, y) in enumerate([(xs[0], xs[1]), (xs[1], xs[0])]):
        S, Ln = dtw64(x.cpu().numpy(), y.cpu().numpy())
        assert got[k, 0] == S and got[k, 1] == Ln
    with pytest.raises(ValueError, match="4097 frames"):
        M.dtw(cepstra([4097], 24, 4), cepstra([4097], 24, 5))


def test_every_pair_gets_the_same_bits_alone_and_in_a_shuffled_batch():
    rng = np.random.default_rng(0)
    lx = [int(v) for v in rng.integers(1, 700, 40)]
    ly = [int(v) for v in rng.integers(1, 700, 40)]
    xs, ys = cepstra(lx, 24, 6), cepstra(ly, 24, 7)
    batch = M.dtw(xs, ys)
    perm = rng.permutation(40)
    shuffled = M.dtw([xs[i] for i in perm], [ys[i] for i in perm])
    assert bits_equal(shuffled, batch[torch.from_numpy(perm).cuda()])
    for i in range(40):
        assert bits_equal(M.dtw([xs[i]], [ys[i]])[0], batch[i])


def test_identities():
    for T in (1, 5, 333):
        x = cepstra([T], 24, T)[0]
        assert M.dtw([x], [x]).cpu().tolist() == [[0.0, float(T)]]
        doubled = x.repeat_interleave(2, dim=0)
        assert M.dtw([x, doubled], [doubled, x]).cpu().tolist() == [[0.0, 2.0 * T], [0.0, 2.0 * T]]


def test_kernel_skips_a_pair_longer_than_the_launch_was_sized_for():
    xs = cepstra([50, 60], 24, 8)
    tab = np.zeros(2, M._PAIR)
    tab["x_off"], tab["y_off"], tab["tx"], tab["ty"] = [0, 0], [0, 0], [50, 50], [50, 60]
    pairs = torch.from_numpy(tab.view(np.uint8)).cuda()
    out = torch.zeros((2, 2), dtype=torch.float64, device="cuda")
    x, y = xs[0].contiguous(), torch.cat(xs).contiguous()
    d = L.DtwDesc(n_pairs=2, dims=24, max_short=49, pairs=pairs.data_ptr(), x=x.data_ptr(), y=y.data_ptr(), out=out.data_ptr())
    L.check(L.load().avc_dtw(d, torch.cuda.current_stream().cuda_stream), "avc_dtw")
    got = out.cpu()
    assert torch.isnan(got[:, 0]).all() and (got[:, 1] == 0).all()


# ----------------------------------------------------------------------------- the shortest inputs
def test_min_frames_is_what_the_engine_accepts():
    from adaptive_voice_conversion_b200.model import AE
    cfg = default_config(80)
    torch.manual_seed(0)
    model = AE(cfg).cuda().eval()
    src, ref = M.min_frames(cfg)
    assert (src, ref) == (17, 9)
    g = torch.Generator().manual_seed(0)
    x = lambda T: torch.randn((1, 80, T), generator=g).cuda()
    assert model.inference(x(src), x(ref)).shape == (1, 80, 24)
    for a, b in ((src - 1, ref), (src, ref - 1)):
        with pytest.raises(L.AvcError):
            model.inference(x(a), x(b))
            torch.cuda.synchronize()


# ----------------------------------------------------------------------------- end to end
SENTENCES = 6


def make_set(n_mels, seed):
    """4 speakers reading SENTENCES shared lines (lines 3 and up skipped now and then) and 2 lines of their own;
    p302_001 is too short to be a source and p303_002 too short for either role; p301's reading of line 0 is p300's
    frames exactly; p302_900 has no transcript."""
    rng = np.random.default_rng(seed)
    data, texts = {}, {}
    for s in range(4):
        for k in range(SENTENCES + 2):
            if 3 <= k < SENTENCES and rng.random() < 0.3:
                continue
            u = f"p{300 + s}_{k:03d}.wav"
            data[u] = rng.standard_normal((int(rng.integers(17, 260)), n_mels)).astype(np.float32)
            texts[u] = f"Line number {k}." if k < SENTENCES else f"Speaker {s}'s own line {k}!"
    data["p302_001.wav"] = data["p302_001.wav"][:10]
    data["p303_002.wav"] = data["p303_002.wav"][:5]
    data["p301_000.wav"] = data["p300_000.wav"].copy()
    data["p302_900.wav"] = rng.standard_normal((90, n_mels)).astype(np.float32)
    return data, texts


def make_model(c_in, sn):
    from adaptive_voice_conversion_b200.model import AE
    cfg = default_config(c_in)
    cfg["Decoder"]["sn"] = sn
    torch.manual_seed(c_in + sn)
    return AE(cfg).cuda()


@pytest.mark.parametrize("c_in", [80, 512])
@pytest.mark.parametrize("sn", [False, True], ids=["plain", "sn"])
def test_evaluate_mcd_end_to_end(tmp_path, c_in, sn):
    from adaptive_voice_conversion_b200.inference import Inferencer
    data, raw_texts = make_set(c_in, c_in + sn)
    tdir = tmp_path / "txt"
    for u, t in raw_texts.items():
        p = tdir / u.split("_")[0] / (u[:-4] + ".txt")
        p.parent.mkdir(parents=True, exist_ok=True)
        p.write_text(t + "\n")
    texts = M.read_transcripts(str(tdir), data)
    assert texts["p300_000.wav"] == "line number 0" and "p302_900.wav" not in texts
    attr = make_attr(c_in, 11)
    model = make_model(c_in, sn)
    model.train()
    buffers = {k: v.clone() for k, v in model.named_buffers()}
    res = M.evaluate_mcd(model, data, attr, texts, per_triplet=True)
    assert model.training and all(bits_equal(v, buffers[k]) for k, v in model.named_buffers())
    trip, n_short = M.parallel_triplets(list(data), texts, {u: len(v) for u, v in data.items()}, 0, 0, 17, 9)
    assert res["n"] == len(trip) > 10 and res["n_short"] == n_short > 0 and res["dims"] == 24
    assert [t[:3] for t in res["triplets"]] == [list(t) for t in trip]

    # the conversions are inference_ragged's, bit for bit
    model.eval()
    inf = Inferencer.__new__(Inferencer)
    inf.config, inf.model, inf.attr = model.config, model, None
    dev = {u: torch.from_numpy(v).cuda() for u, v in data.items()}
    srcs, refs = [dev[s] for s, _, _ in trip], [dev[r] for _, r, _ in trip]
    ragged = [o[: s.shape[0]] for o, s in zip(inf.inference_ragged(srcs, refs), srcs)]
    seen = 0
    for idx, decs in M.converted(model, srcs, refs):
        for i, d in zip(idx, decs):
            assert bits_equal(d.contiguous(), ragged[i].contiguous()), trip[i]
            seen += 1
    assert seen == len(trip)

    # the numbers are the float64 restatement on the device's cepstra, exactly
    conv = M.mel_cepstrum(ragged, attr)
    plain = {u: c.cpu().numpy() for u, c in zip(dev, M.mel_cepstrum(list(dev.values()), attr))}
    rows = []
    for (s, r, g), c in zip(trip, conv):
        S, Ln = dtw64(c.cpu().numpy(), plain[g])
        S0, L0 = dtw64(plain[s], plain[g])
        rows.append((MCD_SCALE * S / Ln, MCD_SCALE * S0 / L0))
    assert [t[3:] for t in res["triplets"]] == [list(r) for r in rows]
    tot = np.float64(0)
    tot0 = np.float64(0)
    for a, b in rows:
        tot += a
        tot0 += b
    assert res["mcd"] == float(tot / len(rows)) and res["mcd_source"] == float(tot0 / len(rows))
    assert sum(v["n"] for v in res["speakers"].values()) == len(trip)
    assert list(res["speakers"]) == list(dict.fromkeys(g.split("_")[0] for _, _, g in trip))
    # identical parallel recordings: no distortion before conversion
    same = [t for t in res["triplets"] if {t[0], t[2]} == {"p300_000.wav", "p301_000.wav"}]
    assert len(same) == 2 and all(t[4] == 0.0 for t in same) and all(t[3] > 0.0 for t in same)

    again = M.evaluate_mcd(model, data, attr, texts, per_triplet=True)
    assert json.dumps(again) == json.dumps(res)
    capped = M.evaluate_mcd(model, data, attr, texts, max_pairs=5, seed=3)
    assert capped["n"] == 5 and "triplets" not in capped
    none = M.evaluate_mcd(model, {u: data[u] for u in data if u.startswith("p300")}, attr, texts)
    assert none == {"n": 0, "n_short": 0, "dims": 24, "speakers": {}}
