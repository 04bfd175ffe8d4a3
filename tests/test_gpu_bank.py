"""GPU: speaker code banks.

* avc_time_sum_varlen against float64 (lengths 1 to 4097 at len_div 8, NaN in every padded frame, sentinels); sum *
  (1.f / L) is avc_time_mean_varlen_fwd's row bit for bit;
* avc_pooled_group_mean bit-identical to avc_time_mean_grouped_fwd on random groupings, and to a sequential float32
  numpy restatement for groups of 1, 64, 65 and 1000 rows (a -0 row included);
* AE.speaker_codes_from_sums(AE.get_speaker_sums(...)) bit-identical to get_speaker_embeddings(groups=) at c_in 80 and
  512, fp32 and TF32 (sn: True once), for a 64-member set spread over 1 to 8 batches in different packings; a
  300-member set within the few-shot tests' bound of the float64 layer restatement;
* avc_spk_identify: scores equal one-member avc_spk_group_mean bit for bit, the tie rule on duplicated rows, ranks
  against literal loops, bad descriptors rejected before any launch, a second launch giving the same bits;
* Inferencer.inference_with_codes bit-identical to inference_padded with sets, graph replay equal to eager, a mix with
  weight 1 on one speaker equal to that speaker's conversion;
* end to end: speaker_bank.py, inference.py -bank -speaker and -pairs with @ fields, evaluate.py -spk -bank against a
  host recomputation from the device scores.
"""
import ctypes as C
import json
import os
import pickle
import subprocess
import sys

import numpy as np
import pytest
import torch

import oracle.ae_oracle as orc
from _sn_ref import sn_config
from adaptive_voice_conversion_b200 import _lib as L
from adaptive_voice_conversion_b200 import speaker_bank as SB
from adaptive_voice_conversion_b200 import speaker_eval as S
from adaptive_voice_conversion_b200.evaluate import speaker_of
from test_gpu_fewshot import _checkpoint, a4, bits_equal, oracle_codes, tol, write_eval_dir
from test_gpu_padded_inference import REL, _inferencer, make_model, padded, relerr

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SENTINEL = -7777.0


@pytest.fixture(params=["fp32", "tf32"])
def precision(request, monkeypatch):
    monkeypatch.setenv("AVC_PRECISION", request.param)
    return request.param


# ----------------------------------------------------------------------------- the pooling kernels
def varlen_batch(seed, B, Cc, div):
    g = torch.Generator().manual_seed(seed)
    lens = torch.randint(1, 4098, (B,), generator=g)
    lens[:3] = torch.tensor([1, 4097, 8])
    T = -(-4097 // div)
    Lm = [-(-int(v) // div) for v in lens]
    x = torch.randn((B, Cc, T), generator=g) + 1.5
    for b in range(B):
        x[b, :, Lm[b]:] = float("nan")
    return x, lens, Lm, T


def sum_varlen(xa, B, Cc, T, lt, div):
    lib = L.load()
    sums = torch.full((B * Cc + 8,), SENTINEL, device="cuda")
    counts = torch.full((B + 2,), -5, dtype=torch.int32, device="cuda")
    assert lib.avc_time_sum_varlen(xa.data_ptr(), xa[0].numel(), sums.data_ptr(), counts.data_ptr(), B, Cc, T, lt.data_ptr(),
                                   div, 1, None) == 0, L.last_error()
    return sums, counts


def test_time_sum_varlen_kernel():
    lib = L.load()
    B, Cc, div = 40, 32, 8
    x, lens, Lm, T = varlen_batch(5, B, Cc, div)
    xa, lt = a4(x), lens.to(torch.int32).cuda()
    s1, c1 = sum_varlen(xa, B, Cc, T, lt, div)
    s2, c2 = sum_varlen(xa, B, Cc, T, lt, div)
    assert torch.equal(s1, s2) and torch.equal(c1, c2)
    s1, c1 = s1.cpu(), c1.cpu()
    assert bool((s1[B * Cc:] == SENTINEL).all()) and c1[B:].tolist() == [-5, -5]
    assert c1[:B].tolist() == Lm
    sums = s1[:B * Cc].view(B, Cc)
    worst = 0.0
    for b in range(B):
        ref = x[b, :, :Lm[b]].double().sum(dim=1)
        worst = max(worst, relerr(sums[b], ref))
    assert worst < 1e-5, worst
    print(f"time_sum_varlen: worst relative error against float64 {worst:.3g}")
    mean = torch.full((B * Cc,), SENTINEL, device="cuda")
    assert lib.avc_time_mean_varlen_fwd(xa.data_ptr(), xa[0].numel(), mean.data_ptr(), B, Cc, T, lt.data_ptr(), div, 1,
                                        None) == 0
    mean = mean.cpu().view(B, Cc)
    inv = torch.tensor([1.0 / np.float32(n) for n in Lm], dtype=torch.float32)
    assert bits_equal((sums * inv[:, None]).numpy(), mean.numpy())
    n0 = L.launch_count()
    for Bx, Cx, Tx, dv in ((0, Cc, T, div), (B, 6, T, div), (B, Cc, 0, div), (B, Cc, T, 0)):
        assert lib.avc_time_sum_varlen(xa.data_ptr(), xa[0].numel(), mean.data_ptr(), c1.data_ptr(), Bx, Cx, Tx,
                                       lt.data_ptr(), dv, 1, None) == L.ERR_INVALID
    assert lib.avc_time_sum_varlen(xa.data_ptr(), xa[0].numel(), None, c1.data_ptr(), B, Cc, T, lt.data_ptr(), div, 1,
                                   None) == L.ERR_INVALID
    assert L.launch_count() == n0


def pooled(sums, counts, offs, Cc):
    lib = L.load()
    G = len(offs) - 1
    out = torch.full((G * Cc + 8,), SENTINEL, device="cuda")
    o = torch.tensor(offs, dtype=torch.int64).cuda()
    assert lib.avc_pooled_group_mean(sums.data_ptr(), counts.data_ptr(), counts.shape[0], Cc, o.data_ptr(), G,
                                     out.data_ptr(), None) == 0, L.last_error()
    out = out.cpu()
    assert bool((out[G * Cc:] == SENTINEL).all())
    return out[:G * Cc].view(G, Cc)


def test_pooled_group_mean_is_grouped_mean():
    lib = L.load()
    B, Cc, div = 64, 32, 8
    x, lens, Lm, T = varlen_batch(9, B, Cc, div)
    xa, lt = a4(x), lens.to(torch.int32).cuda()
    s, c = sum_varlen(xa, B, Cc, T, lt, div)
    sums, counts = s[:B * Cc].view(B, Cc), c[:B].contiguous()
    rng = np.random.default_rng(1)
    for trial in range(6):
        cuts = sorted(rng.choice(np.arange(1, B), size=int(rng.integers(0, 20)), replace=False).tolist())
        offs = [0] + cuts + [B]
        G = len(offs) - 1
        want = torch.full((G * Cc,), SENTINEL, device="cuda")
        o32 = torch.tensor(offs, dtype=torch.int32).cuda()
        assert lib.avc_time_mean_grouped_fwd(xa.data_ptr(), xa[0].numel(), want.data_ptr(), B, Cc, T, lt.data_ptr(), div, 1,
                                             o32.data_ptr(), G, None) == 0
        assert bits_equal(pooled(sums, counts, offs, Cc).numpy(), want.cpu().view(G, Cc).numpy()), trial
    # argument errors before any launch
    o = torch.tensor([0, B], dtype=torch.int64).cuda()
    out = torch.empty(B, Cc, device="cuda")
    n0 = L.launch_count()
    for n, Cx, G in ((0, Cc, 1), (B, 6, 1), (B, Cc, 0), (B, Cc, B + 1)):
        assert lib.avc_pooled_group_mean(sums.data_ptr(), counts.data_ptr(), n, Cx, o.data_ptr(), G, out.data_ptr(),
                                         None) == L.ERR_INVALID
    assert lib.avc_pooled_group_mean(sums.data_ptr(), counts.data_ptr(), B, Cc, None, 1, out.data_ptr(), None) == L.ERR_INVALID
    assert L.launch_count() == n0


def test_pooled_group_mean_sequential_float32():
    rng = np.random.default_rng(3)
    sizes = [1, 64, 65, 1000, 1, 7]
    N, Cc = sum(sizes), 64
    sums = (rng.standard_normal((N, Cc)) * 50).astype(np.float32)
    counts = rng.integers(1, 5000, N).astype(np.int32)
    sums[0, :5] = np.float32(-0.0)      # a one-member group of -0: assigned, so -0 stays -0
    offs = np.concatenate([[0], np.cumsum(sizes)]).tolist()
    got = pooled(torch.from_numpy(sums).cuda(), torch.from_numpy(counts).cuda(), offs, Cc).numpy()
    for g, n in enumerate(sizes):
        a, b = offs[g], offs[g + 1]
        acc = sums[a].copy()
        for m in range(a + 1, b):
            acc = (acc + sums[m]).astype(np.float32)
        inv = np.float32(1.0) / np.float32(int(counts[a:b].sum()))
        assert bits_equal(got[g], (acc * inv).astype(np.float32)), (g, n)
    assert np.signbit(got[0, :5]).all()


# ----------------------------------------------------------------------------- the model
def spread(m, refs, T, batches, order):
    """speaker_sums of refs in `batches` (lists of indices, in `order` within each batch), rows put back in ref order."""
    c_h = m.config["SpeakerEncoder"]["c_h"]
    sums = torch.empty(len(refs), c_h, device="cuda")
    counts = torch.empty(len(refs), dtype=torch.int32, device="cuda")
    for idx in batches:
        idx = [idx[k] for k in order(len(idx))]
        s, c = m.get_speaker_sums(padded([refs[i] for i in idx], T, "nan"),
                                  lengths=torch.tensor([refs[i].shape[1] for i in idx]).cuda())
        rows = torch.tensor(idx).cuda()
        sums.index_copy_(0, rows, s)
        counts.index_copy_(0, rows, c)
    return sums, counts


@pytest.mark.parametrize("cfg_name", ["c80", "c512", "sn"])
def test_codes_from_sums_are_grouped_codes(precision, cfg_name):
    if cfg_name == "sn" and precision == "fp32":
        pytest.skip("sn: True once, in TF32")
    cfg = {"c80": lambda: orc.default_config(80), "c512": lambda: orc.default_config(512), "sn": lambda: sn_config(80)}[cfg_name]()
    c_in = cfg["SpeakerEncoder"]["c_in"]
    m = make_model(cfg)
    g = torch.Generator().manual_seed(c_in)
    lens = torch.randint(9, 600, (64,), generator=g).tolist()
    refs = [torch.randn((c_in, t), generator=g) for t in lens]
    T = 640
    sizes = [1, 20, 3, 40]
    groups = torch.tensor([0] + sizes).cumsum(0)
    with torch.no_grad():
        want = m.get_speaker_embeddings(padded(refs, T, "zeros"), lengths=torch.tensor(lens).cuda(), groups=groups.cuda())
        whole = m.get_speaker_embeddings(padded(refs, T, "zeros"), lengths=torch.tensor(lens).cuda(),
                                         groups=torch.tensor([0, 64]).cuda())
    rng = np.random.default_rng(7)
    for nb in (1, 2, 3, 5, 8):
        perm = rng.permutation(64).tolist()
        cuts = sorted(rng.choice(np.arange(1, 64), size=nb - 1, replace=False).tolist())
        batches = [perm[a:b] for a, b in zip([0] + cuts, cuts + [64])]
        order = (lambda n: list(range(n))) if nb % 2 else (lambda n: list(reversed(range(n))))
        sums, counts = spread(m, refs, T, batches, order)
        codes = m.speaker_codes_from_sums(sums, counts, groups=groups)
        assert bits_equal(codes.cpu().numpy(), want.cpu().numpy()), nb
        one = m.speaker_codes_from_sums(sums, counts, groups=torch.tensor([0, 64]))
        assert bits_equal(one.cpu().numpy(), whole.cpu().numpy()), nb
    with pytest.raises(L.AvcError, match="offsets"):
        m.speaker_codes_from_sums(sums, counts, groups=torch.tensor([0, 63]))
    with pytest.raises(L.AvcError, match="counts"):
        m.speaker_codes_from_sums(sums, counts.long(), groups=torch.tensor([0, 64]))
    m.engine("cuda:0").check_tc_status()


def test_large_set_against_float64(precision):
    cfg = orc.default_config(80)
    m = make_model(cfg)
    g = torch.Generator().manual_seed(300)
    lens = torch.randint(9, 160, (300,), generator=g).tolist()
    refs = [torch.randn((80, t), generator=g) for t in lens]
    batches = [list(range(a, min(a + 64, 300))) for a in range(0, 300, 64)]
    sums, counts = spread(m, refs, 160, batches, lambda n: list(range(n)))
    code = m.speaker_codes_from_sums(sums, counts, groups=torch.tensor([0, 300]))
    err = relerr(code[0], oracle_codes(cfg, refs, [300])[0])
    print(f"300-member code ({precision}): relative error against float64 {err:.3g}")
    assert err < tol(precision, REL, 8e-3)


# ----------------------------------------------------------------------------- identification
def test_identify_against_group_mean():
    rng = np.random.default_rng(11)
    s, m, d = 50, 40, 128
    bank = rng.standard_normal((s, d)).astype(np.float32)
    bank[7] = bank[3]                       # a duplicated row: ties go to the lower index
    bank[20] = 0.0                          # a zero row scores 0
    Q = rng.standard_normal((m, d)).astype(np.float32)
    Q[:5] = bank[[3, 7, 10, 20, 49]]
    targets = rng.integers(0, s, m).astype(np.int32)
    targets[5], targets[6], targets[7] = -1, s, 7
    qd, bd = torch.from_numpy(Q).cuda(), torch.from_numpy(bank).cuda()
    got = S.identify(qd, bd, targets)
    again = S.identify(qd, bd, targets)
    for k in got:
        assert bits_equal(got[k], again[k]), k
    # the score matrix, column by column, from one-member avc_spk_group_mean groups
    score = np.stack([S.group_means(qd, np.zeros(m, np.int32), np.full(m, -1, np.int32), bd[v:v + 1], [0]).cpu().numpy()
                      for v in range(s)], axis=1)
    best = np.argmax(score, axis=1)        # the first maximum: the lowest index among ties
    assert got["best"].tolist() == best.tolist()
    assert got["best"][0] == 3 and got["best"][1] == 3
    assert bits_equal(got["best_score"], score[np.arange(m), best])
    has = (targets >= 0) & (targets < s)
    ts = np.where(has, score[np.arange(m), np.clip(targets, 0, s - 1)], np.nan)
    assert bits_equal(got["target_score"], ts)
    rank = [int(sum(score[i, v] > ts[i] for v in range(s))) if has[i] else -1 for i in range(m)]
    assert got["target_rank"].tolist() == rank
    none = S.identify(qd, bd)
    assert np.isnan(none["target_score"]).all() and (none["target_rank"] == -1).all()
    assert none["best"].tolist() == got["best"].tolist()
    # bad descriptors: nothing launched
    lib = L.load()
    fake = 0x10000
    n0 = L.launch_count()
    base = dict(m=4, s=10, dims=8, queries=fake, bank=fake, q_target=None, best=fake, best_score=fake, target_score=fake,
                target_rank=fake)
    for bad, code in (({"m": 0}, L.ERR_INVALID), ({"s": 0}, L.ERR_INVALID), ({"dims": -1}, L.ERR_INVALID),
                      ({"bank": None}, L.ERR_INVALID), ({"best": None}, L.ERR_INVALID),
                      ({"target_rank": None}, L.ERR_INVALID), ({"s": L.SPK_MAX_N + 1}, L.ERR_UNSUPPORTED),
                      ({"dims": L.SPK_MAX_DIMS + 1}, L.ERR_UNSUPPORTED)):
        desc = L.SpkIdentifyDesc(**dict(base, **bad))
        assert lib.avc_spk_identify(C.byref(desc), None) == code, bad
    assert lib.avc_spk_identify(None, None) == L.ERR_INVALID
    assert L.launch_count() == n0


# ----------------------------------------------------------------------------- conversion with codes
def test_inference_with_codes(precision, monkeypatch):
    cfg = orc.default_config(80)
    inf = _inferencer(cfg)
    g = torch.Generator().manual_seed(17)
    xs = [torch.randn((int(t), 80), generator=g).cuda() for t in torch.randint(17, 301, (20,), generator=g)]
    cs = [torch.randn((int(t), 80), generator=g).cuda() for t in torch.randint(9, 301, (12,), generator=g)]
    sets = [cs[0:3], cs[3:4], cs[4:12]]
    per_pair = [sets[i % 3] for i in range(len(xs))]
    monkeypatch.setenv("AVC_INFER_GRAPH", "1")
    want = inf.inference_padded(xs, per_pair, batch_max=8)
    codes = inf.embed_speakers(sets)
    got = inf.inference_with_codes(xs, codes[torch.tensor([i % 3 for i in range(len(xs))]).cuda()], batch_max=8)
    monkeypatch.setenv("AVC_INFER_GRAPH", "0")
    eager = inf.inference_with_codes(xs, [codes[i % 3] for i in range(len(xs))], batch_max=8)
    for a, b, e in zip(want, got, eager):
        assert bits_equal(a.cpu().numpy(), b.cpu().numpy()) and bits_equal(b.cpu().numpy(), e.cpu().numpy())
    # a bank of three speakers: weight 1 on one speaker is that speaker's conversion
    mels = {f"p{300 + k}_{j:03d}": c for k, s in enumerate(sets) for j, c in enumerate(s)}
    bank = SB.build_bank(inf.model, mels)
    assert bank.speakers == ["p300", "p301", "p302"] and bank.n_utts == [3, 1, 8]
    assert bits_equal(bank.codes.cpu().numpy(), codes.cpu().numpy())     # the sets, packed differently
    monkeypatch.setenv("AVC_INFER_GRAPH", "1")
    one = inf.inference_with_codes(xs[:5], torch.stack([bank.code("p301")] * 5))
    mix = inf.inference_with_codes(xs[:5], torch.stack([bank.code("p300:0,p301:1,p302:0")] * 5))
    for a, b in zip(one, mix):
        assert bits_equal(a.cpu().numpy(), b.cpu().numpy())
    with pytest.raises(ValueError, match="codes must be"):
        inf.inference_with_codes(xs[:2], codes[:1])


# ----------------------------------------------------------------------------- the CLIs, end to end
def write_train(root, n_mels, seed=5):
    """train.pkl: the four speakers of write_eval_dir's in_test, with utterance ids of their own, and one short one."""
    rng = np.random.default_rng(seed)
    data = {f"p{300 + s}_{100 + k:03d}.wav": (rng.standard_normal((int(rng.integers(60, 300)), n_mels)) + 0.3 * s
                                              ).astype(np.float32) for s in range(4) for k in range(9)}
    data["p303_199.wav"] = np.zeros((4, n_mels), np.float32)
    with open(root / "train.pkl", "wb") as f:
        pickle.dump(data, f)
    return data


def test_bank_cli_end_to_end(tmp_path):
    cfg = orc.default_config(80)
    cfg_path, ckpt = _checkpoint(tmp_path, cfg)
    test_data = write_eval_dir(tmp_path, 80)
    train = write_train(tmp_path, 80)
    env = dict(os.environ, PYTHONPATH=ROOT)
    bank_path = str(tmp_path / "bank.pt")
    run = subprocess.run([sys.executable, os.path.join(ROOT, "speaker_bank.py"), "-c", cfg_path, "-m", ckpt, "-d",
                          str(tmp_path), "-set", "train", "-o", bank_path], check=True, env=env, cwd=str(tmp_path),
                         capture_output=True, text=True)
    assert "4 speakers, 36 utterances pooled, 1 skipped" in run.stdout, run.stdout
    inf = _inferencer(cfg)
    bank = SB.SpeakerBank.load(bank_path, inf.model)
    want = SB.build_bank(inf.model, {u: torch.from_numpy(v).cuda() for u, v in train.items()})
    assert bits_equal(bank.codes.cpu().numpy(), want.codes.cpu().numpy())

    rng = np.random.default_rng(1)
    files = {}
    for name, T in (("s1", 140), ("s2", 97), ("c", 230)):
        files[name] = str(tmp_path / f"{name}.npy")
        np.save(files[name], rng.standard_normal((T, 80)).astype(np.float32))
    base = [sys.executable, os.path.join(ROOT, "inference.py"), "-c", cfg_path, "-m", ckpt]
    subprocess.run(base + ["-s", files["s1"], "-bank", bank_path, "-speaker", "p301:0.25,p302:0.75", "-o",
                           str(tmp_path / "t.npy")], check=True, env=env, cwd=str(tmp_path))
    mel = {k: torch.from_numpy(np.load(v)).cuda() for k, v in files.items()}
    one = inf.inference_with_codes([mel["s1"]], bank.code("p301:0.25,p302:0.75")[None])[0]
    assert bits_equal(np.load(tmp_path / "t.npy"), one.cpu().numpy())
    pf = tmp_path / "pairs.txt"
    pf.write_text(f"{files['s1']} @p300 o0.npy\n{files['s2']} @p301:1,p303:1 o1.npy\n{files['s2']} {files['c']} o2.npy\n")
    subprocess.run(base + ["-pairs", str(pf), "-bank", bank_path, "-o", str(tmp_path / "out")], check=True, env=env,
                   cwd=str(tmp_path))
    banked = inf.inference_with_codes([mel["s1"], mel["s2"]], torch.stack([bank.code("p300"), bank.code("p301:1,p303:1")]))
    plain = inf.inference_padded([mel["s2"]], [mel["c"]])
    for k, w in enumerate(banked + plain):
        assert bits_equal(np.load(tmp_path / "out" / f"o{k}.npy"), w.cpu().numpy()), k

    if ROOT not in sys.path:
        sys.path.insert(0, ROOT)
    import evaluate as cli
    ev = ["-c", cfg_path, "-m", ckpt, "-d", str(tmp_path), "-eval_sets", "in_test", "-spk", "-max_pairs", "12"]
    cli.main(ev + ["-o", str(tmp_path / "plain.json")])
    cli.main(ev + ["-bank", bank_path, "-o", str(tmp_path / "bank.json")])
    cli.main(ev + ["-bank", bank_path, "-n_refs", "3", "-o", str(tmp_path / "bank3.json")])
    plain = json.loads((tmp_path / "plain.json").read_text())["in_test"]["spk"]
    withb = json.loads((tmp_path / "bank.json").read_text())["in_test"]["spk"]
    new = {"id_target", "id_source", "id_real", "n_banked", "n_unbanked", "bank_speakers"}
    assert not new & set(plain["conversion"]) and new <= set(withb["conversion"])
    assert {k: v for k, v in withb["conversion"].items() if k not in new} == plain["conversion"]
    assert withb["eer"] == plain["eer"]
    c = withb["conversion"]
    assert c["bank_speakers"] == 4 and c["n_banked"] == c["n"] and c["n_unbanked"] == 0
    k3 = json.loads((tmp_path / "bank3.json").read_text())["in_test"]["spk"]["conversion"]
    assert k3["n_refs"] == 3 and new <= set(k3)

    # the id_* shares against a host recomputation from the device's scores
    from adaptive_voice_conversion_b200.model import AE
    model = AE(cfg).cuda()
    model.load_state_dict(torch.load(ckpt))
    model.eval()
    res = S.evaluate_speakers(model, test_data, max_pairs=12, per_pair=True, bank=bank)["conversion"]
    pairs = [(p[0], p[1]) for p in res["pairs"]]
    dev = {u: torch.from_numpy(v).cuda() for u, v in test_data.items()}
    y = S.converted_embeddings(model, [dev[u] for u, _ in pairs], [dev[r] for _, r in pairs])
    utts = sorted(test_data)
    E = S.representations(model, [dev[u] for u in utts])["speaker"]
    score = np.stack([S.group_means(torch.cat([y, E]), np.zeros(len(pairs) + len(utts), np.int32),
                                    np.full(len(pairs) + len(utts), -1, np.int32), bank.codes[v:v + 1], [0]).cpu().numpy()
                      for v in range(len(bank))], axis=1)
    best = np.argmax(score, axis=1)
    P = len(pairs)
    assert res["id_target"] == float(np.mean(best[:P] == [bank.index(speaker_of(r)) for _, r in pairs]))
    assert res["id_source"] == float(np.mean(best[:P] == [bank.index(speaker_of(u)) for u, _ in pairs]))
    assert res["id_real"] == float(np.mean(best[P:] == [bank.index(speaker_of(u)) for u in utts]))
    print(f"bank identification on random weights: {res['id_target']} {res['id_source']} {res['id_real']}")

    # a bank that pooled evaluated utterances is refused
    leaky = tmp_path / "leaky.pt"
    SB.build_bank(model, {u: dev[u] for u in utts[:5]}).save(str(leaky))
    with pytest.raises(ValueError, match="pooled 5 of the evaluated"):
        cli.main(ev + ["-bank", str(leaky)])
