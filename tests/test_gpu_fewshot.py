"""GPU: few-shot conversion, a speaker code pooled over several references of the target speaker.

* avc_time_mean_grouped_fwd against a float64 restatement (groups of 1, 2, 7 and 64 members, lengths 1 to 4097 at
  len_div 8, NaN in every padded frame, sentinels around out, two launches giving the same bits); a one-member group
  is avc_time_mean_varlen_fwd's row bit for bit;
* avc_spk_group_mean_multi against literal loops (n_exclude 1, 3 and 64, duplicate and out-of-range entries), and
  n_exclude = 1 giving avc_spk_group_mean's bits;
* AE.get_speaker_embeddings(groups=) in fp32 and TF32 at c_in 80 and 512: against the float64 oracle's speaker-encoder
  layers run per reference, pooled over the union of the valid frames, then dense; one-member groups bit-identical to
  the rows of get_speaker_embeddings(lengths=); permuting whole groups permutes the rows bit for bit;
* AE.inference_from_embeddings bit-identical to AE.inference, unpadded and padded (once with sn: True);
* Inferencer.inference_padded with reference sets: graph replay against eager, no capture on a second call, one-element
  sets within the padded path's bound of the single-reference call;
* inference.py -t with several files and -pairs with sets against the Python API; evaluate.py -n_refs 1 against a run
  without the flag; n_refs 3 against a float64 recomputation.
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
import torch.nn.functional as F

import _spk_ref as R
import oracle.ae_oracle as orc
from _sn_ref import sn_config
from adaptive_voice_conversion_b200 import _lib as L
from adaptive_voice_conversion_b200 import speaker_eval as S
from adaptive_voice_conversion_b200.evaluate import speaker_of
from test_gpu_padded_inference import REL, TOL_FP32, TOL_TF32, _inferencer, make_model, padded, relerr

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SENTINEL = -7777.0


@pytest.fixture(params=["fp32", "tf32"])
def precision(request, monkeypatch):
    monkeypatch.setenv("AVC_PRECISION", request.param)
    return request.param


def tol(precision, fp32, tf32):
    return fp32 if precision == "fp32" else tf32


def bits_equal(a, b):
    a, b = np.ascontiguousarray(a), np.ascontiguousarray(b)
    return a.shape == b.shape and a.dtype == b.dtype and a.tobytes() == b.tobytes()


def a4(x):
    """planar [B][C][T] -> A4 [B][C/4][T][4] on the device, bit-exact."""
    B, Cc, T = x.shape
    return x.reshape(B, Cc // 4, 4, T).permute(0, 1, 3, 2).contiguous().cuda()


# ----------------------------------------------------------------------------- the kernels
def test_grouped_time_mean_kernel():
    lib = L.load()
    g = torch.Generator().manual_seed(21)
    sizes = [1, 2, 7, 64, 1, 7]
    B, Cc, div = sum(sizes), 32, 8
    lens = torch.randint(1, 4098, (B,), generator=g)
    lens[:3] = torch.tensor([1, 4097, 8])
    T = -(-4097 // div)
    Lm = [-(-int(v) // div) for v in lens]
    x = torch.randn((B, Cc, T), generator=g) + 1.5
    for b in range(B):
        x[b, :, Lm[b]:] = float("nan")
    xa, lt = a4(x), lens.to(torch.int32).cuda()
    offs = torch.tensor([0] + sizes).cumsum(0).to(torch.int32).cuda()
    G = len(sizes)
    outs = []
    for _ in range(2):
        out = torch.full((G * Cc + 8,), SENTINEL, device="cuda")
        assert lib.avc_time_mean_grouped_fwd(xa.data_ptr(), xa[0].numel(), out.data_ptr(), B, Cc, T, lt.data_ptr(), div, 1,
                                             offs.data_ptr(), G, None) == 0, L.last_error()
        outs.append(out.cpu())
    assert torch.equal(outs[0], outs[1])
    out = outs[0]
    assert bool((out[G * Cc:] == SENTINEL).all())
    x64, row = x.double(), 0
    for gi, n in enumerate(sizes):
        ref = sum(x64[m, :, :Lm[m]].sum(dim=1) for m in range(row, row + n)) / sum(Lm[row:row + n])
        assert relerr(out[gi * Cc:(gi + 1) * Cc], ref) < 1e-5, (gi, n)   # float32 sums of up to 33 000 frames
        row += n
    # one-member groups: avc_time_mean_varlen_fwd's rows bit for bit
    single = torch.full((B * Cc,), SENTINEL, device="cuda")
    assert lib.avc_time_mean_varlen_fwd(xa.data_ptr(), xa[0].numel(), single.data_ptr(), B, Cc, T, lt.data_ptr(), div, 1,
                                        None) == 0
    single = single.cpu().view(B, Cc)
    assert torch.equal(out[:Cc], single[0]) and torch.equal(out[4 * Cc:5 * Cc], single[sum(sizes[:4])])
    ones = torch.arange(B + 1, dtype=torch.int32).cuda()
    every = torch.full((B * Cc,), SENTINEL, device="cuda")
    assert lib.avc_time_mean_grouped_fwd(xa.data_ptr(), xa[0].numel(), every.data_ptr(), B, Cc, T, lt.data_ptr(), div, 1,
                                         ones.data_ptr(), B, None) == 0
    assert torch.equal(every.cpu().view(B, Cc), single)
    # argument errors before any launch
    n0 = L.launch_count()
    for args in ((B, Cc, T, 0), (B, Cc, T, B + 1), (B, 6, T, G), (0, Cc, T, 1)):
        Bx, Cx, Tx, Gx = args
        assert lib.avc_time_mean_grouped_fwd(xa.data_ptr(), xa[0].numel(), out.data_ptr(), Bx, Cx, Tx, lt.data_ptr(), div,
                                             1, offs.data_ptr(), Gx, None) == L.ERR_INVALID, args
    assert lib.avc_time_mean_grouped_fwd(xa.data_ptr(), xa[0].numel(), out.data_ptr(), B, Cc, T, lt.data_ptr(), div, 1,
                                         None, G, None) == L.ERR_INVALID
    assert L.launch_count() == n0


def group_mean_multi64(q, q_label, ex, V, labels):
    """Mean of s(q, V[v]) over v with labels[v] == q_label and v not in ex, ascending v (the literal loop)."""
    keep = [v for v in range(len(V)) if labels[v] == q_label and v not in set(int(e) for e in ex)]
    if not keep:
        return float("nan")
    # group_mean64 with one exclusion skips nothing when given -1: restrict the set instead, keeping the order
    return R.group_mean64(q, q_label, -1, V[keep], labels[keep])


@pytest.mark.parametrize("n_ex", [1, 3, 64])
def test_group_mean_multi(n_ex):
    rng = np.random.default_rng(n_ex)
    n, d = 300, 128
    V = rng.standard_normal((n, d)).astype(np.float32)
    labels = rng.integers(0, 6, n).astype(np.int32)
    Q = np.concatenate([rng.standard_normal((12, d)).astype(np.float32), V[:4]])
    ql = rng.integers(0, 7, len(Q)).astype(np.int32)          # label 6: no member -> NaN
    ex = rng.integers(-5, n + 5, (len(Q), n_ex)).astype(np.int32)
    ex[:, 0] = [int(np.nonzero(labels == ql[m])[0][0]) if (labels == ql[m]).any() else -1 for m in range(len(Q))]
    if n_ex > 1:
        ex[:, 1] = ex[:, 0]                                     # a duplicate
        ex[0] = np.nonzero(labels == ql[0])[0][:n_ex].tolist() + [-1] * max(0, n_ex - int((labels == ql[0]).sum()))
    got = S.group_means(torch.from_numpy(Q).cuda(), ql, torch.from_numpy(ex), torch.from_numpy(V).cuda(), labels)
    got = got.cpu().numpy()
    ref = np.array([group_mean_multi64(Q[m], ql[m], ex[m], V, labels) for m in range(len(Q))])
    assert bits_equal(got, ref)
    if n_ex == 1:
        one = S.group_means(torch.from_numpy(Q).cuda(), ql, ex[:, 0], torch.from_numpy(V).cuda(), labels).cpu().numpy()
        assert bits_equal(got, one)
    lib = L.load()
    fake = 0x10000
    desc = L.SpkGroupDesc(m=4, n=10, dims=8, queries=fake, q_labels=fake, q_exclude=fake, set=fake, labels=fake, out=fake)
    n0 = L.launch_count()
    for k in (0, 65):
        assert lib.avc_spk_group_mean_multi(C.byref(desc), k, None) == L.ERR_INVALID and "n_exclude" in L.last_error()
    assert L.launch_count() == n0


# ----------------------------------------------------------------------------- the model
def oracle_codes(cfg, refs, sizes):
    """float64: the oracle's speaker-encoder conv layers per reference, pooled over the union of each group's frames,
    then its dense layers."""
    sd = {k: v.double() for k, v in orc.init_state(cfg, 0).items()}
    p, sub = "speaker_encoder", cfg["SpeakerEncoder"]["subsample"]
    feats = []
    for r in refs:
        out = orc.conv_bank_cat(r[None].double(), sd, p, orc._count(sd, p + ".conv_bank.{}.weight"))
        out = F.relu(orc.reflect_conv1d(out, sd[f"{p}.in_conv_layer.weight"], sd[f"{p}.in_conv_layer.bias"]))
        for l, s in enumerate(sub):
            y = F.relu(orc.reflect_conv1d(out, sd[f"{p}.first_conv_layers.{l}.weight"], sd[f"{p}.first_conv_layers.{l}.bias"]))
            y = F.relu(orc.reflect_conv1d(y, sd[f"{p}.second_conv_layers.{l}.weight"], sd[f"{p}.second_conv_layers.{l}.bias"],
                                          stride=s))
            if s > 1:
                out = F.avg_pool1d(out, kernel_size=s, ceil_mode=True)
            out = y + out
        feats.append(out[0])
    codes, row = [], 0
    for n in sizes:
        h = torch.cat(feats[row:row + n], dim=1).mean(dim=1)[None]
        row += n
        for l in range(orc._count(sd, p + ".first_dense_layers.{}.weight")):
            y = F.relu(F.linear(h, sd[f"{p}.first_dense_layers.{l}.weight"], sd[f"{p}.first_dense_layers.{l}.bias"]))
            y = F.relu(F.linear(y, sd[f"{p}.second_dense_layers.{l}.weight"], sd[f"{p}.second_dense_layers.{l}.bias"]))
            h = y + h
        codes.append(F.linear(h, sd[f"{p}.output_layer.weight"], sd[f"{p}.output_layer.bias"])[0])
    return torch.stack(codes)


@pytest.mark.parametrize("c_in", [80, 512])
def test_grouped_speaker_embeddings(precision, c_in):
    cfg = orc.default_config(c_in)
    m = make_model(cfg)
    g = torch.Generator().manual_seed(c_in)
    sizes = [1, 3, 2, 1, 5]
    lens = [9, 145, 33, 600, 301, 17, 128, 77, 129, 200, 450, 60]
    refs = [torch.randn((c_in, t), generator=g) for t in lens]
    T = 640
    lc = torch.tensor(lens).cuda()
    offs = torch.tensor([0] + sizes).cumsum(0).cuda()
    with torch.no_grad():
        codes = m.get_speaker_embeddings(padded(refs, T, "nan"), lengths=lc, groups=offs)
        rows = m.get_speaker_embeddings(padded(refs, T, "noise"), lengths=lc)
    assert codes.shape == (len(sizes), cfg["SpeakerEncoder"]["c_out"])
    ref = oracle_codes(cfg, refs, sizes)
    for gi in range(len(sizes)):
        assert relerr(codes[gi], ref[gi]) < tol(precision, REL, 8e-3), gi
    # one-member groups are the rows of the lengths call
    assert torch.equal(codes[0], rows[0]) and torch.equal(codes[3], rows[6])
    # permuting whole groups permutes the codes
    order = [4, 0, 3, 1, 2]
    starts = [sum(sizes[:k]) for k in range(len(sizes))]
    perm = [starts[k] + j for k in order for j in range(sizes[k])]
    poffs = torch.tensor([0] + [sizes[k] for k in order]).cumsum(0).cuda()
    with torch.no_grad():
        pc = m.get_speaker_embeddings(padded([refs[i] for i in perm], T, "zeros"), lengths=lc[perm], groups=poffs)
    assert torch.equal(pc, codes[order])
    # lengths=None with groups: every row full length
    with torch.no_grad():
        full = m.get_speaker_embeddings(padded(refs[:3], 145), groups=torch.tensor([0, 1, 3]))
        one = m.get_speaker_embeddings(padded(refs[:1], 145))
    assert relerr(full[0], one[0]) < tol(precision, TOL_FP32, TOL_TF32)
    m.engine("cuda:0").check_tc_status()


@pytest.mark.parametrize("cfg_name,prec", [("c80", "fp32"), ("c80", "tf32"), ("c512", "tf32"), ("sn", "tf32")])
def test_inference_from_embeddings_is_inference(monkeypatch, cfg_name, prec):
    monkeypatch.setenv("AVC_PRECISION", prec)
    cfg = {"c80": lambda: orc.default_config(80), "c512": lambda: orc.default_config(512), "sn": lambda: sn_config(80)}[cfg_name]()
    m = make_model(cfg)
    n_mels = cfg["SpeakerEncoder"]["c_in"]
    g = torch.Generator().manual_seed(3)
    x, c = torch.randn((3, n_mels, 200), generator=g).cuda(), torch.randn((3, n_mels, 150), generator=g).cuda()
    lx, lc = torch.tensor([17, 200, 131]), torch.tensor([9, 150, 64]).cuda()
    with torch.no_grad():
        a = m.inference(x, c)
        b = m.inference_from_embeddings(x, m.get_speaker_embeddings(c))
        pa = m.inference(x, c, lengths=lx, cond_lengths=lc)
        pb = m.inference_from_embeddings(x, m.get_speaker_embeddings(c, lengths=lc), lengths=lx)
    assert torch.equal(a, b) and torch.equal(pa, pb)
    with pytest.raises(L.AvcError):
        m.inference_from_embeddings(x, torch.zeros(2, 128, device="cuda"))


def test_inference_padded_with_sets(precision, monkeypatch):
    cfg = orc.default_config(80)
    inf = _inferencer(cfg)
    g = torch.Generator().manual_seed(13)
    src = torch.randint(100, 301, (30,), generator=g).tolist() + [17, 129]
    ref = torch.randint(100, 301, (40,), generator=g).tolist() + [9, 600]
    xs = [torch.randn((t, 80), generator=g).cuda() for t in src]
    cs = [torch.randn((t, 80), generator=g).cuda() for t in ref]
    shared = cs[:3]
    sets = [shared if i % 4 == 0 else cs[i % 40:i % 40 + 1 + i % 5] for i in range(len(xs))]
    monkeypatch.setenv("AVC_INFER_GRAPH", "1")
    got = inf.inference_padded(xs, sets, batch_max=16)
    caps = inf.padded_captures
    assert caps > 0
    again = inf.inference_padded(xs, sets, batch_max=16)
    assert inf.padded_captures == caps
    monkeypatch.setenv("AVC_INFER_GRAPH", "0")
    eager = inf.inference_padded(xs, sets, batch_max=16)
    for a, b, e in zip(got, again, eager):
        assert torch.equal(a, b) and torch.equal(a, e)
    # a pair's conversion is inference_from_embeddings with its set's code
    codes = inf.embed_speakers([sets[0], sets[1]])
    with torch.no_grad():
        for i, k in ((0, 0), (1, 1)):
            want = inf.model.inference_from_embeddings(xs[i].t()[None].contiguous(), codes[k:k + 1])[0].t()
            assert relerr(got[i], want) < tol(precision, TOL_FP32, TOL_TF32), i
    # one-element sets: the single-reference call within the padded path's bound
    monkeypatch.setenv("AVC_INFER_GRAPH", "1")
    single = inf.inference_padded(xs, cs[:len(xs)])
    ones = inf.inference_padded(xs, [[c] for c in cs[:len(xs)]])
    for i, (a, b) in enumerate(zip(ones, single)):
        assert a.shape == b.shape and relerr(a, b) < tol(precision, TOL_FP32, TOL_TF32), i
    with pytest.raises(ValueError, match="set 0 has 65"):
        inf.embed_speakers([cs[:1] * 65])


# ----------------------------------------------------------------------------- the CLIs
def _checkpoint(tmp_path, cfg):
    import yaml
    from adaptive_voice_conversion_b200.model import AE
    cfg_path = tmp_path / "config.yaml"
    cfg_path.write_text(yaml.safe_dump(cfg))
    m = AE(cfg)
    m.load_state_dict(orc.init_state(cfg, seed=0))
    torch.save(m.state_dict(), tmp_path / "model.ckpt")
    return str(cfg_path), str(tmp_path / "model.ckpt")


def test_inference_cli_with_sets(tmp_path):
    cfg = orc.default_config(80)
    cfg_path, ckpt = _checkpoint(tmp_path, cfg)
    rng = np.random.default_rng(0)
    files = {}
    for name, T in (("s1", 140), ("s2", 97), ("a", 120), ("b", 61), ("c", 230)):
        files[name] = str(tmp_path / f"{name}.npy")
        np.save(files[name], rng.standard_normal((T, 80)).astype(np.float32))
    env = dict(os.environ, PYTHONPATH=ROOT)
    base = [sys.executable, os.path.join(ROOT, "inference.py"), "-c", cfg_path, "-m", ckpt]
    subprocess.run(base + ["-s", files["s1"], "-t", files["a"], files["b"], files["c"], "-o", str(tmp_path / "t.npy")],
                   check=True, env=env, cwd=str(tmp_path))
    pf = tmp_path / "pairs.txt"
    ab = f"{files['a']},{files['b']}"
    pf.write_text(f"{files['s1']} {ab} o0.npy\n{files['s2']} {ab} o1.npy\n{files['s2']} {files['c']} o2.npy\n")
    subprocess.run(base + ["-pairs", str(pf), "-o", str(tmp_path / "out")], check=True, env=env, cwd=str(tmp_path))

    inf = _inferencer(cfg)
    mel = {k: torch.from_numpy(np.load(v)).cuda() for k, v in files.items()}
    _, want = inf.inference_one_utterance(mel["s1"], [mel["a"], mel["b"], mel["c"]])
    assert bits_equal(np.load(tmp_path / "t.npy"), want)
    pair = [mel["a"], mel["b"]]
    sets = inf.inference_padded([mel["s1"], mel["s2"]], [pair, pair])
    one = inf.inference_padded([mel["s2"]], [mel["c"]])
    for k, w in enumerate(sets + one):
        assert bits_equal(np.load(tmp_path / "out" / f"o{k}.npy"), w.cpu().numpy()), k


SENTENCES = 6


def write_eval_dir(root, n_mels, seed=0):
    """A data directory with one parallel set (4 speakers reading SENTENCES shared lines and two of their own), its
    crop index, attr.pkl and transcripts."""
    rng = np.random.default_rng(seed)
    data, txt = {}, root / "txt"
    for s in range(4):
        for k in range(SENTENCES + 2):
            u = f"p{300 + s}_{k:03d}.wav"
            data[u] = (rng.standard_normal((int(rng.integers(130, 260)), n_mels)) + 0.3 * s).astype(np.float32)
            p = txt / u[:4] / (u[:-4] + ".txt")
            p.parent.mkdir(parents=True, exist_ok=True)
            p.write_text(f"Line number {k}.\n" if k < SENTENCES else f"Speaker {s}'s own line {k}.\n")
    with open(root / "in_test.pkl", "wb") as f:
        pickle.dump(data, f)
    with open(root / "in_test_samples_128.json", "w") as f:
        json.dump([[u, 0] for u in sorted(data)[:8]], f)
    with open(root / "attr.pkl", "wb") as f:
        pickle.dump({"mean": rng.standard_normal(n_mels).astype(np.float32) * 0.1 + 0.4,
                     "std": np.abs(rng.standard_normal(n_mels)).astype(np.float32) * 0.1 + 0.2}, f)
    return data


def test_evaluate_n_refs(tmp_path):
    cfg = orc.default_config(80)
    cfg_path, ckpt = _checkpoint(tmp_path, cfg)
    data = write_eval_dir(tmp_path, 80)
    if ROOT not in sys.path:
        sys.path.insert(0, ROOT)
    import evaluate as cli
    base = ["-c", cfg_path, "-m", ckpt, "-d", str(tmp_path), "-eval_sets", "in_test", "-spk", "-mcd", "-transcripts",
            str(tmp_path / "txt"), "-max_pairs", "10"]
    runs = {}
    for k, extra in (("plain", []), ("k1", ["-n_refs", "1"]), ("k3", ["-n_refs", "3"])):
        out = tmp_path / f"{k}.json"
        cli.main(base + extra + ["-o", str(out)])
        runs[k] = out.read_text()
    assert runs["plain"] == runs["k1"]
    plain, k3 = json.loads(runs["plain"])["in_test"], json.loads(runs["k3"])["in_test"]
    assert "n_refs" not in plain["spk"]["conversion"] and "n_few" not in plain["mcd"]
    assert k3["spk"]["conversion"]["n_refs"] == 3 and k3["mcd"]["n_refs"] == 3
    assert k3["spk"]["conversion"]["n"] + k3["spk"]["conversion"]["n_few"] == plain["spk"]["conversion"]["n"]
    assert k3["mcd"]["n"] + k3["mcd"]["n_few"] == plain["mcd"]["n"]
    assert k3["spk"]["eer"] == plain["spk"]["eer"]

    # sim_target of n_refs 3 against a host float64 recomputation from the device's embeddings
    from adaptive_voice_conversion_b200.model import AE
    model = AE(cfg).cuda()
    model.load_state_dict(torch.load(ckpt))
    model.eval()
    res = S.evaluate_speakers(model, data, n_refs=3, per_pair=True, seed=2)
    conv = res["conversion"]
    assert conv["n"] > 5 and all(len(p[1]) == 3 for p in conv["pairs"])
    utts = sorted(data)
    speakers = sorted({speaker_of(u) for u in utts})
    labels = np.array([speakers.index(speaker_of(u)) for u in utts], np.int32)
    dev = {u: torch.from_numpy(v).cuda() for u, v in data.items()}
    E = S.representations(model, [dev[u] for u in utts])["speaker"].cpu().numpy()
    pairs = [(p[0], p[1]) for p in conv["pairs"]]
    y = S.converted_embeddings(model, [dev[u] for u, _ in pairs], [[dev[r] for r in refs] for _, refs in pairs])
    idx = {u: i for i, u in enumerate(utts)}
    for (u, refs), yv, row in zip(pairs, y.cpu().numpy(), conv["pairs"]):
        st = group_mean_multi64(yv, speakers.index(speaker_of(refs[0])), [idx[r] for r in refs], E, labels)
        assert row[2] == st, (u, refs)
        ss = R.group_mean64(yv, speakers.index(speaker_of(u)), idx[u], E, labels)
        assert row[3] == ss and row[4] == bool(st > ss)
