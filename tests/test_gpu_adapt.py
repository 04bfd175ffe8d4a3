"""GPU: speaker adaptation (adaptive_voice_conversion_b200/adapt.py).

1. bit anchor: on B copies of one segment (one speaker code c0 for every sample), the adaptation step with c = c0 gives
   FusedTrainer's decoder gradient slice and dec bit for bit, and AE.forward's dec (bit for bit in fp32, within the TF32
   bound in TF32, where AE.forward re-packs the latent's planar mu and log_sigma rounded to TF32);
2. one step against the float64 oracle (autograd on the decoder and c, encoders detached, then clip_and_adam), fp32 at
   c_in 80 with clipping active and inactive, and once with sn: True;
3. frozen means frozen: every encoder parameter and state_dict entry keeps its bits; the adapted bank loads against the
   adapted model with the base fingerprint;
4. K graph-replayed steps equal K eager steps bit for bit, across epoch boundaries (every batch is full, and every
   step's reported loss equals the eager run's); two runs with one seed give the same checkpoint and code;
5. avc_rec_loss_varlen against a float64 numpy restatement of its summation order, bit for bit;
6. evaluate_mcd(target_codes=) against the default path, per triplet, bit for bit;
7. 200 steps on a seeded synthetic speaker lower the training L1;
8. adapt.py -wav -holdout end to end, then inference.py -bank -speaker against Inferencer.inference_with_codes.
"""
import os
import pickle
import subprocess
import sys
import types

import numpy as np
import pytest
import torch

import oracle.ae_oracle as orc
from _sn_ref import power_iteration64, sn_config
from adaptive_voice_conversion_b200 import _lib as L
from adaptive_voice_conversion_b200 import adapt as A
from adaptive_voice_conversion_b200 import speaker_bank as SB

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
ENC = ("speaker_encoder.", "content_encoder.")


def bits_equal(a, b):
    a, b = np.ascontiguousarray(a), np.ascontiguousarray(b)
    return a.shape == b.shape and a.dtype == b.dtype and a.tobytes() == b.tobytes()


def tbits(a, b):
    return bits_equal(a.detach().cpu().numpy(), b.detach().cpu().numpy())


def rel_l2(a, b):
    a, b = a.detach().double().cpu().flatten(), b.detach().double().cpu().flatten()
    return float((a - b).norm() / (b.norm() + 1e-30))


def make_model(cfg, seed=0):
    from adaptive_voice_conversion_b200.model import AE
    torch.manual_seed(seed)
    m = AE(cfg)        # Decoder.sn: torch's default init, with its u and v
    if not cfg["Decoder"].get("sn", False):
        m.load_state_dict(orc.init_state(cfg, seed=seed), strict=True)
    return m.cuda()


def small_cfg(c_in=80, B=8, sn=False):
    cfg = sn_config(c_in) if sn else orc.default_config(c_in)
    cfg["data_loader"]["batch_size"] = B
    return cfg


@pytest.fixture(params=["fp32", "tf32"])
def precision(request, monkeypatch):
    monkeypatch.setenv("AVC_PRECISION", request.param)
    return request.param


# ----------------------------------------------------------------------------- 1. bit anchor
def test_bit_anchor_against_the_training_step(precision):
    from adaptive_voice_conversion_b200.optim import FusedAdam
    from adaptive_voice_conversion_b200.trainer import FusedTrainer
    cfg = small_cfg(80, 8)
    B = 8
    seg = torch.randn((1, 80, 128), generator=torch.Generator().manual_seed(3))
    x = seg.expand(B, -1, -1).contiguous().cuda()
    eps = torch.randn((B, 128, 16), generator=torch.Generator().manual_seed(4)).cuda()
    ref = make_model(cfg)
    ref.flatten_parameters()
    o = cfg["optimizer"]
    opt = FusedAdam(ref, lr=o["lr"], betas=(o["beta1"], o["beta2"]), amsgrad=o["amsgrad"], weight_decay=o["weight_decay"],
                    max_norm=o["grad_norm"])
    ft = FusedTrainer(ref, opt, cfg)
    _, _, emb, dec_ref = ft.step(x, 1.0, eps=eps, return_outputs=True)
    emb = emb.cpu()
    assert all(tbits(emb[b], emb[0]) for b in range(B))      # B copies of one segment: one code
    n_enc = sum(p.numel() for n, p in ref.named_parameters() if n.startswith(ENC))
    g_ref = opt.flat_g[n_enc:].clone()

    model = make_model(cfg)
    tr = A.make_trainer(model, emb[0], cfg)
    _, _, _, dec = tr.step(x, 0.0, eps=eps, return_outputs=True)
    n_dec = tr.opt.flat_g.numel() - emb.shape[1]
    assert n_dec == g_ref.numel() and tr.code.data_ptr() == tr.opt.flat_p[n_dec:].data_ptr()   # decoder, then c
    assert tbits(tr.opt.flat_g[:n_dec], g_ref)
    assert tbits(dec, dec_ref)
    _, _, _, dec_fwd = make_model(cfg)(x, eps=eps)
    if precision == "fp32":
        assert tbits(dec, dec_fwd)
    else:   # AE.forward hands mu and log_sigma to the decoder as planar tensors and re-packs them rounded to TF32 (as the
        # training step's dec against AE.forward's): test_gpu_model.py's TF32 bound
        err = float((dec - dec_fwd.detach()).abs().max() / dec_fwd.detach().abs().max())
        assert err < 8e-3, err
    tr.eng.check_tc_status()


# ----------------------------------------------------------------------------- 2. against the float64 oracle
def oracle_step(model, cfg, x, eps, code, sn):
    """(grads, updated values) of one adaptation step in float64: autograd on the decoder (weight_orig with sn, u and v
    after one power iteration held constant) and the code; encoders detached; then clip_and_adam on that set."""
    sd = {k: v.detach().double().cpu() for k, v in model.state_dict().items()}
    names = [n for n, _ in model.named_parameters() if n.startswith("decoder.")]
    leaves = {n: sd[n].clone().requires_grad_(True) for n in names}
    c = code.detach().double().cpu().clone().requires_grad_(True)
    st = dict(sd)
    st.update(leaves)
    for n in [n for n in names if n.endswith(".weight_orig")]:
        base = n[: -len(".weight_orig")]
        u, v, _, _ = power_iteration64(sd[n], sd[base + ".weight_u"], sd[base + ".weight_v"], iterate=True)
        W = leaves[n]
        st[base + ".weight"] = W / (u @ (W.reshape(W.shape[0], -1) @ v))
    xd, ed = x.double().cpu(), eps.double().cpu()
    with torch.no_grad():
        mu, ls = orc.content_encoder(sd, xd, cfg["ContentEncoder"]["subsample"])
    z = mu + torch.exp(ls / 2) * ed
    dec = orc.decoder(st, z, c.expand(x.shape[0], -1), cfg["Decoder"]["upsample"])
    loss = cfg["lambda"]["lambda_rec"] * (dec - xd).abs().mean()
    gs = torch.autograd.grad(loss, [leaves[n] for n in names] + [c])
    grads = dict(zip(names + ["code"], gs))
    vals = {n: sd[n].clone() for n in names}
    vals["code"] = code.detach().double().cpu().clone()
    gn = orc.clip_and_adam(vals, grads, orc.AdamState(vals), cfg["optimizer"])
    return grads, vals, gn


@pytest.mark.parametrize("case", ["clip", "noclip", "sn"])
def test_one_step_against_the_oracle(monkeypatch, case):
    monkeypatch.setenv("AVC_PRECISION", "fp32")
    B = 4
    cfg = small_cfg(80, B, sn=case == "sn")
    cfg["optimizer"]["grad_norm"] = 1e-3 if case != "noclip" else 1e9
    model = make_model(cfg)
    g = torch.Generator().manual_seed(11)
    x = torch.randn((B, 80, 128), generator=g)
    eps = torch.randn((B, 128, 16), generator=g)
    code = torch.randn(128, generator=g) * 0.5
    grads, _, gn_ref = oracle_step(model, cfg, x, eps, code, case == "sn")
    tr = A.make_trainer(model, code, cfg)
    names = [n for n, _ in model.named_parameters() if n.startswith("decoder.")]
    before = {n: p.detach().double().cpu().clone() for n, p in model.named_parameters() if n in names}
    tr.step(x.cuda(), 0.0, eps=eps.cuda())
    _, _, gnorm = tr.losses()
    G = {n: tr.G[n].detach().double().cpu() for n in names}
    G["code"] = tr.code_grad.detach().double().cpu()
    # the existing fp32 step tests' gradient bounds (tests/test_gpu_model.py assert_grads_close)
    num = den = 0.0
    for k in names + ["code"]:
        r = grads[k]
        num += float((G[k] - r).pow(2).sum())
        den += float(r.pow(2).sum())
        if float(r.norm()) > 1e-4:
            assert rel_l2(G[k], r) < 5e-2, (k, rel_l2(G[k], r))
    assert (num / den) ** 0.5 < 1e-2
    assert rel_l2(G["code"], grads["code"]) < 1e-2, rel_l2(G["code"], grads["code"])
    assert abs(gnorm - gn_ref) / gn_ref < 1e-2
    # the oracle's clip + Adam on OUR gradients lands on OUR updated values; the flat layout is decoder then code
    before["code"] = code.double()
    gn = orc.clip_and_adam(before, G, orc.AdamState(before), cfg["optimizer"])
    assert abs(gn - gnorm) / gn < 1e-4
    after = dict((n, p.detach().double().cpu()) for n, p in model.named_parameters() if n in names)
    after["code"] = tr.code.detach().double().cpu()
    for k in before:
        assert float((after[k] - before[k]).abs().max()) < 2e-6, k
    print(f"{case}: code gradient rel L2 {rel_l2(G['code'], grads['code']):.3g}, grad norm {gnorm:.6g} vs {gn_ref:.6g}")


# ----------------------------------------------------------------------------- 3./4. frozen, graph, seed
def synthetic_clips(n, seed, n_mels=80, lo=130, hi=400, lengths=None):
    rng = np.random.default_rng(seed)
    base = rng.standard_normal(n_mels).astype(np.float32)
    lengths = lengths or [int(rng.integers(lo, hi)) for _ in range(n)]
    return {f"syn_{k:03d}": (rng.standard_normal((T, n_mels)) * 0.5 + base).astype(np.float32) for k, T in enumerate(lengths)}


# 6 clips of 130..135 frames: 3 + 4 + ... + 8 = 33 crops of 128 frames, 2 batches of 16 per epoch (one crop dropped)
EPOCH_CLIPS = [130, 131, 132, 133, 134, 135]


def test_frozen_encoders_graph_and_seed(tmp_path, monkeypatch):
    cfg = small_cfg(80, 16)
    clips = synthetic_clips(6, 1, lengths=EPOCH_CLIPS)     # 7 steps cross three epoch boundaries
    clips["syn_short"] = np.zeros((100, 80), np.float32)
    heldout = {u.replace("syn", "held"): v for u, v in synthetic_clips(3, 2, lo=17, hi=200).items()}
    heldout["held_tiny"] = np.zeros((9, 80), np.float32)
    base = make_model(cfg)
    base_sd = {k: v.detach().clone() for k, v in base.state_dict().items()}
    fp0 = SB.fingerprint(base)
    runs = {}
    for name, graph in (("graph", "1"), ("eager", "0"), ("graph2", "1")):
        monkeypatch.setenv("AVC_GRAPH", graph)
        m = make_model(cfg)
        res = A.adapt(m, cfg, "syn", clips, 7, seed=5, heldout=heldout)
        A.save(res, m, str(tmp_path / name))
        runs[name] = (m, res)
    m, res = runs["graph"]
    r = res["report"]
    assert r["clips"]["used"] == [f"syn_{k:03d}" for k in range(6)] and r["clips"]["skipped"] == ["syn_short"]
    assert [e["step"] for e in r["losses"]] == [0, 6]
    h = r["heldout"]
    assert h["before"]["rec"]["n"] == 3 and h["before"]["rec"]["skipped"] == ["held_tiny"]
    assert h["after"]["rec"]["rec"] is not None
    # frozen: every encoder entry keeps its bits, the decoder moved
    sd = m.state_dict()
    for k, v in base_sd.items():
        if k.startswith(ENC):
            assert tbits(sd[k], v), k
    assert any(not tbits(sd[k], v) for k, v in base_sd.items() if k.startswith("decoder."))
    ck = torch.load(tmp_path / "graph.ckpt")
    assert list(ck) == list(base_sd)
    for k in base_sd:
        if k.startswith(ENC):
            assert tbits(ck[k], base_sd[k]), k
    assert SB.fingerprint(m) == fp0
    loaded = make_model(cfg)
    loaded.load_state_dict(ck, strict=True)
    bank = SB.SpeakerBank.load(str(tmp_path / "graph.bank.pt"), loaded)
    assert bank.speakers == ["syn"] and bank.n_utts == [6] and bank.n_skipped == 1
    assert bank.fingerprint == fp0 and tbits(bank.codes[0], res["code"])
    # the code started from the pooled bank code of the adaptation clips and moved
    code0 = SB.build_bank(base, {u: v for u, v in clips.items() if u != "syn_short"}, speaker_of=lambda u: "syn").codes[0]
    assert not tbits(res["code"], code0)
    # graph replay == eager, and one seed gives one result
    for other in ("eager", "graph2"):
        m2, res2 = runs[other]
        assert tbits(res2["code"], res["code"]), other
        sd2 = m2.state_dict()
        assert all(tbits(sd2[k], sd[k]) for k in sd), other
        assert res2["report"]["losses"] == r["losses"], other
    m3 = make_model(cfg)
    res3 = A.adapt(m3, cfg, "syn", clips, 7, seed=6)
    assert not tbits(res3["code"], res["code"])


def test_every_batch_is_full_and_the_graph_reports_as_eager(monkeypatch):
    """Across epoch boundaries every batch has the same shape, so the captured graph replays every step after the
    third, and each step's reported loss equals the eager run's (whose normaliser is set by every step)."""
    cfg = small_cfg(80, 16)
    clips = synthetic_clips(6, 1, lengths=EPOCH_CLIPS)
    ds, _, _ = A.segments(clips, cfg, 16, 3, "cuda")
    assert (ds.sampler.n, ds.sampler.batch_size, ds.sampler.batches_per_epoch) == (33, 16, 2)
    assert all(tuple(next(ds).shape) == (16, 80, 128) for _ in range(9))
    small, _, _ = A.segments(clips, cfg, 64, 3, "cuda")       # fewer crops than the batch: one batch of all of them
    assert small.sampler.batch_size == 33 and tuple(next(small).shape) == (33, 80, 128)
    logs = {}
    for name, graph in (("graph", "1"), ("eager", "0")):
        monkeypatch.setenv("AVC_GRAPH", graph)
        ds, _, _ = A.segments(clips, cfg, 16, 3, "cuda")
        tr = A.make_trainer(make_model(cfg), torch.zeros(128), cfg)
        torch.manual_seed(3)
        logs[name] = A.train(tr, iter(ds), 10, log_every=1)
        assert (tr._graphs is not None) == (graph == "1")
    assert [e["step"] for e in logs["graph"]] == list(range(10))
    assert logs["graph"] == logs["eager"]


# ----------------------------------------------------------------------------- 5. the kernel
def rec_varlen64(dec, x, lens, threads=512):
    """The kernel's order: thread i adds units i, i + 512, ... of (c, t < L) in row-major order, in float64; then the
    warp xor-butterflies and the 16 warp sums, padded to 32 with zeros, butterflied again."""
    out = []
    lane = np.arange(32)
    for b, Lb in enumerate(lens):
        terms = np.abs(dec[b, :, :Lb].astype(np.float64) - x[b, :, :Lb].astype(np.float64)).reshape(-1)
        acc = np.zeros(threads)
        for k in range(0, len(terms), threads):
            part = terms[k:k + threads]
            acc[:len(part)] = acc[:len(part)] + part
        p = acc.reshape(threads // 32, 32)
        for o in (16, 8, 4, 2, 1):
            p = p + p[:, lane ^ o]
        w = np.zeros(32)
        w[:threads // 32] = p[:, 0]
        for o in (16, 8, 4, 2, 1):
            w = w + w[lane ^ o]
        out.append(w[0])
    return np.array(out)


def test_rec_loss_varlen_kernel():
    lib = L.load()
    g = torch.Generator().manual_seed(21)
    B, Cc, T = 11, 80, 333
    lens = torch.randint(1, T + 1, (B,), generator=g)
    lens[0], lens[1], lens[2] = 1, T, 2
    dec = torch.randn((B, Cc, T), generator=g)
    x = torch.randn((B, Cc, T), generator=g) * 2
    for b in range(B):
        dec[b, :, lens[b]:] = float("nan")
        x[b, :, lens[b]:] = float("inf")
    want = rec_varlen64(dec.numpy(), x.numpy(), lens.tolist())
    dg, xg = dec.cuda(), x.cuda()
    got = A.rec_loss_varlen(dg, xg, lens.to(torch.int32).cuda())
    again = A.rec_loss_varlen(dg, xg, lens.cuda())
    assert bits_equal(got.cpu().numpy(), want)
    assert tbits(got, again)
    # whatever the padding holds
    dg2, xg2 = dg.clone(), xg.clone()
    for b in range(B):
        dg2[b, :, lens[b]:] = 3.0
        xg2[b, :, lens[b]:] = -1e30
    assert tbits(A.rec_loss_varlen(dg2, xg2, lens.cuda()), got)
    lt = lens.to(torch.int32).cuda()
    out = torch.full((B,), -5.0, dtype=torch.float64, device="cuda")
    n0 = L.launch_count()
    good = dict(B=B, C=Cc, T=T, dec=dg.data_ptr(), x=xg.data_ptr(), lengths=lt.data_ptr(), out=out.data_ptr())
    for bad in (dict(B=0), dict(C=0), dict(T=0), dict(B=-1), dict(dec=None), dict(x=None), dict(lengths=None), dict(out=None)):
        d = L.RecVarlenDesc(**dict(good, **bad))
        assert lib.avc_rec_loss_varlen(d, None) == L.ERR_INVALID, bad
    assert lib.avc_rec_loss_varlen(None, None) == L.ERR_INVALID
    assert L.launch_count() == n0
    torch.cuda.synchronize()
    assert bool((out == -5.0).all())
    with pytest.raises(ValueError, match="lengths"):
        A.rec_loss_varlen(dg, xg, torch.full((B,), T + 1))


# ----------------------------------------------------------------------------- 6. target_codes
def parallel_set(root, n_mels=80, seed=0):
    """3 speakers, each reading one shared line and one line of their own: every target has one possible reference."""
    rng = np.random.default_rng(seed)
    data, texts = {}, {}
    for s in range(3):
        for k, line in ((0, "the shared line"), (1, f"own line of speaker {s}")):
            u = f"p{300 + s}_{k:03d}.wav"
            data[u] = (rng.standard_normal((int(rng.integers(130, 260)), n_mels)) * 0.3 + 0.4 + 0.05 * s).astype(np.float32)
            texts[u] = line
    return data, texts


def test_evaluate_mcd_target_codes(precision):
    from adaptive_voice_conversion_b200.mcd import evaluate_mcd
    cfg = small_cfg(80, 8)
    model = make_model(cfg).eval()
    data, texts = parallel_set(None)
    attr = {"mean": np.zeros(80, np.float32), "std": np.ones(80, np.float32)}
    plain = evaluate_mcd(model, data, attr, texts, per_triplet=True)
    assert plain == evaluate_mcd(model, data, attr, texts, per_triplet=True, target_codes=None)
    assert plain["n"] == 6
    codes = {}
    with torch.no_grad():
        for s, r, g, *_ in plain["triplets"]:
            codes[g.split("_")[0]] = model.get_speaker_embeddings(torch.from_numpy(data[r]).t()[None].contiguous().cuda())[0]
    coded = evaluate_mcd(model, data, attr, texts, per_triplet=True, target_codes=codes)
    assert coded["n"] == 6 and coded["n_no_code"] == 0
    for a, b in zip(plain["triplets"], coded["triplets"]):
        assert a == b
    assert {k: v for k, v in coded.items() if k != "n_no_code"} == plain
    one = evaluate_mcd(model, data, attr, texts, per_triplet=True, target_codes={"p301": codes["p301"]})
    assert one["n"] == 2 and one["n_no_code"] == 4 and set(one["speakers"]) == {"p301"}
    assert one["triplets"] == [t for t in plain["triplets"] if t[2].startswith("p301")]


# ----------------------------------------------------------------------------- 7./8. a synthetic speaker
def write_wavs(root, name, n, seed, sr=24000, seconds=2.5):
    """n seeded recordings of one synthetic voice: a harmonic tone at a speaker-specific pitch with a slow vibrato and
    a little noise."""
    from scipy.io import wavfile
    rng = np.random.default_rng(seed)
    f0 = 110.0 + 20.0 * (seed % 5)
    paths = []
    for k in range(n):
        t = np.arange(int(sr * seconds * rng.uniform(0.8, 1.2))) / sr
        f = f0 * (1.0 + 0.05 * np.sin(2 * np.pi * rng.uniform(2, 5) * t))
        ph = 2 * np.pi * np.cumsum(f) / sr
        y = sum(np.sin(h * ph) / h for h in range(1, 12)) * (0.5 + 0.5 * np.sin(2 * np.pi * rng.uniform(0.5, 2) * t) ** 2)
        y = 0.2 * y + 0.01 * rng.standard_normal(len(t))
        p = root / f"{name}_{k}.wav"
        wavfile.write(str(p), sr, (y / np.abs(y).max() * 0.5 * 32767).astype(np.int16))
        paths.append(str(p))
    return paths


def wav_mels(paths):
    from adaptive_voice_conversion_b200.vocoder import Vocoder, load_wav
    voc = Vocoder(n_mels=80)
    return {p: m for p, (m, _) in zip(paths, voc.wav_to_mel([torch.from_numpy(load_wav(p, voc.hp.sr)).cuda()
                                                              for p in paths]))}


def test_adaptation_lowers_the_training_loss(tmp_path):
    cfg = small_cfg(80, 32)
    paths = write_wavs(tmp_path, "syn", 6, seed=3)
    mels = wav_mels(paths)
    mean = torch.cat(list(mels.values())).mean(0)
    std = torch.cat(list(mels.values())).std(0) + 1e-3
    mels = {u: (m - mean) / std for u, m in mels.items()}
    model = make_model(cfg)
    ds, used, _ = A.segments(mels, cfg, 32, 0, "cuda")
    assert len(used) == 6
    tr = A.make_trainer(model, torch.zeros(128), cfg)
    with torch.no_grad():
        tr.code.copy_(SB.build_bank(model, mels, speaker_of=lambda u: "syn").codes[0])
    torch.manual_seed(0)
    log = A.train(tr, iter(ds), 200, log_every=1)
    losses = np.array([e["loss_rec"] for e in log])
    first, last = float(losses[:10].mean()), float(losses[-10:].mean())
    print(f"training L1: first 10 steps {first:.4f}, last 10 steps {last:.4f}, ratio {last / first:.3f}")
    assert last < 0.7 * first, (first, last)     # measured on an H100: 0.8300 -> 0.4942 (ratio 0.595)


def test_adapt_cli_end_to_end(tmp_path):
    import yaml
    cfg = small_cfg(80, 16)
    cfg_path = tmp_path / "config.yaml"
    cfg_path.write_text(yaml.safe_dump(cfg))
    base = make_model(cfg)
    torch.save(base.state_dict(), tmp_path / "base.ckpt")
    wavs = write_wavs(tmp_path, "alice", 4, seed=1)
    held = write_wavs(tmp_path, "alice_held", 2, seed=2)
    with open(tmp_path / "attr.pkl", "wb") as f:
        pickle.dump({"mean": np.full(80, 0.4, np.float32), "std": np.full(80, 0.2, np.float32)}, f)
    env = dict(os.environ, PYTHONPATH=ROOT)
    out = str(tmp_path / "alice_model")
    run = subprocess.run([sys.executable, os.path.join(ROOT, "adapt.py"), "-c", str(cfg_path), "-m", str(tmp_path / "base.ckpt"),
                          "-a", str(tmp_path / "attr.pkl"), "-speaker", "alice", "-wav", *wavs, "-holdout", *held, "-o", out,
                          "-steps", "12", "-batch_size", "8"], env=env, cwd=str(tmp_path), capture_output=True, text=True)
    assert run.returncode == 0, run.stderr[-3000:]
    for sfx in (".ckpt", ".bank.pt", ".json"):
        assert os.path.isfile(out + sfx), sfx
    import json
    rep = json.loads(open(out + ".json").read())
    assert tuple(rep) == A.REPORT_KEYS and rep["clips"]["used"] == wavs
    assert rep["settings"]["steps"] == 12 and rep["settings"]["batch_size"] == 8
    assert rep["heldout"]["before"]["rec"]["n"] == 2 and rep["heldout"]["after"]["rec"]["n"] == 2
    # the checkpoint strict-loads into the reference-layout AE; the encoders are the base's
    from adaptive_voice_conversion_b200.inference import Inferencer
    ck = torch.load(out + ".ckpt")
    assert [k for k, _ in orc.param_shapes(cfg)] == list(ck)
    for k, v in base.state_dict().items():
        if k.startswith(ENC):
            assert tbits(ck[k], v), k
    args = types.SimpleNamespace(attr=None, model=None, source=None, target=None, output=None, sample_rate=24000)
    inf = Inferencer(cfg, args)
    inf.model.load_state_dict(ck, strict=True)
    bank = SB.SpeakerBank.load(out + ".bank.pt", inf.model)
    assert bank.speakers == ["alice"] and bank.n_utts == [4] and bank.utterances == [sorted(wavs)]
    src = np.random.default_rng(7).standard_normal((150, 80)).astype(np.float32)
    np.save(tmp_path / "src.npy", src)
    subprocess.run([sys.executable, os.path.join(ROOT, "inference.py"), "-c", str(cfg_path), "-m", out + ".ckpt", "-s",
                    str(tmp_path / "src.npy"), "-bank", out + ".bank.pt", "-speaker", "alice", "-o", str(tmp_path / "t.npy")],
                   check=True, env=env, cwd=str(tmp_path))
    want = inf.inference_with_codes([torch.from_numpy(src).cuda()], bank.code("alice")[None])[0]
    assert bits_equal(np.load(tmp_path / "t.npy"), want.cpu().numpy())
