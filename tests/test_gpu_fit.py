"""GPU: speaker-code fitting (adaptive_voice_conversion_b200/fit.py, csrc/fit.cu).

1. anchor on speaker adaptation: one speaker, m = B, the same crops and eps = 0 in AdaptTrainer (z = mu + 0 is mu bit
   for bit): its ddec equals avc_group_l1's and its code gradient equals the fitting step's g_s, both bit for bit (g_s
   is formed in avc_bias_grad's order);
2. one step against the float64 oracle (autograd on oracle/ae_oracle.py with respect to the codes only, then per-code
   clip + L2 decay + Adam(amsgrad)): two speakers, fp32 at c_in 80, clipping active and inactive, and once with sn;
3. the kernels against the float64 restatement (tests/_fit_ref.py): avc_group_l1's sums (bit for bit) and gradient for
   unequal groups, avc_code_adam over several steps with one code clipped beside one that is not, and its emb rows;
4. frozen means frozen: every state_dict entry and weight pack keeps its bits; need_wgrad=False runs no weight-gradient
   entry point, writes no gradient buffer, and gives the full backward's dz and demb bit for bit;
5. independence: a speaker's code after K steps does not depend on its wave partners (bit for bit), and its first-step
   gradient alone and in a wave of three agrees within float32 reassociation (fp32) or the TF32 bound (tf32);
6. graph replay equals eager across an epoch boundary of a speaker's crop order; one seed gives the same bank bytes;
7. 200 steps lower each synthetic speaker's training L1 and held-out rec;
8. speaker_bank.py -fit_steps end to end, inference.py -bank -speaker, evaluate.py -spk -bank, and the refusal of the
   fitted bank by a model with a changed decoder weight.
"""
import json
import os
import subprocess
import sys

import numpy as np
import pytest
import torch

import oracle.ae_oracle as orc
from _fit_ref import CodeAdamState, a4_of, code_adam_ref, group_l1_ref, oracle_codes_step
from _sn_ref import sn_config
from adaptive_voice_conversion_b200 import _lib as L
from adaptive_voice_conversion_b200 import adapt as A
from adaptive_voice_conversion_b200 import fit as F
from adaptive_voice_conversion_b200 import speaker_bank as SB
from adaptive_voice_conversion_b200.engine import A4

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def tbits(a, b):
    a, b = a.detach().cpu().contiguous(), b.detach().cpu().contiguous()
    return a.shape == b.shape and a.dtype == b.dtype and a.numpy().tobytes() == b.numpy().tobytes()


def rel_l2(a, b):
    a, b = torch.as_tensor(a).double().flatten(), torch.as_tensor(b).double().flatten()
    return float((a - b).norm() / (b.norm() + 1e-30))


def make_model(cfg, seed=0):
    from adaptive_voice_conversion_b200.model import AE
    torch.manual_seed(seed)
    m = AE(cfg)
    if not cfg["Decoder"].get("sn", False):
        m.load_state_dict(orc.init_state(cfg, seed=seed), strict=True)
    return m.cuda()


def small_cfg(sn=False):
    return sn_config(80) if sn else orc.default_config(80)


@pytest.fixture(params=["fp32", "tf32"])
def precision(request, monkeypatch):
    monkeypatch.setenv("AVC_PRECISION", request.param)
    return request.param


def speakers(n, seed, n_clips=3, lo=130, hi=260, n_mels=80):
    """{speaker: {id: [T, n_mels]}} of n seeded synthetic speakers (a per-speaker mean spectrum plus noise)."""
    rng = np.random.default_rng(seed)
    out = {}
    for s in range(n):
        base = rng.standard_normal(n_mels).astype(np.float32)
        out[f"p{300 + s}"] = {f"p{300 + s}_{k:03d}": (rng.standard_normal((int(rng.integers(lo, hi)), n_mels)) * 0.5 + base
                                                      ).astype(np.float32) for k in range(n_clips)}
    return out


def flat(sp):
    return {u: v for d in sp.values() for u, v in d.items()}


def spk_of(u):
    return u.split("_")[0]


def wave(model, cfg, sp, names, m, steps, seed=0, lr=None, tr=None):
    """(trainer, WaveCorpus, pooled codes [S, c_out]) of one wave of `names`."""
    mels = flat({s: sp[s] for s in names})
    bank = SB.build_bank(model, mels, speaker_of=spk_of)
    per, unfitted = F.plan(bank.speakers, bank.utterances, {u: v.shape[0] for u, v in mels.items()}, 128, m)
    assert not unfitted
    index = [e for s in names for e in per[s]["index"]]
    order = F.order_table([per[s]["n_crops"] for s in names], m, steps, seed, names)
    corpus = F.WaveCorpus(mels, index, order, cfg, "cuda")
    tr = tr or F.CodeFitTrainer(model, cfg, len(names), m, lr)
    return tr, corpus, torch.stack([bank.codes[bank.index(s)] for s in names])


# ----------------------------------------------------------------------------- 1. anchor on adaptation
def test_anchor_on_adaptation(precision):
    cfg = small_cfg()
    B = 8
    sp = speakers(1, 1)
    model = make_model(cfg)
    tr, corpus, codes0 = wave(model, cfg, sp, ["p300"], B, 1)
    tr.reset(codes0)
    ad = A.make_trainer(make_model(cfg), codes0[0], cfg)
    assert ad.eng is not tr.eng
    seen = {}

    def spy(eng, key):
        bwd = eng.decoder_bwd

        def f(P, G, ctx, ddec4, **kw):
            seen[key] = ddec4.to_planar().clone()
            return bwd(P, G, ctx, ddec4, **kw)
        eng.decoder_bwd = f
    spy(tr.eng, "fit")
    spy(ad.eng, "adapt")
    try:
        x = tr._x
        corpus.gather(x, 0, B)
        x = x.clone()
        tr.step(x, 0.0)
        ad.step(x, 0.0, eps=torch.zeros(B, 128, 16, device="cuda"))
    finally:
        del tr.eng.decoder_bwd, ad.eng.decoder_bwd
    d_fit, d_ad = seen["fit"], seen["adapt"]
    assert tbits(d_fit, d_ad)
    assert tbits(tr.grad[0], ad.code_grad)        # bit for bit: g_s follows avc_bias_grad's order
    tr.eng.check_tc_status()


# ----------------------------------------------------------------------------- 2. against the float64 oracle
@pytest.mark.parametrize("case", ["clip", "noclip", "sn"])
def test_one_step_against_the_oracle(monkeypatch, case):
    monkeypatch.setenv("AVC_PRECISION", "fp32")
    cfg = small_cfg(sn=case == "sn")
    cfg["optimizer"]["grad_norm"] = 1e-4 if case != "noclip" else 1e9
    model = make_model(cfg)
    m = 3
    g = torch.Generator().manual_seed(11)
    x = torch.randn((2 * m, 80, 128), generator=g)
    codes = torch.randn((2, 128), generator=g) * 0.5
    g_ref, n_ref, _, _ = oracle_codes_step(model, cfg, x, codes, m)
    tr = F.CodeFitTrainer(model, cfg, 2, m)
    tr.reset(codes.cuda())
    tr.step(x.cuda(), 0.0)
    for s in range(2):
        print(f"{case}: code {s} gradient rel L2 {rel_l2(tr.grad[s].cpu(), g_ref[s]):.3g}")
        assert rel_l2(tr.grad[s].cpu(), g_ref[s]) < 5e-3, (s, rel_l2(tr.grad[s].cpu(), g_ref[s]))
        assert abs(float(tr.gnorm[s]) - n_ref[s]) / n_ref[s] < 5e-3
    clipped = n_ref > cfg["optimizer"]["grad_norm"]
    assert clipped.all() == (case != "noclip")
    # the float64 update on OUR gradient lands on OUR codes
    vals = codes.double().numpy().copy()
    code_adam_ref(vals, np.repeat(tr.grad.double().cpu().numpy() / m, m, axis=0), m, CodeAdamState(2, 128),
                  cfg["optimizer"])
    assert float(np.abs(tr.codes.double().cpu().numpy() - vals).max()) < 2e-6
    # the expanded rows of the next step
    assert tbits(tr.emb, tr.codes.repeat_interleave(m, 0))


# ----------------------------------------------------------------------------- 3. the kernels
def group_l1_gpu(dec, x, m, lam, rnd, total=True):
    B, Cc, T = dec.shape
    dec4 = torch.from_numpy(a4_of(dec)).cuda()
    xg = torch.from_numpy(np.ascontiguousarray(x)).cuda()
    hp = torch.tensor([lam], dtype=torch.float32).cuda()
    ddec = torch.full_like(dec4, float("nan"))
    part = torch.zeros(B, dtype=torch.float64, device="cuda")
    sums = torch.zeros(B // m, dtype=torch.float64, device="cuda")
    tot = torch.zeros(1, device="cuda")
    d = L.GroupL1Desc(B=B, C=Cc, T=T, m=m, round_tf32=int(rnd), dec=dec4.data_ptr(), x=xg.data_ptr(), hp=hp.data_ptr(),
                      ddec=ddec.data_ptr(), part=part.data_ptr(), sums=sums.data_ptr(),
                      total=tot.data_ptr() if total else None)
    L.check(L.load().avc_group_l1(d, None), "avc_group_l1")
    torch.cuda.synchronize()
    ddec = ddec.cpu().numpy().transpose(0, 1, 3, 2).reshape(B, Cc, T)
    return ddec, part.cpu().numpy(), sums.cpu().numpy(), float(tot.cpu()[0])


@pytest.mark.parametrize("rnd", [0, 1])
def test_group_l1_kernel(rnd):
    rng = np.random.default_rng(5)
    m, G, Cc, T = 3, 4, 80, 128
    dec = rng.standard_normal((m * G, Cc, T)).astype(np.float32)
    x = (rng.standard_normal((m * G, Cc, T)) * np.arange(1, m * G + 1)[:, None, None]).astype(np.float32)
    x[0, :7, :5] = dec[0, :7, :5]                              # ties: a zero gradient
    x[4] = dec[4]                                              # one whole sample at zero loss
    lam = 10.0
    g, part, sums, tot = group_l1_gpu(dec, x, m, lam, rnd)
    g_ref, part_ref, sums_ref, tot_ref = group_l1_ref(dec, x, m, lam, bool(rnd))
    assert part.tobytes() == part_ref.tobytes()
    assert sums.tobytes() == sums_ref.tobytes() and len(set(sums.tolist())) == G
    assert np.float32(tot).tobytes() == tot_ref.tobytes()
    assert g.tobytes() == g_ref.tobytes()
    assert (g[0, :7, :5] == 0).all() and (g[4] == 0).all()
    # a group's sum does not depend on what the other groups hold
    dec2 = dec.copy()
    dec2[m:] = rng.standard_normal(dec2[m:].shape)
    _, _, sums2, _ = group_l1_gpu(dec2, x, m, lam, rnd, total=False)
    assert sums2[0].tobytes() == sums[0].tobytes()
    lib = L.load()
    n0 = L.launch_count()
    good = dict(B=4, C=80, T=8, m=2, dec=1, x=1, hp=1, ddec=1, part=1, sums=1)
    for bad in (dict(B=0), dict(m=0), dict(C=6), dict(m=3), dict(dec=None), dict(hp=None), dict(sums=None)):
        assert lib.avc_group_l1(L.GroupL1Desc(**dict(good, **bad)), None) == L.ERR_INVALID, bad
    assert L.launch_count() == n0


def code_adam_gpu(S, m, Cc, opt, lr):
    from adaptive_voice_conversion_b200.optim import FusedAdam
    hp = torch.zeros(16)
    hp[2], hp[3], hp[4], hp[5], hp[6] = 1.0, lr, opt["beta1"], opt["beta2"], 1e-8
    hp[7], hp[8], hp[9] = opt["weight_decay"], opt["grad_norm"], 1.0
    t = {k: torch.zeros(S, Cc, device="cuda") for k in ("codes", "exp_avg", "exp_avg_sq", "max_exp_avg_sq", "grad")}
    t["steps"], t["gnorm"] = torch.zeros(S, device="cuda"), torch.zeros(S, device="cuda")
    t["emb"] = torch.full((S * m, Cc), float("nan"), device="cuda")
    t["hp"] = hp.cuda()
    return t


def test_code_adam_kernel():
    S, m, Cc = 3, 1100, 128                 # m > 1024: a thread adds two rows
    opt = {"beta1": 0.9, "beta2": 0.999, "weight_decay": 1e-4, "grad_norm": 1.0, "amsgrad": True}
    lr = 1e-2
    t = code_adam_gpu(S, m, Cc, opt, lr)
    rng = np.random.default_rng(2)
    codes = rng.standard_normal((S, Cc)).astype(np.float32)
    t["codes"].copy_(torch.from_numpy(codes))
    ref = codes.astype(np.float64)
    st = CodeAdamState(S, Cc)
    lib = L.load()
    for k in range(4):
        demb = rng.standard_normal((S * m, Cc)).astype(np.float32) * 1e-4
        demb[m:2 * m] *= 1e3                 # code 1 clipped (norm ~ 37), codes 0 and 2 not (~ 0.04)
        dg = torch.from_numpy(demb).cuda()
        d = L.CodeAdamDesc(S=S, m=m, C=Cc, demb=dg.data_ptr(), **{k2: v.data_ptr() for k2, v in t.items()})
        L.check(lib.avc_code_adam(d, None), "avc_code_adam")
        g_ref, n_ref = code_adam_ref(ref, demb, m, st, opt, lr)
        assert (n_ref[[0, 2]] < 1.0).all() and n_ref[1] > 1.0
        # g_s in avc_bias_grad's order at T = 1, bit for bit
        for s in range(S):
            gb = torch.zeros(Cc, device="cuda")
            L.check(lib.avc_bias_grad(dg[s * m].data_ptr(), Cc, gb.data_ptr(), m, Cc, 1, None), "bias_grad")
            assert tbits(t["grad"][s], gb), (k, s)
        assert rel_l2(t["grad"].cpu(), g_ref) < 1e-6
        assert np.abs(t["gnorm"].cpu().numpy() - n_ref).max() / n_ref.max() < 1e-5
        assert np.abs(t["codes"].cpu().numpy() - ref).max() < 2e-6, k
        assert (t["steps"].cpu().numpy() == k + 1).all()
        assert tbits(t["emb"], t["codes"].repeat_interleave(m, 0))
    n0 = L.launch_count()
    good = dict(S=1, m=1, C=8, demb=16, **{k2: 16 for k2 in t})
    for bad in (dict(S=0), dict(m=0), dict(C=6), dict(C=L.CODE_MAX_C + 4), dict(demb=None), dict(steps=None),
                dict(emb=None), dict(hp=None), dict(demb=20)):
        assert lib.avc_code_adam(L.CodeAdamDesc(**dict(good, **bad)), None) == L.ERR_INVALID, bad
    assert L.launch_count() == n0


# ----------------------------------------------------------------------------- 4. frozen
def test_frozen_and_data_gradient_only(precision, monkeypatch):
    cfg = small_cfg()
    sp = speakers(2, 2)
    model = make_model(cfg)
    sd0 = {k: v.detach().clone() for k, v in model.state_dict().items()}
    tr, corpus, codes0 = wave(model, cfg, sp, ["p300", "p301"], 4, 6)
    packs0 = {(n, k): v.clone() for n, d in tr.eng.packed.items() for k, v in d.items() if isinstance(v, torch.Tensor)}
    tr.reset(codes0)

    def boom(*a, **k):
        raise AssertionError("a weight-gradient launch in a data-gradient-only backward")
    with monkeypatch.context() as mp:
        mp.setattr(type(tr.eng), "wgrad", boom)
        for k in range(6):
            tr.run_step(corpus, k)
    torch.cuda.synchronize()
    assert tr._graphs is not None or os.environ.get("AVC_GRAPH") == "0"
    sd = model.state_dict()
    assert all(tbits(sd[k], v) for k, v in sd0.items())
    for key, v in packs0.items():
        assert tbits(tr.eng.packed[key[0]][key[1]], v), key
    assert not tbits(tr.codes, codes0)
    # need_wgrad=False against the full backward, on one batch: dz and demb bit for bit, a sentinel gradient buffer
    # untouched
    eng, P = tr.eng, tr.P
    x = tr._x
    corpus.gather(x, 0, tr.B)
    mu4, ls4, _ = eng.content_fwd(P, x, False)
    _, _, z4 = eng.reparam_fwd(mu4, ls4, None, want_planar=False)
    dec4, cd = eng.decoder_fwd(P, z4, tr.emb, True)
    dd = torch.randn(dec4.B, dec4.C, dec4.T, device="cuda")
    ddec4 = A4.empty(dec4.B, dec4.C, dec4.T, "cuda")
    eng.pack_a4(dd, ddec4)
    names = [n for n, _ in model.named_parameters() if n.startswith("decoder.")]
    sentinel = {n: torch.full_like(p, 7.25) for n, p in model.named_parameters() if n in names}
    G0 = {n: v.clone() for n, v in sentinel.items()}
    with monkeypatch.context() as mp:
        mp.setattr(type(eng), "wgrad", boom)
        dz_a, demb_a = eng.decoder_bwd(P, sentinel, cd, ddec4, need_wgrad=False)
        dz_b, demb_b = eng.decoder_bwd(P, None, cd, ddec4, need_wgrad=False)
    G = {n: torch.zeros_like(p) for n, p in model.named_parameters() if n in names}
    eng.prepare_tables(P, G)
    dz_f, demb_f = eng.decoder_bwd(P, G, cd, ddec4)
    eng.join_wgrad()
    eng.flush_wgrad()
    torch.cuda.synchronize()
    assert all(tbits(sentinel[n], G0[n]) for n in names)
    assert any(float(G[n].abs().max()) > 0 for n in names)
    for dz, demb in ((dz_a, demb_a), (dz_b, demb_b)):
        assert tbits(dz.t, dz_f.t) and tbits(demb, demb_f)


# ----------------------------------------------------------------------------- 5. independence
def test_independence(precision):
    cfg = small_cfg()
    sp = speakers(4, 3)
    K, m = 5, 4
    model = make_model(cfg)
    got = []
    for partner in ("p301", "p302"):
        tr, corpus, codes0 = wave(model, cfg, sp, ["p300", partner], m, K)
        codes, _ = F.fit_wave(tr, corpus, codes0, K)
        got.append(codes[0])
    assert tbits(got[0], got[1])
    # first-step g_A alone and in a wave of three
    g = {}
    for names in (["p300"], ["p300", "p302", "p303"]):
        tr, corpus, codes0 = wave(model, cfg, sp, names, m, 1)
        F.fit_wave(tr, corpus, codes0, 1)
        g[len(names)] = tr.grad[0].clone()
    err = rel_l2(g[3].cpu(), g[1].cpu())
    print(f"{precision}: first-step g_A alone vs in a wave of three: rel L2 {err:.3g}")
    assert err < (1e-4 if precision == "fp32" else 8e-3), err


# ----------------------------------------------------------------------------- 6. graph replay, seed
def test_graph_equals_eager_and_seed(monkeypatch, tmp_path):
    cfg = small_cfg()
    sp = speakers(2, 4, n_clips=2, lo=130, hi=134)       # 2 clips of 130..133 frames: 6..12 crops, m = 4
    K, m = 7, 4
    res = {}
    for name, graph in (("graph", "1"), ("eager", "0")):
        monkeypatch.setenv("AVC_GRAPH", graph)
        model = make_model(cfg)
        tr, corpus, codes0 = wave(model, cfg, sp, ["p300", "p301"], m, K)
        codes, log = F.fit_wave(tr, corpus, codes0, K, log_every=1)
        assert (tr._graphs is not None) == (graph == "1")
        res[name] = (codes, log)
    n = [sum(v.shape[0] - 127 for v in sp[s].values()) for s in ("p300", "p301")]
    assert min(n) // m < K                                  # an epoch boundary of a speaker's crop order
    assert tbits(res["graph"][0], res["eager"][0])
    for (k1, s1, g1), (k2, s2, g2) in zip(res["graph"][1], res["eager"][1]):
        assert k1 == k2 and s1.tobytes() == s2.tobytes() and g1.tobytes() == g2.tobytes()
    monkeypatch.setenv("AVC_GRAPH", "1")
    blobs = []
    for run in range(2):
        model = make_model(cfg)
        mels = flat(sp)
        bank = SB.build_bank(model, mels, speaker_of=spk_of)
        fitted, _ = F.fit_bank(model, bank, mels, K, crops=m, speakers_per_wave=2, seed=9)
        path = tmp_path / "bank.pt"        # (torch.save writes the file's name into the archive)
        fitted.save(str(path))
        blobs.append(path.read_bytes())
    assert blobs[0] == blobs[1]


# ----------------------------------------------------------------------------- 7. fitting helps its own objective
def test_fitting_lowers_the_loss():
    cfg = small_cfg()
    every = speakers(3, 7, n_clips=8, lo=140, hi=300)
    sp = {s: dict(list(d.items())[:5]) for s, d in every.items()}
    held = {s: dict(list(d.items())[5:]) for s, d in every.items()}    # the same voices, other clips
    model = make_model(cfg)
    mels = flat(sp)
    bank = SB.build_bank(model, mels, speaker_of=spk_of)
    fitted, rep = F.fit_bank(model, bank, mels, 200, lr=1e-2, crops=16, speakers_per_wave=3, seed=0, heldout=held,
                             log_every=10)
    for s in bank.speakers:
        r = rep["speakers"][s]
        first = np.mean([e["loss_rec"] for e in r["losses"][:2]])
        last = np.mean([e["loss_rec"] for e in r["losses"][-2:]])
        hb, ha = r["heldout"]["before"]["rec"]["rec"], r["heldout"]["after"]["rec"]["rec"]
        print(f"{s}: training L1 {first:.4f} -> {last:.4f}, held-out rec {hb:.4f} -> {ha:.4f}")
        assert last < first and ha < hb, s
    assert rep["unfitted"] == [] and rep["n_waves"] == 1


# ----------------------------------------------------------------------------- 8. end to end
def test_fit_cli_end_to_end(tmp_path):
    from test_gpu_bank import write_train
    from test_gpu_fewshot import _checkpoint, write_eval_dir
    from test_gpu_padded_inference import _inferencer
    cfg = orc.default_config(80)
    cfg_path, ckpt = _checkpoint(tmp_path, cfg)
    write_eval_dir(tmp_path, 80)
    train = write_train(tmp_path, 80)
    env = dict(os.environ, PYTHONPATH=ROOT)
    bank_path, rep_path = str(tmp_path / "bank.pt"), str(tmp_path / "fit.json")
    run = subprocess.run([sys.executable, os.path.join(ROOT, "speaker_bank.py"), "-c", cfg_path, "-m", ckpt, "-d",
                          str(tmp_path), "-set", "train", "-o", bank_path, "-fit_steps", "20", "-fit_crops", "4",
                          "-fit_speakers", "3", "-holdout_set", "in_test", "-transcripts", str(tmp_path / "txt"),
                          "-report", rep_path],
                         env=env, cwd=str(tmp_path), capture_output=True, text=True)
    assert run.returncode == 0, run.stderr[-3000:]
    rep = json.loads(open(rep_path).read())
    assert tuple(rep) == F.REPORT_KEYS and rep["n_waves"] == 2 and rep["settings"]["steps"] == 20
    for s, r in rep["speakers"].items():
        assert tuple(r) == F.SPEAKER_KEYS and r["fitted"] and [e["step"] for e in r["losses"]] == [0, 19]
        assert r["heldout"]["before"]["rec"]["n"] > 0 and r["heldout"]["after"]["rec"]["rec"] is not None
        assert r["heldout"]["before"]["mcd"]["n"] > 0 and r["heldout"]["after"]["mcd"]["mcd"] is not None
    assert rep["mcd"]["before"]["n"] == rep["mcd"]["after"]["n"] > 0
    inf = _inferencer(cfg)
    bank = SB.SpeakerBank.load(bank_path, inf.model)
    pooled = SB.build_bank(inf.model, {u: torch.from_numpy(v).cuda() for u, v in train.items()})
    assert bank.fitted is not None and bank.fitted["steps"] == 20 and bank.speakers == pooled.speakers
    assert not tbits(bank.codes, pooled.codes)
    src = np.random.default_rng(7).standard_normal((150, 80)).astype(np.float32)
    np.save(tmp_path / "src.npy", src)
    subprocess.run([sys.executable, os.path.join(ROOT, "inference.py"), "-c", cfg_path, "-m", ckpt, "-s",
                    str(tmp_path / "src.npy"), "-bank", bank_path, "-speaker", "p301", "-o", str(tmp_path / "t.npy")],
                   check=True, env=env, cwd=str(tmp_path))
    want = inf.inference_with_codes([torch.from_numpy(src).cuda()], bank.code("p301")[None])[0]
    assert np.load(tmp_path / "t.npy").tobytes() == want.cpu().numpy().tobytes()
    if ROOT not in sys.path:
        sys.path.insert(0, ROOT)
    import evaluate as cli
    cli.main(["-c", cfg_path, "-m", ckpt, "-d", str(tmp_path), "-eval_sets", "in_test", "-spk", "-max_pairs", "8",
              "-bank", bank_path, "-o", str(tmp_path / "ev.json")])
    assert json.loads((tmp_path / "ev.json").read_text())["in_test"]["spk"]["conversion"]["bank_speakers"] == 4
    # a changed decoder weight refuses the fitted bank; an unfitted bank of the same speaker encoder still loads
    changed = make_model(cfg)
    changed.load_state_dict(torch.load(ckpt))
    with torch.no_grad():
        changed.decoder.out_conv_layer.bias[0] += 1e-3
    with pytest.raises(ValueError, match="fitted to a different"):
        SB.SpeakerBank.load(bank_path, changed)
    plain = str(tmp_path / "plain.pt")
    pooled.save(plain)
    assert SB.SpeakerBank.load(plain, changed).fitted is None
