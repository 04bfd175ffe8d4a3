"""Model-level parity (GPU): the drop-in AE / Solver / Inferencer against (a) the fixtures
generated from the unmodified reference (tests/golden, oracle/make_golden.py) and (b) the
CPU oracle on seeded inputs, at BASELINE.json's sizes.

Tolerance (north_star): 1e-3 relative fp32 on the mel reconstruction and the KL loss; we
additionally check elementwise outputs relative to each tensor's max.
"""
import os
import types

import pytest
import torch

import oracle.ae_oracle as orc
from oracle.make_golden import load_fixture, pick

pytestmark = pytest.mark.gpu

REL = 1e-3   # north_star: mel reconstruction (L1) and KL loss within 1e-3 relative


@pytest.fixture(params=["fp32", "tf32"])
def precision(request, monkeypatch):
    """Both arithmetic modes of the conv blocks: exact FFMA kernels and tensor-core TF32."""
    monkeypatch.setenv("AVC_PRECISION", request.param)
    return request.param


def tol(precision, fp32, tf32):
    return fp32 if precision == "fp32" else tf32


def relerr(a, b):
    a, b = a.detach().float().cpu(), b.detach().float().cpu()
    return float((a - b).abs().max() / (b.abs().max() + 1e-12))


def rel_l2(a, b):
    a, b = a.detach().double().cpu().flatten(), b.detach().double().cpu().flatten()
    return float((a - b).norm() / (b.norm() + 1e-30))


def assert_grads_close(grads, ref, names, per_tensor=5e-2, overall=1e-2):
    """Gradient parity metric.  A ReLU pre-activation within ~1e-6 of zero takes a different
    branch in two fp32 implementations (or fp32 vs fp64); one such flip moves a conv weight
    gradient by ~1/sqrt(B*T) of its max (measured: 1e-2..6e-2 on single tensors at B=8 while
    every kernel is exact to 1e-6 on identical inputs -- DESIGN.md section 6).  Elementwise max
    error is therefore not a usable parity metric for full-network gradients; relative L2
    error per tensor and over the whole gradient is."""
    num = den = 0.0
    for k in names:
        g, r = pick(grads[k].detach().double().cpu(), ref[k])
        r = r.double()
        num += float((g - r).pow(2).sum())
        den += float(r.pow(2).sum())
        if float(r.norm()) > 1e-4:
            assert rel_l2(g, r) < per_tensor, (k, rel_l2(g, r))
    assert (num / den) ** 0.5 < overall, (num / den) ** 0.5


def load(golden_dir, name):
    return load_fixture(os.path.join(golden_dir, name))


def make_model(c_in):
    from adaptive_voice_conversion_b200.model import AE
    cfg = orc.default_config(c_in)
    m = AE(cfg)
    m.load_state_dict(orc.init_state(cfg, seed=0), strict=True)
    return m.cuda(), cfg


@pytest.mark.parametrize("name", ["train_c80_b1.pt", "train_c80_b4.pt", "train_c512_b2.pt", "train_c80_b2_t256.pt"])
def test_forward_backward_vs_reference_fixture(golden_dir, name, precision):
    """BASELINE config 1 (single segment) and friends: AE.forward + recon/KL + grads through
    loss.backward() (the autograd path) vs the reference's own outputs."""
    fx = load(golden_dir, name)
    rec = fx["steps"][0]
    model, cfg = make_model(fx["c_in"])
    x = fx["x"].cuda()
    mu, ls, emb, dec = model(x, eps=rec["eps"].cuda())
    for k, v in (("mu", mu), ("log_sigma", ls), ("emb", emb), ("dec", dec)):
        assert relerr(v, rec[k]) < tol(precision, REL, 8e-3), (k, relerr(v, rec[k]))   # elementwise, of max
    loss_rec = torch.nn.L1Loss()(dec, x)
    loss_kl = 0.5 * torch.mean(torch.exp(ls) + mu ** 2 - 1 - ls)
    assert abs(float(loss_rec) - float(rec["loss_rec"])) / float(rec["loss_rec"]) < REL
    assert abs(float(loss_kl) - float(rec["loss_kl"])) / float(rec["loss_kl"]) < REL
    loss = cfg["lambda"]["lambda_rec"] * loss_rec + fx["lambda_kl"] * loss_kl
    loss.backward()
    grads = {k: p.grad for k, p in model.named_parameters()}
    assert all(g is not None for g in grads.values())
    gl2 = torch.stack([grads[k].norm() for k in fx["names"]]).cpu()
    # tf32: ~0.1% of ReLU masks differ from the fp32 reference -> ~3e-2 relative L2 on gradients
    assert torch.allclose(gl2, rec["grad_l2"], rtol=tol(precision, 3e-2, 2e-1), atol=1e-5), float(((gl2 - rec["grad_l2"]).abs() / (rec["grad_l2"] + 1e-5)).max())
    assert_grads_close(grads, rec["grad_small"], list(rec["grad_small"]), per_tensor=tol(precision, 5e-2, 3e-1), overall=tol(precision, 1e-2, 1e-1))
    total = torch.sqrt(sum((g.double() ** 2).sum() for g in grads.values()))
    assert abs(float(total) - float(rec["grad_norm"])) / float(rec["grad_norm"]) < tol(precision, 5e-3, 3e-2)
    model.engine(x.device).check_tc_status()


@pytest.mark.parametrize("name", ["infer_c80.pt", "infer_c80_t512.pt"])
def test_inference_vs_reference_fixture(golden_dir, name, precision):
    """AE.inference incl. odd lengths and T_cond != T (output length 8*ceil(T/8))."""
    fx = load(golden_dir, name)
    model, _ = make_model(fx["c_in"])
    dec = model.inference(fx["x"].cuda(), fx["x_cond"].cuda())
    assert dec.shape == fx["dec"].shape
    assert relerr(dec, fx["dec"]) < tol(precision, REL, 8e-3), relerr(dec, fx["dec"])
    assert rel_l2(dec, fx["dec"]) < tol(precision, 1e-4, 3e-3)
    emb = model.get_speaker_embeddings(fx["x_cond"].cuda())
    assert relerr(emb, fx["emb"]) < tol(precision, REL, 8e-3)


def test_forward_batch256_vs_oracle(precision):
    """BASELINE config 2: batch=256 synthetic 80x128 segments, fused forward vs oracle."""
    model, cfg = make_model(80)
    g = torch.Generator().manual_seed(1)
    x = torch.randn((256, 80, 128), generator=g)
    eps = torch.randn((256, 128, 16), generator=torch.Generator().manual_seed(2))
    sd = orc.init_state(cfg, seed=0)
    with torch.no_grad():
        mu_r, ls_r, emb_r, dec_r = orc.ae_forward(sd, cfg, x, eps)
        rec_r, kl_r = orc.ae_losses(x, mu_r, ls_r, dec_r)
        mu, ls, emb, dec = model(x.cuda(), eps=eps.cuda())
    for k, a, b in (("mu", mu, mu_r), ("log_sigma", ls, ls_r), ("emb", emb, emb_r), ("dec", dec, dec_r)):
        assert relerr(a, b) < tol(precision, REL, 8e-3), (k, relerr(a, b))
        assert rel_l2(a, b) < tol(precision, 1e-4, 3e-3), (k, rel_l2(a, b))
    rec, kl = orc.ae_losses(x, mu.cpu(), ls.cpu(), dec.cpu())
    assert abs(float(rec) - float(rec_r)) / float(rec_r) < REL
    assert abs(float(kl) - float(kl_r)) / float(kl_r) < REL


def _solver_args(tmp_path):
    return types.SimpleNamespace(data_dir="synthetic", train_set="train", train_index_file="", logdir=str(tmp_path / "log"),
                                 load_model=False, load_opt=False, store_model_path=str(tmp_path / "model"),
                                 load_model_path=str(tmp_path / "model"), summary_steps=1, save_steps=1000, tag="t", iters=0)


def test_solver_step_vs_oracle(tmp_path, precision):
    """BASELINE config 3 semantics at a small batch: Solver.ae_step (fused fwd+bwd+clip+Adam)
    vs the oracle's ae_train_step: losses, grad norm, gradients and post-step weights."""
    from adaptive_voice_conversion_b200.solver import Solver
    cfg = orc.default_config(80)
    cfg["data_loader"]["batch_size"] = 8
    solver = Solver(cfg, _solver_args(tmp_path))
    sd = orc.init_state(cfg, seed=0)
    solver.model.load_state_dict(sd, strict=True)
    solver.trainer.eng.pack_weights(solver.trainer.P, need_dgrad=True)
    st = orc.AdamState(sd)
    x = torch.randn((8, 80, 128), generator=torch.Generator().manual_seed(1))
    for it in range(2):
        eps = torch.randn((8, 128, 16), generator=torch.Generator().manual_seed(50 + it))
        before = {k: v.detach().cpu().clone() for k, v in solver.model.state_dict().items()}
        res = orc.ae_train_step(sd, st, cfg, x, eps, 0.37)
        meta = solver.ae_step(x, 0.37, eps=eps.cuda())
        t_ = REL if it == 0 else 2e-2   # see tests/test_oracle_golden.py on Adam's sign sensitivity
        assert abs(meta["loss_rec"] - res["loss_rec"]) / res["loss_rec"] < t_
        assert abs(meta["loss_kl"] - res["loss_kl"]) / res["loss_kl"] < t_
        assert abs(meta["grad_norm"] - res["grad_norm"]) / res["grad_norm"] < tol(precision, 10 * t_, 5e-2)
        if it == 0:
            G = {k: v.detach().cpu().clone() for k, v in solver.trainer.G.items()}
            assert_grads_close(G, res["grads"], list(sd), per_tensor=tol(precision, 5e-2, 3e-1), overall=tol(precision, 1e-2, 1e-1))
            # optimizer integration (flat-buffer order, clip coefficient, bias correction, amsgrad):
            # the oracle's clip+Adam applied to OUR gradients must land on OUR post-step weights
            st2 = orc.AdamState(before)
            gn = orc.clip_and_adam(before, G, st2, cfg["optimizer"])
            assert abs(gn - meta["grad_norm"]) / gn < 1e-4
            for k, p in solver.model.state_dict().items():
                assert float((p.cpu() - before[k]).abs().max()) < 2e-6, k
    # checkpoint round trip in the reference's formats (.ckpt state_dict, .opt Adam state_dict)
    solver.save_model(0)
    ck = torch.load(str(tmp_path / "model.ckpt"), map_location="cpu")
    assert list(ck) == list(sd) and all(ck[k].shape == sd[k].shape for k in sd)
    opt_sd = torch.load(str(tmp_path / "model.opt"), map_location="cpu")
    ref_opt = torch.optim.Adam([torch.nn.Parameter(v.clone()) for v in sd.values()], lr=5e-4, amsgrad=True, weight_decay=1e-4)
    ref_opt.load_state_dict(opt_sd)     # loads into a stock torch Adam => format compatible
    assert float(ref_opt.state_dict()["state"][0]["step"]) == 2.0


def test_solver_step_b256_vs_oracle(tmp_path):
    """BASELINE config 3 at FULL size: one Solver.ae_step on batch=256 (the fused step, default precision) vs the
    oracle's train step on the same x / eps: losses within the 1e-3 contract, gradient norm, gradient (relative
    L2) and post-step weights."""
    from adaptive_voice_conversion_b200.solver import Solver
    B = 256
    cfg = orc.default_config(80)
    cfg["data_loader"]["batch_size"] = B
    solver = Solver(cfg, _solver_args(tmp_path))
    sd = orc.init_state(cfg, seed=0)
    solver.model.load_state_dict(sd, strict=True)
    solver.trainer.eng.pack_weights(solver.trainer.P, need_dgrad=True)
    st = orc.AdamState(sd)
    x = torch.randn((B, 80, 128), generator=torch.Generator().manual_seed(1))
    eps = torch.randn((B, 128, 16), generator=torch.Generator().manual_seed(2))
    before = {k: v.detach().cpu().clone() for k, v in solver.model.state_dict().items()}
    res = orc.ae_train_step(sd, st, cfg, x, eps, 1.0)          # sd is updated in place
    meta = solver.ae_step(x, 1.0, eps=eps.cuda())
    prec = solver.trainer.eng.precision
    assert abs(meta["loss_rec"] - res["loss_rec"]) / res["loss_rec"] < REL
    assert abs(meta["loss_kl"] - res["loss_kl"]) / res["loss_kl"] < REL
    assert abs(meta["grad_norm"] - res["grad_norm"]) / res["grad_norm"] < tol(prec, 1e-2, 3e-2)
    G = {k: v.detach().cpu().clone() for k, v in solver.trainer.G.items()}
    assert_grads_close(G, res["grads"], list(sd), per_tensor=tol(prec, 5e-2, 3e-1), overall=tol(prec, 1e-2, 1e-1))
    # the optimizer applied to OUR gradients lands on OUR weights (clip coefficient, bias correction, amsgrad, wd)
    st2 = orc.AdamState(before)
    gn = orc.clip_and_adam(before, G, st2, cfg["optimizer"])
    assert abs(gn - meta["grad_norm"]) / gn < 1e-4
    after = solver.model.state_dict()
    for k in before:
        assert float((after[k].cpu() - before[k]).abs().max()) < 2e-6, k
    # and the reference's post-step weights: one Adam step moves every element by <= lr, so two correct
    # implementations differ by at most 2*lr where the gradient sign is noise
    lr = cfg["optimizer"]["lr"]
    for k in sd:
        assert float((after[k].cpu() - sd[k]).abs().max()) <= 2.05 * lr, k
    solver.trainer.eng.check_tc_status()


def test_graph_step_matches_eager(tmp_path):
    """CUDA-graph replay of the fused step == the eager step, step by step, on injected eps (the graph reads
    x and eps from static buffers refilled by step())."""
    from adaptive_voice_conversion_b200.solver import Solver
    outs = []
    for use_graph in (False, True):
        cfg = orc.default_config(80)
        cfg["data_loader"]["batch_size"] = 4
        solver = Solver(cfg, _solver_args(tmp_path))
        solver.model.load_state_dict(orc.init_state(cfg, seed=0), strict=True)
        solver.trainer.eng.pack_weights(solver.trainer.P, need_dgrad=True)
        xs = [torch.randn((4, 80, 128), generator=torch.Generator().manual_seed(10 + i)).cuda() for i in range(3)]
        es = [torch.randn((4, 128, 16), generator=torch.Generator().manual_seed(20 + i)).cuda() for i in range(3)]
        if use_graph:
            solver.trainer.capture(xs[0], warmup=0, eps_example=es[0])
        rec = []
        for i in range(3):
            solver.trainer.step(xs[i], 1.0, eps=es[i])
            rec.append(solver.trainer.losses() + (solver.opt.flat_g.detach().cpu().clone(), solver.opt.flat_p.detach().cpu().clone()))
        if use_graph:
            assert solver.trainer._graphs is not None
        outs.append(rec)
    for i, ((l0, k0, n0, g0, p0), (l1, k1, n1, g1, p1)) in enumerate(zip(*outs)):
        # the same kernels on the same data, every reduction in a fixed order: the same bits at every step
        assert (l0, k0, n0) == (l1, k1, n1), (i, l0, l1, k0, k1, n0, n1)
        assert torch.equal(g0, g1), (i, int((g0 != g1).sum()))
        assert torch.equal(p0, p1), (i, int((p0 != p1).sum()))


def test_plain_training_loop_gets_the_graph_path(tmp_path, monkeypatch):
    """Solver.ae_step in a plain loop (what train.sh runs): the third step on the same batch shape is recorded into
    CUDA graphs and later ones replay them; a different batch shape falls back to eager launches without dropping the
    graphs; AVC_GRAPH=0 keeps everything eager."""
    from adaptive_voice_conversion_b200.solver import Solver
    cfg = orc.default_config(80)
    cfg["data_loader"]["batch_size"] = 8
    monkeypatch.setenv("AVC_GRAPH", "1")
    solver = Solver(cfg, _solver_args(tmp_path))
    tr = solver.trainer
    x = torch.randn((8, 80, 128), generator=torch.Generator().manual_seed(1))
    seen = []
    for i in range(5):
        meta = solver.ae_step(x, 1.0)
        seen.append(tr._graphs is not None)
        assert all(v == v and abs(v) < 1e4 for v in meta.values()), meta      # finite
    assert seen == [False, False, True, True, True]
    assert meta["loss_rec"] < 1.5
    solver.ae_step(x[:4], 1.0)                                                  # odd batch: eager, graphs kept
    assert tr._graphs is not None and tuple(tr._static.shape) == (8, 80, 128)
    solver.ae_step(x, 1.0)
    tr.eng.check_tc_status()
    monkeypatch.setenv("AVC_GRAPH", "0")
    s2 = Solver(cfg, _solver_args(tmp_path))
    for i in range(4):
        s2.ae_step(x, 1.0)
    assert s2.trainer._graphs is None


def test_resume_restores_the_annealing_position(tmp_path):
    """save_model writes <path>.iter next to the reference-format .ckpt/.opt; a new Solver with load_model
    continues the KL annealing where the first one stopped (the reference restarts it, solver.py:100-104)."""
    from adaptive_voice_conversion_b200.solver import Solver
    cfg = orc.default_config(80)
    cfg["data_loader"]["batch_size"] = 4
    cfg["annealing_iters"] = 10
    a = _solver_args(tmp_path)
    a.save_steps = 3
    s1 = Solver(cfg, a)
    lams = []
    s1.run_steps(3, lambda_of=lambda it: lams.append(it) or 0.1 * (it + 1))
    assert lams == [0, 1, 2] and s1.iteration == 3
    s1.save_model(iteration=2)
    a2 = _solver_args(tmp_path)
    a2.load_model = True
    s2 = Solver(cfg, a2)
    assert s2.iteration == 3
    lams2 = []
    s2.run_steps(2, lambda_of=lambda it: lams2.append(it) or 0.1 * (it + 1))
    assert lams2 == [3, 4]
    for k, v in s1.model.state_dict().items():      # same weights were loaded before the two extra steps
        assert v.shape == s2.model.state_dict()[k].shape
    assert float(s2.opt.step_dev.item()) == 5.0     # Adam's step counter resumed too (3 loaded + 2)


def test_inference_ragged_batch_equals_per_utterance(precision):
    """Inferencer.inference_ragged: (src, tgt) pairs of different lengths, bucketed by exact length, each utterance
    identical to converting it alone and within tolerance of the reference (inference.py:62-65, model.py:387-391)."""
    from adaptive_voice_conversion_b200.inference import Inferencer
    cfg = orc.default_config(80)
    args = types.SimpleNamespace(attr=None, model=None, source=None, target=None, output=None, sample_rate=24000)
    inf = Inferencer(cfg, args)
    inf.model.load_state_dict(orc.init_state(cfg, seed=0), strict=True)
    lens = [(301, 173), (128, 96), (301, 173), (64, 301), (128, 96), (301, 173), (77, 50)]
    xs = [torch.randn((t, 80), generator=torch.Generator().manual_seed(10 + i)).cuda() for i, (t, _) in enumerate(lens)]
    cs = [torch.randn((tc, 80), generator=torch.Generator().manual_seed(40 + i)).cuda() for i, (_, tc) in enumerate(lens)]
    outs = inf.inference_ragged(xs, cs)
    assert [o.shape[0] for o in outs] == [8 * ((t + 7) // 8) for t, _ in lens]
    for i, (x, c) in enumerate(zip(xs, cs)):
        _, mel = inf.inference_one_utterance(x, c)
        # same kernels, per-sample arithmetic (bit-identical wherever the tile plan does not depend on the batch;
        # a different InstanceNorm summation order is amplified to the TF32 noise floor, tests/test_gpu_properties.py)
        assert relerr(outs[i].cpu(), torch.from_numpy(mel)) < tol(precision, 1e-5, 2e-3), i
        if i in (0, 3, 6):
            with torch.no_grad():
                ref = orc.ae_inference(orc.init_state(cfg, 0), cfg, x.cpu().t()[None], c.cpu().t()[None])
            assert relerr(outs[i].t()[None], ref) < tol(precision, REL, 8e-3), i


def test_inference_graph_replay_equals_eager(monkeypatch):
    """Inferencer.inference_batch replays a captured CUDA graph (two streams inside): a replay on NEW inputs equals
    the eager call bit for bit (same kernels, same launch order per stream), and an in-place parameter update
    invalidates the graph (the packs it reads belong to the old weights)."""
    from adaptive_voice_conversion_b200.inference import Inferencer
    cfg = orc.default_config(80)
    args = types.SimpleNamespace(attr=None, model=None, source=None, target=None, output=None, sample_rate=24000)
    inf = Inferencer(cfg, args)
    inf.model.load_state_dict(orc.init_state(cfg, seed=0), strict=True)
    mk = lambda seed, t: torch.randn((4, 80, t), generator=torch.Generator().manual_seed(seed)).cuda()
    x0, c0, x1, c1 = mk(1, 128), mk(2, 96), mk(3, 128), mk(4, 96)
    monkeypatch.setenv("AVC_INFER_GRAPH", "1")        # (the suite may run with the switch off)
    inf.inference_batch(x0, c0)                       # captures
    got = inf.inference_batch(x1, c1)                 # replays on new inputs
    assert len(inf._graphs) == 1
    monkeypatch.setenv("AVC_INFER_GRAPH", "0")
    want = inf.inference_batch(x1, c1)
    assert torch.equal(got, want)
    monkeypatch.setenv("AVC_INFER_GRAPH", "1")
    with torch.no_grad():
        inf.model.decoder.out_conv_layer.bias.add_(1.0)
    got2 = inf.inference_batch(x1, c1)
    assert len(inf._graphs) == 2
    assert float((got2 - want - 1.0).abs().max()) < 1e-5
    inf.model.engine(x0.device).check_tc_status()


def test_inferencer_api(tmp_path, precision):
    from adaptive_voice_conversion_b200.inference import Inferencer
    cfg = orc.default_config(80)
    args = types.SimpleNamespace(attr=None, model=None, source=None, target=None, output=None, sample_rate=24000)
    inf = Inferencer(cfg, args)
    inf.model.load_state_dict(orc.init_state(cfg, seed=0), strict=True)
    x = torch.randn((301, 80), generator=torch.Generator().manual_seed(3))
    xc = torch.randn((173, 80), generator=torch.Generator().manual_seed(4))
    wav, mel = inf.inference_one_utterance(x.cuda(), xc.cuda())
    assert wav is None and mel.shape == (304, 80)
    with torch.no_grad():
        ref = orc.ae_inference(orc.init_state(cfg, 0), cfg, x.t()[None], xc.t()[None])
    assert relerr(torch.from_numpy(mel).t()[None], ref) < tol(precision, REL, 8e-3)
    with pytest.raises(RuntimeError):
        inf.inference_from_path()
