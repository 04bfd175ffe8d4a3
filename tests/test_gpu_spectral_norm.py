"""GPU: the decoder's spectral norm (Decoder.sn).  The kernels against the float64 restatement (tests/_sn_ref.py) on
the same fp32 inputs; their determinism; and the model, solver, inferencer, graph, resume and data-parallel paths
against the fixtures of the unmodified reference (tools/make_golden_sn.py) or against themselves."""
import os
import socket
import subprocess
import sys
import types

import pytest
import torch

from _sn_ref import adjoint64, power_iteration64, sn_config, state_checksum
from oracle.make_golden import load_fixture, pick

pytestmark = pytest.mark.gpu
HERE = os.path.dirname(os.path.abspath(__file__))
REL = 1e-3
KERNEL_TOL = 1e-5       # relative to each tensor's max, fp32 kernels against float64

# (h, w) of every wrapped decoder layer at c_in 80 and 512 (in_conv, first / second convs, affine, out_conv) + a sweep
DECODER_SHAPES = [(128, 128, 1), (128, 128, 5), (256, 128, 5), (256, 128), (80, 128, 1), (512, 128, 1)]
SWEEP_SHAPES = [(1, 1), (3, 7), (17, 33), (16, 4096), (4096, 1), (1000, 3, 3), (4096, 4096)]


def relmax(a, b):
    a, b = a.detach().double().cpu(), b.detach().double().cpu()
    return float((a - b).abs().max() / (b.abs().max() + 1e-30))


def rel_l2(a, b):
    a, b = a.detach().double().cpu().flatten(), b.detach().double().cpu().flatten()
    return float((a - b).norm() / (b.norm() + 1e-30))


def run_kernels(Ws, us, vs, mode, grads=None):
    """avc_spectral_norm (and avc_spectral_norm_bwd with grads) on one item table; u, v, grads change in place.
    -> (sigma [n], W_bar list).  The scratch starts as NaN: a read of a slot no kernel wrote would show."""
    from adaptive_voice_conversion_b200 import _lib as L
    lib = L.load()
    n = len(Ws)
    shapes = [(W.shape[0], W[0].numel()) for W in Ws]
    sizes = [int(lib.avc_spectral_norm_scratch_floats(h, w)) for h, w in shapes]
    scratch = torch.full((sum(sizes),), float("nan"), device="cuda")
    sigma = torch.zeros(n, device="cuda")
    wbar = [torch.full_like(W, float("nan")) for W in Ws]
    items = (L.SnItem * n)()
    off = 0
    for i, (W, (h, w), sz) in enumerate(zip(Ws, shapes, sizes)):
        it = items[i]
        it.weight, it.w_bar, it.u, it.v = W.data_ptr(), wbar[i].data_ptr(), us[i].data_ptr(), vs[i].data_ptr()
        it.sigma, it.grad = sigma.data_ptr() + 4 * i, grads[i].data_ptr() if grads is not None else None
        it.scratch_off, it.h, it.w = off, h, w
        off += sz
    raw = torch.frombuffer(bytearray(bytes(items)), dtype=torch.uint8).cuda()
    st = torch.cuda.current_stream().cuda_stream
    mh, mw = max(h for h, _ in shapes), max(w for _, w in shapes)
    L.check(lib.avc_spectral_norm(raw.data_ptr(), n, mh, mw, mode, scratch.data_ptr(), st), "spectral_norm")
    if grads is not None:
        L.check(lib.avc_spectral_norm_bwd(raw.data_ptr(), n, mh, mw, scratch.data_ptr(), st), "spectral_norm_bwd")
    torch.cuda.synchronize()
    return sigma, wbar


def make_inputs(shape, seed):
    g = torch.Generator().manual_seed(seed)
    W = torch.randn(shape, generator=g) * 0.05
    h, w = shape[0], W[0].numel()
    u = torch.nn.functional.normalize(torch.randn(h, generator=g), dim=0, eps=1e-12)
    v = torch.nn.functional.normalize(torch.randn(w, generator=g), dim=0, eps=1e-12)
    G = torch.randn(shape, generator=g)
    return W, u, v, G


@pytest.mark.parametrize("shape", DECODER_SHAPES + SWEEP_SHAPES, ids=lambda s: "x".join(map(str, s)))
@pytest.mark.parametrize("iterate", [True, False], ids=["iterate", "fixed"])
def test_kernels_vs_float64(shape, iterate):
    from adaptive_voice_conversion_b200 import _lib as L
    W, u0, v0, G = make_inputs(shape, seed=sum(shape))
    u, v, g = u0.cuda(), v0.cuda(), G.cuda()
    sigma, wbar = run_kernels([W.cuda()], [u], [v], L.SN_ITERATE if iterate else L.SN_FIXED, grads=[g])
    u64, v64, s64, wbar64 = power_iteration64(W, u0, v0, iterate=iterate)
    assert relmax(u, u64) < KERNEL_TOL and relmax(v, v64) < KERNEL_TOL, (relmax(u, u64), relmax(v, v64))
    if not iterate:
        assert torch.equal(u.cpu(), u0) and torch.equal(v.cpu(), v0)      # eval mode never writes them
    assert abs(float(sigma[0]) - float(s64)) <= KERNEL_TOL * abs(float(s64))
    assert relmax(wbar[0], wbar64) < KERNEL_TOL
    # the backward against the float64 adjoint at the kernel's own u, v, sigma and W_bar
    want = adjoint64(G, wbar[0].cpu(), u.cpu(), v.cpu(), float(sigma[0]))
    scale = float(G.abs().max()) / float(sigma[0])     # the size of the adjoint's terms (the result may cancel to 0)
    err = float((g.cpu().double() - want).abs().max()) / scale
    assert err < KERNEL_TOL, err


def test_kernels_are_deterministic_and_item_independent():
    """Repeated calls give the same bits, and every item gets the same bits alone or in a launch with the others."""
    from adaptive_voice_conversion_b200 import _lib as L
    shapes = DECODER_SHAPES + [(17, 33), (1000, 3, 3)]
    ins = [make_inputs(s, seed=7 + i) for i, s in enumerate(shapes)]
    for mode in (L.SN_ITERATE, L.SN_FIXED):
        outs = []
        for _ in range(2):
            us, vs, gs = [u.cuda() for _, u, _, _ in ins], [v.cuda() for _, _, v, _ in ins], [G.cuda() for *_, G in ins]
            sigma, wbar = run_kernels([W.cuda() for W, *_ in ins], us, vs, mode, grads=gs)
            outs.append((sigma.cpu(), [t.cpu() for t in wbar], [t.cpu() for t in us], [t.cpu() for t in vs], [t.cpu() for t in gs]))
        (s0, w0, u0, v0, g0), (s1, w1, u1, v1, g1) = outs
        assert torch.equal(s0, s1) and all(torch.equal(a, b) for a, b in zip(w0 + u0 + v0 + g0, w1 + u1 + v1 + g1))
        for i, (W, u, v, G) in enumerate(ins):
            us, vs, gs = [u.cuda()], [v.cuda()], [G.cuda()]
            sigma, wbar = run_kernels([W.cuda()], us, vs, mode, grads=gs)
            assert torch.equal(sigma.cpu()[0], s0[i]) and torch.equal(wbar[0].cpu(), w0[i]), (mode, i)
            assert torch.equal(us[0].cpu(), u0[i]) and torch.equal(vs[0].cpu(), v0[i]) and torch.equal(gs[0].cpu(), g0[i]), (mode, i)


# ------------------------------------------------------------------ the model against the reference's fixtures
@pytest.fixture(params=["fp32", "tf32"])
def precision(request, monkeypatch):
    monkeypatch.setenv("AVC_PRECISION", request.param)
    return request.param


def tol(precision, fp32, tf32):
    return fp32 if precision == "fp32" else tf32


def fixture(golden_dir, name):
    return load_fixture(os.path.join(golden_dir, name))


def reference_init(fx):
    """The reference's initial state: torch.manual_seed(seed); AE(cfg) (tests/test_spectral_norm_host.py)."""
    from adaptive_voice_conversion_b200.model import AE
    torch.manual_seed(fx["init_seed"])
    m = AE(sn_config(fx["c_in"]))
    assert torch.equal(state_checksum(m.state_dict()), fx["state_checksum"])
    return m


def sn_errors(model, rec, sigma=None):
    """max relative errors of u, v (of max) and sigma against a fixture snapshot {layer: {u, v, sigma}}."""
    mods = dict(model.named_modules())
    eng = model.engine(next(model.parameters()).device)
    names = eng.sn_names()
    eu = ev = es = 0.0
    for n, r in rec.items():
        eu = max(eu, relmax(mods[n].weight_u, r["u"]))
        ev = max(ev, relmax(mods[n].weight_v, r["v"]))
        s = float((sigma if sigma is not None else eng._sn_sigma)[names.index(n)])
        es = max(es, abs(s - float(r["sigma"])) / float(r["sigma"]))
    return eu, ev, es


def test_forward_backward_vs_reference_fixture(golden_dir, precision):
    """AE.forward in training mode (one power iteration), the losses, u / v / sigma, and the weight_orig gradients
    through loss.backward() against the reference's first step."""
    fx = fixture(golden_dir, "train_sn_c80_b4.pt")
    rec = fx["steps"][0]
    model = reference_init(fx).cuda()
    cfg = model.config
    x = fx["x"].cuda()
    mu, ls, emb, dec = model(x, eps=rec["eps"].cuda())
    eu, ev, es = sn_errors(model, rec["sn"])
    print(f"\nsn-error first forward ({precision}): u {eu:.2e} v {ev:.2e} sigma {es:.2e} (relative)")
    assert eu < 1e-5 and ev < 1e-5 and es < 1e-5, (eu, ev, es)    # fp32 weights only: no TF32 in the power iteration
    for k, v in (("mu", mu), ("log_sigma", ls), ("emb", emb), ("dec", dec)):
        assert relmax(v, rec[k]) < tol(precision, REL, 8e-3), (k, relmax(v, rec[k]))
    loss_rec = torch.nn.L1Loss()(dec, x)
    loss_kl = 0.5 * torch.mean(torch.exp(ls) + mu ** 2 - 1 - ls)
    assert abs(float(loss_rec) - float(rec["loss_rec"])) / float(rec["loss_rec"]) < REL
    assert abs(float(loss_kl) - float(rec["loss_kl"])) / float(rec["loss_kl"]) < REL
    (cfg["lambda"]["lambda_rec"] * loss_rec + fx["lambda_kl"] * loss_kl).backward()
    grads = {k: p.grad for k, p in model.named_parameters()}
    gl2 = torch.stack([grads[k].norm() for k in fx["names"]]).cpu()
    assert torch.allclose(gl2, rec["grad_l2"], rtol=tol(precision, 3e-2, 2e-1), atol=1e-5)
    num = den = 0.0
    for k, r in rec["grad_small"].items():
        g, r = pick(grads[k].detach().double().cpu(), r)
        num += float((g - r.double()).pow(2).sum())
        den += float(r.double().pow(2).sum())
        if float(r.norm()) > 1e-4:
            assert rel_l2(g, r) < tol(precision, 5e-2, 3e-1), (k, rel_l2(g, r))
    assert (num / den) ** 0.5 < tol(precision, 1e-2, 1e-1)
    dec_names = [k for k in rec["grad_small"] if k.endswith(".weight_orig")]
    assert len(dec_names) == 3
    total = torch.sqrt(sum((g.double() ** 2).sum() for g in grads.values()))
    assert abs(float(total) - float(rec["grad_norm"])) / float(rec["grad_norm"]) < tol(precision, 5e-3, 3e-2)
    model.engine(x.device).check_tc_status()


def _solver_args(tmp_path, **kw):
    a = types.SimpleNamespace(data_dir="synthetic", train_set="train", train_index_file="", logdir=str(tmp_path / "log"),
                              load_model=False, load_opt=False, store_model_path=str(tmp_path / "model"),
                              load_model_path=str(tmp_path / "model"), summary_steps=1, save_steps=1000, tag="t", iters=0)
    a.__dict__.update(kw)
    return a


def make_solver(tmp_path, fx, batch, **kw):
    from adaptive_voice_conversion_b200.solver import Solver
    cfg = sn_config(fx["c_in"])
    cfg["data_loader"]["batch_size"] = batch
    os.makedirs(tmp_path, exist_ok=True)
    solver = Solver(cfg, _solver_args(tmp_path, **kw))
    if not kw.get("load_model"):
        solver.model.load_state_dict(reference_init(fx).state_dict(), strict=True)
        solver.trainer.eng.pack_weights(solver.trainer.P, need_dgrad=True)
    return solver


def test_solver_steps_vs_reference_fixture(tmp_path, golden_dir, precision):
    """Three Solver.ae_steps (the fused step: power iteration, re-pack, backward correction, clip, Adam on weight_orig)
    against the reference's three Adam steps; u and v after step k are the reference's after its k-th step."""
    fx = fixture(golden_dir, "train_sn_c80_b4.pt")
    solver = make_solver(tmp_path, fx, 4)
    x = fx["x"]
    for i, rec in enumerate(fx["steps"]):
        meta = solver.ae_step(x, fx["lambda_kl"], eps=rec["eps"].cuda())
        t_ = REL if i == 0 else 2e-2      # Adam's sign sensitivity after the first step (tests/test_gpu_model.py)
        assert abs(meta["loss_rec"] - float(rec["loss_rec"])) / float(rec["loss_rec"]) < t_, (i, meta)
        assert abs(meta["loss_kl"] - float(rec["loss_kl"])) / float(rec["loss_kl"]) < t_, (i, meta)
        assert abs(meta["grad_norm"] - float(rec["grad_norm"])) / float(rec["grad_norm"]) < tol(precision, 10 * t_, 5e-2), (i, meta)
        eu, ev, es = sn_errors(solver.model, rec["sn"])
        print(f"\nsn-error after step {i} ({precision}): u {eu:.2e} v {ev:.2e} sigma {es:.2e}")
        # step 0 starts from the reference's weights: u, v and sigma to fp32 rounding.  Later steps start from weights
        # that Adam moved by +-lr where a gradient's sign is rounding noise, and u, v follow W
        if i == 0:
            assert eu < 1e-5 and ev < 1e-5 and es < 1e-5, (i, eu, ev, es)
        else:
            assert eu < tol(precision, 1e-2, 5e-2) and ev < tol(precision, 1e-2, 5e-2), (i, eu, ev)
            assert es < tol(precision, 1e-3, 5e-3), (i, es)
        pl2 = torch.stack([p.detach().norm() for p in solver.model.parameters()]).cpu()
        prt = 1e-3 if i == 0 else tol(precision, 1e-3, 3e-2)
        assert torch.allclose(pl2, rec["param_l2_after"], rtol=prt), (i, float(((pl2 - rec["param_l2_after"]).abs() / rec["param_l2_after"]).max()))
    solver.trainer.eng.check_tc_status()


def test_inference_vs_reference_fixture(golden_dir, precision):
    """Eval mode: sigma from the stored u and v, which do not move.  Training mode: one power iteration per call."""
    fx = fixture(golden_dir, "infer_sn_c80.pt")
    model = reference_init(fx).cuda()
    model.eval()
    x, xc = fx["x"].cuda(), fx["x_cond"].cuda()
    dec = model.inference(x, xc)
    got, want = pick(dec, fx["dec"])
    assert relmax(got, want) < tol(precision, REL, 8e-3), relmax(got, want)
    mods = dict(model.named_modules())
    for n, r in fx["sn_init"].items():
        assert torch.equal(mods[n].weight_u.cpu(), r["u"]) and torch.equal(mods[n].weight_v.cpu(), r["v"]), n
    _, _, es = sn_errors(model, fx["sn_eval"])
    assert es < 1e-5, es
    model.train()
    dec = model.inference(x, xc)
    got, want = pick(dec, fx["dec_train"])
    assert relmax(got, want) < tol(precision, REL, 8e-3), relmax(got, want)
    eu, ev, es = sn_errors(model, fx["sn_train"])
    assert eu < 1e-5 and ev < 1e-5 and es < 1e-5, (eu, ev, es)
    assert not torch.equal(mods["decoder.in_conv_layer"].weight_u.cpu(), fx["sn_init"]["decoder.in_conv_layer"]["u"])


def test_inferencer_graph_sees_new_u_v(golden_dir, monkeypatch):
    """Inferencer.inference_batch replays a captured graph equal to the eager call; a load_state_dict that changes only
    u and v makes it capture again."""
    from adaptive_voice_conversion_b200.inference import Inferencer
    fx = fixture(golden_dir, "infer_sn_c80.pt")
    args = types.SimpleNamespace(attr=None, model=None, source=None, target=None, output=None, sample_rate=24000)
    inf = Inferencer(sn_config(80), args)
    sd = reference_init(fx).state_dict()
    inf.model.load_state_dict(sd, strict=True)
    mk = lambda seed, t: torch.randn((2, 80, t), generator=torch.Generator().manual_seed(seed)).cuda()   # noqa: E731
    x, c = mk(1, 128), mk(2, 96)
    monkeypatch.setenv("AVC_INFER_GRAPH", "1")
    inf.inference_batch(x, c)
    got = inf.inference_batch(x, c)
    monkeypatch.setenv("AVC_INFER_GRAPH", "0")
    assert torch.equal(got, inf.inference_batch(x, c))
    monkeypatch.setenv("AVC_INFER_GRAPH", "1")
    sd2 = dict(sd)
    for k in sd2:
        if k.endswith((".weight_u", ".weight_v")):
            sd2[k] = -sd2[k]          # the power iteration's sign flips; sigma = u . (W v) is unchanged
    sd2["decoder.out_conv_layer.weight_v"] = torch.nn.functional.normalize(torch.ones_like(sd["decoder.out_conv_layer.weight_v"]), dim=0)
    inf.model.load_state_dict(sd2, strict=True)
    got2 = inf.inference_batch(x, c)
    assert len(inf._graphs) == 2
    monkeypatch.setenv("AVC_INFER_GRAPH", "0")
    assert torch.equal(got2, inf.inference_batch(x, c)) and not torch.equal(got, got2)


def _run(solver, xs, es):
    out = []
    for x, e in zip(xs, es):
        solver.trainer.step(x, 1.0, eps=e)
        out.append(solver.trainer.losses() + (solver.opt.flat_p.detach().cpu().clone(),
                                              torch.cat([b.detach().cpu().reshape(-1) for b in solver.model.buffers()])))
    return out


def _same(a, b):
    for i, ((l0, k0, n0, p0, uv0), (l1, k1, n1, p1, uv1)) in enumerate(zip(a, b)):
        assert (l0, k0, n0) == (l1, k1, n1), (i, l0, l1)
        assert torch.equal(p0, p1) and torch.equal(uv0, uv1), (i, int((p0 != p1).sum()), int((uv0 != uv1).sum()))


def test_graph_replay_and_resume_are_bit_identical(tmp_path, golden_dir, precision):
    """Graph replay == eager steps, and a run resumed from .ckpt / .opt / .iter == the uninterrupted run: losses,
    parameters, u and v, bit for bit."""
    fx = fixture(golden_dir, "train_sn_c80_b4.pt")
    xs = [torch.randn((4, 80, 128), generator=torch.Generator().manual_seed(10 + i)).cuda() for i in range(4)]
    es = [torch.randn((4, 128, 16), generator=torch.Generator().manual_seed(20 + i)).cuda() for i in range(4)]
    eager = _run(make_solver(tmp_path / "a", fx, 4), xs, es)
    s = make_solver(tmp_path / "b", fx, 4)
    s.trainer.capture(xs[0], warmup=0, eps_example=es[0])
    graph = _run(s, xs, es)
    assert s.trainer._graphs is not None
    _same(eager, graph)
    s1 = make_solver(tmp_path / "c", fx, 4)
    first = _run(s1, xs[:2], es[:2])
    s1.save_model(1)
    s2 = make_solver(tmp_path / "c", fx, 4, load_model=True)
    _same(eager, first + _run(s2, xs[2:], es[2:]))


def _free_port():
    s = socket.socket()
    s.bind(("127.0.0.1", 0))
    p = s.getsockname()[1]
    s.close()
    return p


def test_two_rank_step_equals_single_process_step(tmp_path, golden_dir):
    """DP: both ranks hold bitwise equal u and v (broadcast at start, then the same power iteration without
    communication), and a 2-rank step equals a 1-rank step on the concatenated batch."""
    per_rank = 8
    fx = fixture(golden_dir, "train_sn_c80_b4.pt")
    ref = make_solver(tmp_path / "ref", fx, 2 * per_rank)
    x = torch.randn((2 * per_rank, 80, 128), generator=torch.Generator().manual_seed(1)).cuda()
    want = []
    for it in range(2):
        eps = torch.randn((2 * per_rank, 128, 16), generator=torch.Generator().manual_seed(50 + it)).cuda()
        ref.trainer.step(x, 0.37, eps=eps)
        lr_, lk_, gn_ = ref.trainer.losses()
        want.append(dict(loss_rec=lr_, loss_kl=lk_, grad_norm=gn_, flat_g=ref.opt.flat_g.detach().cpu().clone(),
                         flat_p=ref.opt.flat_p.detach().cpu().clone(),
                         uv=torch.cat([b.detach().cpu().reshape(-1) for b in ref.model.buffers()])))
    ngpu = torch.cuda.device_count()
    backend = "nccl" if ngpu >= 2 else "gloo"
    port = _free_port()
    procs = []
    for rank in range(2):
        env = dict(os.environ, RANK=str(rank), WORLD_SIZE="2", LOCAL_RANK=str(rank if ngpu >= 2 else 0),
                   MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port))
        procs.append(subprocess.Popen([sys.executable, os.path.join(HERE, "_dp_sn_worker.py"), str(tmp_path), backend, str(per_rank)],
                                      env=env, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True))
    outs = []
    for p in procs:
        try:
            outs.append(p.communicate(timeout=600)[0])
        except subprocess.TimeoutExpired:
            for q in procs:
                q.kill()
            raise
    for p, o in zip(procs, outs):
        assert p.returncode == 0, o[-3000:]
    r0, r1 = torch.load(str(tmp_path / "rank0.pt")), torch.load(str(tmp_path / "rank1.pt"))
    assert torch.equal(r0["init_uv"], r1["init_uv"])
    for it in range(2):
        a, b, s = r0["steps"][it], r1["steps"][it], want[it]
        assert torch.equal(a["uv"], b["uv"]) and torch.equal(a["flat_p"], b["flat_p"]) and torch.equal(a["flat_g"], b["flat_g"])
        if it == 0:     # same weights, same kernels: the power iteration of step 0 is the single process's, bit for bit
            assert torch.equal(a["uv"], s["uv"])
        assert rel_l2(a["uv"], s["uv"]) < 1e-4
        gt, lt = (2e-4, 1e-5) if it == 0 else (1e-1, 2e-3)     # tests/test_gpu_dp.py
        assert rel_l2(0.5 * a["flat_g"], s["flat_g"]) < gt, (it, rel_l2(0.5 * a["flat_g"], s["flat_g"]))
        for k in ("loss_rec", "loss_kl"):
            assert abs(0.5 * (a[k] + b[k]) - s[k]) / s[k] < lt, (it, k)
        assert rel_l2(a["flat_p"], s["flat_p"]) < 1e-3
