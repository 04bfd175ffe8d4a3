"""GPU: held-out evaluation.  avc_eval_losses against float64 torch; the per-segment losses against the float64 oracle
(with and without the decoder's spectral norm); the evaluation's dec against AE.inference bit for bit; training with
evaluations in between against training without them, bit for bit; the value logged at an iteration against a fresh
Solver on the checkpoint of that iteration; and the 2-rank table against the 1-rank table."""
import json
import os
import socket
import subprocess
import sys
import types

import numpy as np
import pytest
import torch

import oracle.ae_oracle as orc
from _eval_data import SEG, write_data_dir
from _sn_ref import power_iteration64, sn_config
from adaptive_voice_conversion_b200 import _lib as L
from adaptive_voice_conversion_b200 import data_utils as D
from adaptive_voice_conversion_b200 import evaluate as E

pytestmark = pytest.mark.gpu
HERE = os.path.dirname(os.path.abspath(__file__))


@pytest.fixture(params=["tf32", "fp32"])
def precision(request, monkeypatch):
    monkeypatch.setenv("AVC_PRECISION", request.param)
    return request.param


def bits_equal(a, b):
    return a.shape == b.shape and a.dtype == b.dtype and torch.equal(a.contiguous().view(torch.uint8), b.contiguous().view(torch.uint8))


# ----------------------------------------------------------------------------- 1. the kernel
def run_kernel(dec4, x, mu4, ls4, out, first):
    B, C, T = x.shape
    d = L.EvalDesc(B=B, C=C, T=T, C_lat=mu4.shape[1] * 4, T_lat=mu4.shape[2], dec=dec4.data_ptr(), x=x.data_ptr(),
                   mu=mu4.data_ptr(), ls=ls4.data_ptr(), out=out.data_ptr(), first=first)
    L.check(L.load().avc_eval_losses(d, torch.cuda.current_stream().cuda_stream), "avc_eval_losses")


def planar(a4):
    B, Cq, T, _ = a4.shape
    return a4.permute(0, 1, 3, 2).reshape(B, Cq * 4, T)


@pytest.mark.parametrize("B", [1, 3, 128])
@pytest.mark.parametrize("C, T", [(80, 128), (512, 128), (80, 64), (512, 64)], ids=["c80", "c512", "c80-frame2", "c512-frame2"])
def test_kernel_matches_float64(B, C, T):
    g = torch.Generator().manual_seed(B * 1000 + C + T)
    n = 2 * B + 1                       # two full batches and a ragged one of 1 at the end of the table
    Tl = T // 8
    dec4 = torch.randn((n, C // 4, T, 4), generator=g)
    x = torch.randn((n, C, T), generator=g)
    mu4 = torch.randn((n, 32, Tl, 4), generator=g)
    ls4 = torch.randn((n, 32, Tl, 4), generator=g) * 0.5
    dev = [t.cuda() for t in (dec4, x, mu4, ls4)]
    outs = []
    for _ in range(2):
        out = torch.full((n, 2), float("nan"), dtype=torch.float64, device="cuda")
        for first in range(0, n, B):
            c = min(B, n - first)
            run_kernel(*(t[first:first + c] for t in dev), out, first)
        outs.append(out.cpu())
    assert bits_equal(outs[0], outs[1])
    rec = (planar(dec4).double() - x.double()).abs().sum((1, 2))
    m, l = mu4.double(), ls4.double()
    kl = (torch.exp(l) + m ** 2 - 1 - l).sum((1, 2, 3))
    got = outs[0]
    assert float(((got[:, 0] - rec).abs() / rec).max()) < 1e-12
    assert float(((got[:, 1] - kl).abs() / kl).max()) < 1e-12
    # a sample's sums do not depend on its batch
    one = torch.full((n, 2), float("nan"), dtype=torch.float64, device="cuda")
    run_kernel(*(t[n - 1:n] for t in dev), one, n - 1)
    assert bits_equal(one[n - 1].cpu(), got[n - 1])


# ----------------------------------------------------------------------------- 2./3. against the oracle and inference
def make_model(sn, c_in=80):
    from adaptive_voice_conversion_b200.model import AE
    cfg = sn_config(c_in) if sn else orc.default_config(c_in)
    cfg["data_loader"]["batch_size"] = 16
    if sn:                # the reference's seeded initialisation (u and v included)
        torch.manual_seed(0)
        model = AE(cfg)
    else:
        model = AE(cfg)
        model.load_state_dict(orc.init_state(cfg, seed=0), strict=True)
    return cfg, model.cuda()


def oracle_state(model):
    """float64 state for the oracle; with the spectral norm, weight = weight_orig / sigma of the stored u, v (eval mode)."""
    sd = {k: v.detach().double().cpu() for k, v in model.state_dict().items()}
    for k in [k for k in sd if k.endswith(".weight_orig")]:
        base = k[: -len(".weight_orig")]
        sd[base + ".weight"] = power_iteration64(sd[k], sd[base + ".weight_u"], sd[base + ".weight_v"], iterate=False)[3]
    return sd


@pytest.mark.parametrize("sn,seg", [(False, SEG), (True, SEG), (False, 256)], ids=["plain", "sn", "plain-seg256"])
def test_per_segment_losses_match_the_oracle(tmp_path, precision, sn, seg):
    cfg, model = make_model(sn)
    cfg["data_loader"]["segment_size"] = seg    # (256: the conv blocks' longer-sequence routes, see test_step_routes_host.py)
    model.train()          # the evaluation is eval mode whatever the flag; it leaves the flag alone
    n = 40                 # batches of 16, 16 and 8
    d = write_data_dir(tmp_path / "data", 80, {"in_test": n}, seg=seg)
    held = E.HeldOut(["in_test"], d, cfg, device="cuda")
    u0 = {k: v.clone() for k, v in model.named_buffers()}
    tab = held.tables(model)["in_test"].cpu()
    assert model.training and all(bits_equal(v, u0[k]) for k, v in model.named_buffers())
    data, index = D.load_corpus(os.path.join(d, "in_test.pkl"), os.path.join(d, f"in_test_samples_{seg}.json"))
    pds = D.PickleDataset.from_loaded(data, index, seg)
    x = D.CollateFn(1)([pds[i] for i in range(n)]).double()
    sd = oracle_state(model)
    with torch.no_grad():
        dec = orc.ae_inference(sd, cfg, x, x)
        mu, ls = orc.content_encoder(sd, x, cfg["ContentEncoder"]["subsample"])
    rec = (dec - x).abs().sum((1, 2))
    kl = (torch.exp(ls) + mu ** 2 - 1 - ls).sum((1, 2))
    tol = 1e-3 if precision == "tf32" else 1e-5
    e_rec = float(((tab[:, 0] - rec).abs() / rec).max())
    e_kl = float(((tab[:, 1] - kl).abs() / kl).max())
    assert e_rec < tol and e_kl < tol, (e_rec, e_kl)
    res = held.evaluate(model)["in_test"]
    assert res["n"] == n
    assert abs(res["loss_rec"] - float(rec.sum()) / (n * 80 * seg)) < tol * res["loss_rec"]
    assert abs(res["loss_kl"] - 0.5 * float(kl.sum()) / (n * 128 * seg // 8)) < tol * res["loss_kl"]


@pytest.mark.parametrize("sn", [False, True], ids=["plain", "sn"])
def test_eval_dec_is_inference_bit_for_bit(precision, sn):
    _, model = make_model(sn)
    x = torch.randn((16, 80, SEG), generator=torch.Generator().manual_seed(5)).cuda()
    eng, P = E.eval_params(model, torch.device("cuda"))
    out = torch.zeros((20, 2), dtype=torch.float64, device="cuda")
    dec = eng.unpack_a4(eng.eval_losses(P, x, out, 4))
    model.eval()
    ref = model.inference(x, x)
    assert bits_equal(dec, ref)
    rec = (ref.double() - x.double()).abs().sum((1, 2)).cpu()
    assert float(((out[4:, 0].cpu() - rec).abs() / rec).max()) < 1e-12
    assert (out[:4] == 0).all()


# ----------------------------------------------------------------------------- 4./5. inside training
# 7 full batches per epoch.  (A short batch is left out: the pipelined loop reads a step's losses after the next step is
# enqueued, and decodes them with that step's element count, so the step before a shape change would report different
# means in a run that drains there.)
N_TRAIN, B_TRAIN = 112, 16


def data_dir(tmp_path):
    return write_data_dir(tmp_path / "data", 80, {"train": N_TRAIN, "in_test": 40, "out_test": 24}, seed=3)


def solver(tmp_path, d, name, cfg, eval_steps=0, load=None, save_steps=10 ** 9):
    from adaptive_voice_conversion_b200.solver import Solver
    args = types.SimpleNamespace(data_dir=d, train_set="train", train_index_file=f"train_samples_{SEG}.json",
                                 logdir=str(tmp_path / "log"), load_model=load is not None, load_opt=False,
                                 store_model_path=str(tmp_path / name), load_model_path=str(tmp_path / (load or name)),
                                 summary_steps=1, save_steps=save_steps, tag="t", iters=0, eval_steps=eval_steps,
                                 eval_sets="in_test,out_test")
    torch.manual_seed(0)
    s = Solver(cfg, args)
    s.losses = []
    orig = s.trainer.losses_async

    def recording():
        get = orig()

        def g():
            v = get()
            s.losses.append(v)
            return v
        return g
    s.trainer.losses_async = recording
    return s


def train_config(sn):
    cfg = sn_config(80) if sn else orc.default_config(80)
    cfg["data_loader"]["batch_size"] = B_TRAIN
    return cfg


@pytest.mark.parametrize("graph", ["1", "0"], ids=["graph", "eager"])
@pytest.mark.parametrize("sn", [False, True], ids=["plain", "sn"])
def test_evaluations_do_not_change_training(tmp_path, monkeypatch, graph, sn):
    monkeypatch.setenv("AVC_GRAPH", graph)
    d = data_dir(tmp_path)
    cfg = train_config(sn)
    runs = []
    for name, k in (("plain", 0), ("eval", 3)):
        s = solver(tmp_path, d, name, cfg, eval_steps=k)
        s.train(9)      # capture at step 3, replay after; evaluations after steps 3, 6 and 9
        assert s.iteration == 9 and len(s.losses) == 9
        assert (s.trainer._graphs is not None) == (graph == "1")
        runs.append(dict(losses=s.losses, p=s.opt.flat_p.cpu(), m=s.opt.flat_m.cpu(), v=s.opt.flat_v.cpu(),
                         vmax=s.opt.flat_vmax.cpu(), buf={k_: b.cpu() for k_, b in s.model.named_buffers()},
                         training=s.model.training))
        del s
    a, b = runs
    assert a["losses"] == b["losses"]
    for k in ("p", "m", "v", "vmax"):
        assert bits_equal(a[k], b[k]), k
    assert a["buf"].keys() == b["buf"].keys() and (len(a["buf"]) > 0) == sn
    assert all(bits_equal(a["buf"][k], b["buf"][k]) for k in a["buf"])
    assert a["training"] == b["training"]
    lines = [json.loads(x) for x in open(tmp_path / "eval.eval.jsonl").read().splitlines()]
    assert [x["iteration"] for x in lines] == [3, 6, 9]
    assert all(set(x["sets"]) == {"in_test", "out_test"} and np.isfinite(x["sets"]["in_test"]["loss_rec"]) for x in lines)


@pytest.mark.parametrize("sn", [False, True], ids=["plain", "sn"])
def test_logged_value_equals_a_fresh_solver_on_the_checkpoint(tmp_path, sn):
    d = data_dir(tmp_path)
    cfg = train_config(sn)
    s = solver(tmp_path, d, "a", cfg, eval_steps=5, save_steps=5)
    s.train(5)            # run_steps(5) returns, then the evaluation at 5; the checkpoint is written at step 5
    logged = json.loads(open(tmp_path / "a.eval.jsonl").read().splitlines()[-1])
    assert logged["iteration"] == 5
    del s
    fresh = solver(tmp_path, d, "b", cfg, load="a")
    assert fresh.iteration == 5 and fresh.held_out is None
    res = fresh.evaluate()
    assert json.loads(json.dumps(res)) == logged["sets"]


# ----------------------------------------------------------------------------- 6. data parallel
def _free_port():
    s = socket.socket()
    s.bind(("127.0.0.1", 0))
    p = s.getsockname()[1]
    s.close()
    return p


def test_two_rank_table_equals_one_rank_table(tmp_path):
    d = write_data_dir(tmp_path / "data", 80, {"in_test": 70, "out_test": 16}, seed=7)   # 70 = 4 x 16 + 6: ragged
    _, model = make_model(False)
    cfg = orc.default_config(80)
    cfg["data_loader"]["batch_size"] = 16
    single = {k: v.cpu() for k, v in E.HeldOut(["in_test", "out_test"], d, cfg, device="cuda").tables(model).items()}
    ngpu = torch.cuda.device_count()
    backend = "nccl" if ngpu >= 2 else "gloo"
    port = _free_port()
    procs = []
    for rank in range(2):
        env = dict(os.environ, RANK=str(rank), WORLD_SIZE="2", LOCAL_RANK=str(rank if ngpu >= 2 else 0),
                   MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port))
        procs.append(subprocess.Popen([sys.executable, os.path.join(HERE, "_dp_eval_worker.py"), str(tmp_path), d, backend],
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
    for rank in range(2):
        got = torch.load(str(tmp_path / f"eval_rank{rank}.pt"))
        assert got.keys() == single.keys()
        for k in single:
            assert bits_equal(got[k], single[k]), (rank, k)
