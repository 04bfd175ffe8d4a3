"""GPU, at BASELINE.json's full size (B=256, 80 mels x 128 frames): properties of the train step
that hold whatever the batch size and need no CPU-sized oracle run --
  * per-sample independence of the forward (InstanceNorm statistics are per sample),
  * batch-permutation invariance of the gradient,
  * homogeneity of the gradient in (lambda_rec, lambda_kl),
  * data-parallel semantics: the gradient of the whole batch is the mean of the gradients of its
    two halves (what the NCCL all-reduce + 1/world scale computes).
Both arithmetic modes.  In tf32 mode activations that feed a tensor-core conv are ROUNDED to a 10-bit mantissa:
rounding is discontinuous, so a 1e-7 difference in an InstanceNorm sum (another summation order for another
tile shape) is amplified layer by layer up to the TF32 noise floor (~5e-4) -- exactly as far as either result is
from the fp32 reference.  Measured in round 2: every kernel is bit-identical or 1e-7
apart per sample across batch sizes, the 14-layer content encoder 5e-4.  Tolerances below reflect that.
"""
import os
import types

import pytest
import torch

import oracle.ae_oracle as orc

pytestmark = pytest.mark.gpu

B, C_IN, T = 256, 80, 128


def rel_l2(a, b):
    a, b = a.detach().double().flatten(), b.detach().double().flatten()
    return float((a - b).norm() / (b.norm() + 1e-30))


@pytest.fixture(scope="module", params=["fp32", "tf32"])
def rig(request, tmp_path_factory):
    from adaptive_voice_conversion_b200.solver import Solver
    mp = pytest.MonkeyPatch()
    mp.setenv("AVC_PRECISION", request.param)
    request.addfinalizer(mp.undo)
    tmp = tmp_path_factory.mktemp("prop")
    cfg = orc.default_config(C_IN)
    cfg["data_loader"]["batch_size"] = B
    args = types.SimpleNamespace(data_dir="synthetic", train_set="train", train_index_file="", logdir=str(tmp / "log"),
                                 load_model=False, load_opt=False, store_model_path=str(tmp / "model"),
                                 load_model_path=str(tmp / "model"), summary_steps=1, save_steps=10 ** 9, tag="t", iters=0)
    solver = Solver(cfg, args)
    solver.model.load_state_dict(orc.init_state(cfg, seed=0), strict=True)
    solver.trainer.eng.pack_weights(solver.trainer.P, need_dgrad=True)
    g = torch.Generator().manual_seed(1)
    x = torch.randn((B, C_IN, T), generator=g).cuda()
    eps = torch.randn((B, 128, T // 8), generator=g).cuda()
    assert solver.trainer.eng.precision == request.param
    return solver, x, eps


def tol(solver, fp32, tf32):
    return fp32 if solver.trainer.eng.precision == "fp32" else tf32


def grad_of(solver, x, eps, lambda_rec=10.0, lambda_kl=1.0):
    """Flat gradient of lambda_rec*L1 + lambda_kl*KL on (x, eps), no optimizer step."""
    tr = solver.trainer
    tr.opt.sync_hparams(lambda_rec=float(lambda_rec), lambda_kl=float(lambda_kl))
    tr._lambda_kl = float(lambda_kl)
    outs = tr._fwd_bwd(x.contiguous(), eps.contiguous())
    torch.cuda.synchronize()
    tr.eng.check_tc_status()
    return tr.opt.flat_g.clone(), outs


def test_forward_is_per_sample(rig):
    solver, x, eps = rig
    with torch.no_grad():
        mu, ls, emb, dec = solver.model(x, eps=eps)
        for i in (0, 101, 255):
            mu1, ls1, emb1, dec1 = solver.model(x[i:i + 1], eps=eps[i:i + 1])
            for a, b in ((mu1, mu[i:i + 1]), (ls1, ls[i:i + 1]), (emb1, emb[i:i + 1]), (dec1, dec[i:i + 1])):
                assert rel_l2(a, b) < 1e-5, (i, rel_l2(a, b))


def test_gradient_is_permutation_invariant(rig):
    solver, x, eps = rig
    g0, _ = grad_of(solver, x, eps)
    perm = torch.randperm(B, generator=torch.Generator().manual_seed(7)).cuda()
    g1, _ = grad_of(solver, x[perm], eps[perm])
    assert rel_l2(g1, g0) < tol(solver, 1e-4, 2e-2), rel_l2(g1, g0)      # same terms, different summation order


def test_gradient_is_homogeneous_in_the_loss_weights(rig):
    solver, x, eps = rig
    g0, _ = grad_of(solver, x, eps, 10.0, 1.0)
    g2, _ = grad_of(solver, x, eps, 20.0, 2.0)
    assert rel_l2(g2, 2.0 * g0) < 1e-5, rel_l2(g2, 2.0 * g0)
    solver.trainer.opt.sync_hparams(lambda_rec=10.0, lambda_kl=1.0)


def test_whole_batch_gradient_is_the_mean_of_the_half_batch_gradients(rig):
    solver, x, eps = rig
    g, _ = grad_of(solver, x, eps)
    h = B // 2
    ga, _ = grad_of(solver, x[:h], eps[:h])
    gb, _ = grad_of(solver, x[h:], eps[h:])
    assert rel_l2(0.5 * (ga + gb), g) < tol(solver, 1e-4, 2e-2), rel_l2(0.5 * (ga + gb), g)
