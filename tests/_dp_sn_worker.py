"""Worker of tests/test_gpu_spectral_norm.py's data-parallel test: one rank of a Decoder.sn FusedTrainer step
(launched as a subprocess per rank; RANK / WORLD_SIZE / LOCAL_RANK / MASTER_* in the environment)."""
import os
import sys
import types

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))

import torch  # noqa: E402
import torch.distributed as dist  # noqa: E402

from _sn_ref import sn_config  # noqa: E402


def main():
    out_dir, backend, per_rank = sys.argv[1], sys.argv[2], int(sys.argv[3])
    rank, world = int(os.environ["RANK"]), int(os.environ["WORLD_SIZE"])
    local = int(os.environ["LOCAL_RANK"])
    torch.cuda.set_device(local)
    dev = torch.device("cuda", local)
    if backend == "nccl":
        dist.init_process_group("nccl", device_id=dev)
    else:
        dist.init_process_group("gloo")
    from adaptive_voice_conversion_b200.solver import Solver
    cfg = sn_config(80)
    cfg["data_loader"]["batch_size"] = per_rank
    args = types.SimpleNamespace(data_dir="synthetic", train_set="train", train_index_file="", logdir=os.path.join(out_dir, "log"),
                                 load_model=False, load_opt=False, store_model_path=os.path.join(out_dir, "model"),
                                 load_model_path=os.path.join(out_dir, "model"), summary_steps=1, save_steps=10 ** 9, tag="t", iters=0)
    import contextlib, io
    torch.manual_seed(1000 + rank)      # different draws per rank: Solver must broadcast rank 0's u and v
    with contextlib.redirect_stdout(io.StringIO()):
        solver = Solver(cfg, args)
    assert solver.world == world
    init = torch.cat([b.detach().cpu().reshape(-1) for b in solver.model.buffers()])
    from adaptive_voice_conversion_b200.model import AE
    torch.manual_seed(0)
    solver.model.load_state_dict(AE(cfg).state_dict(), strict=True)   # the single-process run's start
    solver.trainer.eng.pack_weights(solver.trainer.P, need_dgrad=True)
    n = per_rank * world
    x = torch.randn((n, 80, 128), generator=torch.Generator().manual_seed(1))
    sl = slice(rank * per_rank, (rank + 1) * per_rank)
    tr = solver.trainer
    recs = []
    for it in range(2):
        eps = torch.randn((n, 128, 16), generator=torch.Generator().manual_seed(50 + it))
        tr.step(x[sl].to(dev), 0.37, eps=eps[sl].to(dev))
        lr_, lk_, gn_ = tr.losses()
        recs.append(dict(loss_rec=lr_, loss_kl=lk_, grad_norm=gn_, flat_g=tr.opt.flat_g.detach().cpu().clone(),
                         flat_p=tr.opt.flat_p.detach().cpu().clone(),
                         uv=torch.cat([b.detach().cpu().reshape(-1) for b in solver.model.buffers()])))
    torch.save({"init_uv": init, "steps": recs}, os.path.join(out_dir, f"rank{rank}.pt"))
    dist.barrier()
    dist.destroy_process_group()


if __name__ == "__main__":
    main()
