"""Worker of tests/test_gpu_eval.py: one rank of a data-parallel held-out evaluation (launched as a subprocess per rank;
RANK / WORLD_SIZE / LOCAL_RANK / MASTER_* in the environment).  nccl when every rank has its own GPU, gloo on the CUDA
table when the ranks share one GPU."""
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import torch  # noqa: E402
import torch.distributed as dist  # noqa: E402

import oracle.ae_oracle as orc  # noqa: E402


def main():
    out_dir, data_dir, backend = sys.argv[1], sys.argv[2], sys.argv[3]
    rank, world = int(os.environ["RANK"]), int(os.environ["WORLD_SIZE"])
    dev = torch.device("cuda", int(os.environ["LOCAL_RANK"]))
    torch.cuda.set_device(dev)
    if backend == "nccl":
        dist.init_process_group("nccl", device_id=dev)
    else:
        dist.init_process_group("gloo")
    from adaptive_voice_conversion_b200.evaluate import HeldOut
    from adaptive_voice_conversion_b200.model import AE
    cfg = orc.default_config(80)
    cfg["data_loader"]["batch_size"] = 16
    model = AE(cfg)
    model.load_state_dict(orc.init_state(cfg, seed=0), strict=True)
    model = model.to(dev)
    held = HeldOut(["in_test", "out_test"], data_dir, cfg, rank=rank, world=world, device=dev)
    tabs = {k: v.cpu() for k, v in held.tables(model).items()}
    torch.save(tabs, os.path.join(out_dir, f"eval_rank{rank}.pt"))
    dist.barrier()
    dist.destroy_process_group()


if __name__ == "__main__":
    main()
