"""Worker for tests/test_gpu_tc256.py's two-rank test: each rank evaluates its shard of config 4 at a small size on the
256-wide tensor-core kernel, and the gradient and term losses are summed over the ranks.  Launched with
torch.distributed.run."""
import os
import sys

import numpy as np
import torch
import torch.distributed as dist

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
import neuralpde_jl_b200 as npde          # noqa: E402
import tc256_cases as X                   # noqa: E402
import tc_cases as TC                     # noqa: E402

rank, world = int(os.environ["RANK"]), int(os.environ["WORLD_SIZE"])
torch.cuda.set_device(int(os.environ["LOCAL_RANK"]))
dist.init_process_group("gloo")
out = sys.argv[1]
cfg = X.cfg4_small()
rep = npde.symbolic_discretize(cfg.pde_system, cfg.discretization(dtype=np.float32, mode="tc_bf16",
                                                                  device=int(os.environ["LOCAL_RANK"])),
                               rank=rank, world=world)
uid = [npde.Engine.comm_unique_id() if rank == 0 else None]
dist.broadcast_object_list(uid, src=0)
rep.engine.comm_init(uid[0], rank, world)
tot, terms, g = rep.engine.loss_grad_host(TC.make_theta(cfg), None, True)
if rank == 0:
    np.savez(out, tot=tot, terms=terms, g=g)
dist.barrier()
dist.destroy_process_group()
