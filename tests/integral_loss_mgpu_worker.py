"""Worker for tests/test_gpu_integral_loss.py's two-rank test: each rank evaluates its shard of the pure-Neumann problem;
the zero-mean constraint's whole node set stays on rank 0 (none on rank 1), so the ranks' sum is the one-rank value.
Launched with torch.distributed.run."""
import os
import sys

import numpy as np
import torch
import torch.distributed as dist

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
import neuralpde_jl_b200 as npde          # noqa: E402
import integral_loss_cases as LC          # noqa: E402

rank, world = int(os.environ["RANK"]), int(os.environ["WORLD_SIZE"])
torch.cuda.set_device(int(os.environ["LOCAL_RANK"]))
dist.init_process_group("gloo")
out = sys.argv[1]
case = LC.neumann2d()
rep = npde.symbolic_discretize(case[0], LC.discretization(case, np.float64, device=int(os.environ["LOCAL_RANK"])),
                               rank=rank, world=world)
uid = [npde.Engine.comm_unique_id() if rank == 0 else None]
dist.broadcast_object_list(uid, src=0)
rep.engine.comm_init(uid[0], rank, world)
tot, terms, g = rep.engine.loss_grad_host(rep.flat_init_params, None, True)
if rank == 0:
    np.savez(out, tot=tot, terms=terms, g=g)
dist.barrier()
dist.destroy_process_group()
