"""Worker for tests/test_gpu_quasi_newton.py: every rank runs 10 device-resident L-BFGS iterations on its shard of the
point sets (gradient summed over the ranks by the engine), then the ranks compare theta bit for bit.  Launched with
torch.distributed.run; PINN_B200_NO_P2P=1 selects the ncclAllReduce path."""
import os
import sys

import numpy as np
import torch
import torch.distributed as dist

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import neuralpde_jl_b200 as npde          # noqa: E402
from neuralpde_jl_b200 import configs     # noqa: E402

rank, world = int(os.environ["RANK"]), int(os.environ["WORLD_SIZE"])
local = int(os.environ["LOCAL_RANK"])
torch.cuda.set_device(local)
dist.init_process_group("gloo")
out = sys.argv[1]
cfg = configs.config2(n=48, width=32, hidden=3)
rep = npde.symbolic_discretize(cfg.pde_system, cfg.discretization(dtype=np.float64, device=local), rank=rank, world=world)
uid = [npde.Engine.comm_unique_id() if rank == 0 else None]
dist.broadcast_object_list(uid, src=0)
rep.engine.comm_init(uid[0], rank, world)
fused, _ = rep.engine.comm_info()
rep.engine.qn_begin(rep.flat_init_params, npde.engine.QN_LBFGS)
f, gn, status, it, ev = rep.engine.qn_iterate(10)
theta = rep.engine.qn_theta()
gathered = [None] * world
dist.all_gather_object(gathered, (theta.tobytes(), f, it, ev))
assert all(g == gathered[0] for g in gathered), "replicas diverged"
if rank == 0:
    np.savez(out, theta=theta, f=f, it=it, ev=ev, fused=int(fused))
dist.barrier()
dist.destroy_process_group()
