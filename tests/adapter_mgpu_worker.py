"""Worker for tests/test_gpu_adapter.py's two-rank test: each rank evaluates its contiguous shard of a one-teacher
neural adapter's grid, and the gradient and term losses are summed over the ranks.  Launched with
torch.distributed.run."""
import os
import sys

import numpy as np
import torch
import torch.distributed as dist

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
import neuralpde_jl_b200 as npde                     # noqa: E402
from neuralpde_jl_b200.strategies import adapter_training_set, shard_range   # noqa: E402
import test_gpu_adapter as T                         # noqa: E402

rank, world = int(os.environ["RANK"]), int(os.environ["WORLD_SIZE"])
dev = int(os.environ["LOCAL_RANK"])
torch.cuda.set_device(dev)
dist.init_process_group("gloo")
out = sys.argv[1]
_, _, pt = T._teacher(seed=1)
sys_ = T._system(T._box())
th = T._theta0(T.STUDENT, np.float64)
prob = npde.neural_adapter(npde.NeuralAdapterLoss(T.STUDENT, pt(T.x, T.y)), th, sys_, npde.GridTraining(0.05), device=dev)
eng = prob.representation.engine
pts = adapter_training_set(sys_.domain, 0.05, np.float64)
lo, hi = shard_range(pts.shape[1], rank, world)
eng.set_points_host(0, pts[:, lo:hi])
eng.set_global_count(0, pts.shape[1])
uid = [npde.Engine.comm_unique_id() if rank == 0 else None]
dist.broadcast_object_list(uid, src=0)
eng.comm_init(uid[0], rank, world)
tot, terms, g = eng.loss_grad_host(th, None, True)
if rank == 0:
    np.savez(out, tot=tot, terms=terms, g=g)
dist.barrier()
dist.destroy_process_group()
