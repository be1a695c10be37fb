"""Device-resident step time of one BASELINE config / mode: K steps, each bracketed by CUDA events on the launching
stream, L2 flushed (256 MiB memset) between steps; prints median / min ms and launches per step.  Development aid
(A/B of two library builds via PINN_B200_LIB); the contract bench is bench.py.
usage: step_time.py [cfg2|cfg3|cfg1] [mode] [steps] [n (cfg2 grid size)]"""
import os, sys
import numpy as np
sys.path.insert(0, "."); sys.path.insert(0, "tests")
import torch
import neuralpde_jl_b200 as npde
from neuralpde_jl_b200 import configs
which = sys.argv[1] if len(sys.argv) > 1 else "cfg2"
mode = sys.argv[2] if len(sys.argv) > 2 else "tc_split"
K = int(sys.argv[3]) if len(sys.argv) > 3 else 30
kw = {"n": int(sys.argv[4])} if len(sys.argv) > 4 and which == "cfg2" else {}
cfg = getattr(configs, "config" + which[-1])(**kw)
rep = npde.symbolic_discretize(cfg.pde_system, cfg.discretization(dtype=np.float32, mode=mode))
eng = rep.engine
dev = torch.device("cuda")
th = torch.from_numpy(rep.flat_init_params).to(dev)
g = torch.empty_like(th); terms = torch.empty(eng.n_terms, device=dev); tot = torch.empty(1, device=dev)
flush = torch.empty(256 * 1024 * 1024 // 4, dtype=torch.float32, device=dev)
st = torch.cuda.current_stream().cuda_stream
if hasattr(rep.strategy, "points"):
    rep.loss_functions.full_loss_function(rep.flat_init_params)
for _ in range(5):
    flush.zero_(); eng.loss_grad_device(th, g, terms, tot, None, st)
torch.cuda.synchronize()
l0 = eng.launch_count()
ev = [(torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)) for _ in range(K)]
for a, b in ev:
    flush.zero_(); a.record(); eng.loss_grad_device(th, g, terms, tot, None, st); b.record()
torch.cuda.synchronize()
ms = np.array([a.elapsed_time(b) for a, b in ev])
print("%s %s %s lib=%s: median %.4f ms min %.4f ms launches/step %.1f loss %.8g pts/s %.4g" % (
    which, mode, kw, os.path.basename(os.environ.get("PINN_B200_LIB", "default")), np.median(ms), ms.min(), (eng.launch_count() - l0) / K,
    float(tot.item()), cfg.n_pde_points / (np.median(ms) * 1e-3)), flush=True)
