"""Device-resident loss+grad timing of the BASELINE configs on the parity (FFMA) path (and tensor-core where the
shape is supported).  Development aid; the contract bench is bench.py."""
import sys, time
import numpy as np
sys.path.insert(0, "."); sys.path.insert(0, "tests")
import torch
import neuralpde_jl_b200 as npde
from neuralpde_jl_b200 import configs

cases = [("cfg1", configs.config1(), ["ffma", "tc_split"]),
         ("cfg2", configs.config2(), ["ffma", "tc_split", "tc_bf16"]),
         ("cfg3 (65536 pts, 5x128)", configs.config3(), ["ffma", "tc_bf16"]),
         ("cfg5 (262144 pts = 1M/4 GPUs, 4x128)", configs.config5(points=1 << 18, bcs_points=4096), ["ffma"]),
         ("cfg4 (32^3 nodes, 4 nets 6x256)", configs.config4(nodes=32, bc_nodes=16), ["ffma"])]
dev = torch.device("cuda")
only = sys.argv[1:]
for name, cfg, modes in cases:
    if only and not any(name.startswith(o) for o in only): continue
    for mode in modes:
        try:
            rep = npde.symbolic_discretize(cfg.pde_system, cfg.discretization(dtype=np.float32, mode=mode))
        except Exception as ex:
            print(name, mode, "unsupported:", str(ex)[:100]); continue
        eng = rep.engine
        th = torch.from_numpy(rep.flat_init_params).to(dev)
        g = torch.empty_like(th); terms = torch.empty(eng.n_terms, device=dev); tot = torch.empty(1, device=dev)
        st = torch.cuda.current_stream().cuda_stream
        if hasattr(rep.strategy, "points"):
            rep.loss_functions.full_loss_function(rep.flat_init_params)     # draws the first sample
        for _ in range(2):
            eng.loss_grad_device(th, g, terms, tot, None, st)
        torch.cuda.synchronize()
        n = 5
        t0 = torch.cuda.Event(enable_timing=True); t1 = torch.cuda.Event(enable_timing=True)
        t0.record()
        for _ in range(n):
            eng.loss_grad_device(th, g, terms, tot, None, st)
        t1.record(); torch.cuda.synchronize()
        ms = t0.elapsed_time(t1) / n
        npts = cfg.n_pde_points
        fl = eng.flops_per_eval()
        print("%-42s %-9s %9.3f ms  %10.3e pde-pts/s  %7.2f TFLOP/s (algorithmic)  loss %.6g  finite-grad %s" % (
            name, mode, ms, npts / (ms * 1e-3), fl / (ms * 1e-3) / 1e12, float(tot.item()), bool(torch.isfinite(g).all())), flush=True)
        eng.close()
