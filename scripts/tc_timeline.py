"""Phase timeline of one tile of the tensor-core kernel (CTA 0), from in-kernel clock64() marks."""
import os
os.environ.setdefault("PINN_B200_LIB", os.path.join("neuralpde.jl_b200", "lib", "libpinn_b200_debug.so"))   # build.py --debug
import ctypes as C, sys
import numpy as np
sys.path.insert(0, "."); sys.path.insert(0, "tests")
import neuralpde_jl_b200 as npde
from neuralpde_jl_b200 import configs
mode = sys.argv[1] if len(sys.argv) > 1 else "tc_split"
which = sys.argv[2] if len(sys.argv) > 2 else "cfg2"
n = int(sys.argv[3]) if len(sys.argv) > 3 else 128     # cfg 2 grid size: n^2 / 128 PDE tiles + 4 boundary tiles
cfg = configs.config3() if which == "cfg3" else configs.config2(n=n)
rep = npde.symbolic_discretize(cfg.pde_system, cfg.discretization(dtype=np.float32, mode=mode))
eng = rep.engine
if hasattr(rep.strategy, "points"):
    rep.loss_functions.full_loss_function(rep.flat_init_params)     # draws the first sample
lib = eng.lib
lib.pinn_debug_tc_timeline.argtypes = [C.c_void_p, C.c_void_p]
lib.pinn_debug_tc_timeline.restype = C.c_int
th = rep.flat_init_params
for _ in range(3):
    eng.loss_grad_host(th, None, True)
assert lib.pinn_debug_tc_timeline(eng._h, None) == 0
eng.loss_grad_host(th, None, True)
buf = np.zeros(2000, dtype=np.int64)
assert lib.pinn_debug_tc_timeline(eng._h, buf.ctypes.data) == 0
n = int(buf[999])
ids = (buf[:n] >> 48).astype(int); clk = buf[:n] & ((1 << 48) - 1)
names = {1: "start", 2: "setup done", 3: "tile loaded", 4: "fwd done", 5: "program done", 6: "stash drained", 7: "end",
         10: "F enter", 11: "F l: tiles written+sync", 12: "F l: mma issued", 13: "F l: mma done", 14: "F l: stash read done+sync",
         15: "F epilogues done", 16: "F exit", 20: "B enter", 21: "B l: start (prev. layer's gradient sum)",
         22: "B l: stash loaded", 24: "B l: recompute done+sync", 26: "B l: zbar written+sync", 27: "B l: dgrad done+stored",
         28: "B l: wgrad done, partials exchanged+sync", 29: "B l0 start", 30: "B exit"}
if which == "cfg3":     # marks of the 128-wide kernel (tc_wide_kernel.cu)
    names.update({21: "B l: start", 26: "B l: zbar epilogue+sync", 27: "B l: wgrad issued (issuing lane waits H tiles)",
                  28: "B l: wgrad done", 29: "B l: dgrad done + wgrad flushed"})
t0 = clk[0]
prev = t0
agg = {}
for i, c in zip(ids, clk):
    print("%8d  +%7d  %s" % (c - t0, c - prev, names.get(i, str(i))))
    agg[names.get(i, str(i))] = agg.get(names.get(i, str(i)), 0) + (c - prev)
    prev = c
print("\n--- time attributed to the interval ENDING at each mark (cycles) ---")
for k, v in sorted(agg.items(), key=lambda x: -x[1]):
    print("%8d  %5.1f%%  %s" % (v, 100.0 * v / (clk[-1] - t0), k))

# per-CTA spans
rec = buf[1000:].reshape(-1, 4)
rec = rec[rec[:, 1] > 0]
g0 = rec[:, 0].min()
print("\n--- per-CTA spans: %d CTAs; start skew (ns) min %d max %d; end (ns) min %d max %d; cycles min %d median %d max %d"
      % (len(rec), (rec[:, 0] - g0).min(), (rec[:, 0] - g0).max(), (rec[:, 1] - g0).min(), (rec[:, 1] - g0).max(),
         rec[:, 2].min(), int(np.median(rec[:, 2])), rec[:, 2].max()))
order = np.argsort(rec[:, 2])
print("slowest CTAs (bid, smid, cycles, start ns, end ns):", [(int(i), int(rec[i, 3]), int(rec[i, 2]), int(rec[i, 0] - g0), int(rec[i, 1] - g0)) for i in order[-6:]])
print("fastest CTAs:", [(int(i), int(rec[i, 3]), int(rec[i, 2])) for i in order[:6]])
