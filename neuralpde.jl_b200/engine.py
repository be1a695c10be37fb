"""ctypes binding of the C ABI in include/pinn_b200.h.

This is the Python stand-in for the Julia shim of INTEGRATION.md: it builds a
``pinn_problem_desc`` from plain Python data and calls the library.  There is no CPU
fallback: if the shared library is missing or no CUDA device is present the calls raise.
"""
from __future__ import annotations

import ctypes as C
import os
from dataclasses import dataclass, field
from typing import List, Optional, Sequence

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.environ.get("PINN_B200_LIB") or os.path.join(HERE, "lib", "libpinn_b200.so")

ABI_VERSION = 2
MAX_IN = 8
MAX_TERMS = 32

F32, F64 = 0, 1
# PINN_MODE_*: FFMA (any shape, fp32 / fp64), TC_BF16 (hidden widths up to 64, 64 / 128, or multiples of 64 up to 256),
# TC_SPLIT (hidden widths up to 64), TC_F64 (FFMA's shapes, fp64 only, layer products on DMMA); include/pinn_b200.h lists
# the shapes each tensor-core mode accepts
MODE_FFMA, MODE_TC_BF16, MODE_TC_SPLIT, MODE_TC_F64 = 0, 1, 2, 3
ACT = {"identity": 0, "tanh": 1, "sigmoid": 2, "sin": 3, "softplus": 4, "swish": 5, "gelu": 6, "logcosh": 7,
       "cos": 8}
OP = {
    "const": 0, "coord": 1, "tap": 2, "param": 3, "add": 4, "sub": 5, "mul": 6, "div": 7, "neg": 8,
    "pow": 9, "powi": 10, "sin": 11, "cos": 12, "exp": 13, "log": 14, "tanh": 15, "sqrt": 16, "abs": 17,
    "integral": 18,
}
REDUCE_MEAN, REDUCE_WSUM = 0, 1
# functional terms: g(scale * sum_p w_p v_p), g = |.| or (.)^2 (integral constraints, pinn.IntegralLoss)
REDUCE_ABS_OF_SUM, REDUCE_SQUARE_OF_SUM = 2, 3

# symbols include/pinn_b200.h declares; tests check that the library exports every one
EXPORTS = [
    "pinn_create", "pinn_destroy", "pinn_last_error", "pinn_abi_version", "pinn_set_points",
    "pinn_set_points_host", "pinn_set_global_count", "pinn_loss_grad", "pinn_loss_grad_host",
    "pinn_term_residual", "pinn_term_residual_host", "pinn_comm_unique_id", "pinn_comm_init",
    "pinn_launch_count", "pinn_set_timing", "pinn_last_kernel_ms", "pinn_workspace_bytes",
    "pinn_flops_per_eval", "pinn_adam_begin", "pinn_adam_iterate", "pinn_adam_theta",
    "pinn_term_grad_stats", "pinn_term_grad_stats_host", "pinn_set_sampler", "pinn_resample", "pinn_get_points_host",
    "pinn_comm_info", "pinn_set_sampler_ex", "pinn_qn_begin", "pinn_qn_iterate", "pinn_qn_theta",
    "pinn_hmc_begin", "pinn_hmc_iterate", "pinn_hmc_theta", "pinn_hmc_begin_ex", "pinn_create_ex",
    "pinn_quadrature_nodes", "pinn_create_ex2", "pinn_set_fixed_params", "pinn_set_fixed_params_host",
    "pinn_hmc_begin_ex2", "pinn_set_sampler_kkl",
]

# substitutions of infinite integration bounds (pinn_integral_desc.inf_kind) and the limits of integral terms
INF_NONE, INF_BOTH, INF_UPPER, INF_LOWER = 0, 1, 2, 3
MAX_INTEGRALS = 8
MAX_QUAD = 64
# Gauss-Legendre nodes per integrating dimension the Python layer uses.  16 meet test/Forward/forward__integral.jl's
# rtol = 1e-5 on [0, Inf) with 300x margin (12 are the fewest that do); DESIGN section 4.7.
DEFAULT_QUAD_NODES = 16
# fixed (non-trained) networks per problem: teachers of a neural adapter, registered network functions
MAX_FIXED_NETS = 16

# quasi-Newton optimizer / line search kinds and run states (pinn_qn_options, pinn_qn_iterate)
QN_LBFGS, QN_BFGS = 0, 1
LS_HAGERZHANG, LS_BACKTRACKING = 0, 1
QN_RUNNING, QN_CONVERGED, QN_LS_FAILED = 0, 1, 2

# HMC adaptor / metric kinds (pinn_hmc_options) and the statistics columns of pinn_hmc_iterate
HMC_ADAPT_NONE, HMC_ADAPT_STAN = 0, 1
HMC_METRIC_UNIT, HMC_METRIC_DIAG = 0, 1
# kinds of the per-entry priors of theta's last entries (pinn_hmc_prior)
HMC_PRIOR_NORMAL, HMC_PRIOR_LOGNORMAL, HMC_PRIOR_UNIFORM = 0, 1, 2
# pinn_set_sampler_kkl flags: one coefficient vector per sample path, shared by all its times
KKL_STRONG = 1
# pinn_hmc_begin_ex2 flags: the device samplers draw fresh points before every evaluation of the chain
HMC_REDRAW = 1
HMC_STATS = ("step_size", "acceptance_rate", "is_accept", "log_density", "hamiltonian_energy",
             "hamiltonian_energy_error", "numerical_error", "is_adapt")


class EngineError(RuntimeError):
    """Raised for any nonzero return code of the C ABI (message from pinn_last_error)."""


class _Instr(C.Structure):
    _fields_ = [("op", C.c_int32), ("a", C.c_int32), ("b", C.c_int32), ("_pad", C.c_int32), ("imm", C.c_double)]


class _QnOptions(C.Structure):
    _fields_ = [("kind", C.c_int32), ("m", C.c_int32), ("linesearch", C.c_int32), ("_pad", C.c_int32),
                ("initial_stepnorm", C.c_double)]


class _HmcOptions(C.Structure):
    _fields_ = [("n_leapfrog", C.c_int32), ("adaptor", C.c_int32), ("metric", C.c_int32), ("n_adapts", C.c_int32),
                ("target_accept", C.c_double), ("step_size", C.c_double), ("prior_mean", C.c_double),
                ("prior_std", C.c_double), ("seed", C.c_uint64)]


class _HmcPrior(C.Structure):
    _fields_ = [("kind", C.c_int32), ("a", C.c_double), ("b", C.c_double)]


class _NetDesc(C.Structure):
    _fields_ = [("n_layers", C.c_int32), ("dims", C.POINTER(C.c_int32)), ("acts", C.POINTER(C.c_int32)),
                ("theta_offset", C.c_int64)]


class _FixedNetDesc(C.Structure):
    _fields_ = [("n_layers", C.c_int32), ("dims", C.POINTER(C.c_int32)), ("acts", C.POINTER(C.c_int32))]


class _TapDesc(C.Structure):
    _fields_ = [("net", C.c_int32), ("out", C.c_int32), ("order", C.c_int32), ("dir", C.c_int32 * 4)]


class _TermDesc(C.Structure):
    _fields_ = [("dim", C.c_int32), ("n_taps", C.c_int32), ("taps", C.POINTER(_TapDesc)),
                ("net_rows", C.POINTER(C.c_int32)), ("n_instr", C.c_int32), ("prog", C.POINTER(_Instr)),
                ("reduction", C.c_int32), ("scale", C.c_double)]


class _IntegralDesc(C.Structure):
    _fields_ = [("owner", C.c_int32), ("n_dims", C.c_int32), ("q", C.c_int32), ("row", C.c_int32 * 2),
                ("lb_row", C.c_int32 * 2), ("ub_row", C.c_int32 * 2), ("lb", C.c_double * 2), ("ub", C.c_double * 2),
                ("inf_kind", C.c_int32 * 2), ("shift", C.c_double * 2), ("n_taps", C.c_int32),
                ("taps", C.POINTER(_TapDesc)), ("net_rows", C.POINTER(C.c_int32)), ("n_instr", C.c_int32),
                ("prog", C.POINTER(_Instr))]


class _ProblemDesc(C.Structure):
    _fields_ = [("abi_version", C.c_int32), ("dtype", C.c_int32), ("mode", C.c_int32), ("device", C.c_int32),
                ("n_nets", C.c_int32), ("nets", C.POINTER(_NetDesc)), ("n_terms", C.c_int32),
                ("terms", C.POINTER(_TermDesc)), ("n_params", C.c_int32), ("param_offset", C.c_int64),
                ("n_theta", C.c_int64)]


# ---- plain-data problem description (what the Julia shim would assemble) ---------------------
@dataclass
class NetSpec:
    dims: Sequence[int]                 # in, hidden..., out
    acts: Sequence[str]                 # one per Dense layer
    theta_offset: int = 0

    @property
    def n_params(self) -> int:
        return sum(self.dims[i] * self.dims[i + 1] + self.dims[i + 1] for i in range(len(self.dims) - 1))


@dataclass
class FixedNetSpec:
    """A network whose parameters are not trained (pinn_fixed_net_desc); taps name it as network len(nets) + j."""
    dims: Sequence[int]
    acts: Sequence[str]

    @property
    def n_params(self) -> int:
        return sum(self.dims[i] * self.dims[i + 1] + self.dims[i + 1] for i in range(len(self.dims) - 1))


@dataclass
class TapSpec:
    net: int
    order: int = 0
    dirs: Sequence[int] = ()
    out: int = 0


@dataclass
class TermSpec:
    dim: int
    taps: List[TapSpec]
    prog: List[tuple]                   # (opname, a, b, imm)
    net_rows: Optional[List[List[int]]] = None   # per network: point row feeding input j
    reduction: int = REDUCE_MEAN
    scale: float = 1.0


@dataclass
class IntegralSpec:
    """One integral term (pinn_integral_desc): read by term ``owner``'s program as ("integral", index); the integrand's
    program runs over the node point (the owner's rows with ``rows`` replaced by x(t), then the t rows)."""
    owner: int
    n_dims: int = 1
    q: int = DEFAULT_QUAD_NODES
    rows: List[int] = field(default_factory=lambda: [0, 0])
    lb: List[float] = field(default_factory=lambda: [0.0, 0.0])
    ub: List[float] = field(default_factory=lambda: [0.0, 0.0])
    lb_row: List[int] = field(default_factory=lambda: [-1, -1])
    ub_row: List[int] = field(default_factory=lambda: [-1, -1])
    inf_kind: List[int] = field(default_factory=lambda: [0, 0])
    shift: List[float] = field(default_factory=lambda: [0.0, 0.0])
    taps: List[TapSpec] = field(default_factory=list)
    prog: List[tuple] = field(default_factory=list)
    net_rows: Optional[List[List[int]]] = None


@dataclass
class ProblemSpec:
    nets: List[NetSpec]
    terms: List[TermSpec]
    n_params: int = 0
    param_offset: int = 0
    n_theta: int = 0
    dtype: str = "float32"
    mode: int = MODE_FFMA
    device: int = 0
    integrals: List[IntegralSpec] = field(default_factory=list)   # non-empty: created with pinn_create_ex
    fixed: List[FixedNetSpec] = field(default_factory=list)       # non-empty: created with pinn_create_ex2
    _keep: list = field(default_factory=list, repr=False)


_lib = None


def load_library():
    """Load libpinn_b200.so and declare prototypes.  Raises if the library is not built."""
    global _lib
    if _lib is not None:
        return _lib
    if not os.path.exists(LIB_PATH):
        raise EngineError(
            "libpinn_b200.so is not built (%s); run `python __graft_entry__.py build` -- "
            "this engine has no CPU fallback" % LIB_PATH)
    lib = C.CDLL(LIB_PATH)
    vp, i32, i64, dbl = C.c_void_p, C.c_int32, C.c_int64, C.c_double
    lib.pinn_create.argtypes = [C.POINTER(_ProblemDesc), C.POINTER(vp)]
    lib.pinn_create.restype = C.c_int
    lib.pinn_create_ex.argtypes = [C.POINTER(_ProblemDesc), C.POINTER(_IntegralDesc), C.c_int32, C.POINTER(vp)]
    lib.pinn_create_ex.restype = C.c_int
    lib.pinn_create_ex2.argtypes = [C.POINTER(_ProblemDesc), C.POINTER(_IntegralDesc), C.c_int32, C.POINTER(_FixedNetDesc),
                                    C.c_int32, C.POINTER(vp)]
    lib.pinn_create_ex2.restype = C.c_int
    lib.pinn_set_fixed_params.argtypes = [vp, i32, vp]
    lib.pinn_set_fixed_params.restype = C.c_int
    lib.pinn_set_fixed_params_host.argtypes = [vp, i32, vp, vp]
    lib.pinn_set_fixed_params_host.restype = C.c_int
    lib.pinn_quadrature_nodes.argtypes = [C.c_int32, C.POINTER(C.c_double), C.POINTER(C.c_double)]
    lib.pinn_quadrature_nodes.restype = C.c_int
    lib.pinn_destroy.argtypes = [vp]
    lib.pinn_destroy.restype = C.c_int
    lib.pinn_last_error.argtypes = []
    lib.pinn_last_error.restype = C.c_char_p
    lib.pinn_abi_version.argtypes = []
    lib.pinn_abi_version.restype = C.c_int
    lib.pinn_set_points.argtypes = [vp, i32, vp, i64, vp]
    lib.pinn_set_points.restype = C.c_int
    lib.pinn_set_points_host.argtypes = [vp, i32, vp, i64, vp, vp]
    lib.pinn_set_points_host.restype = C.c_int
    lib.pinn_set_global_count.argtypes = [vp, i32, i64]
    lib.pinn_set_global_count.restype = C.c_int
    lib.pinn_loss_grad.argtypes = [vp, vp, C.POINTER(dbl), vp, vp, vp, vp]
    lib.pinn_loss_grad.restype = C.c_int
    lib.pinn_loss_grad_host.argtypes = [vp, vp, C.POINTER(dbl), vp, vp, vp]
    lib.pinn_loss_grad_host.restype = C.c_int
    lib.pinn_set_sampler.argtypes = [vp, i32, i64, C.POINTER(dbl), C.POINTER(dbl), C.c_uint64, vp]
    lib.pinn_set_sampler.restype = C.c_int
    lib.pinn_set_sampler_ex.argtypes = [vp, i32, i32, i64, C.POINTER(dbl), C.POINTER(dbl), C.c_uint64, vp]
    lib.pinn_set_sampler_ex.restype = C.c_int
    lib.pinn_set_sampler_kkl.argtypes = [vp, i32, i64, i32, i32, dbl, dbl, C.c_uint32, C.c_uint64, vp]
    lib.pinn_set_sampler_kkl.restype = C.c_int
    lib.pinn_resample.argtypes = [vp, vp]
    lib.pinn_resample.restype = C.c_int
    lib.pinn_get_points_host.argtypes = [vp, i32, vp]
    lib.pinn_get_points_host.restype = C.c_int
    lib.pinn_term_grad_stats.argtypes = [vp, i32, vp, C.POINTER(dbl), C.POINTER(dbl), vp]
    lib.pinn_term_grad_stats.restype = C.c_int
    lib.pinn_term_grad_stats_host.argtypes = [vp, i32, vp, C.POINTER(dbl), C.POINTER(dbl)]
    lib.pinn_term_grad_stats_host.restype = C.c_int
    lib.pinn_term_residual.argtypes = [vp, i32, vp, vp, vp]
    lib.pinn_term_residual.restype = C.c_int
    lib.pinn_term_residual_host.argtypes = [vp, i32, vp, vp]
    lib.pinn_term_residual_host.restype = C.c_int
    lib.pinn_comm_unique_id.argtypes = [vp]
    lib.pinn_comm_unique_id.restype = C.c_int
    lib.pinn_comm_init.argtypes = [vp, vp, i32, i32]
    lib.pinn_comm_init.restype = C.c_int
    lib.pinn_comm_info.argtypes = [vp, C.POINTER(i32)]
    lib.pinn_comm_info.restype = C.c_char_p
    lib.pinn_launch_count.argtypes = [vp]
    lib.pinn_launch_count.restype = i64
    lib.pinn_set_timing.argtypes = [vp, i32]
    lib.pinn_set_timing.restype = C.c_int
    lib.pinn_last_kernel_ms.argtypes = [vp]
    lib.pinn_last_kernel_ms.restype = dbl
    lib.pinn_workspace_bytes.argtypes = [vp]
    lib.pinn_workspace_bytes.restype = i64
    lib.pinn_flops_per_eval.argtypes = [vp]
    lib.pinn_flops_per_eval.restype = dbl
    lib.pinn_adam_begin.argtypes = [vp, vp, dbl, dbl, dbl, dbl]
    lib.pinn_adam_begin.restype = C.c_int
    lib.pinn_adam_iterate.argtypes = [vp, i32, C.POINTER(dbl), vp, vp]
    lib.pinn_adam_iterate.restype = C.c_int
    lib.pinn_adam_theta.argtypes = [vp, vp]
    lib.pinn_adam_theta.restype = C.c_int
    lib.pinn_qn_begin.argtypes = [vp, vp, C.POINTER(_QnOptions), C.POINTER(dbl)]
    lib.pinn_qn_begin.restype = C.c_int
    lib.pinn_qn_iterate.argtypes = [vp, i32, C.POINTER(dbl), C.POINTER(dbl), C.POINTER(i32), C.POINTER(i64), C.POINTER(i64)]
    lib.pinn_qn_iterate.restype = C.c_int
    lib.pinn_qn_theta.argtypes = [vp, vp]
    lib.pinn_qn_theta.restype = C.c_int
    lib.pinn_hmc_begin.argtypes = [vp, C.POINTER(dbl), C.POINTER(_HmcOptions), C.POINTER(dbl), dbl, C.POINTER(dbl)]
    lib.pinn_hmc_begin.restype = C.c_int
    lib.pinn_hmc_begin_ex.argtypes = [vp, C.POINTER(dbl), C.POINTER(_HmcOptions), C.POINTER(dbl), dbl,
                                      C.POINTER(_HmcPrior), i32, C.POINTER(dbl)]
    lib.pinn_hmc_begin_ex.restype = C.c_int
    lib.pinn_hmc_begin_ex2.argtypes = [vp, C.POINTER(dbl), C.POINTER(_HmcOptions), C.POINTER(dbl), dbl,
                                       C.POINTER(_HmcPrior), i32, C.POINTER(dbl), C.c_uint32, C.POINTER(dbl)]
    lib.pinn_hmc_begin_ex2.restype = C.c_int
    lib.pinn_hmc_iterate.argtypes = [vp, i32, C.POINTER(dbl), C.POINTER(dbl)]
    lib.pinn_hmc_iterate.restype = C.c_int
    lib.pinn_hmc_theta.argtypes = [vp, C.POINTER(dbl)]
    lib.pinn_hmc_theta.restype = C.c_int
    _lib = lib
    return lib


def quadrature_nodes(q: int):
    """(nodes, weights) of the q-point Gauss-Legendre rule on [-1, 1] that integral terms use (host only)."""
    lib = load_library()
    x, w = np.empty(int(q)), np.empty(int(q))
    _check(lib.pinn_quadrature_nodes(int(q), x.ctypes.data_as(C.POINTER(C.c_double)),
                                     w.ctypes.data_as(C.POINTER(C.c_double))))
    return x, w


def _check(rc: int):
    if rc != 0:
        raise EngineError(load_library().pinn_last_error().decode("utf-8", "replace"))


def _np_dtype(dtype: str):
    return np.float64 if dtype in ("float64", "f64") else np.float32


def _ptr(x) -> C.c_void_p:
    """Device/host pointer of a numpy array, torch tensor, int address or None."""
    if x is None:
        return C.c_void_p(0)
    if isinstance(x, int):
        return C.c_void_p(x)
    if isinstance(x, np.ndarray):
        return C.c_void_p(x.ctypes.data)
    if hasattr(x, "data_ptr"):
        return C.c_void_p(x.data_ptr())
    raise TypeError("cannot take a pointer of %r" % type(x))


def _marshal_body(spec: ProblemSpec, taps_l, prog_l, net_rows_l, keep):
    """taps / net_rows / program arrays of a term or an integrand"""
    taps = (_TapDesc * max(1, len(taps_l)))()
    for i, tp in enumerate(taps_l):
        taps[i].net, taps[i].out, taps[i].order = int(tp.net), int(tp.out), int(tp.order)
        d = list(tp.dirs) + [0, 0, 0, 0]
        for q in range(4):
            taps[i].dir[q] = int(d[q])
    all_nets = list(spec.nets) + list(spec.fixed)
    rows = (C.c_int32 * (len(all_nets) * MAX_IN))(*([-1] * (len(all_nets) * MAX_IN)))
    for k, n in enumerate(all_nets):
        r = net_rows_l[k] if net_rows_l is not None and k < len(net_rows_l) and net_rows_l[k] is not None \
            else list(range(n.dims[0]))
        for j, v in enumerate(r):
            rows[k * MAX_IN + j] = int(v)
    prog = (_Instr * max(1, len(prog_l)))()
    for i, ins in enumerate(prog_l):
        op, a, b, imm = (list(ins) + [0, 0, 0.0])[:4]
        prog[i].op, prog[i].a, prog[i].b, prog[i].imm = OP[op], int(a), int(b), float(imm)
    keep += [taps, rows, prog]
    return taps, rows, prog


def build_integrals(spec: ProblemSpec):
    """Marshal spec.integrals into a pinn_integral_desc array (kept alive on the spec)."""
    arr = (_IntegralDesc * max(1, len(spec.integrals)))()
    for i, it in enumerate(spec.integrals):
        d = arr[i]
        d.owner, d.n_dims, d.q = int(it.owner), int(it.n_dims), int(it.q)
        for k in range(2):
            d.row[k], d.lb_row[k], d.ub_row[k] = int(it.rows[k]), int(it.lb_row[k]), int(it.ub_row[k])
            d.lb[k], d.ub[k], d.shift[k] = float(it.lb[k]), float(it.ub[k]), float(it.shift[k])
            d.inf_kind[k] = int(it.inf_kind[k])
        d.taps, d.net_rows, d.prog = _marshal_body(spec, it.taps, it.prog, it.net_rows, spec._keep)
        d.n_taps, d.n_instr = len(it.taps), len(it.prog)
    spec._keep.append(arr)
    return arr


def build_fixed(spec: ProblemSpec):
    """Marshal spec.fixed into a pinn_fixed_net_desc array (kept alive on the spec)."""
    arr = (_FixedNetDesc * max(1, len(spec.fixed)))()
    for j, f in enumerate(spec.fixed):
        dims = (C.c_int32 * len(f.dims))(*[int(v) for v in f.dims])
        acts = (C.c_int32 * len(f.acts))(*[ACT[a] for a in f.acts])
        arr[j].n_layers, arr[j].dims, arr[j].acts = len(f.acts), dims, acts
        spec._keep += [dims, acts]
    spec._keep.append(arr)
    return arr


def build_desc(spec: ProblemSpec) -> _ProblemDesc:
    """Marshal a ProblemSpec into the C descriptor (buffers are kept alive on the spec)."""
    keep = spec._keep
    keep.clear()
    nets = (_NetDesc * len(spec.nets))()
    for k, n in enumerate(spec.nets):
        dims = (C.c_int32 * len(n.dims))(*[int(v) for v in n.dims])
        acts = (C.c_int32 * len(n.acts))(*[ACT[a] for a in n.acts])
        keep += [dims, acts]
        nets[k].n_layers = len(n.acts)
        nets[k].dims = dims
        nets[k].acts = acts
        nets[k].theta_offset = int(n.theta_offset)
    terms = (_TermDesc * len(spec.terms))()
    for t, tm in enumerate(spec.terms):
        taps = (_TapDesc * max(1, len(tm.taps)))()
        for i, tp in enumerate(tm.taps):
            taps[i].net, taps[i].out, taps[i].order = int(tp.net), int(tp.out), int(tp.order)
            d = list(tp.dirs) + [0, 0, 0, 0]
            for q in range(4):
                taps[i].dir[q] = int(d[q])
        all_nets = list(spec.nets) + list(spec.fixed)
        rows = (C.c_int32 * (len(all_nets) * MAX_IN))(*([-1] * (len(all_nets) * MAX_IN)))
        for k, n in enumerate(all_nets):
            r = tm.net_rows[k] if tm.net_rows is not None and k < len(tm.net_rows) and tm.net_rows[k] is not None \
                else list(range(n.dims[0]))
            for j, v in enumerate(r):
                rows[k * MAX_IN + j] = int(v)
        prog = (_Instr * max(1, len(tm.prog)))()
        for i, ins in enumerate(tm.prog):
            op, a, b, imm = (list(ins) + [0, 0, 0.0])[:4]
            prog[i].op, prog[i].a, prog[i].b, prog[i].imm = OP[op], int(a), int(b), float(imm)
        keep += [taps, rows, prog]
        terms[t].dim = int(tm.dim)
        terms[t].n_taps = len(tm.taps)
        terms[t].taps = taps
        terms[t].net_rows = rows
        terms[t].n_instr = len(tm.prog)
        terms[t].prog = prog
        terms[t].reduction = int(tm.reduction)
        terms[t].scale = float(tm.scale)
    keep += [nets, terms]
    d = _ProblemDesc()
    d.abi_version = ABI_VERSION
    d.dtype = F64 if _np_dtype(spec.dtype) is np.float64 else F32
    d.mode = int(spec.mode)
    d.device = int(spec.device)
    d.n_nets, d.nets = len(spec.nets), nets
    d.n_terms, d.terms = len(spec.terms), terms
    d.n_params, d.param_offset = int(spec.n_params), int(spec.param_offset)
    d.n_theta = int(spec.n_theta)
    return d


class Engine:
    """One engine handle (one GPU rank).  Thin, explicit wrapper over the C ABI."""

    def __init__(self, spec: ProblemSpec):
        self.lib = load_library()
        self.spec = spec
        self.np_dtype = _np_dtype(spec.dtype)
        self.n_terms = len(spec.terms)
        self.n_theta = int(spec.n_theta)
        self._h = C.c_void_p(0)
        desc = build_desc(spec)
        if spec.fixed:
            _check(self.lib.pinn_create_ex2(C.byref(desc), build_integrals(spec), len(spec.integrals), build_fixed(spec),
                                            len(spec.fixed), C.byref(self._h)))
        elif spec.integrals:
            _check(self.lib.pinn_create_ex(C.byref(desc), build_integrals(spec), len(spec.integrals), C.byref(self._h)))
        else:
            _check(self.lib.pinn_create(C.byref(desc), C.byref(self._h)))
        self._keep_pts = {}

    def close(self):
        if self._h:
            self.lib.pinn_destroy(self._h)
            self._h = C.c_void_p(0)

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    # -- fixed networks ---------------------------------------------------------------------------
    def set_fixed_params(self, j: int, dev_params):
        """Alias a device buffer (torch CUDA tensor or raw pointer) as fixed network j's parameters."""
        self._keep_pts[("fixed", int(j))] = dev_params
        _check(self.lib.pinn_set_fixed_params(self._h, int(j), _ptr(dev_params)))

    def set_fixed_params_host(self, j: int, params: np.ndarray, stream: int = 0):
        """Copy fixed network j's parameters (flat Lux layout) into engine memory."""
        p = np.ascontiguousarray(params, dtype=self.np_dtype).reshape(-1)
        if not 0 <= int(j) < len(self.spec.fixed):
            raise ValueError("fixed network %d out of range [0, %d)" % (int(j), len(self.spec.fixed)))
        if p.size != self.spec.fixed[int(j)].n_params:
            raise ValueError("fixed network %d has %d parameters, got %d" % (int(j), self.spec.fixed[int(j)].n_params,
                                                                               p.size))
        _check(self.lib.pinn_set_fixed_params_host(self._h, int(j), _ptr(p), C.c_void_p(stream)))

    # -- points ---------------------------------------------------------------------------------
    def set_points(self, term: int, dev_pts, n: int, dev_weights=None):
        """Alias device-resident points (torch CUDA tensor or raw pointer), d x n column-major."""
        self._keep_pts[term] = (dev_pts, dev_weights)
        _check(self.lib.pinn_set_points(self._h, term, _ptr(dev_pts), int(n), _ptr(dev_weights)))

    def set_points_host(self, term: int, pts: np.ndarray, weights: Optional[np.ndarray] = None, stream: int = 0):
        """Upload a host (d, n) array (any memory order; converted to d x n column-major)."""
        pts = np.asarray(pts, dtype=self.np_dtype)
        if pts.ndim != 2:
            raise ValueError("points must be a (d, n) matrix")
        if pts.shape[0] != self.spec.terms[term].dim:
            raise ValueError("term %d expects %d rows per point (coordinates + hoisted rows), got %d"
                             % (term, self.spec.terms[term].dim, pts.shape[0]))
        buf = np.asfortranarray(pts)          # column-major: one point = d contiguous scalars
        flat = buf.ravel(order="F")
        w = None if weights is None else np.ascontiguousarray(weights, dtype=self.np_dtype)
        _check(self.lib.pinn_set_points_host(self._h, term, _ptr(flat), int(pts.shape[1]), _ptr(w), C.c_void_p(stream)))

    def set_sampler(self, term: int, n: int, lb, ub, seed: int = 0, stream: int = 0, kind: str = "uniform"):
        """Register a device-side sampler for a term (box lb..ub per point row) and draw the first sample.
        kind "uniform": StochasticTraining; "lhs": Latin hypercube (QuasiRandomTraining's default algorithm)."""
        lb = np.ascontiguousarray(lb, dtype=np.float64); ub = np.ascontiguousarray(ub, dtype=np.float64)
        dim = self.spec.terms[term].dim
        if lb.shape != (dim,) or ub.shape != (dim,):
            raise ValueError("term %d expects %d bounds per side, got %s / %s" % (term, dim, lb.shape, ub.shape))
        _check(self.lib.pinn_set_sampler_ex(self._h, int(term), {"uniform": 0, "lhs": 1}[kind], int(n),
                                            lb.ctypes.data_as(C.POINTER(C.c_double)), ub.ctypes.data_as(C.POINTER(C.c_double)),
                                            C.c_uint64(int(seed) & (2 ** 64 - 1)), C.c_void_p(stream)))
        self._n_pts = getattr(self, "_n_pts", {})
        self._n_pts[int(term)] = int(n)

    def set_sampler_kkl(self, term: int, n_times: int, sub_batch: int, t_lb: float, t_ub: float, seed: int = 0,
                        strong: bool = False, stream: int = 0):
        """Register NNSDE's device sampler for a term with rows (t, z_1..z_n_z): n_times uniform times in [t_lb, t_ub],
        each with sub_batch N(0, 1) coefficient vectors, independent per point, or with strong=True one per sample s
        shared by all times (include/pinn_b200.h gives the formula).  Draws the first sample."""
        dim = self.spec.terms[term].dim
        _check(self.lib.pinn_set_sampler_kkl(self._h, int(term), int(n_times), int(sub_batch), dim - 1, float(t_lb),
                                             float(t_ub), KKL_STRONG if strong else 0,
                                             C.c_uint64(int(seed) & (2 ** 64 - 1)), C.c_void_p(stream)))
        self._n_pts = getattr(self, "_n_pts", {})
        self._n_pts[int(term)] = int(n_times) * int(sub_batch)

    def resample(self, stream: int = 0):
        """Draw the next sample of every term that has a device-side sampler."""
        _check(self.lib.pinn_resample(self._h, C.c_void_p(stream)))

    def get_points_host(self, term: int, n: int) -> np.ndarray:
        """Current (d, n) point set of a term, copied from the device."""
        dim = self.spec.terms[term].dim
        buf = np.empty(int(n) * dim, dtype=self.np_dtype)
        _check(self.lib.pinn_get_points_host(self._h, int(term), _ptr(buf)))
        return buf.reshape(int(n), dim).T.copy()

    def set_global_count(self, term: int, n_global: int):
        _check(self.lib.pinn_set_global_count(self._h, term, int(n_global)))

    # -- hot path -------------------------------------------------------------------------------
    def _weights(self, weights):
        if weights is None:
            return None
        w = np.ascontiguousarray(weights, dtype=np.float64)
        if w.shape != (self.n_terms,):
            raise ValueError("need %d term weights" % self.n_terms)
        return w

    def loss_grad_device(self, dev_theta, dev_grad, dev_term_losses, dev_total, weights=None, stream: int = 0):
        w = self._weights(weights)
        wp = w.ctypes.data_as(C.POINTER(C.c_double)) if w is not None else None
        _check(self.lib.pinn_loss_grad(self._h, _ptr(dev_theta), wp, _ptr(dev_grad), _ptr(dev_term_losses),
                                       _ptr(dev_total), C.c_void_p(stream)))

    def loss_grad_host(self, theta: np.ndarray, weights=None, want_grad: bool = True):
        """Host-buffer call: returns (total, term_losses, grad or None)."""
        th = np.ascontiguousarray(theta, dtype=self.np_dtype)
        if th.shape != (self.n_theta,):
            raise ValueError("theta must have length %d" % self.n_theta)
        grad = np.empty(self.n_theta, dtype=self.np_dtype) if want_grad else None
        terms = np.empty(self.n_terms, dtype=self.np_dtype)
        total = np.empty(1, dtype=self.np_dtype)
        w = self._weights(weights)
        wp = w.ctypes.data_as(C.POINTER(C.c_double)) if w is not None else None
        _check(self.lib.pinn_loss_grad_host(self._h, _ptr(th), wp, _ptr(grad), _ptr(terms), _ptr(total)))
        return float(total[0]), terms, grad

    def term_residual_host(self, term: int, theta: np.ndarray, n: int) -> np.ndarray:
        th = np.ascontiguousarray(theta, dtype=self.np_dtype)
        r = np.empty(int(n), dtype=self.np_dtype)
        _check(self.lib.pinn_term_residual_host(self._h, term, _ptr(th), _ptr(r)))
        return r

    def term_grad_stats_host(self, term: int, theta: np.ndarray):
        """(max |g|, mean |g|) of the gradient of term `term`'s unweighted loss (GradientScaleAdaptiveLoss)."""
        th = np.ascontiguousarray(theta, dtype=self.np_dtype)
        mx, mn = C.c_double(0.0), C.c_double(0.0)
        _check(self.lib.pinn_term_grad_stats_host(self._h, int(term), _ptr(th), C.byref(mx), C.byref(mn)))
        return float(mx.value), float(mn.value)

    def term_residual_device(self, term: int, dev_theta, dev_r, stream: int = 0):
        _check(self.lib.pinn_term_residual(self._h, term, _ptr(dev_theta), _ptr(dev_r), C.c_void_p(stream)))

    # -- device-resident Adam loop ----------------------------------------------------------------------
    def adam_begin(self, theta0: np.ndarray, lr=1e-3, beta1=0.9, beta2=0.999, eps=1e-8):
        th = np.ascontiguousarray(theta0, dtype=self.np_dtype)
        _check(self.lib.pinn_adam_begin(self._h, _ptr(th), float(lr), float(beta1), float(beta2), float(eps)))

    def adam_iterate(self, n_steps: int, weights=None):
        """Run n_steps fused iterations on the device; returns (loss, term_losses) of the last evaluated theta."""
        terms = np.empty(self.n_terms, dtype=self.np_dtype)
        total = np.empty(1, dtype=self.np_dtype)
        w = self._weights(weights)
        wp = w.ctypes.data_as(C.POINTER(C.c_double)) if w is not None else None
        _check(self.lib.pinn_adam_iterate(self._h, int(n_steps), wp, _ptr(total), _ptr(terms)))
        return float(total[0]), terms

    def adam_theta(self) -> np.ndarray:
        th = np.empty(self.n_theta, dtype=self.np_dtype)
        _check(self.lib.pinn_adam_theta(self._h, _ptr(th)))
        return th

    # -- device-resident quasi-Newton (BFGS / L-BFGS) ---------------------------------------------------------
    def qn_begin(self, theta0: np.ndarray, kind: int = QN_LBFGS, m: int = 10, linesearch: int = LS_HAGERZHANG,
                 initial_stepnorm: Optional[float] = None, weights=None):
        """Start a quasi-Newton run at theta0 (one loss / gradient evaluation); weights stay fixed for the run."""
        th = np.ascontiguousarray(theta0, dtype=self.np_dtype)
        if th.shape != (self.n_theta,):
            raise ValueError("theta must have length %d" % self.n_theta)
        opt = _QnOptions(int(kind), int(m), int(linesearch), 0, float(initial_stepnorm or 0.0))
        w = self._weights(weights)
        wp = w.ctypes.data_as(C.POINTER(C.c_double)) if w is not None else None
        _check(self.lib.pinn_qn_begin(self._h, _ptr(th), C.byref(opt), wp))

    def qn_iterate(self, n_iters: int):
        """Up to n_iters iterations; returns (loss, ||g||_inf, status, iterations, evaluations), the counts since
        qn_begin.  status: QN_RUNNING, QN_CONVERGED or QN_LS_FAILED."""
        f, gn = C.c_double(0.0), C.c_double(0.0)
        st, it, ev = C.c_int32(0), C.c_int64(0), C.c_int64(0)
        _check(self.lib.pinn_qn_iterate(self._h, int(n_iters), C.byref(f), C.byref(gn), C.byref(st), C.byref(it),
                                        C.byref(ev)))
        return float(f.value), float(gn.value), int(st.value), int(it.value), int(ev.value)

    def qn_theta(self) -> np.ndarray:
        th = np.empty(self.n_theta, dtype=self.np_dtype)
        _check(self.lib.pinn_qn_theta(self._h, _ptr(th)))
        return th

    # -- device-resident HMC sampler ------------------------------------------------------------------------
    def hmc_begin(self, theta0: np.ndarray, n_leapfrog: int = 30, adaptor: int = HMC_ADAPT_STAN,
                  metric: int = HMC_METRIC_DIAG, n_adapts: int = 0, target_accept: float = 0.8, step_size: float = 0.0,
                  prior_mean: float = 0.0, prior_std: float = 1.0, seed: int = 0, weights=None,
                  ll_const: float = 0.0, tail_priors=None, tail_logabs=None, redraw: bool = False) -> float:
        """Start a chain at theta0 (float64) for the log density sum_k w_k L_k + ll_const + log N(theta; prior);
        step_size <= 0 runs find_good_stepsize.  Returns the initial step size.  ``tail_priors``: a list of
        (HMC_PRIOR_*, a, b) for the last len(tail_priors) entries of theta, which the Normal prior then leaves out
        (pinn_hmc_begin_ex); None calls pinn_hmc_begin.  ``tail_logabs``: c_j per tail entry, adding
        c_j log|theta_tail_j| to the log density; ``redraw``: the device samplers draw fresh points before every
        evaluation (PINN_HMC_REDRAW).  Either one calls pinn_hmc_begin_ex2."""
        th = np.ascontiguousarray(theta0, dtype=np.float64)
        if th.shape != (self.n_theta,):
            raise ValueError("theta must have length %d" % self.n_theta)
        opt = _HmcOptions(int(n_leapfrog), int(adaptor), int(metric), int(n_adapts), float(target_accept),
                          float(step_size), float(prior_mean), float(prior_std), int(seed) & (2 ** 64 - 1))
        w = self._weights(weights)
        wp = w.ctypes.data_as(C.POINTER(C.c_double)) if w is not None else None
        eps = C.c_double(0.0)
        if tail_logabs is not None or redraw:
            tp = list(tail_priors or [])
            tail = (_HmcPrior * max(1, len(tp)))(*[_HmcPrior(int(k), float(a), float(b)) for k, a, b in tp])
            la = None
            if tail_logabs is not None:
                la = np.ascontiguousarray(tail_logabs, dtype=np.float64)
                if la.shape != (len(tp),):
                    raise ValueError("tail_logabs needs one entry per tail prior (%d), got %s" % (len(tp), la.shape))
            _check(self.lib.pinn_hmc_begin_ex2(self._h, th.ctypes.data_as(C.POINTER(C.c_double)), C.byref(opt), wp,
                                               float(ll_const), tail, len(tp),
                                               None if la is None else la.ctypes.data_as(C.POINTER(C.c_double)),
                                               HMC_REDRAW if redraw else 0, C.byref(eps)))
        elif tail_priors is None:
            _check(self.lib.pinn_hmc_begin(self._h, th.ctypes.data_as(C.POINTER(C.c_double)), C.byref(opt), wp,
                                           float(ll_const), C.byref(eps)))
        else:
            tail = (_HmcPrior * max(1, len(tail_priors)))(*[_HmcPrior(int(k), float(a), float(b))
                                                            for k, a, b in tail_priors])
            _check(self.lib.pinn_hmc_begin_ex(self._h, th.ctypes.data_as(C.POINTER(C.c_double)), C.byref(opt), wp,
                                              float(ll_const), tail, len(tail_priors), C.byref(eps)))
        return float(eps.value)

    def hmc_iterate(self, n: int):
        """n transitions: (samples [n, n_theta] float64, stats [n, 8] with the columns of HMC_STATS)."""
        samples = np.empty((int(n), self.n_theta), dtype=np.float64)
        stats = np.empty((int(n), len(HMC_STATS)), dtype=np.float64)
        dp = C.POINTER(C.c_double)
        _check(self.lib.pinn_hmc_iterate(self._h, int(n), samples.ctypes.data_as(dp), stats.ctypes.data_as(dp)))
        return samples, stats

    def hmc_theta(self) -> np.ndarray:
        th = np.empty(self.n_theta, dtype=np.float64)
        _check(self.lib.pinn_hmc_theta(self._h, th.ctypes.data_as(C.POINTER(C.c_double))))
        return th

    # -- multi-GPU --------------------------------------------------------------------------------
    @staticmethod
    def comm_unique_id() -> bytes:
        buf = (C.c_char * 128)()
        _check(load_library().pinn_comm_unique_id(C.cast(buf, C.c_void_p)))
        return bytes(buf)

    def comm_init(self, unique_id: bytes, rank: int, nranks: int):
        buf = (C.c_char * 128).from_buffer_copy(unique_id)
        _check(self.lib.pinn_comm_init(self._h, C.cast(buf, C.c_void_p), int(rank), int(nranks)))

    def comm_info(self):
        """(fused_p2p, reason): whether the multi-GPU gradient sum runs inside the fused kernel over peer memory,
        and why not when it fell back to ncclAllReduce."""
        flag = C.c_int32(0)
        why = self.lib.pinn_comm_info(self._h, C.byref(flag))
        return bool(flag.value), (why or b"").decode("utf-8", "replace")

    # -- introspection ------------------------------------------------------------------------------
    def launch_count(self) -> int:
        return int(self.lib.pinn_launch_count(self._h))

    def set_timing(self, on: bool):
        _check(self.lib.pinn_set_timing(self._h, 1 if on else 0))

    def last_kernel_ms(self) -> float:
        return float(self.lib.pinn_last_kernel_ms(self._h))

    def workspace_bytes(self) -> int:
        return int(self.lib.pinn_workspace_bytes(self._h))

    def flops_per_eval(self) -> float:
        return float(self.lib.pinn_flops_per_eval(self._h))
