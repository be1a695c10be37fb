"""Problems for the 256-wide tensor-core kernel (csrc/tc_x256_kernel.cu): the channel structures, shapes, networks and terms
of tests/tc_cases.py with hidden widths that are multiples of 64 up to 256, so that the planner sends them to that kernel.
Each builder returns a Config (neuralpde_jl_b200.configs)."""
import sympy as sp

from neuralpde_jl_b200 import configs
from neuralpde_jl_b200.configs import Config
from neuralpde_jl_b200.strategies import GridTraining, QuadratureTraining
from neuralpde_jl_b200.symbolic import Differential, Eq, In, PDESystem, parameters, variables

import tc_cases as TC
import tc_model as M

# (kernel, n1, n2, pure, ak) of every instantiation of PINN_TC_DISPATCH in tx_loss_grad_kernel: the wide kernel's set
X256_DISPATCH = {("tx",) + k[1:] for k in M.WIDE_DISPATCH}
WIDTHS = [[256, 256], [256, 192, 128], [64, 256], [192, 192]]


def x256_keys(model):
    """TcModel.dispatch_keys of a model of a 256-wide problem, named for this kernel."""
    return {("tx",) + k[1:] for k in model.dispatch_keys()}


def structure_case(name, generic):
    """Config of structure `name` (tc_cases.STRUCTURES, one that fits 4 channels per pass) on 256-wide networks."""
    build, _ = TC.STRUCTURES[name]
    i = sorted(TC.STRUCTURES).index(name)
    sys_, dx = build()
    widths = WIDTHS[i % len(WIDTHS)]
    chain = TC.net(len(sys_.ivs), widths, TC._acts(i, len(widths), generic))
    return Config("%s_x256_%s" % (name, "generic" if generic else "tanh"), sys_, [chain], GridTraining(dx))


def matrix():
    """(id, Config factory) of every structure x activation kind the 256-wide kernel runs."""
    out = []
    for name, (_, wide_ok) in sorted(TC.STRUCTURES.items()):
        if wide_ok:
            for generic in (False, True):
                out.append(("%s-x256-%s" % (name, "generic" if generic else "tanh"),
                            (lambda n=name, g=generic: structure_case(n, g))))
    return out


def burgers_depth(tl, widths=None):
    """Burgers on 2 -> 256 x (tl + 1) -> 1 (tl tensor layers), or on the given hidden widths."""
    sys_, _ = TC._burgers()
    widths = widths or [256] * (tl + 1)
    return Config("burgers_x256_%s" % "_".join(map(str, widths)), sys_, [TC.net(2, widths, ["tanh"] * len(widths))],
                  GridTraining(0.1))


def coupled():
    """Two networks of different widths and depths (256 / 192 / 64), one term taps both."""
    t, x = parameters("t x")
    u, v = variables("u v")
    U, V = u(t, x), v(t, x)
    Dt, Dx = Differential(t), Differential(x)
    eqs = [Eq(Dt(U) + V * Dx(U), 0.0), Eq((Dx ** 2)(V), U)]
    bcs = [Eq(u(0, x), sp.sin(sp.pi * x)), Eq(v(t, 0), 0.0)]
    sys_ = PDESystem(eqs, bcs, [In(t, 0.0, 1.0), In(x, 0.0, 1.0)], [t, x], [U, V])
    chains = [TC.net(2, [256, 256], ["tanh", "tanh"]), TC.net(2, [64, 192, 256], ["tanh", "softplus", "sin"])]
    return Config("coupled_x256", sys_, chains, GridTraining(0.05), multioutput=True)


def cfg4_small(width=256, hidden=3):
    """BASELINE config 4 (four coupled networks, momentum terms with 10 taps split into three passes) at a small size."""
    return configs.config4(nodes=5, bc_nodes=3, width=width, hidden=hidden)


def quadrature():
    """2-D Poisson (two passes) with Gauss-Legendre quadrature weights (WSUM terms)."""
    sys_, _ = TC._poisson()
    chain = TC.net(2, [256, 256], ["tanh", "sigmoid"])
    return Config("poisson_quadrature_x256", sys_, [chain], QuadratureTraining(nodes_per_dim=20, bc_nodes_per_dim=12))


def heat_param_estim():
    """u_t = a u_xx with a in theta.p and a DataLoss term, on a 256-wide network."""
    cfg = TC.heat_param_estim()
    cfg.chains = [TC.net(2, [256, 256], ["tanh", "tanh"])]
    cfg.name = "heat_param_estim_x256"
    return cfg


def many_rows():
    """3-D transport whose PDE term has a 7-row point matrix (hoisted coordinate rows)."""
    cfg = TC.many_rows("tw")
    cfg.chains = [TC.net(3, [256, 256], ["tanh", "softplus"])]
    cfg.name = "many_rows_x256"
    return cfg


def point_count():
    """1-D u_xx; the tests set the PDE term's point count."""
    sys_, _ = TC._uxx()
    return Config("uxx_points_x256", sys_, [TC.net(1, [256, 256], ["tanh", "tanh"])], GridTraining(1.0 / 99))
