"""NNDAE host side (no GPU): the lowered per-point value Σ_k f_k² against the float64 oracle, the grid, the term's
reduction, scale and weight, the exact-derivative deviation at θ0, the refusals, cos's derivatives against autograd,
the solution's output times and indexing, and the sm_90a compile (reference src/dae_solve.jl)."""
import math
import os
import shutil
import subprocess

import numpy as np
import pytest
import sympy as sp
import torch

import neuralpde_jl_b200 as npde
from neuralpde_jl_b200 import dae as D
from neuralpde_jl_b200 import engine as E
from neuralpde_jl_b200.build import CSRC, INCLUDE, NVCC_FLAGS, _nvcc
from neuralpde_jl_b200.ode import ComponentVector, OptimizationSolution
from nndae_oracle import DT, NNDAEOracle, case_i, case_ii, mlp

torch.set_default_dtype(torch.float64)


# ---- problems beyond the reference's two ------------------------------------------------------------------------------
def algebraic_du():
    """f reads du of its algebraic component: du_2 is 0, so 0 = u₂ - e^{-t} + du₂"""
    f = lambda du, u, p, t: [du[0] + u[0] * u[1], u[1] - sp.exp(-t) + du[1]]   # noqa: E731
    prob = npde.DAEProblem(f, [0.0, 0.0], [1.0, 1.0], (0.0, 2.0), differential_vars=[True, False])
    return prob, npde.Chain(npde.Dense(1, 8, "tanh"), npde.Dense(8, 2))


def scalar():
    """a scalar u0: f sees 1-element lists for du and u"""
    f = lambda du, u, p, t: [du[0] - sp.cos(t) * u[0]]   # noqa: E731
    prob = npde.DAEProblem(f, 0.0, 0.5, (0.0, 1.5), differential_vars=[True])
    return prob, npde.Chain(npde.Dense(1, 6, "cos"), npde.Dense(6, 1))


def with_p():
    """a problem that reads p"""
    f = lambda du, u, p, t: [du[0] - p[0] * u[0] + p[1] * u[1], u[0] + u[1] - p[2] * t]   # noqa: E731
    prob = npde.DAEProblem(f, [0.0, 0.0], [0.3, -0.3], (0.0, 1.0), [1.5, 0.5, 2.0], differential_vars=[True, False])
    return prob, npde.Chain(npde.Dense(1, 10, "cos"), npde.Dense(10, 10, "gelu"), npde.Dense(10, 2))


CASES = {"case_i": case_i, "case_ii": case_ii, "algebraic_du": algebraic_du, "scalar": scalar, "with_p": with_p}


def theta(chain, seed):
    return npde.initialparameters(np.random.default_rng(seed), chain, np.float64)


def rep_of(prob, chain, dt=DT, **kw):
    return D.NNDAERepresentation(prob, npde.NNDAE(chain, npde.Adam(0.01), **kw), dt=dt)


# ---- the lowered program against the oracle -------------------------------------------------------------------------------
_OPS = {"add": lambda a, b: a + b, "sub": lambda a, b: a - b, "mul": lambda a, b: a * b, "div": lambda a, b: a / b,
        "pow": lambda a, b: a ** b, "neg": lambda a, b: -a, "sin": lambda a, b: torch.sin(a),
        "cos": lambda a, b: torch.cos(a), "exp": lambda a, b: torch.exp(a), "log": lambda a, b: torch.log(a),
        "tanh": lambda a, b: torch.tanh(a), "sqrt": lambda a, b: torch.sqrt(a), "abs": lambda a, b: torch.abs(a)}


def run_term(spec, chain, th, t):
    """the term's program on the host, its taps (value and d/dt of output k) by autograd"""
    tt = torch.tensor(t).requires_grad_(True)
    N = mlp(torch.tensor(th), chain.dims, chain.acts, tt[None, :])
    taps = []
    for tp in spec.taps:
        v = N[tp.out]
        for _ in tp.dirs:
            v = torch.autograd.grad(v.sum(), tt, create_graph=True)[0]
        taps.append(v.detach())
    val = []
    for op, a, b, imm in spec.prog:
        if op == "const":
            val.append(torch.full((t.size,), imm))
        elif op == "coord":
            val.append(torch.tensor(t))
        elif op == "tap":
            val.append(taps[a])
        elif op == "powi":
            val.append(val[a] ** int(imm))
        else:
            val.append(_OPS[op](val[a], val[b] if b < len(val) else None))
    return val[-1].numpy()


@pytest.mark.parametrize("name", sorted(CASES))
@pytest.mark.parametrize("seed", [0, 5])
def test_lowered_value_matches_oracle(name, seed):
    prob, chain = CASES[name]()
    rep = rep_of(prob, chain)
    th = theta(chain, seed)
    mine = run_term(rep.specs[0], chain, th, rep.ts)
    ref = NNDAEOracle(prob, chain).per_point(torch.tensor(th), torch.tensor(rep.ts), "exact").detach().numpy()
    np.testing.assert_allclose(mine, ref, rtol=1e-13, atol=1e-13 * np.abs(ref).max())


def test_algebraic_component_gets_zero_derivative():
    """f reads du₂ of the algebraic u₂: the program has no d/dt tap of output 1"""
    prob, chain = algebraic_du()
    spec = rep_of(prob, chain).specs[0]
    assert sorted((tp.out, tp.order) for tp in spec.taps) == [(0, 0), (0, 1), (1, 0)]


# ---- grid, term, θ ---------------------------------------------------------------------------------------------------------
def test_grid_and_term():
    """tspan[1]:dt:tspan[2] with Float32 tspan and dt = 1/100f0; one functional term: (1/n Σ_i v_i)², no weights"""
    for case, n in ((case_i, 101), (case_ii, 158)):
        prob, chain = case()
        rep = rep_of(prob, chain)
        assert rep.ts.size == n and rep.ts[0] == 0.0 and rep.ts[-1] <= prob.tspan[1]
        np.testing.assert_allclose(np.diff(rep.ts), DT, rtol=1e-12)
        assert len(rep.specs) == 1 and rep.term_names == ["loss"]
        spec = rep.specs[0]
        assert spec.reduction == E.REDUCE_SQUARE_OF_SUM and spec.scale == 1.0 / n
        assert list(rep.term_weights) == [1.0] and rep.quad_weights == [None]
        np.testing.assert_array_equal(rep.point_sets[0], rep.ts[None, :])
        assert rep.flat_init_params.shape == (chain.n_params,) and rep.flat_init_params.p.size == 0
        assert rep.spec.n_params == 0 and rep.dtype == np.float64
    prob, chain = case_i()
    assert rep_of(prob, chain, init_params=theta(chain, 1).astype(np.float32)).dtype == np.float32


@pytest.mark.parametrize("case", [case_i, case_ii])
def test_exact_derivative_against_forward_difference(case):
    """the deviation of the exact d/dt from the reference's forward difference, pinned at θ0 in float64 (measured
    2e-9 and 4e-9)"""
    prob, chain = case()
    th, t = torch.tensor(rep_of(prob, chain).flat_init_params), torch.tensor(rep_of(prob, chain).ts)
    orc = NNDAEOracle(prob, chain)
    ex, fd = orc.loss(th, t, "exact").item(), orc.loss(th, t, "fd").item()
    rel = abs(ex - fd) / abs(ex)
    print("%s exact vs forward difference at θ0: relative %.2e" % (case.__name__, rel))
    assert rel < 1e-7


# ---- refusals --------------------------------------------------------------------------------------------------------------
def test_refusals():
    f = lambda du, u, p, t: [du[0] - u[1], u[1] - t]   # noqa: E731
    with pytest.raises(ValueError, match="needs differential_vars"):
        npde.DAEProblem(f, [0.0, 0.0], [0.0, 0.0], (0.0, 1.0))
    with pytest.raises(ValueError, match="differential_vars has 3 entries, u0 has 2"):
        npde.DAEProblem(f, [0.0, 0.0], [0.0, 0.0], (0.0, 1.0), differential_vars=[True, False, False])
    with pytest.raises(ValueError, match="complex"):
        npde.DAEProblem(f, [0.0, 0.0], [0.0, 1j], (0.0, 1.0), differential_vars=[True, False])
    with pytest.raises(ValueError, match="complex"):
        npde.DAEProblem(f, [0.0, 0.0], [0.0, 0.0], (0.0, 1.0), [1 + 2j], differential_vars=[True, False])
    with pytest.raises(ValueError, match=r"The NNODE solver only supports out-of-place DAE definitions, i.e. du=f\(u,p,t\)\."):
        npde.DAEProblem(lambda out, du, u, p, t: None, [0.0, 0.0], [0.0, 0.0], (0.0, 1.0), differential_vars=[True, False])
    prob = npde.DAEProblem(f, [0.0, 0.0], [0.0, 0.0], (0.0, 1.0), differential_vars=[True, False])
    chain = npde.Chain(npde.Dense(1, 4, "cos"), npde.Dense(4, 2))
    with pytest.raises(ValueError, match="only GridTraining"):
        rep_of(prob, chain, strategy=npde.GridTraining(0.1))
    with pytest.raises(ValueError, match="`dt` is not defined"):
        rep_of(prob, chain, dt=None)
    with pytest.raises(ValueError, match="autodiff not supported for GridTraining."):
        rep_of(prob, chain, autodiff=True)
    with pytest.raises(ValueError, match="1 input and 2 outputs"):
        rep_of(prob, npde.Chain(npde.Dense(1, 4, "cos"), npde.Dense(4, 3)))
    for mode in ("tc_bf16", "tc_split"):
        with pytest.raises(ValueError, match="NNDAE runs on the FFMA kernel"):
            npde.NNDAE(chain, npde.Adam(0.01), mode=mode)
    with pytest.raises(ValueError, match="needs float64 parameters"):
        rep_of(prob, chain, init_params=theta(chain, 0).astype(np.float32), mode="tc_f64")
    with pytest.raises(TypeError, match="takes no callback or chunk"):
        npde.solve(prob, npde.NNDAE(chain, npde.Adam(0.01)), maxiters=10, dt=0.1, callback=lambda *a: False)
    with pytest.raises(TypeError, match="needs maxiters"):
        npde.solve(prob, npde.NNDAE(chain, npde.Adam(0.01)), dt=0.1)
    with pytest.raises(TypeError, match="alg must be an NNDAE"):
        D.NNDAERepresentation(prob, npde.NNODE(chain, npde.Adam(0.01)), dt=0.1)
    with pytest.raises(ValueError, match="could not be traced with symbolic du, u, p and t"):
        rep_of(npde.DAEProblem(lambda du, u, p, t: [float(du[0]), u[1]], [0.0, 0.0], [0.0, 0.0], (0.0, 1.0),
                               differential_vars=[True, False]), chain)
    with pytest.raises(ValueError, match="returns 1 components, u0 has 2"):
        rep_of(npde.DAEProblem(lambda du, u, p, t: [du[0]], [0.0, 0.0], [0.0, 0.0], (0.0, 1.0),
                               differential_vars=[True, False]), chain)


# ---- cos ---------------------------------------------------------------------------------------------------------------------
def test_cos_derivatives_against_autograd():
    """the closed form the kernel evaluates (ffma_kernel.cuh act_eval4, PINN_ACT_COS): cos, -sin, -cos, sin, cos"""
    z = torch.cat([torch.linspace(-40.0, 40.0, 801), torch.tensor([-1e-8, 0.0, 1e-8, 17.3, -23.9])]).requires_grad_(True)
    ds = [torch.cos(z)]
    for _ in range(4):
        ds.append(torch.autograd.grad(ds[-1].sum(), z, create_graph=True)[0])
    zn = z.detach().numpy()
    mine = [np.cos(zn), -np.sin(zn), -np.cos(zn), np.sin(zn), np.cos(zn)]
    for k, (a, b) in enumerate(zip(mine, ds)):
        np.testing.assert_allclose(a, b.detach().numpy(), rtol=1e-15, atol=1e-15, err_msg="derivative %d" % k)
    assert npde.Dense(1, 3, "cos").activation == "cos" and E.ACT["cos"] == 8


# ---- solution ----------------------------------------------------------------------------------------------------------------
class _FakeRep:
    """the solution's view of a representation, with φ evaluated by the oracle instead of the device"""

    def __init__(self, prob, chain, alg):
        self.prob, self.alg, self.orc = prob, alg, NNDAEOracle(prob, chain)

    def trial(self, theta, X):
        t = torch.tensor(np.ravel(np.asarray(X, dtype=np.float64)))
        return self.orc.phi(torch.tensor(np.asarray(theta, dtype=np.float64)), t).detach().numpy()


def _solution(case, saveat=None, dt=None, save_everystep=True, analytic=None):
    prob, chain = case()
    if analytic is not None:
        prob = npde.DAEProblem(npde.DAEFunction(prob.f.f, analytic), prob.du0, prob.u0, prob.tspan, prob.p,
                               differential_vars=prob.differential_vars)
    th = ComponentVector(theta(chain, 3), chain.n_params)
    res = OptimizationSolution(th, 0.25, 7, "Success")
    rep = _FakeRep(prob, chain, npde.NNDAE(chain, npde.Adam(0.01)))
    ts = D._save_times(*prob.tspan, saveat, dt, save_everystep)
    return D.DAESolution(rep, res, ts), rep, th


def test_solution_times_and_indexing():
    sol, rep, th = _solution(case_i, dt=DT)
    assert sol.t.size == 101 and sol.resid == 0.25 and sol.retcode == "Success" and sol.k.u.p.size == 0
    U = rep.trial(th, sol.t)
    np.testing.assert_array_equal(np.stack(sol.u, axis=1), U)
    np.testing.assert_array_equal(sol(0.37), rep.trial(th, [0.37])[:, 0])
    assert sol(0.37, idxs=1) == rep.trial(th, [0.37])[1, 0]
    np.testing.assert_array_equal(sol(np.array([0.1, 0.2])), rep.trial(th, [0.1, 0.2]))
    assert _solution(case_i, saveat=0.25)[0].t.tolist() == [0.0, 0.25, 0.5, 0.75, 1.0]
    assert _solution(case_i, saveat=[0.1, 0.3])[0].t.tolist() == [0.1, 0.3]
    assert _solution(case_i)[0].t.size == 100
    assert _solution(case_i, save_everystep=False)[0].t.tolist() == [0.0, 1.0]
    sol, rep, th = _solution(scalar, saveat=0.5)
    assert all(isinstance(v, float) for v in sol.u) and len(sol.u) == 4
    assert sol(0.5) == rep.trial(th, [0.5])[0, 0]


def test_solution_errors_with_analytic():
    """DAEFunction's analytic(du0, u0, p, t): SciMLBase's timeseries errors"""
    seen = []

    def an(du0, u0, p, t):
        seen.append((du0, u0))
        return [1 + math.sin(2 * math.pi * t) / (2 * math.pi), -math.cos(2 * math.pi * t)]

    sol, rep, th = _solution(case_i, saveat=0.5, analytic=an)
    A = np.array([an([0.0, 0.0], [1.0, -1.0], None, t) for t in sol.t]).T
    E_ = rep.trial(th, sol.t) - A
    assert seen[0] == ([0.0, 0.0], [1.0, -1.0])
    assert sol.errors["l∞"] == pytest.approx(np.abs(E_).max(), rel=1e-15)
    assert sol.errors["final"] == pytest.approx(np.abs(E_[:, -1]).mean(), rel=1e-15)
    assert sol.errors["l2"] == pytest.approx(np.sqrt(np.mean(E_ ** 2)), rel=1e-15)
    assert _solution(case_i, saveat=0.5)[0].errors == {}


# ---- the sm_90a compile ----------------------------------------------------------------------------------------------------
@pytest.mark.skipif(shutil.which("nvcc") is None and not os.path.exists("/usr/local/cuda/bin/nvcc"), reason="no nvcc")
def test_cos_activation_compiles_for_sm90a(tmp_path):
    """the planner (cos's range check and tensor-core refusal) and the FFMA kernel, where cos joins act_eval4"""
    assert "PINN_ACT_COS = 8" in open(os.path.join(INCLUDE, "pinn_b200.h")).read()
    for src, defs in (("plan.cu", []), ("ffma_inst.cu", ["-DPINN_INST_REAL=double", "-DPINN_INST_BUFS=1"])):
        r = subprocess.run([_nvcc(), *NVCC_FLAGS, *defs, "-c", os.path.join(CSRC, src), "-o", str(tmp_path / "x.o")],
                           capture_output=True, text=True)
        assert r.returncode == 0, r.stderr
