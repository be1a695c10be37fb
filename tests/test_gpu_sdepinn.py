"""SDEPINN on the device: the norm term (a weighted-sum owner of an integral) on its own, then loss, term losses and
gradient of the whole problem against the float64 oracle, tc_f64 against ffma, logcosh's value, first and third
derivative taps against autograd, the launch count and reproducibility, device BFGS against the float64 quasi-Newton
oracle, and the reference's test/NNSDE2 problems (reference src/NN_SDE_weaksolve.jl)."""
import dataclasses
import math

import numpy as np
import pytest
import torch
from scipy import stats

import neuralpde_jl_b200 as npde
from neuralpde_jl_b200 import engine as E
from neuralpde_jl_b200.lowering import lower_equation, term_spec
from neuralpde_jl_b200.sde_weak import SDEPINNProblem
from neuralpde_jl_b200.symbolic import get_vars
from sdepinn_oracle import SDEPINNOracle, act
from test_sdepinn_host import chain, make, theta
import qn_oracle as Q

pytestmark = pytest.mark.gpu
torch.set_default_dtype(torch.float64)


def rel(a, b):
    a, b = np.asarray(a, dtype=np.float64), np.asarray(b, dtype=np.float64)
    return float(np.linalg.norm(a - b) / max(np.linalg.norm(b), 1e-300))


def _rep(name, dtype=np.float64, seed=0, mode="ffma", **kw):
    prob, alg0, case = make(name)
    th = theta(alg0.chain, seed)
    prob, alg, case = make(name, initial_parameters=th.astype(dtype), mode=mode, **kw)
    opt_prob = SDEPINNProblem(prob, alg).discretize()
    return opt_prob, alg, case, th


def _weights(rep):
    w = rep.weights
    return np.concatenate([w["pde"], w["bc"], w["add"]])


def _oracle(case, alg, th64, **kw):
    return SDEPINNOracle(case, alg.chain.dims, alg.chain.acts, lam=alg.λ_norm, **kw).loss_and_grad(th64)


# ---- the norm term on its own --------------------------------------------------------------------------------------------
@pytest.mark.parametrize("dtype, ltol, gtol", [(np.float64, 1e-10, 1e-9), (np.float32, 1e-5, 5e-4)])
@pytest.mark.parametrize("name", ["ou", "gbm"])
def test_norm_term_alone(name, dtype, ltol, gtol):
    """one weighted-sum term whose program is INTEGRAL 0 - 1, on its own in an engine problem: Σ_t (∫ p̂ dx - 1)² over
    the 21 grid times with 64 Gauss-Legendre nodes"""
    prob, alg, case = make(name)
    s = SDEPINNProblem(prob, alg)
    norm = s.discretization.additional_loss
    vi = get_vars(s.pde_system.ivs, s.pde_system.dvs)
    lt = lower_equation(norm.eq, vi)
    integ = [dataclasses.replace(it, owner=0, q=64) for it in lt.integrals]
    ch = alg.chain
    th = theta(ch, 4)
    spec = E.ProblemSpec(nets=[E.NetSpec(ch.dims, ch.acts, 0)], terms=[term_spec(lt, E.REDUCE_WSUM, 1.0)],
                         n_theta=th.size, dtype=np.dtype(dtype).name, integrals=integ)
    eng = E.Engine(spec)
    eng.set_points_host(0, norm.points.astype(dtype), np.ones(norm.points.shape[1], dtype=dtype))
    total, terms, grad = eng.loss_grad_host(th.astype(dtype), None, True)
    orc = SDEPINNOracle(case, ch.dims, ch.acts)
    t = torch.tensor(th).requires_grad_(True)
    L = orc.term_losses(t)[-1]
    (G,) = torch.autograd.grad(L, t)
    assert abs(total - float(L)) <= ltol * float(L), (total, float(L))
    assert rel(grad, G.numpy()) <= gtol


# ---- the whole problem ----------------------------------------------------------------------------------------------
@pytest.mark.parametrize("dtype, ltol, gtol", [(np.float64, 1e-10, 1e-9), (np.float32, 1e-5, 5e-4)])
@pytest.mark.parametrize("seed", [0, 7])
@pytest.mark.parametrize("name", ["ou", "gbm"])
def test_loss_terms_and_gradient_against_oracle(name, seed, dtype, ltol, gtol):
    opt_prob, alg, case, th = _rep(name, dtype, seed)
    rep = opt_prob.representation
    total, terms, grad = rep.engine.loss_grad_host(opt_prob.u0, _weights(rep), True)
    L, T, G = _oracle(case, alg, th)
    assert rep.term_names == ["pde_1"] + ["bc_%d" % (j + 1) for j in range(len(T) - 2)] + ["additional"]
    assert abs(total - L) <= ltol * L, (total, L)
    np.testing.assert_allclose(terms, T, rtol=ltol * 10, atol=ltol * L)
    assert rel(grad, G) <= gtol
    f, g = opt_prob.f.grad(opt_prob.u0, None)
    assert f == total and np.array_equal(g, grad)


def test_lambda_norm_is_the_norm_term_weight():
    opt_prob, alg, case, th = _rep("ou", λ_norm=2.5)
    rep = opt_prob.representation
    total, terms, grad = rep.engine.loss_grad_host(opt_prob.u0, _weights(rep), True)
    L, T, G = _oracle(case, alg, th)
    assert abs(total - L) <= 1e-10 * L and abs(total - (sum(terms[:-1]) + 2.5 * terms[-1])) <= 1e-12 * L
    assert rel(grad, G) <= 1e-9


@pytest.mark.parametrize("name", ["ou", "gbm"])
def test_tc_f64_matches_ffma(name):
    out = []
    for mode in ("ffma", "tc_f64"):
        opt_prob, _, _, _ = _rep(name, np.float64, 3, mode=mode)
        rep = opt_prob.representation
        out.append(rep.engine.loss_grad_host(opt_prob.u0, _weights(rep), True))
    assert abs(out[1][0] - out[0][0]) <= 1e-12 * abs(out[0][0])
    np.testing.assert_allclose(out[1][1], out[0][1], rtol=1e-12)
    assert rel(out[1][2], out[0][2]) <= 1e-12


@pytest.mark.parametrize("mode", ["tc_split", "tc_bf16"])
def test_tensor_core_modes_refuse_logcosh(mode):
    """the engine refuses a logcosh layer on the tensor-core kernels (SDEPINN itself refuses the modes first)"""
    dims, acts = [2, 16, 16, 1], ["logcosh", "tanh", "identity"]
    term = E.TermSpec(dim=2, taps=[E.TapSpec(net=0, order=0)], prog=[("tap", 0, 0, 0.0)], net_rows=[[0, 1]])
    with pytest.raises(E.EngineError, match="logcosh layers run on the FFMA path"):
        E.Engine(E.ProblemSpec(nets=[E.NetSpec(dims, acts, 0)], terms=[term], n_theta=16 * 3 + 16 * 17 + 17,
                               dtype="float32", mode=E.MODE_TC_SPLIT if mode == "tc_split" else E.MODE_TC_BF16))


# ---- logcosh taps -------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("dtype, ltol, gtol", [(np.float64, 1e-10, 1e-9), (np.float32, 1e-5, 5e-4)])
def test_logcosh_value_first_and_third_derivative_taps(dtype, ltol, gtol):
    """a PDE-style term on a logcosh network: r = u + ∂u/∂x + ∂³u/∂y³ - x y over a 2-D point set (the reverse sweep of
    the third-derivative tap takes logcosh's fourth derivative); weights scaled so that some pre-activations pass 20"""
    dims, acts = [2, 12, 12, 1], ["logcosh", "logcosh", "logcosh"]
    ch = npde.Chain(npde.Dense(2, 12, "logcosh"), npde.Dense(12, 12, "logcosh"), npde.Dense(12, 1, "logcosh"))
    theta_ = npde.initialparameters(np.random.default_rng(5), ch, np.float64) * 3.0
    taps = [E.TapSpec(net=0, order=0), E.TapSpec(net=0, order=1, dirs=(0,)), E.TapSpec(net=0, order=3, dirs=(1, 1, 1))]
    prog = [("tap", 0, 0, 0.0), ("tap", 1, 0, 0.0), ("add", 0, 1, 0.0), ("tap", 2, 0, 0.0), ("add", 2, 3, 0.0),
            ("coord", 0, 0, 0.0), ("coord", 1, 0, 0.0), ("mul", 5, 6, 0.0), ("sub", 4, 7, 0.0)]
    term = E.TermSpec(dim=2, taps=taps, prog=prog, net_rows=[[0, 1]])
    eng = E.Engine(E.ProblemSpec(nets=[E.NetSpec(dims, acts, 0)], terms=[term], n_theta=theta_.size,
                                 dtype=np.dtype(dtype).name))
    X = np.random.default_rng(1).uniform(-3, 3, size=(2, 300))
    eng.set_points_host(0, X.astype(dtype))
    total, _, grad = eng.loss_grad_host(theta_.astype(dtype), None, True)
    th = torch.tensor(theta_).requires_grad_(True)
    x = torch.tensor(X).requires_grad_(True)
    h = x
    o = 0
    pre = []
    for a, (i, j) in zip(acts, zip(dims[:-1], dims[1:])):
        W = th[o:o + i * j].reshape(i, j).T
        b = th[o + i * j:o + i * j + j]
        o += i * j + j
        z = W @ h + b[:, None]
        pre.append(float(z.abs().max()))
        h = act(a, z)
    u = h[0]
    assert max(pre) > 20.0           # the large-|z| branch is exercised
    (gx,) = torch.autograd.grad(u.sum(), x, create_graph=True)
    d3 = gx[1]
    for _ in range(2):
        (gg,) = torch.autograd.grad(d3.sum(), x, create_graph=True)
        d3 = gg[1]
    L = ((u + gx[0] + d3 - x[0] * x[1]) ** 2).mean()
    (G,) = torch.autograd.grad(L, th)
    assert abs(total - float(L)) <= ltol * float(L), (total, float(L))
    assert rel(grad, G.numpy()) <= gtol


# ---- launches, reproducibility, BFGS ------------------------------------------------------------------------------------
def test_one_launch_per_evaluation_and_bit_reproducible():
    opt_prob, _, _, _ = _rep("ou")
    rep = opt_prob.representation
    eng = rep.engine
    out = []
    for _ in range(3):
        l0 = eng.launch_count()
        out.append(eng.loss_grad_host(opt_prob.u0, _weights(rep), True))
        assert eng.launch_count() - l0 == 1
    for r in out[1:]:
        assert r[0] == out[0][0] and np.array_equal(r[1], out[0][1]) and np.array_equal(r[2], out[0][2])


@pytest.mark.parametrize("name", ["ou", "gbm"])
def test_device_bfgs_against_oracle(name):
    opt_prob, alg, case, th = _rep(name, np.float64, 0)
    eng = opt_prob.representation.engine
    eng.qn_begin(opt_prob.u0, E.QN_BFGS, linesearch=E.LS_HAGERZHANG, weights=_weights(opt_prob.representation))
    f0, _, _, _, _ = eng.qn_iterate(0)
    traj = []
    for _ in range(6):
        f, _, status, it, ev = eng.qn_iterate(1)
        if it == len(traj):
            break
        traj.append((eng.qn_theta().astype(np.float64), f, ev))
        if status != E.QN_RUNNING:
            break
    orc = SDEPINNOracle(case, alg.chain.dims, alg.chain.acts, lam=alg.λ_norm)
    fg = lambda t: orc.loss_and_grad(t)[0::2]          # noqa: E731
    res = Q.minimize(fg, th, method="bfgs", linesearch="hagerzhang", maxiters=6)
    assert abs(f0 - fg(th)[0]) <= 1e-10 * abs(f0)
    assert len(traj) == len(res.history) >= 3
    for k, ((th_e, f_e, ev_e), (th_o, f_o, ev_o)) in enumerate(zip(traj, res.history)):
        assert rel(th_e, th_o) <= 1e-6, (k, rel(th_e, th_o))
        assert abs(f_e - f_o) <= 1e-8 * abs(f_o), (k, f_e, f_o)
        assert ev_e == ev_o
    assert traj[-1][1] < f0


# ---- the reference's test/NNSDE2 ------------------------------------------------------------------------------------------
def _mse(phi, u, x_0, x_end, dx, pdf):
    xs = np.arange(int(round((x_end - x_0) / dx)) + 1) * dx + x_0
    err = []
    for t in (0.1, 0.2, 0.4, 0.6, 0.8, 1.0):
        pred = phi(np.vstack([xs, np.full(xs.size, t)]), u)[0]
        err.append((pdf(xs, t) - pred) ** 2)
    return float(np.mean(np.concatenate(err)))


def test_reference_ou_process():
    """nn_sde_weaksolve__ou_process.jl: BFGS, maxiters 300, MSE < 1e-2 against the OU density"""
    prob, _, _ = make("ou")
    alg = npde.SDEPINN(chain=chain(), optimalg=npde.BFGS(), x_0=-4.0, x_end=4.0, distrib=npde.Normal(0.5, 0.05))
    res, phi = npde.solve(prob, alg, maxiters=300)
    pdf = lambda x, t: stats.norm(0.5 * math.exp(-t), math.sqrt(0.5 * (1 - math.exp(-2 * t)))).pdf(x)   # noqa: E731
    mse = _mse(phi, res.u, -4.0, 4.0, 0.02, pdf)
    print("OU: objective %.6g after %d iterations (%s), MSE %.4g" % (res.objective, res.iterations, res.retcode, mse))
    assert np.isfinite(res.objective)
    assert mse < 1e-2


def test_reference_gbm():
    """nn_sde_weaksolve__gbm_sde.jl: BFGS, maxiters 400, MSE < 5e-2 against the GBM (log-normal) density"""
    prob, _, _ = make("gbm")
    alg = npde.SDEPINN(chain=chain(), optimalg=npde.BFGS(), x_0=0.0, x_end=3.0,
                       distrib=npde.LogNormal(math.log(1.0), 0.05))
    res, phi = npde.solve(prob, alg, maxiters=400)
    pdf = lambda x, t: stats.lognorm(math.sqrt(t) * 0.3, scale=math.exp((0.2 - 0.045) * t)).pdf(x)   # noqa: E731
    mse = _mse(phi, res.u, 0.0, 3.0, 0.01, pdf)
    print("GBM: objective %.6g after %d iterations (%s), MSE %.4g" % (res.objective, res.iterations, res.retcode, mse))
    assert np.isfinite(res.objective)
    assert mse < 5e-2
