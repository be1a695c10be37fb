"""NNSDE host side (no GPU): tracing and lowering of f and g, point layout and weights of every strategy, weak / strong
and batch on / off, the Euler-Maruyama terms, loss assembly against the float64 oracle, the exact-vs-FD d/dt
distance, the KKL sampler replay's own invariants, the refusals, and the kernel sources' compile for sm_90a
(reference src/NN_SDE_solve.jl)."""
import math
import os
import shutil
import subprocess

import numpy as np
import pytest
import sympy as sp
import torch

import neuralpde_jl_b200 as npde
from neuralpde_jl_b200.engine import REDUCE_MEAN, REDUCE_WSUM
from nnode_oracle import mlp
from nnsde_oracle import NNSDEOracle, kkl_points

torch.set_default_dtype(torch.float64)


# ---- problems ------------------------------------------------------------------------------------------------------
def gbm(tspan=(0.0, 1.0)):                # test/NNSDE1 test 1 / 2
    return npde.SDEProblem(lambda u, p, t: 1.2 * u, lambda u, p, t: 1.1 * u, 0.5, tspan)


def additive():                           # test 3
    return npde.SDEProblem(lambda u, p, t: 0.05 / sp.sqrt(1 + t) - u / ((1 + t) * 2),
                           lambda u, p, t: 0.05 * 0.1 / sp.sqrt(1 + t), 0.5, (0.0, 1.0))


def vector2():
    return npde.SDEProblem(lambda u, p, t: [-u[0] + u[1] * sp.sin(t), p[0] * u[0] - u[1]],
                           lambda u, p, t: [0.1 * u[0], p[1] * u[1] ** 2], [1.0, 0.5], (0.5, 2.0), [0.7, 0.3])


def gbm_inverse(p=(0.0, 0.0)):            # test 4
    return npde.SDEProblem(lambda u, p, t: p[0] * u, lambda u, p, t: p[1] * u, 0.5, (0.0, 1.0), list(p))


def chain(n_in, n_out, width=6, act="tanh"):
    return npde.Chain(npde.Dense(n_in, width, act), npde.Dense(width, width, act), npde.Dense(width, n_out))


def dataset(n_paths=3, n_t=11, seed=5):
    rng = np.random.default_rng(seed)
    t = np.linspace(0.0, 1.0, n_t)
    dW = rng.standard_normal((n_paths, n_t - 1)) * np.sqrt(np.diff(t))
    W = np.concatenate([np.zeros((n_paths, 1)), np.cumsum(dW, axis=1)], axis=1)
    return [[0.5 * np.exp((1.5 - 0.125) * t + 0.5 * w) for w in W], t]


def _run_prog(spec, rows, taps, params):
    val = []
    for op, a, b, imm in spec.prog:
        f = {"const": lambda: np.full(rows.shape[1], imm), "coord": lambda: rows[a], "tap": lambda: taps[a],
             "param": lambda: np.full(rows.shape[1], params[a]),
             "add": lambda: val[a] + val[b], "sub": lambda: val[a] - val[b], "mul": lambda: val[a] * val[b],
             "div": lambda: val[a] / val[b], "neg": lambda: -val[a], "powi": lambda: val[a] ** int(imm),
             "pow": lambda: val[a] ** val[b], "sin": lambda: np.sin(val[a]), "cos": lambda: np.cos(val[a]),
             "exp": lambda: np.exp(val[a]), "log": lambda: np.log(val[a]), "tanh": lambda: np.tanh(val[a]),
             "sqrt": lambda: np.sqrt(val[a]), "abs": lambda: np.abs(val[a])}[op]
        val.append(f())
    return val[-1]


def oracle_taps(spec, orc, th, X):
    """N_k and dN_k/dt at the (1 + n_z, m) points, from the oracle's MLP"""
    t = torch.tensor(X[0]).requires_grad_(True)
    N = mlp(th, orc.dims, orc.acts, torch.cat([t[None, :], torch.tensor(X[1:])]))
    dN = torch.stack([torch.autograd.grad(N[k].sum(), t, retain_graph=True)[0] for k in range(orc.n)])
    return [(dN if tp.order else N)[tp.out].detach().numpy() for tp in spec.taps]


def host_terms(rep, orc, theta, point_sets=None):
    """every term's loss, the engine's reduction restated on the host, from the program run on oracle taps"""
    th = torch.tensor(np.asarray(theta, dtype=np.float64))
    out = []
    for i, spec in enumerate(rep.specs):
        X = (point_sets or rep.point_sets)[i]
        r = _run_prog(spec, X, oracle_taps(spec, orc, th, X) if spec.taps else [], np.asarray(theta)[rep.n_net:])
        if spec.reduction == REDUCE_MEAN:
            out.append(np.mean(r ** 2))
        else:
            w = rep.quad_weights[i] if rep.quad_weights[i] is not None else np.ones(X.shape[1])
            out.append(spec.scale * np.sum(w * r ** 2))
    return np.array(out)


def per_time(X, S):
    """the reference's Vector of (1 + n_z) x S input matrices from the engine's point layout p = i S + s"""
    return [torch.tensor(X[:, i * S:(i + 1) * S]) for i in range(X.shape[1] // S)]


def oracle_total(rep, orc, theta, alg, point_sets=None, derivative="exact"):
    """the reference's total_loss at θ (a tensor to differentiate, or an array)"""
    th = theta if isinstance(theta, torch.Tensor) else torch.tensor(np.asarray(theta, dtype=np.float64))
    tt = "sum" if alg.strong_loss else "mean"
    X = (point_sets or rep.point_sets)[0]
    if isinstance(rep.strategy, npde.QuadratureTraining):
        L = orc.quadrature_loss(th, torch.tensor(X), torch.tensor(rep.quad_weights[0]), tt, derivative)
    else:
        L = orc.grid_loss(th, per_time(X, alg.sub_batch), alg.batch, tt, derivative)
    if alg.param_estim and alg.dataset:
        L = L + orc.em_loss(th, alg.dataset)
    return L


def cases():
    ds = dataset()
    out = []
    for strong in (False, True):
        for batch in (True, False):
            for S in (1, 4):
                out += [("grid", gbm(), dict(strategy=npde.GridTraining(0.1), sub_batch=S, strong_loss=strong, batch=batch)),
                        ("wit", vector2(), dict(strategy=npde.WeightedIntervalTraining([0.5, 0.5], 8), sub_batch=S,
                                                strong_loss=strong, batch=batch)),
                        ("estim", gbm_inverse((1.1, 0.4)), dict(strategy=npde.GridTraining(0.25), sub_batch=S,
                                                                strong_loss=strong, batch=batch, param_estim=True,
                                                                dataset=ds))]
        out += [("quad", additive(), dict(strong_loss=strong)), ("quad_vec", vector2(), dict(strong_loss=strong))]
    return out


def make(i, n_z=3, dtype=np.float64):
    name, prob, akw = cases()[i]
    n = 1 if np.ndim(prob.u0) == 0 else len(prob.u0)
    ch = chain(1 + n_z, n)
    alg = npde.NNSDE(ch, npde.Adam(0.1), seed=i, **akw)
    if dtype != np.float64:
        init = npde.NNSDERepresentation(prob, alg).flat_init_params
        alg = npde.NNSDE(ch, npde.Adam(0.1), np.asarray(init, dtype=dtype), seed=i, **akw)
    return name, prob, alg, npde.NNSDERepresentation(prob, alg)


# ---- tracing and lowering ----------------------------------------------------------------------------------------
@pytest.mark.parametrize("prob, estim", [(gbm(), False), (additive(), False), (vector2(), False),
                                         (gbm_inverse((1.5, 0.5)), True), (gbm((0.5, 2.0)), False)])
def test_lowered_program_matches_oracle_residual(prob, estim):
    n = 1 if np.ndim(prob.u0) == 0 else len(prob.u0)
    ch = chain(4, n)
    ds = dataset() if estim else []
    alg = npde.NNSDE(ch, npde.Adam(0.1), param_estim=estim, dataset=ds, sub_batch=3)
    rep = npde.NNSDERepresentation(prob, alg, dt=0.1)
    theta = np.asarray(rep.flat_init_params, dtype=np.float64).copy()
    if alg.param_estim:
        theta[rep.n_net:] += np.linspace(0.1, 0.3, theta.size - rep.n_net)
    orc = NNSDEOracle(prob, ch, param_estim=alg.param_estim)
    X = rep.point_sets[0]
    R = orc.residual(torch.tensor(theta), torch.tensor(X)).detach().numpy()
    for k in range(n):
        spec = rep.specs[k]
        assert [tp.net for tp in spec.taps] == [0] * len(spec.taps) and {tp.out for tp in spec.taps} <= set(range(n))
        assert {tp.dirs for tp in spec.taps} <= {(), (0,)} and spec.net_rows == [[0, 1, 2, 3]]
        r = _run_prog(spec, X, oracle_taps(spec, orc, torch.tensor(theta), X), theta[rep.n_net:])
        np.testing.assert_allclose(-r, R[k], rtol=1e-13, atol=1e-13)


def test_time_rescaling_and_ensemble_draw_shapes():
    rep = npde.NNSDERepresentation(gbm((0.5, 2.0)), npde.NNSDE(chain(4, 1), npde.Adam(0.1), sub_batch=2), dt=0.3)
    assert rep.tspan_scale == (0.25, 1.0) and rep.dt == pytest.approx(0.4)
    np.testing.assert_allclose(rep.training_sets[0][0], [0.25, 0.25])
    np.testing.assert_allclose([m[0, 0] for m in rep.training_sets], [0.25, 0.65])
    rep = npde.NNSDERepresentation(gbm(), npde.NNSDE(chain(4, 1), npde.Adam(0.1)), dt=0.1)
    assert rep.n_z == 3 and rep.point_sets[0].shape == (4, 11)


# ---- point layout and weights ------------------------------------------------------------------------------------
def test_point_layout_and_weights_of_every_row():
    prob, ch = vector2(), chain(4, 2)
    S = 4
    for strong in (False, True):
        for batch in (True, False):
            alg = npde.NNSDE(ch, npde.Adam(0.1), strategy=npde.GridTraining(0.1), sub_batch=S, strong_loss=strong,
                             batch=batch)
            rep = npde.NNSDERepresentation(prob, alg)
            X = rep.point_sets[0]
            nt = len(rep.training_sets)
            assert X.shape == (4, nt * S) and np.array_equal(X, np.concatenate(rep.training_sets, axis=1))
            np.testing.assert_allclose(X[0], np.repeat([m[0, 0] for m in rep.training_sets], S))
            zs = X[1:].reshape(3, nt, S)
            if strong:        # one z per path, bit-identical across times
                assert all(np.array_equal(zs[:, i], zs[:, 0]) for i in range(nt))
            else:             # an independent draw per point
                assert len({tuple(c) for c in X[1:].T}) == nt * S
            spec = rep.specs[0]
            if not strong and batch:
                assert spec.reduction == REDUCE_MEAN
            else:
                assert spec.reduction == REDUCE_WSUM
                assert spec.scale == {(False, False): 1 / S, (True, True): 1 / nt, (True, False): 1.0}[(strong, batch)]
            np.testing.assert_array_equal(rep.term_weights, [1.0, 1.0])
            assert rep.point_sets[0] is rep.point_sets[1] or np.array_equal(rep.point_sets[0], rep.point_sets[1])
            # StochasticTraining: MEAN terms on the device sampler, weight 1 / N_t / S / N_t S
            st = npde.StochasticTraining(7)
            rep = npde.NNSDERepresentation(prob, npde.NNSDE(ch, npde.Adam(0.1), strategy=st, sub_batch=S,
                                                            strong_loss=strong, batch=batch))
            assert rep.point_sets == [None, None] and rep.sampled == [0, 1]
            assert all(s.reduction == REDUCE_MEAN for s in rep.specs)
            w = {(False, True): 1, (False, False): 7, (True, True): S, (True, False): 7 * S}[(strong, batch)]
            np.testing.assert_array_equal(rep.term_weights, [w, w])
    # Quadrature: one Gauss-Legendre term on the scaled span, z once per node, residual Σ_k r_k^2
    rep = npde.NNSDERepresentation(prob, npde.NNSDE(ch, npde.Adam(0.1)))
    g, w = np.polynomial.legendre.leggauss(16)
    np.testing.assert_allclose(rep.point_sets[0][0], 0.375 * g + 0.625)
    np.testing.assert_allclose(rep.quad_weights[0], 0.375 * w)
    assert rep.term_names == ["quadrature"] and rep.specs[0].scale == 1.0 and rep.training_sets == []


@pytest.mark.parametrize("i", range(len(cases())))
def test_loss_assembly_matches_oracle(i):
    name, prob, alg, rep = make(i)
    orc = NNSDEOracle(prob, alg.chain, param_estim=alg.param_estim)
    theta = rep.flat_init_params
    terms = host_terms(rep, orc, theta)
    total = float(np.dot(rep.term_weights, terms)) + rep.loss_const
    ref = float(oracle_total(rep, orc, theta, alg).detach())
    assert abs(total - ref) <= 1e-12 * abs(ref), (name, total, ref)
    th = torch.tensor(np.asarray(theta, dtype=np.float64))
    tt = "sum" if alg.strong_loss else "mean"
    for k, nm in enumerate(rep.term_names):       # each term against its reference piece
        if nm.startswith("residual"):
            one = NNSDEOracle(prob, alg.chain, param_estim=alg.param_estim)
            Xs = per_time(rep.point_sets[k], alg.sub_batch)
            r2 = [(one.residual(th, X)[int(nm[-1]) - 1] ** 2) for X in Xs]
            red = [(q.mean() if tt == "mean" else q.sum()) for q in r2]
            piece = sum(red) / len(red) if alg.batch else sum(red)
            piece = float(piece.detach())
            assert abs(terms[k] * rep.term_weights[k] - piece) <= 1e-12 * piece, (name, nm)


def test_em_terms_and_constant_em():
    ds = dataset()
    ch = chain(4, 1)
    rep = npde.NNSDERepresentation(gbm_inverse((1.2, 0.3)), npde.NNSDE(ch, npde.Adam(0.1), param_estim=True, dataset=ds),
                                   dt=0.25)
    assert rep.term_names == ["residual_1", "em_1", "em_2"] and rep.loss_const == 0.0
    assert rep.specs[1].taps == [] and rep.specs[1].net_rows is None and rep.point_sets[1].shape == (4, 30)
    orc = NNSDEOracle(rep.prob, ch, param_estim=True)
    th = torch.tensor(np.asarray(rep.flat_init_params))
    em = float(host_terms(rep, orc, rep.flat_init_params)[1:].sum())
    assert abs(em - float(orc.em_loss(th, ds))) <= 1e-12 * em
    # f and g do not read θ.p: both EM terms are constants of the objective
    prob = npde.SDEProblem(lambda u, p, t: 1.5 * u, lambda u, p, t: 0.5 * u, 0.5, (0.0, 1.0), [1.0])
    rep = npde.NNSDERepresentation(prob, npde.NNSDE(ch, npde.Adam(0.1), param_estim=True, dataset=ds), dt=0.25)
    assert rep.term_names == ["residual_1"]
    ref = float(NNSDEOracle(prob, ch, param_estim=True).em_loss(torch.tensor(np.asarray(rep.flat_init_params)), ds))
    assert abs(rep.loss_const - ref) <= 1e-12 * ref
    # only g reads θ.p: the first term is a constant, the second a parameter-only term
    prob = npde.SDEProblem(lambda u, p, t: 1.5 * u, lambda u, p, t: p[0] * u, 0.5, (0.0, 1.0), [0.4])
    rep = npde.NNSDERepresentation(prob, npde.NNSDE(ch, npde.Adam(0.1), param_estim=True, dataset=ds), dt=0.25)
    assert rep.term_names == ["residual_1", "em_2"] and rep.loss_const > 0
    orc = NNSDEOracle(prob, ch, param_estim=True)
    th = np.asarray(rep.flat_init_params)
    total = host_terms(rep, orc, th)[1] + rep.loss_const
    assert abs(total - float(orc.em_loss(torch.tensor(th), ds))) <= 1e-12 * total


def test_fd_and_exact_time_derivative_distance():
    """at θ0 the exact d/dt moves the loss by a relative 1e-12 .. 1e-7 against the reference's forward difference"""
    for i in (0, 1, 2, len(cases()) - 2):
        name, prob, alg, rep = make(i)
        orc = NNSDEOracle(prob, alg.chain, param_estim=alg.param_estim)
        ex = float(oracle_total(rep, orc, rep.flat_init_params, alg).detach())
        fd = float(oracle_total(rep, orc, rep.flat_init_params, alg, derivative="fd").detach())
        assert 1e-13 < abs(ex - fd) / abs(ex) < 1e-6, (name, ex, fd)


def test_kkl_replay_invariants():
    weak = kkl_points(5, 3, 3, 0.2, 1.0, 9, 4, False)
    strong = kkl_points(5, 3, 3, 0.2, 1.0, 9, 4, True)
    np.testing.assert_array_equal(weak[0], strong[0])
    assert np.all((weak[0] >= 0.2) & (weak[0] < 1.0)) and np.all(weak[0].reshape(5, 3) == weak[0][::3, None])
    z = strong[1:].reshape(3, 5, 3)
    assert all(np.array_equal(z[:, i], z[:, 0]) for i in range(5))
    assert not np.array_equal(kkl_points(5, 3, 3, 0.2, 1.0, 9, 5, False), weak)
    big = kkl_points(200, 20, 2, 0.0, 1.0, 1, 0, False)
    assert abs(big[1:].mean()) < 0.05 and abs(big[1:].var() - 1) < 0.05


# ---- refusals ----------------------------------------------------------------------------------------------------
def test_refusals():
    ch = chain(4, 1)
    adam = npde.Adam(0.1)
    with pytest.raises(ValueError, match="out-of-place"):
        npde.SDEProblem(lambda du, u, p, t: None, lambda u, p, t: u, 0.5, (0.0, 1.0))
    with pytest.raises(ValueError, match="complex"):
        npde.SDEProblem(lambda u, p, t: u, lambda u, p, t: u, 0.5 + 1j, (0.0, 1.0))
    with pytest.raises(ValueError, match="complex"):
        npde.SDEProblem(lambda u, p, t: u, lambda u, p, t: u, 0.5, (0.0, 1.0), [1j])
    with pytest.raises(ValueError, match="tspan\\[end\\] = 0"):
        npde.SDEProblem(lambda u, p, t: u, lambda u, p, t: u, 0.5, (-1.0, 0.0))
    for st in (npde.GridTraining(0.1), npde.StochasticTraining(10), npde.WeightedIntervalTraining([1.0], 10)):
        with pytest.raises(ValueError, match="autodiff not supported for %s." % type(st).__name__):
            npde.NNSDERepresentation(gbm(), npde.NNSDE(ch, adam, strategy=st, autodiff=True))
    with pytest.raises(ValueError, match="QuasiRandomTraining is not supported"):
        npde.NNSDERepresentation(gbm(), npde.NNSDE(ch, adam, strategy=npde.QuasiRandomTraining(10)))
    with pytest.raises(ValueError, match="Dataset or an additional loss is required"):
        npde.NNSDERepresentation(gbm_inverse(), npde.NNSDE(ch, adam, param_estim=True), dt=0.1)
    for bad in ([[np.ones(3)]], [np.ones(3), np.ones(3)], [[np.ones(4)], np.linspace(0, 1, 3)]):
        with pytest.raises(ValueError, match="Invalid dataset"):
            npde.NNSDERepresentation(gbm_inverse(), npde.NNSDE(ch, adam, param_estim=True, dataset=bad), dt=0.1)
    with pytest.raises(ValueError, match="scalar process"):
        npde.NNSDERepresentation(vector2(), npde.NNSDE(chain(4, 2), adam, param_estim=True, dataset=dataset()), dt=0.1)
    with pytest.raises(ValueError, match="moment_loss"):
        npde.NNSDE(ch, adam, moment_loss=True)
    with pytest.raises(ValueError, match="closures"):
        npde.NNSDE(ch, adam, additional_loss=lambda phi, th: 0.0)
    with pytest.raises(ValueError, match="tstops"):
        npde.NNSDERepresentation(gbm(), npde.NNSDE(ch, adam), dt=0.1, tstops=[0.5])
    for mode in ("tc_bf16", "tc_split"):
        with pytest.raises(ValueError, match="FFMA kernel"):
            npde.NNSDE(ch, adam, mode=mode)
    with pytest.raises(ValueError, match="sub_batch > 1"):
        npde.NNSDERepresentation(gbm(), npde.NNSDE(ch, adam, sub_batch=2))
    with pytest.raises(ValueError, match="PINN_MAX_DIM"):
        npde.NNSDERepresentation(gbm(), npde.NNSDE(chain(9, 1), adam), dt=0.1)
    with pytest.raises(ValueError, match="1 outputs|needs 1 outputs"):
        npde.NNSDERepresentation(gbm(), npde.NNSDE(chain(4, 2), adam), dt=0.1)
    with pytest.raises(ValueError, match="g returns 1 components, u0 has 2"):
        npde.NNSDERepresentation(npde.SDEProblem(lambda u, p, t: [u[0], u[1]], lambda u, p, t: u[0], [1.0, 1.0],
                                                 (0.0, 1.0)), npde.NNSDE(chain(4, 2), adam), dt=0.1)
    with pytest.raises(ValueError, match="tc_f64"):
        npde.NNSDERepresentation(gbm(), npde.NNSDE(ch, adam, np.zeros(ch.n_params, np.float32), mode="tc_f64"), dt=0.1)
    with pytest.raises(TypeError, match="needs maxiters"):
        npde.solve(gbm(), npde.NNSDE(ch, adam))


# ---- the kernel sources compile ----------------------------------------------------------------------------------
@pytest.mark.skipif(shutil.which("nvcc") is None and not os.path.exists("/usr/local/cuda/bin/nvcc"), reason="no nvcc")
def test_kkl_sampler_and_planner_compile_for_sm90a(tmp_path):
    from neuralpde_jl_b200 import build as B
    for src in ("ffma_launch.cu", "plan.cu", "pinn_abi.cu"):
        r = subprocess.run([B._nvcc(), *B.NVCC_FLAGS, "-c", os.path.join(B.CSRC, src), "-o", str(tmp_path / "x.o")],
                           capture_output=True, text=True)
        assert r.returncode == 0, r.stderr
