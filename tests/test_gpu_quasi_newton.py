"""Device-resident BFGS / L-BFGS (pinn_qn_*, npde.BFGS / npde.LBFGS): trajectory parity with the float64 oracle
(tests/qn_oracle.py, two-loop L-BFGS and dense BFGS), descent in fp32 and tensor-core modes, bit-reproducibility, the
reference's BFGS solves through npde.solve, the refusals, and the replicated multi-GPU run."""
import os
import subprocess
import sys

import numpy as np
import pytest
import torch

import neuralpde_jl_b200 as npde
from neuralpde_jl_b200 import configs, engine as E
from helpers import oracle_eval, rel
import qn_oracle as Q

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
LS = {"hagerzhang": E.LS_HAGERZHANG, "backtracking": E.LS_BACKTRACKING}


def _rep(cfg, dtype=np.float64, mode="ffma"):
    return npde.symbolic_discretize(cfg.pde_system, cfg.discretization(dtype=dtype, mode=mode))


def _engine_trajectory(rep, method, ls, iters, m=5):
    eng = rep.engine
    kind = E.QN_LBFGS if method == "lbfgs" else E.QN_BFGS
    eng.qn_begin(rep.flat_init_params, kind, m=m, linesearch=LS[ls])
    f0, _, _, _, ev0 = eng.qn_iterate(0)
    out = []
    for _ in range(iters):
        f, gn, status, it, ev = eng.qn_iterate(1)
        if it == len(out):
            break
        out.append((eng.qn_theta().astype(np.float64), f, ev))
        if status != E.QN_RUNNING:
            break
    return f0, ev0, out, status


@pytest.mark.parametrize("method,ls", [("lbfgs", "hagerzhang"), ("lbfgs", "backtracking"), ("bfgs", "hagerzhang"),
                                       ("bfgs", "backtracking")])
@pytest.mark.parametrize("cfg_name", ["cfg1", "cfg2_small"])
def test_trajectory_matches_float64_oracle(cfg_name, method, ls):
    cfg = configs.config1() if cfg_name == "cfg1" else configs.config2(n=16, width=16, hidden=3)
    rep = _rep(cfg)
    sets = [rep.point_sets[i] for i in range(len(rep.point_sets))]
    f0, ev0, traj, status = _engine_trajectory(rep, method, ls, 15)
    fg = lambda th: oracle_eval(cfg, th, "exact", sets)[0::2]          # noqa: E731  (loss, grad)
    res = Q.minimize(fg, rep.flat_init_params.astype(np.float64), method=method, m=5, linesearch=ls, maxiters=15)
    assert ev0 == 1 and abs(f0 - fg(rep.flat_init_params)[0]) <= 1e-12 * abs(f0)
    assert len(traj) == len(res.history), (len(traj), len(res.history), res.retcode)
    assert len(traj) >= 5
    for k, ((th_e, f_e, ev_e), (th_o, f_o, ev_o)) in enumerate(zip(traj, res.history)):
        assert rel(th_e, th_o) <= 1e-7, (k, rel(th_e, th_o))
        assert abs(f_e - f_o) <= 1e-9 * abs(f_o), (k, f_e, f_o)
        assert ev_e == ev_o, (k, ev_e, ev_o)
    assert traj[-1][1] < f0


@pytest.mark.parametrize("ls", ["hagerzhang", "backtracking"])
def test_fp32_lbfgs_descends_on_its_own_loss(ls):
    rep = _rep(configs.config2(n=32, width=32, hidden=3), np.float32)
    eng = rep.engine
    eng.qn_begin(rep.flat_init_params, E.QN_LBFGS, linesearch=LS[ls])
    f_prev = eng.qn_iterate(0)[0]
    f_start = f_prev
    for _ in range(50):
        f, gn, status, it, ev = eng.qn_iterate(1)
        # an accepted step meets Armijo (BackTracking) or Wolfe / approximate Wolfe (HagerZhang, phi <= phi0 + 1e-6 |phi0|)
        assert f <= f_prev + (0.0 if ls == "backtracking" else 1e-6 * abs(f_prev)), (it, f, f_prev)
        f_prev = f
        if status != E.QN_RUNNING:
            break
    assert np.isfinite(f_prev) and f_prev < 0.5 * f_start
    # tc_split: 20 iterations end finite and below the start
    rep_t = _rep(configs.config2(n=32, width=32, hidden=3), np.float32, "tc_split")
    rep_t.engine.qn_begin(rep_t.flat_init_params, E.QN_LBFGS, linesearch=LS[ls])
    f0 = rep_t.engine.qn_iterate(0)[0]
    f, _, status, it, _ = rep_t.engine.qn_iterate(20)
    assert np.isfinite(f) and f < f0 and status != E.QN_LS_FAILED, (f, f0, status, it)
    assert np.all(np.isfinite(rep_t.engine.qn_theta()))


@pytest.mark.parametrize("dtype,method", [(np.float64, "lbfgs"), (np.float32, "lbfgs"), (np.float64, "bfgs")])
def test_two_runs_are_bit_identical(dtype, method):
    cfg = configs.config2(n=24, width=16, hidden=3)
    runs = []
    for _ in range(2):
        rep = _rep(cfg, dtype)
        rep.engine.qn_begin(rep.flat_init_params, E.QN_LBFGS if method == "lbfgs" else E.QN_BFGS)
        f, _, _, it, ev = rep.engine.qn_iterate(12)
        runs.append((rep.engine.qn_theta(), f, it, ev))
    assert np.array_equal(runs[0][0], runs[1][0]) and runs[0][1:] == runs[1][1:]


def test_third_order_ode_with_bfgs_as_the_reference_states_it():
    """reference test/NNPDE1/nnpde__pde_iii_3rd_order_ode.jl:54-130 with the reference's optimizer, BFGS(), through
    npde.solve: the same system, chains and bounds as the scipy-driven test in test_gpu_properties.py."""
    import sympy as sp
    x = npde.parameters("x")
    u, Dxu, Dxxu, O1, O2 = npde.variables("u Dxu Dxxu O1 O2")
    Dx = npde.Differential(x)
    eq = npde.Eq(Dx(Dxxu(x)), sp.cos(sp.pi * x))
    ep = float(np.cbrt(np.finfo(np.float64).eps)) ** 2 / 6
    bcs = [npde.Eq(u(0.0), 0.0), npde.Eq(u(1.0), -1.0), npde.Eq(Dxu(1.0), 1.0),
           npde.Eq(Dxu(x), Dx(u(x)) + ep * O1(x)), npde.Eq(Dxxu(x), Dx(Dxu(x)) + ep * O2(x))]
    sys_ = npde.PDESystem(eq, bcs, [npde.In(x, 0.0, 1.0)], [x], [u(x), Dxu(x), Dxxu(x), O1(x), O2(x)])
    chains = [npde.Chain(npde.Dense(1, 12, "tanh"), npde.Dense(12, 12, "tanh"), npde.Dense(12, 1)) for _ in range(3)] + \
             [npde.Chain(npde.Dense(1, 4, "tanh"), npde.Dense(4, 1)) for _ in range(2)]
    rng = np.random.default_rng(100)
    theta0 = np.concatenate([npde.initialparameters(rng, c, np.float64) for c in chains])
    strategy = npde.QuasiRandomTraining(100, resampling=False, minibatch=1, seed=7)
    prob = npde.discretize(sys_, npde.PhysicsInformedNN(chains, strategy, init_params=theta0))
    res = npde.solve(prob, npde.BFGS(), maxiters=2000)
    xs = np.arange(0.0, 1.0001, 0.01)
    analytic = (np.pi * xs * (-xs + np.pi ** 2 * (2 * xs - 3) + 1) - np.sin(np.pi * xs)) / np.pi ** 3
    pred = prob.representation.phi[0](xs.reshape(1, -1), res.u)[0]
    print("3rd-order ODE system, device BFGS: loss %.3e after %d iterations (%s), max |u - analytic| %.2e"
          % (res.objective, res.iterations, res.retcode, np.max(np.abs(pred - analytic))))
    assert res.objective < 1e-6, (res.objective, res.retcode)
    np.testing.assert_allclose(pred, analytic, atol=1e-4)


@pytest.mark.parametrize("kind", ["grid", "stochastic"])
def test_2d_poisson_with_the_reference_bfgs_polish(kind):
    """reference test/NNPDE1/nnpde__pde_ii_2d_poisson.jl:57-97: Adam(0.01) for 1000 iterations, then
    BFGS(linesearch = BackTracking()) for 1000, `u_predict ≈ u_real atol = 2.0` on the 101 x 101 lattice (norm-wise)."""
    import sympy as sp
    x, y = npde.parameters("x y")
    u = npde.variables("u")
    eq = npde.Eq((npde.Differential(x) ** 2)(u(x, y)) + (npde.Differential(y) ** 2)(u(x, y)), -sp.sin(sp.pi * x) * sp.sin(sp.pi * y))
    bcs = [npde.Eq(u(0, y), 0.0), npde.Eq(u(1, y), 0.0), npde.Eq(u(x, 0), 0.0), npde.Eq(u(x, 1), 0.0)]
    sys_ = npde.PDESystem(eq, bcs, [npde.In(x, 0.0, 1.0), npde.In(y, 0.0, 1.0)], [x, y], [u(x, y)])
    chain = npde.Chain(npde.Dense(2, 12, "sigmoid"), npde.Dense(12, 12, "sigmoid"), npde.Dense(12, 1))
    strategy = npde.GridTraining(0.1) if kind == "grid" else npde.StochasticTraining(100, bcs_points=50, seed=1)
    if kind != "grid":
        strategy.device_sampler = True
    theta0 = npde.initialparameters(np.random.default_rng(0), chain, np.float64)
    prob = npde.discretize(sys_, npde.PhysicsInformedNN(chain, strategy, init_params=theta0))
    res = npde.solve(prob, npde.Adam(0.01), maxiters=1000, device_loop=True, chunk=250)
    adam_loss = prob.f.f(res.u, None) if kind == "grid" else None
    prob.u0 = res.u
    res2 = npde.solve(prob, npde.BFGS(linesearch=npde.BackTracking()), maxiters=1000)
    xs = np.arange(0.0, 1.0001, 0.01)
    X, Y = np.meshgrid(xs, xs, indexing="ij")
    pred = prob.representation.phi(np.stack([X.ravel(), Y.ravel()]), res2.u)[0]
    real = np.sin(np.pi * X.ravel()) * np.sin(np.pi * Y.ravel()) / (2 * np.pi ** 2)
    err = float(np.linalg.norm(pred - real))
    print("2-D Poisson (%s) + BFGS(BackTracking) polish: loss %.3e after %d iterations (%s), ||u_predict - u_real|| = %.3f"
          % (kind, res2.objective, res2.iterations, res2.retcode, err))
    assert err < 2.0 and np.isfinite(res2.objective)
    if kind == "grid":
        assert res2.objective <= adam_loss


def test_callback_sees_every_iteration_and_can_halt():
    cfg = configs.config2(n=16, width=16, hidden=3)
    prob = npde.discretize(cfg.pde_system, cfg.discretization(dtype=np.float64))
    seen = []
    res = npde.solve(prob, npde.LBFGS(), maxiters=20, callback=lambda st, l: seen.append((st["iter"], l)) or st["iter"] == 4)
    assert [s[0] for s in seen] == [1, 2, 3, 4] and res.iterations == 4 and res.retcode == "Terminated"
    assert res.objective == seen[-1][1]
    prob2 = npde.discretize(cfg.pde_system, cfg.discretization(dtype=np.float64))
    res2 = npde.solve(prob2, npde.LBFGS(), maxiters=4)
    assert res2.retcode == "MaxIters" and np.array_equal(res2.u, res.u) and res2.objective == res.objective


def test_refusals_name_the_problem():
    cfg_big = configs.config2(n=8, width=128, hidden=5)
    big = _rep(cfg_big, np.float32)
    assert big.engine.n_theta > 16384
    with pytest.raises(npde.EngineError, match="call pinn_qn_begin first"):
        big.engine.qn_iterate(1)
    with pytest.raises(npde.EngineError, match="exceeds 16384.*use L-BFGS"):
        big.engine.qn_begin(big.flat_init_params, E.QN_BFGS)
    prob = npde.discretize(cfg_big.pde_system, cfg_big.discretization(dtype=np.float32))
    with pytest.raises(npde.EngineError, match="use L-BFGS"):
        npde.solve(prob, npde.BFGS(), maxiters=1)
    cfg = configs.config2(n=16, width=16, hidden=2)
    prob_a = npde.discretize(cfg.pde_system, cfg.discretization(adaptive_loss=npde.SoftAdaptAdaptiveLoss(10)))
    with pytest.raises(ValueError, match="NonAdaptiveLoss"):
        npde.solve(prob_a, npde.LBFGS(), maxiters=2)
    cfg3 = configs.config3(points=256, bcs_points=32, width=16, hidden=2)
    prob_s = npde.discretize(cfg3.pde_system, cfg3.discretization(dtype=np.float32))
    with pytest.raises(ValueError, match="point sets that live on the device"):
        npde.solve(prob_s, npde.BFGS(), maxiters=2)
    with pytest.raises(ValueError, match="default parameters"):
        npde.solve(npde.discretize(cfg.pde_system, cfg.discretization()), npde.LBFGS(linesearch=npde.HagerZhang(sigma=0.5)))


def test_device_sampled_lbfgs_draws_every_evaluation():
    cfg = configs.config3(points=1000, bcs_points=100, width=16, hidden=2)
    cfg.strategy.device_sampler = True
    rep = _rep(cfg)
    eng = rep.engine
    pts0 = eng.get_points_host(0, 1000)
    eng.qn_begin(rep.flat_init_params, E.QN_LBFGS)
    f, _, status, it, ev = eng.qn_iterate(5)
    assert not np.array_equal(eng.get_points_host(0, 1000), pts0)
    assert np.isfinite(f) and it >= 1 and ev > it


@pytest.mark.skipif(torch.cuda.device_count() < 2, reason="needs 2 GPUs")
@pytest.mark.parametrize("path", ["p2p", "nccl"])
def test_two_rank_lbfgs_is_replicated_and_matches_one_rank(tmp_path, path):
    out = str(tmp_path / "qn.npz")
    cmd = [sys.executable, "-m", "torch.distributed.run", "--nnodes=1", "--nproc-per-node", "2", "--master-addr", "127.0.0.1",
           "--master-port", "29563", os.path.join(ROOT, "tests", "qn_mgpu_worker.py"), out]
    env = dict(os.environ)
    if path == "nccl":
        env["PINN_B200_NO_P2P"] = "1"
    r = subprocess.run(cmd, capture_output=True, text=True, timeout=300, env=env)
    assert r.returncode == 0, r.stderr[-2000:]
    res = np.load(out)
    assert int(res["fused"]) == (1 if path == "p2p" else 0)
    rep = _rep(configs.config2(n=48, width=32, hidden=3))
    rep.engine.qn_begin(rep.flat_init_params, E.QN_LBFGS)
    f, _, _, it, ev = rep.engine.qn_iterate(10)
    assert int(res["it"]) == it and int(res["ev"]) == ev
    assert rel(res["theta"], rep.engine.qn_theta()) <= 1e-8
