"""The 256-wide tensor-core kernel (csrc/tc_x256_kernel.cu, hidden widths multiples of 64 up to 256) against the precision
model (tests/tc_model.py, tw_bf16 mode: the kernel rounds where the 128-wide kernel does), with the bounds of
test_gpu_tc_model.py: loss and term losses 1e-5, gradient rel L2 5e-4, each W / b block 2e-3 max(||block||, 1e-3 ||g||),
residual probe 1e-5 max |r|, each plus 4x the model's noise floor of the same quantity.  The matrix runs every
(n1, n2, pure, activation kind) instantiation of PINN_TC_DISPATCH in the kernel (asserted below)."""
import numpy as np
import pytest

import neuralpde_jl_b200 as npde
import tc256_cases as X
import tc_cases as TC
import test_gpu_tc_model as G
from cases import FULL_CASES, point_sets
from helpers import engine_eval_sets, rel
from neuralpde_jl_b200 import engine as E
from neuralpde_jl_b200 import pinn

pytestmark = pytest.mark.gpu

MATRIX = X.matrix()
_covered = set()
for _id, _build in MATRIX:
    _covered |= X.x256_keys(TC.capture(_build())[1].model("tw_bf16"))
assert _covered == X.X256_DISPATCH and len(X.X256_DISPATCH) == 14


def check(cfg, draws=16, **kw):
    """test_gpu_tc_model.check in tc_bf16 with twice its noise draws: a 256-wide layer has twice the neurons whose bf16
    rounding an fp32-level difference can flip, and a one-point boundary term sees each flip undiluted."""
    rep, eng, model, th, res, fl = G.check(cfg, "tc_bf16", draws=draws, **kw)
    assert eng.spec.nets and any(d > 128 for n in eng.spec.nets for d in n.dims[1:-1])
    return rep, eng, model, th, res, fl


# ---- every dispatch structure x activation kind ----------------------------------------------------------------------------
@pytest.mark.parametrize("case", [m[0] for m in MATRIX])
def test_dispatch_matrix(case):
    check(dict(MATRIX)[case](), label=case)


# ---- shapes -------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("tl", [1, 2, 3, 4, 5, 6])
def test_depth(tl):
    check(X.burgers_depth(tl))


@pytest.mark.parametrize("widths", [[192, 192, 192], [256, 128, 64, 256], [64, 192, 256, 128]])
def test_widths(widths):
    check(X.burgers_depth(0, widths))


# ---- networks and terms ----------------------------------------------------------------------------------------------------
def test_two_networks_coupled():
    check(X.coupled())


def test_cfg4_four_networks_multi_pass():
    """Config 4 at a small size: four coupled 256-wide networks; the momentum terms (10 taps, 7 channels) run as three
    passes {v, x, xx}, {v, y, yy}, {v, z, zz}."""
    rep, eng, model, th, res, fl = check(X.cfg4_small())
    slots, taps = model.plans[0]
    assert len(slots) == 6 and len(taps) == 10


def test_quadrature_weighted_terms():
    check(X.quadrature())


def test_param_estim_and_data_loss():
    check(X.heat_param_estim())


def test_point_matrix_with_seven_rows():
    rep, eng, model, th, res, fl = check(X.many_rows())
    assert eng.spec.terms[0].dim == 7


@pytest.mark.parametrize("n", [1, 63, 64, 65, 1000])
def test_point_counts(n):
    """Half tiles, partial tiles and the per-element staging path (1000 = 7 full tiles + 104)."""
    x = np.random.default_rng(n).random((1, n))
    check(X.point_count(), sets=[x], label="n=%d" % n)


# ---- loss-only calls and the residual probe -----------------------------------------------------------------------------------
@pytest.mark.parametrize("case", ["burgers-x256-generic", "poisson-x256-tanh"])
def test_loss_only_and_residual_probe(case):
    cfg = dict(MATRIX)[case]()
    rep, eng, model = G.run(cfg, "tc_bf16")
    th = TC.make_theta(cfg)
    total, terms, grad = eng.loss_grad_host(th, None, False)
    res = model.evaluate(th.astype(np.float64), want_grad=False)
    fl = model.noise_floor(th.astype(np.float64), draws=G.FLOOR_DRAWS, base=res)
    ltol, ttol = G.LOSS_TOL + 4 * fl.total, G.LOSS_TOL + 4 * fl.terms
    assert grad is None
    assert np.max(np.abs(terms - res.terms) / np.abs(res.terms) / ttol) <= 1
    assert abs(total - res.total) / abs(res.total) / ltol <= 1
    for t in range(eng.n_terms):
        n = eng.points[t].shape[1]
        r = eng.term_residual_host(t, th, n).astype(np.float64)
        err = np.max(np.abs(r - res.resid[t]))
        bound = G.RESID_TOL * np.max(np.abs(res.resid[t])) + 4 * fl.resid[t]
        assert err <= bound, (t, err, bound)


def test_one_fused_launch_and_one_pack_launch_per_evaluation():
    cfg = X.burgers_depth(2)
    rep, eng, model = G.run(cfg, "tc_bf16")
    th = TC.make_theta(cfg)
    eng.loss_grad_host(th, None, True)
    n0 = eng.launch_count()
    eng.loss_grad_host(th, None, True)
    assert eng.launch_count() - n0 == 2


# ---- refusals ------------------------------------------------------------------------------------------------------------------
def _refused(cfg, mode, match):
    with pytest.raises(npde.EngineError, match=match):
        pinn.symbolic_discretize(cfg.pde_system, cfg.discretization(dtype=np.float32, mode=mode))


def test_tc_split_refuses_256_wide_layers():
    _refused(X.burgers_depth(1), "tc_split", "widths up to 64")


@pytest.mark.parametrize("widths", [[256, 320], [256, 200], [256, 96]])
def test_widths_not_multiples_of_64_up_to_256_are_refused(widths):
    _refused(X.burgers_depth(0, widths), "tc_bf16", "multiple of 64 up to 256")


def test_single_hidden_layer_is_refused():
    _refused(X.burgers_depth(0, [256]), "tc_bf16", "at least one hidden->hidden layer")


def test_seven_tensor_layers_are_refused():
    _refused(X.burgers_depth(7), "tc_bf16", "hidden->hidden layers")


def _many_taps_spec(n_taps):
    """One 2 -> 256 x 2 -> 1 network, one term with 4 channels (u, u_x, u_y, u_xy) and n_taps taps in all (the value tap
    repeated), summed by the program."""
    net = E.NetSpec([2, 256, 256, 1], ["tanh", "tanh", "identity"])
    taps = [E.TapSpec(net=0), E.TapSpec(net=0, order=1, dirs=[0]), E.TapSpec(net=0, order=1, dirs=[1]),
            E.TapSpec(net=0, order=2, dirs=[0, 1])]
    taps += [E.TapSpec(net=0)] * (n_taps - len(taps))
    prog = [("tap", 0, 0, 0.0)]
    for i in range(1, n_taps):
        prog += [("tap", i, 0, 0.0), ("add", len(prog) - 1, len(prog), 0.0)]
    term = E.TermSpec(dim=2, taps=taps, prog=prog, net_rows=[[0, 1]])
    return E.ProblemSpec(nets=[net], terms=[term], n_theta=net.n_params, dtype="float32", mode=E.MODE_TC_BF16)


def test_shared_memory_past_the_limit_is_refused():
    """Four channels fill 128 KB of operand tiles; with 24 taps the per-point tap arrays no longer fit next to them."""
    with pytest.raises(npde.EngineError, match="shared memory per CTA.*too many channels or taps for the 256-wide"):
        E.Engine(_many_taps_spec(24))


def test_float64_is_refused():
    cfg = X.burgers_depth(1)
    with pytest.raises(npde.EngineError, match="PINN_F32"):
        pinn.symbolic_discretize(cfg.pde_system, cfg.discretization(dtype=np.float64, mode="tc_bf16"))


# ---- the BASELINE shape ------------------------------------------------------------------------------------------------------
def test_cfg4_w256_matches_oracle():
    """Config 4 at 256 wide (4 networks, quadrature weights) against the committed float64 golden, at the tc_bf16
    tolerances of DESIGN section 3 (loss 1e-2, gradient 2e-2)."""
    g, cfg, theta, sets, qw = __import__("test_gpu_golden")._full("cfg4_w256")
    rep, total, terms, grad = engine_eval_sets(cfg, np.float32, sets, qw, mode="tc_bf16", theta=theta)
    L = float(g["total"])
    err, gerr = abs(total - L) / abs(L), rel(grad, g["grad"])
    print("cfg4_w256 tc_bf16: loss rel %.3e grad rel %.3e" % (err, gerr))
    assert err <= 1e-2, (total, L)
    np.testing.assert_allclose(terms, g["terms"], rtol=1e-1, atol=1e-12)
    assert gerr < 2e-2


def test_cfg4_w256_against_the_model():
    cfg = FULL_CASES["cfg4_w256"]()
    sets, qw, _ = point_sets(cfg)
    theta = cfg.init_params(np.float64, seed=1).astype(np.float32)
    check(cfg, sets=[s if qw is None else (s, qw[i]) for i, s in enumerate(sets)], theta=theta, draws=G.FULL_FLOOR_DRAWS)


# ---- two ranks ---------------------------------------------------------------------------------------------------------------
@pytest.mark.skipif(__import__("torch").cuda.device_count() < 2, reason="needs 2 GPUs")
def test_two_ranks_reproduce_one_rank(tmp_path):
    import os
    import subprocess
    import sys
    import socket
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    out = str(tmp_path / "r0.npz")
    with socket.socket() as sk:          # a port nothing else on the host is using
        sk.bind(("127.0.0.1", 0))
        port = sk.getsockname()[1]
    cmd = [sys.executable, "-m", "torch.distributed.run", "--nnodes=1", "--nproc-per-node", "2", "--master-addr",
           "127.0.0.1", "--master-port", str(port), os.path.join(root, "tests", "tc256_mgpu_worker.py"), out]
    r = subprocess.run(cmd, capture_output=True, text=True, timeout=600)
    assert r.returncode == 0, r.stderr[-2000:]
    res = np.load(out)
    cfg = X.cfg4_small()
    rep = pinn.symbolic_discretize(cfg.pde_system, cfg.discretization(dtype=np.float32, mode="tc_bf16"))
    tot, terms, g = rep.engine.loss_grad_host(TC.make_theta(cfg), None, True)
    assert abs(float(res["tot"]) - tot) <= 2e-6 * abs(tot)
    np.testing.assert_allclose(res["terms"], terms, rtol=2e-6)
    assert rel(res["g"], g) < 2e-6
