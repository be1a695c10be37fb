"""GPU parity against the committed golden vectors (float64 oracle) for every case: multi-network
systems, parameter estimation + data loss, quadrature weights, mixed derivatives, Neumann conditions,
non-tanh activations.  All calls go through the C ABI."""
import numpy as np
import pytest

import neuralpde_jl_b200 as npde
from cases import CASES
from helpers import engine_eval_sets, load_golden, rel

pytestmark = pytest.mark.gpu


@pytest.mark.parametrize("name", sorted(CASES))
def test_ffma_fp64_matches_golden(name):
    g, sets, qw = load_golden(name)
    rep, total, terms, grad = engine_eval_sets(CASES[name](), np.float64, sets, qw, theta=g["theta"])
    assert abs(total - float(g["total"])) <= 1e-10 * abs(float(g["total"]))
    np.testing.assert_allclose(terms, g["terms"], rtol=1e-9, atol=1e-300)
    assert rel(grad, g["grad"]) < 1e-9


@pytest.mark.parametrize("name", sorted(CASES))
def test_ffma_fp32_loss_rtol_1e5(name):
    g, sets, qw = load_golden(name)
    rep, total, terms, grad = engine_eval_sets(CASES[name](), np.float32, sets, qw, theta=g["theta"])
    assert abs(total - float(g["total"])) <= 1e-5 * abs(float(g["total"]))
    assert rel(grad, g["grad"]) < 5e-4
    # and against the reference's finite-difference semantics in float64
    assert abs(total - float(g["total_fd"])) <= 1e-5 * abs(float(g["total_fd"]))


TC_CASES = ["cfg1", "cfg2_small", "cfg3_small", "neumann_sin"]


@pytest.mark.parametrize("name", TC_CASES)
def test_tc_split_loss_rtol_1e5(name):
    """tensor-core path, forward operands split hi+lo (3 MMAs per product): loss rtol 1e-5 (north star); the reverse
    sweep uses bf16 operands, gradient relative L2 error stated at 1e-2."""
    g, sets, qw = load_golden(name)
    rep, total, terms, grad = engine_eval_sets(CASES[name](), np.float32, sets, qw, mode="tc_split", theta=g["theta"])
    assert abs(total - float(g["total"])) <= 1e-5 * abs(float(g["total"])), (total, float(g["total"]))
    assert rel(grad, g["grad"]) < 1e-2


@pytest.mark.parametrize("name", TC_CASES)
def test_tc_bf16_loss_rtol_1e2(name):
    """plain bf16 operands: BASELINE.md section 3 measured 1.3e-3 on config 2; stated tolerance 1e-2 / 2e-2."""
    g, sets, qw = load_golden(name)
    rep, total, terms, grad = engine_eval_sets(CASES[name](), np.float32, sets, qw, mode="tc_bf16", theta=g["theta"])
    assert abs(total - float(g["total"])) <= 1e-2 * abs(float(g["total"]))
    assert rel(grad, g["grad"]) < 2e-2


WIDE_CASES = ["burgers_wide", "poisson1d_wide", "cfg5_wide"]     # cfg5_wide: 6 channels -> two passes over the network


@pytest.mark.parametrize("name", WIDE_CASES)
def test_tc_wide_bf16_loss_rtol_1e2(name):
    """128-wide layers on the tensor-core path (bf16 operands, streamed weights, fp32 pre-activation stash; BASELINE config 3
    names this mode): same stated tolerance as the narrow bf16 mode, loss 1e-2 / gradient 2e-2."""
    g, sets, qw = load_golden(name)
    rep, total, terms, grad = engine_eval_sets(CASES[name](), np.float32, sets, qw, mode="tc_bf16", theta=g["theta"])
    assert abs(total - float(g["total"])) <= 1e-2 * abs(float(g["total"])), (total, float(g["total"]))
    np.testing.assert_allclose(terms, g["terms"], rtol=2e-2)
    assert rel(grad, g["grad"]) < 2e-2


@pytest.mark.parametrize("name", WIDE_CASES)
def test_tc_wide_loss_only_and_residual_probe(name):
    """loss-only evaluation (no gradient, no stash) and the per-point residual probe on the wide path"""
    g, sets, qw = load_golden(name)
    cfg = CASES[name]()
    rep, total, terms, grad = engine_eval_sets(cfg, np.float32, sets, qw, mode="tc_bf16", theta=g["theta"], want_grad=False)
    assert grad is None
    assert abs(total - float(g["total"])) <= 1e-2 * abs(float(g["total"]))
    r = rep.engine.term_residual_host(0, np.asarray(g["theta"], dtype=np.float32), sets[0].shape[1])
    assert r.shape == (sets[0].shape[1],) and np.isfinite(r).all()
    assert abs(float(np.mean(r.astype(np.float64) ** 2)) - float(g["terms"][0])) <= 2e-2 * float(g["terms"][0])


def test_tc_split_rejects_wide_layers_loudly():
    g, sets, qw = load_golden("burgers_wide")
    with pytest.raises(npde.EngineError, match="widths up to 64"):
        engine_eval_sets(CASES["burgers_wide"](), np.float32, sets, qw, mode="tc_split", theta=g["theta"])


@pytest.mark.parametrize("name", ["mixed", "cfg4_tiny", "cfg5_small"])
def test_tc_rejects_unsupported_shapes_loudly(name):
    """More than 5 propagated channels per network: the tensor-core path refuses (no silent fallback)."""
    g, sets, qw = load_golden(name)
    with pytest.raises(npde.EngineError, match="channels|taps"):
        engine_eval_sets(CASES[name](), np.float32, sets, qw, mode="tc_split", theta=g["theta"])


def test_param_estim_gradient_entry():
    """theta.p sits at the end of theta (reference src/discretize.jl:464); its gradient comes from the residual program."""
    g, sets, qw = load_golden("cfg5_small")
    rep, total, terms, grad = engine_eval_sets(CASES["cfg5_small"](), np.float64, sets, qw, theta=g["theta"])
    assert abs(grad[-1] - g["grad"][-1]) <= 1e-9 * abs(g["grad"][-1]) and abs(g["grad"][-1]) > 0
    assert len(terms) == len(g["terms"]) == 1 + 5 + 1          # pde + 5 bcs + data loss


# ---- the shapes BASELINE.json names (tests/golden/make_golden_full.py) -------------------------------------------------------
from cases import FULL_CASES, point_sets      # noqa: E402


def _full(name):
    import hashlib
    g = np.load(__import__("os").path.join(__import__("os").path.dirname(__import__("os").path.abspath(__file__)), "golden", name + ".npz"))
    cfg = FULL_CASES[name]()
    theta = cfg.init_params(np.float64, seed=1)
    sets, qw, qs = point_sets(cfg)
    sha = lambda a: hashlib.sha256(np.ascontiguousarray(a, dtype=np.float64).tobytes()).hexdigest()      # noqa: E731
    assert sha(theta) == str(g["theta_sha"]) and sha(sets[0]) == str(g["set0_sha"]), "regenerated inputs differ from the golden's"
    return g, cfg, theta, sets, qw


@pytest.mark.parametrize("name,mode,ltol,gtol", [
    ("cfg2_full", "tc_split", 1e-5, 1e-2),     # the headline kernel at the headline shape: 128^2 + 4 x 128 points, 4x64
    ("cfg2_full", "tc_bf16", 1e-2, 2e-2),
    ("cfg2_full", "ffma", 1e-5, 5e-4),
    ("cfg3_full", "tc_bf16", 1e-2, 2e-2),      # 128-wide kernel, 65 536 + 3 x 4 096 points, 5x128: 608 dynamically claimed tiles
    ("cfg3_full", "ffma", 1e-5, 5e-4),
    ("cfg5_full", "tc_bf16", 1e-2, 2e-2),      # 4x128, 6 channels -> two passes, data loss + theta.p, 65 536 points
    ("cfg5_full", "ffma", 1e-5, 5e-4),
    ("cfg4_w256", "ffma", 1e-5, 5e-4),         # 4 coupled networks, 256-wide layers, 7 channels, quadrature weights
])
def test_full_shape_matches_oracle(name, mode, ltol, gtol):
    """Loss, per-term losses and gradient against the float64 oracle at the shapes BASELINE.json names.  Stated tolerances:
    FFMA fp32 loss 1e-5 / gradient 5e-4; tc_split loss 1e-5 / gradient 1e-2 (its reverse sweep uses bf16 operands);
    tc_bf16 loss 1e-2 / gradient 2e-2."""
    g, cfg, theta, sets, qw = _full(name)
    rep, total, terms, grad = engine_eval_sets(cfg, np.float32, sets, qw, mode=mode, theta=theta)
    L = float(g["total"])
    err, gerr = abs(total - L) / abs(L), rel(grad, g["grad"])
    print("%s %s: loss rel %.3e grad rel %.3e" % (name, mode, err, gerr))
    assert err <= ltol, (total, L)
    np.testing.assert_allclose(terms, g["terms"], rtol=max(10 * ltol, 1e-4), atol=1e-12)
    assert gerr < gtol
