"""The precision model of the tensor-core kernels (tests/tc_model.py), checked without a GPU: its bf16 rounding, its
`exact` mode against the float64 oracle, the size of its rounding error against DESIGN section 9's measurement, and the
coverage of the dispatch matrix the GPU tests run (tests/test_gpu_tc_model.py)."""
import numpy as np
import pytest
import torch

import tc_cases as TC
import tc_model as M
from cases import CASES, FULL_CASES, point_sets
from helpers import oracle_eval, rel


# ---- bf16 ---------------------------------------------------------------------------------------------------------
def test_bf16_matches_torch_conversion():
    rng = np.random.default_rng(0)
    v = np.concatenate([rng.standard_normal(20000) * 10.0 ** rng.integers(-8, 8, 20000), [0.0, -0.0, 1.0, -3.5]])
    v32 = v.astype(np.float32)
    want = torch.tensor(v32).to(torch.bfloat16).to(torch.float64).numpy()
    np.testing.assert_array_equal(M.bf16(v32), want)


def test_bf16_rounds_ties_to_even():
    # 1 + 2^-8 lies halfway between bf16 1 and 1 + 2^-7: even mantissa (1) wins; 1 + 3 * 2^-8 rounds up to 1 + 2^-6
    assert M.bf16(1 + 2.0 ** -8) == 1.0
    assert M.bf16(1 + 3 * 2.0 ** -8) == 1 + 2.0 ** -6
    assert M.bf16(-(1 + 2.0 ** -8)) == -1.0
    assert M.bf16(1 + 2.0 ** -8 + 2.0 ** -20) == 1 + 2.0 ** -7          # above the tie: up


def test_split_reconstructs_to_2e_17():
    v = np.random.default_rng(1).standard_normal(100000).astype(np.float32).astype(np.float64)
    hi, lo = M.split(v)
    assert np.all(np.abs(hi + lo - v) <= 2.0 ** -17 * np.abs(v))
    assert np.array_equal(hi, M.bf16(v)) and np.array_equal(lo, M.bf16(v - hi))


# ---- exact mode against the float64 oracle ---------------------------------------------------------------------------
ORDER2_CASES = sorted(n for n in CASES if not n.startswith("third_order"))
MATRIX = TC.matrix()
EXTRA = {"coords_above_one": TC.coords_above_one, "coupled_narrow": TC.coupled_narrow, "coupled_wide": TC.coupled_wide,
         "quadrature": TC.quadrature, "heat_param_estim": TC.heat_param_estim, "many_rows_tc": TC.many_rows, "wide_deep": TC.wide_deep,
         "poisson_tl0": lambda: TC.poisson_depth(0), "poisson_tl6": lambda: TC.poisson_depth(6)}


def _exact_vs_oracle(cfg):
    rep, rec = TC.capture(cfg, mode="ffma", dtype=np.float64)
    rep.resample()                          # Stochastic / QuasiRandom strategies upload their points here
    n_pde, n_bc = len(cfg.pde_system.eqs), len(cfg.pde_system.bcs)
    sets = [np.asarray(rep.point_sets[i], dtype=np.float64) for i in range(n_pde + n_bc)]
    quad = None
    if any(w is not None for w in rep.quad_weights[:n_pde + n_bc]):
        quad = (rep.quad_weights[:n_pde + n_bc], [rec.spec.terms[i].scale for i in range(n_pde + n_bc)])
    theta = TC.make_theta(cfg).astype(np.float64)
    L, T, G = oracle_eval(cfg, theta, "exact", sets, quad)
    res = rec.model("exact").evaluate(theta)
    assert abs(res.total - L) <= 1e-12 * abs(L), (res.total, L)
    np.testing.assert_allclose(res.terms, T, rtol=1e-12, atol=1e-300)
    assert rel(res.grad, G) <= 1e-11, rel(res.grad, G)


@pytest.mark.parametrize("name", ORDER2_CASES)
def test_exact_model_matches_oracle_cases(name):
    _exact_vs_oracle(CASES[name]())


@pytest.mark.parametrize("name", [m[0] for m in MATRIX] + sorted(EXTRA))
def test_exact_model_matches_oracle_matrix(name):
    cfg = dict((m[0], m[2]) for m in MATRIX)[name]() if name in dict((m[0], m[2]) for m in MATRIX) else EXTRA[name]()
    _exact_vs_oracle(cfg)


# ---- coverage of the GPU matrix ---------------------------------------------------------------------------------------
def test_matrix_covers_every_dispatch_instantiation():
    got = set()
    for _, kernel, build in MATRIX:
        rep, rec = TC.capture(build(), mode="tc_bf16")
        got |= rec.model("tw_bf16" if kernel == "tw" else "tc_bf16").dispatch_keys()
    assert len(M.NARROW_DISPATCH) == 24 and len(M.WIDE_DISPATCH) == 14
    assert got == M.NARROW_DISPATCH | M.WIDE_DISPATCH, (sorted(M.NARROW_DISPATCH | M.WIDE_DISPATCH - got), sorted(got - M.NARROW_DISPATCH - M.WIDE_DISPATCH))


def test_noise_floor_of_a_deep_bf16_network():
    """With six bf16 tensor layers, 1e-7 of activation noise (the accuracy of the kernels' approximate tanh) flips enough
    roundings to move a boundary term by 7e-3 relative: the floor the GPU tests add to their fp32-grade bound."""
    cfg = TC.poisson_depth(6)
    rep, rec = TC.capture(cfg)
    model = rec.model("tc_bf16")
    th = TC.make_theta(cfg).astype(np.float64)
    fl = model.noise_floor(th, draws=8, want_grad=True)
    assert fl.terms.max() > 1e-3 and len(fl.resid) == len(fl.terms) and fl.grad > 0
    assert set(fl.blocks) == {name for name, _ in model.blocks()}
    fl0 = model.noise_floor(th, eps=0.0, want_grad=True)
    assert fl0.total == 0 and not fl0.terms.any() and not any(fl0.resid) and fl0.grad == 0 and not any(fl0.blocks.values())


def test_coordinates_above_one_all_round_down():
    """The case for the coordinates' lo: every x rounds to bf16 1.0 and leaves a positive lo at every point."""
    rep, rec = TC.capture(TC.coords_above_one(), mode="tc_split")
    x = rec.points[0][0].astype(np.float64)
    hi, lo = M.split(x)
    assert np.all(hi == 1.0) and np.all(lo > 2.0 ** -10)


# ---- the rounded model's error is the size the kernel's is ----------------------------------------------------------------
def test_split_model_error_matches_design_measurement():
    """cfg 2 at 128^2 / 4x64 in tc_split: DESIGN section 9 measured the kernel against float64 at loss 5.7e-6, gradient
    2.1e-3.  The model, which rounds where the kernel rounds, must show errors of that size (within a factor of 3)."""
    cfg = FULL_CASES["cfg2_full"]()
    sets, _, _ = point_sets(cfg)
    theta = cfg.init_params(np.float64, seed=1).astype(np.float32).astype(np.float64)
    rep, rec = TC.capture(cfg, mode="tc_split")
    for i, s in enumerate(sets):
        rep.set_points(i, s)
    L, T, G = oracle_eval(cfg, theta, "exact", sets, None)
    res = rec.model("tc_split").evaluate(theta)
    err, gerr = abs(res.total - L) / abs(L), rel(res.grad, G)
    print("cfg2_full tc_split model vs float64: loss %.2e gradient %.2e" % (err, gerr))
    assert 5.7e-6 / 3 <= err <= 5.7e-6 * 3
    assert 2.1e-3 / 3 <= gerr <= 2.1e-3 * 3
