"""Tensor-core kernels against the precision model (tests/tc_model.py): the same operation in the same precision, so the
kernels are held to fp32-grade tolerances instead of the bf16 noise of the float64 comparisons (test_gpu_golden.py).

Tolerances (kernel against the model in the same mode):
  loss and every term loss   rel <= 1e-5
  gradient, whole vector     rel L2 <= 5e-4
  gradient, per block        ||d|| <= 2e-3 max(||block||, 1e-3 ||g||), a block = one layer's W, one layer's b, theta.p
  residual probe             max |dr| <= 1e-5 max |r|
Every bound adds 4x the model's noise floor of the same quantity (TcModel.noise_floor: the largest change over 8 draws, 4
at the full shapes, in which every activation moves by 1e-7 and every reverse-sweep adjoint by 1e-7 relative before the
bf16 roundings).  The floor matters where a term's residual is small against its inputs and in deep bf16 networks; it is
what keeps the six-layer wide network's blocks, whose own rounding noise is 1e-3 of their norm, from failing on an
fp32-level change that is not a defect.  Worst measured margins, measured / bound over the whole file, on one NVIDIA
H100 80GB HBM3: loss 0.43, gradient 0.20, block 0.19, residual probe 0.22; cfg 3 at full shape measured loss 2.4e-6,
term losses <= 1.6e-5, gradient 4.7e-5.  The model dominates the file's run time (about 6 minutes, mostly the noise floors
of cfg 3 and cfg 5).  The matrix runs every (n1, n2, pure, activation kind) instantiation of PINN_TC_DISPATCH on both kernels (asserted below, and without a GPU in
test_tc_model.py::test_matrix_covers_every_dispatch_instantiation)."""
import numpy as np
import pytest

import neuralpde_jl_b200 as npde
import tc_cases as TC
import tc_model as M
from cases import FULL_CASES, point_sets
from neuralpde_jl_b200 import pinn

pytestmark = pytest.mark.gpu

LOSS_TOL, GRAD_TOL, BLOCK_TOL, RESID_TOL = 1e-5, 5e-4, 2e-3, 1e-5
FLOOR_DRAWS, FULL_FLOOR_DRAWS = 8, 4     # noise draws of TcModel.noise_floor (full shapes: fewer, the model is slow there)
WORST = {"loss": 0.0, "grad": 0.0, "block": 0.0, "resid": 0.0}
RAISED = {"terms": 0, "terms_of": 0, "grad": 0, "grad_of": 0, "blocks": 0, "blocks_of": 0}   # bounds the floor raised

MATRIX = TC.matrix()
_covered = set()
for _id, _kernel, _build in MATRIX:
    _covered |= TC.capture(_build())[1].model("tw_bf16" if _kernel == "tw" else "tc_bf16").dispatch_keys()
assert _covered == M.NARROW_DISPATCH | M.WIDE_DISPATCH and len(M.NARROW_DISPATCH) == 24 and len(M.WIDE_DISPATCH) == 14


@pytest.fixture(scope="module", autouse=True)
def _report():
    yield
    print("\nworst margins (measured / bound): " + ", ".join("%s %.3f" % kv for kv in WORST.items()))
    print("bounds the noise floor raised by more than 10 %%: term losses %d of %d, gradients %d of %d, blocks %d of %d"
          % tuple(RAISED[k] for k in ("terms", "terms_of", "grad", "grad_of", "blocks", "blocks_of")))


def _note(kind, ratio):
    WORST[kind] = max(WORST[kind], ratio)
    return ratio


def _raised(kind, base, bound):
    RAISED[kind] += int(np.sum(np.asarray(bound) > 1.1 * np.asarray(base)))
    RAISED[kind + "_of"] += np.size(bound)


def run(cfg, mode, sets=None, want_grad=True):
    """(rep, engine, model) of a Config in `mode`; `sets` replaces the point sets of the first terms."""
    with TC.engine_class(M.RecordingEngine):
        rep = pinn.symbolic_discretize(cfg.pde_system, cfg.discretization(dtype=np.float32, mode=mode))
        for i, s in enumerate(sets or []):
            if s is not None:
                rep.set_points(i, *s) if isinstance(s, tuple) else rep.set_points(i, s)
    eng = rep.engine
    model_mode = "tw_bf16" if any(d > 64 for n in eng.spec.nets for d in n.dims[1:-1]) else mode
    return rep, eng, eng.model(model_mode)


def check(cfg, mode, sets=None, theta=None, label="", draws=FLOOR_DRAWS):
    """Loss, term losses, gradient and gradient blocks of the engine against the model.  Every bound is the fp32-grade
    bound plus 4x the model's noise floor (TcModel.noise_floor) of the same quantity."""
    rep, eng, model = run(cfg, mode, sets)
    th = TC.make_theta(cfg) if theta is None else np.asarray(theta, dtype=np.float32)
    total, terms, grad = eng.loss_grad_host(th, None, True)
    res = model.evaluate(th.astype(np.float64))
    fl = model.noise_floor(th.astype(np.float64), draws=draws, want_grad=True, base=res)
    g = res.grad
    gn = np.linalg.norm(g)
    ltol = LOSS_TOL + 4 * fl.total
    ttol = LOSS_TOL + 4 * fl.terms
    gtol = GRAD_TOL + 4 * fl.grad
    lerr = abs(total - res.total) / abs(res.total)
    terr = np.abs(terms - res.terms) / np.abs(res.terms)
    gerr = np.linalg.norm(grad - g) / gn
    blk = {}
    for name, sl in model.blocks():
        base = BLOCK_TOL * max(np.linalg.norm(g[sl]), 1e-3 * gn)
        bound = base + 4 * fl.blocks[name]
        _raised("blocks", base, bound)
        blk[name] = np.linalg.norm(grad[sl] - g[sl]) / bound
    _raised("terms", np.full(len(ttol), LOSS_TOL), ttol)
    _raised("grad", GRAD_TOL, gtol)
    bname = max(blk, key=blk.get)
    print("%s %s: loss %.2e terms %.2e grad %.2e (bound %.2e) worst block %s at %.2f of its bound"
          % (label or cfg.name, mode, lerr, terr.max(), gerr, gtol, bname, blk[bname]))
    assert _note("loss", max(lerr / ltol, np.max(terr / ttol))) <= 1, (lerr, ltol, terr, ttol)
    assert _note("grad", gerr / gtol) <= 1, (gerr, gtol)
    assert _note("block", blk[bname]) <= 1, {k: v for k, v in blk.items() if v > 1}
    return rep, eng, model, th, res, fl


def _modes(kernel):
    return ("tc_bf16", "tc_split") if kernel == "tc" else ("tc_bf16",)


# ---- every dispatch structure x activation kind ----------------------------------------------------------------------------
@pytest.mark.parametrize("case,mode", [(m[0], mode) for m in MATRIX for mode in _modes(m[1])])
def test_dispatch_matrix(case, mode):
    check(dict((m[0], m[2]) for m in MATRIX)[case](), mode, label=case)


# ---- shapes -------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("tl,mode", [(tl, "tc_split") for tl in range(4)] + [(tl, "tc_bf16") for tl in range(4, 7)])
def test_narrow_depth(tl, mode):
    """2-D Poisson (5 channels): 0 to 3 tensor layers with the split weights resident, up to 6 with bf16 weights."""
    check(TC.poisson_depth(tl), mode)


def test_narrow_depth_past_shared_memory_is_refused():
    """Four split tensor layers at 5 channels need more shared memory than an H100 CTA has: a loud error."""
    with pytest.raises(npde.EngineError, match="shared memory per CTA"):
        run(TC.poisson_depth(4), "tc_split")


def test_wide_six_tensor_layers():
    check(TC.wide_deep(), "tc_bf16")


# ---- networks and terms ----------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("mode", ["tc_bf16", "tc_split"])
def test_narrow_two_networks_coupled(mode):
    check(TC.coupled_narrow(), mode)


def test_wide_two_networks_coupled():
    check(TC.coupled_wide(), "tc_bf16")


@pytest.mark.parametrize("width,mode", [(32, "tc_split"), (128, "tc_bf16")])
def test_quadrature_weighted_terms(width, mode):
    check(TC.quadrature(width), mode)


@pytest.mark.parametrize("mode", ["tc_bf16", "tc_split"])
def test_narrow_param_estim_and_data_loss(mode):
    check(TC.heat_param_estim(), mode)


@pytest.mark.parametrize("kernel", ["tc", "tw"])
def test_point_matrix_with_seven_rows(kernel):
    rep, eng, model, th, res, fl = check(TC.many_rows(kernel), "tc_split" if kernel == "tc" else "tc_bf16")
    assert eng.spec.terms[0].dim == 7


@pytest.mark.parametrize("mode", ["tc_bf16", "tc_split"])
def test_narrow_coordinates_lo_in_first_layer_gradient(mode):
    """Every x rounds down to bf16 1.0 here (tc_cases.coords_above_one), so the coordinates' lo enters the first layer's
    weight gradient with one sign.  Without it that block moves by 2.1e-3 of its norm in the model, about the size of the
    generic block bound; this case holds the block to 2e-4 of its norm plus 4x its noise floor."""
    rep, eng, model, th, res, fl = check(TC.coords_above_one(), mode)
    grad = eng.loss_grad_host(th, None, True)[2]
    sl = dict(model.blocks())["net0.W0"]
    err = np.linalg.norm(grad[sl] - res.grad[sl])
    assert _note("block", err / (2e-4 * np.linalg.norm(res.grad[sl]) + 4 * fl.blocks["net0.W0"])) <= 1


@pytest.mark.parametrize("kernel,n", [("tc", n) for n in (1, 127, 128, 129, 1000)] + [("tw", n) for n in (1, 129, 1000)])
def test_point_counts(kernel, n):
    """Partial, exact and multi-tile point counts (1000 = 7 full tiles + 104)."""
    x = np.random.default_rng(n).random((1, n))
    check(TC.point_count(kernel), "tc_split" if kernel == "tc" else "tc_bf16", sets=[x], label="n=%d" % n)


# ---- loss-only calls and the residual probe -----------------------------------------------------------------------------------
@pytest.mark.parametrize("case,mode", [("poisson-tc-tanh", "tc_split"), ("mixed22-tc-generic", "tc_bf16"),
                                       ("burgers-tw-generic", "tc_bf16"), ("poisson-tw-tanh", "tc_bf16")])
def test_loss_only_and_residual_probe(case, mode):
    cfg = dict((m[0], m[2]) for m in MATRIX)[case]()
    rep, eng, model = run(cfg, mode)
    th = TC.make_theta(cfg)
    total, terms, grad = eng.loss_grad_host(th, None, False)
    res = model.evaluate(th.astype(np.float64), want_grad=False)
    fl = model.noise_floor(th.astype(np.float64), draws=FLOOR_DRAWS, base=res)
    ltol, ttol, rfloor = LOSS_TOL + 4 * fl.total, LOSS_TOL + 4 * fl.terms, [4 * r for r in fl.resid]
    assert grad is None
    assert _note("loss", np.max(np.abs(terms - res.terms) / np.abs(res.terms) / ttol)) <= 1
    assert _note("loss", abs(total - res.total) / abs(res.total) / ltol) <= 1
    for t in range(eng.n_terms):
        n = eng.points[t].shape[1]
        r = eng.term_residual_host(t, th, n).astype(np.float64)
        err = np.max(np.abs(r - res.resid[t]))
        bound = RESID_TOL * np.max(np.abs(res.resid[t])) + rfloor[t]
        assert _note("resid", err / bound) <= 1, (t, err, bound)


# ---- the BASELINE shapes ---------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("name,mode", [("cfg2_full", "tc_split"), ("cfg2_full", "tc_bf16"), ("cfg3_full", "tc_bf16"),
                                       ("cfg5_full", "tc_bf16")])
def test_full_shapes(name, mode):
    """cfg 2 at 128^2 / 4x64 on the narrow kernel; cfg 3 (65 536 + 3 x 4 096 points, 5x128: dynamically claimed tiles) and
    cfg 5 (4x128, two passes, data loss, theta.p) on the wide kernel."""
    cfg = FULL_CASES[name]()
    sets, qw, _ = point_sets(cfg)
    theta = cfg.init_params(np.float64, seed=1).astype(np.float32)
    check(cfg, mode, sets=[s if qw is None else (s, qw[i]) for i, s in enumerate(sets)], theta=theta,
          draws=FULL_FLOOR_DRAWS)
