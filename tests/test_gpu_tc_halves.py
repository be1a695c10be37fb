"""The narrow tensor-core kernel's reverse sweep runs the tensor layers of a 128-point tile as two 64-point halves
(csrc/tc_kernel.cu, net_backward): point counts that end a term inside either half or at its edge, several tensor layers
at the smallest channel counts (one and three: the fewest tiles of shared memory the halves have to share), two networks
of one term (the forward is recomputed between their reverse sweeps) and loss-only calls, each against the precision
model at the tolerances of test_gpu_tc_model.py."""
import numpy as np
import pytest

import tc_cases as TC
from neuralpde_jl_b200.configs import Config
from neuralpde_jl_b200.strategies import GridTraining
from test_gpu_tc_model import FLOOR_DRAWS, LOSS_TOL, check, run

pytestmark = pytest.mark.gpu

HALF_EDGES = (1, 63, 64, 65, 127, 129, 192, 193)


@pytest.mark.parametrize("n", HALF_EDGES)
def test_point_counts_at_half_edges(n):
    """1-D u_xx (three channels, one tensor layer): a term of n points ends in the first half, at its edge or in the second."""
    x = np.random.default_rng(n).random((1, n))
    check(TC.point_count("tc"), "tc_split", sets=[x], label="n=%d" % n)


def _deep(structure, width=64, depth=4):
    sys_, dx = TC.STRUCTURES[structure][0]()
    chain = TC.net(len(sys_.ivs), [width] * depth, ["tanh"] * depth)
    return Config("%s_tl%d" % (structure, depth - 1), sys_, [chain], GridTraining(dx))


@pytest.mark.parametrize("structure,n", [("value", 65), ("value", 193), ("transport2", 63), ("transport2", 129)])
@pytest.mark.parametrize("mode", ["tc_bf16", "tc_split"])
def test_three_tensor_layers_few_channels(structure, n, mode):
    """One channel (value only) and three channels (value and two first derivatives) through three 64-wide tensor
    layers, with the PDE term cut at n points."""
    x = np.random.default_rng(n).random((2, n))
    check(_deep(structure), mode, sets=[x], label="%s n=%d" % (structure, n))


@pytest.mark.parametrize("n", [65, 129])
@pytest.mark.parametrize("mode", ["tc_bf16", "tc_split"])
def test_two_networks_in_one_term(n, mode):
    """Two networks of different width and depth tapped by the same terms; the first term cut at n points."""
    x = np.random.default_rng(n).random((2, n))
    check(TC.coupled_narrow(), mode, sets=[x], label="coupled n=%d" % n)


@pytest.mark.parametrize("n", [63, 193])
def test_loss_only(n):
    cfg = _deep("transport2")
    rep, eng, model = run(cfg, "tc_split", [np.random.default_rng(n).random((2, n))])
    th = TC.make_theta(cfg)
    total, terms, grad = eng.loss_grad_host(th, None, False)
    res = model.evaluate(th.astype(np.float64), want_grad=False)
    fl = model.noise_floor(th.astype(np.float64), draws=FLOOR_DRAWS, base=res)
    assert grad is None
    assert np.max(np.abs(terms - res.terms) / np.abs(res.terms)) <= LOSS_TOL + 4 * np.max(fl.terms)
    assert abs(total - res.total) / abs(res.total) <= LOSS_TOL + 4 * fl.total
