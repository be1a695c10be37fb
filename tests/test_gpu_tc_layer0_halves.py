"""The narrow tensor-core kernel's reverse sweep runs layer 0 per 64-point half as well (csrc/tc_kernel.cu, net_backward):
the half's input adjoints of the lowest tensor layer stay in shared memory, Z̄⁰ and the augmented-coordinate tiles go to
region Q, and the layer-0 gradient is one m64n16 MMA per warpgroup (16 points each) whose four partials are summed in a
fixed order.  Checked against the precision model at the tolerances of test_gpu_tc_model.py: point counts at and around
the half edges, every channel structure of PINN_TC_DISPATCH in both modes with one tensor layer (all tanh) and three
(generic activations), two networks in one term, and loss-only calls."""
import numpy as np
import pytest

import tc_cases as TC
from neuralpde_jl_b200.configs import Config
from neuralpde_jl_b200.strategies import GridTraining
from test_gpu_tc_model import FLOOR_DRAWS, LOSS_TOL, check, run

pytestmark = pytest.mark.gpu


@pytest.mark.parametrize("n", (1, 63, 64, 65, 127, 128, 129, 1000))
def test_point_counts(n):
    """1-D u_xx (three channels): a term of n points ends in the first half, at its edge, in the second or after 7 tiles."""
    x = np.random.default_rng(n).random((1, n))
    check(TC.point_count("tc"), "tc_split", sets=[x], label="n=%d" % n)


def _structure(name, tensor_layers):
    """Structure `name` on a narrow network with `tensor_layers` tensor layers: all tanh and 48 wide with one, generic
    activations and a 16-wide first layer (one granule pair per thread in the layer-0 loop) with three."""
    sys_, dx = TC.STRUCTURES[name][0]()
    depth = tensor_layers + 1
    if tensor_layers == 1:
        widths, acts = [48] * depth, ["tanh"] * depth
    else:
        widths, acts = [16] + [64] * (depth - 1), [TC.GENERIC[k % len(TC.GENERIC)] for k in range(depth)]
    chain = TC.net(len(sys_.ivs), widths, acts)
    return Config("%s_tl%d" % (name, tensor_layers), sys_, [chain], GridTraining(dx))


@pytest.mark.parametrize("tensor_layers", [1, 3])
@pytest.mark.parametrize("mode", ["tc_bf16", "tc_split"])
@pytest.mark.parametrize("name", sorted(TC.STRUCTURES))
def test_every_structure(name, mode, tensor_layers):
    check(_structure(name, tensor_layers), mode, label="%s tl=%d" % (name, tensor_layers))


@pytest.mark.parametrize("n", [64, 1000])
@pytest.mark.parametrize("mode", ["tc_bf16", "tc_split"])
def test_two_networks_in_one_term(n, mode):
    """Two networks of different width and depth tapped by the same terms; the first term cut at n points."""
    x = np.random.default_rng(n).random((2, n))
    check(TC.coupled_narrow(), mode, sets=[x], label="coupled n=%d" % n)


@pytest.mark.parametrize("n", [64, 129])
@pytest.mark.parametrize("mode", ["tc_bf16", "tc_split"])
def test_loss_only(n, mode):
    cfg = _structure("poisson", 3)
    rep, eng, model = run(cfg, mode, [np.random.default_rng(n).random((2, n))])
    th = TC.make_theta(cfg)
    total, terms, grad = eng.loss_grad_host(th, None, False)
    res = model.evaluate(th.astype(np.float64), want_grad=False)
    fl = model.noise_floor(th.astype(np.float64), draws=FLOOR_DRAWS, base=res)
    assert grad is None
    assert np.max(np.abs(terms - res.terms) / np.abs(res.terms)) <= LOSS_TOL + 4 * np.max(fl.terms)
    assert abs(total - res.total) / abs(res.total) <= LOSS_TOL + 4 * fl.total
