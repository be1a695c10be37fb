"""The model side of the 256-wide tensor-core kernel, checked without a GPU: the precision model (tests/tc_model.py) in
`exact` mode against the float64 oracle on 256-wide problems, config 4's pass split, and the coverage of the dispatch
matrix that tests/test_gpu_tc256.py runs."""
import numpy as np
import pytest

import tc256_cases as X
import tc_cases as TC
import tc_model as M
from test_tc_model import _exact_vs_oracle


@pytest.mark.parametrize("name,build", [("burgers_tl1", lambda: X.burgers_depth(1)),
                                        ("burgers_mixed_widths", lambda: X.burgers_depth(0, [256, 128, 64, 192])),
                                        ("coupled", X.coupled), ("cfg4_small", lambda: X.cfg4_small(hidden=2))])
def test_exact_model_matches_oracle(name, build):
    _exact_vs_oracle(build())


def test_cfg4_pass_split():
    """A momentum term of config 4 taps u, u_x, u_y, u_z, u_xx, u_yy, u_zz, v, w and p_x (10 taps, u with 7 channels): u
    runs as three passes {value, x, xx}, {value, y, yy}, {value, z, zz} beside v, w and p, 6 slots in all."""
    cfg = X.cfg4_small()
    rep, rec = TC.capture(cfg)
    model = rec.model("tw_bf16")
    slots, taps = model.plans[0]
    assert len(rec.spec.terms[0].taps) == 10
    assert [s.net for s in slots] == [0, 0, 0, 1, 2, 3]
    for k in range(3):
        assert slots[k].dir1 == [k] and slots[k].pairs == [(0, 0)] and slots[k].pure and slots[k].C == 3
    assert all(s.C <= M.TW_MAX_C for s in slots)
    # every u tap reads the pass of its direction: value from the first, d/dx_k and d2/dx_k^2 from pass k
    u_taps = [(tp, st) for tp, st in zip(rec.spec.terms[0].taps, taps) if tp.net == 0]
    for tp, (s, c) in u_taps:
        if tp.order == 0:
            assert (s, c) == (0, 0)
        else:
            assert s == tp.dirs[0] and c == tp.order


def test_matrix_covers_every_dispatch_instantiation():
    got = set()
    for _, build in X.matrix():
        got |= X.x256_keys(TC.capture(build())[1].model("tw_bf16"))
    assert len(X.X256_DISPATCH) == 14 and got == X.X256_DISPATCH


def test_tw_model_rounds_a_256_wide_network():
    """The tw_bf16 model differs from exact on a 256-wide network by bf16-sized amounts, not more."""
    cfg = X.burgers_depth(2)
    rep, rec = TC.capture(cfg)
    th = TC.make_theta(cfg).astype(np.float64)
    ex = rec.model("exact").evaluate(th)
    bf = rec.model("tw_bf16").evaluate(th)
    err = abs(bf.total - ex.total) / abs(ex.total)
    assert 1e-6 < err < 1e-1
