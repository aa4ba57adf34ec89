"""The PPO at every shape the C ABI accepts, without a GPU: the float64 oracle against torch autograd at each shape of
CASES on inputs where the clipped surrogate takes both branches, the weight initialiser and input builders
(tests/ppo_cases.py), and the parameter layout / workspace queries at A = 1..4 and odd sizes."""
import ctypes as C

import numpy as np
import pytest

from harness import lib, library_state  # noqa: F401
from helpers import Box, rel_l2
from ppo_cases import CASES, CLIPPED, KINK_MARGIN, bounds, clip_groups, make_batch, ppo_config, shape_net
from ppo_restatement import init_params, pre_activations, relu_margin

# ------------------------------------------------------------------------------------------------------------ tests
@pytest.mark.parametrize("case", list(CASES))
def test_oracle_backward_matches_autograd_with_clipped_rows(case):
    """The hand-written backward of ppo_oracle against an independent torch-autograd derivation at this shape, on a
    minibatch whose rows fill all five branches of the clipped surrogate."""
    from oracle import ppo_oracle as po, torch_ref as tr
    S, A, H1, H2 = CASES[case]
    low, high = bounds(A)
    p, old, s, a, ret, adv = make_batch(shape_net(S, A, H1, H2), 128, 4, init_seed=3, **CLIPPED)
    ref = po.loss_and_grads(p, old, s, a, ret, adv, low, high, 0.2, 1.0, 0.01)
    auto = tr.ppo_loss_and_grads(p, old, s, a, ret, adv, low, high, 0.2, 1.0, 0.01)
    groups = clip_groups(ref["ratio"], adv)
    assert all(g.any() for g in groups.values()), {k: int(g.sum()) for k, g in groups.items()}
    for key in ("loss", "policy_loss", "value_loss", "entropy_loss", "mean_ratio"):
        assert abs(ref[key] - auto[key]) < 1e-10, key
    assert set(ref["grads"]) == set(po.PPO_TENSORS)
    for name, g in ref["grads"].items():
        assert g.shape == p[name].shape, name
        assert rel_l2(g, auto["grads"][name]) < 1e-10, name


@pytest.mark.parametrize("case", ["a1", "a4", "tiny", "odd"])
def test_initialiser_follows_the_ppo_class(tmp_path, case):
    """init_params draws what PPO._initial_weights draws for the same seed and shapes (the class reads its shapes from
    cpb_ppo_layout, which only needs the session; they are set directly here)."""
    from carla_ppo_b200.ppo import PPO
    from oracle.ppo_oracle import param_shapes
    S, A, H1, H2 = CASES[case]
    m = PPO((S,), Box(*bounds(A)), model_dir=str(tmp_path / "ppo"), seed=7)
    shapes = param_shapes(S, A, (H1, H2), (H1, H2))
    m._names, m._shapes = list(shapes), dict(shapes)
    got, ref = m._initial_weights(), init_params(*shape_net(S, A, H1, H2), seed=7)
    assert list(got) == list(ref)
    for k in ref:
        assert got[k].dtype == ref[k].dtype and np.array_equal(got[k], ref[k]), k


@pytest.mark.parametrize("case", list(CASES))
def test_biases_keep_pre_activations_off_the_relu_kink(case):
    for batch in (1, 9, 256):
        p, _, s = make_batch(shape_net(*CASES[case]), batch, batch, init_seed=0)[:3]
        assert relu_margin(p, s) > KINK_MARGIN, batch
        if batch >= 4:                                          # every unit active on some rows and off on others
            for z in pre_activations(p, s):
                assert (z > 0).any(axis=0).all() and (z < 0).any(axis=0).all(), batch


LAYOUT_SHAPES = list(CASES.values()) + [(67, 1, 500, 300), (67, 3, 500, 300), (2, 4, 3, 2), (1030, 1, 1, 7)]


@pytest.mark.parametrize("shape", LAYOUT_SHAPES, ids=["S%d_A%d_%dx%d" % s for s in LAYOUT_SHAPES])
def test_layout_matches_oracle_shapes(lib, shape):
    from oracle.ppo_oracle import param_shapes, PPO_TENSORS
    S, A, H1, H2 = shape
    cfg = ppo_config(*shape)
    n = lib.cpb_ppo_num_tensors()
    offs = (C.c_int64 * n)(); sizes = (C.c_int64 * n)(); shapes = (C.c_int32 * (2 * n))(); total = C.c_int64()
    assert lib.cpb_ppo_layout(C.byref(cfg), offs, sizes, shapes, C.byref(total)) == 0
    ref = param_shapes(S, A, (H1, H2), (H1, H2))
    assert [lib.cpb_ppo_tensor_name(i).decode() for i in range(n)] == PPO_TENSORS == list(ref)
    spans = []
    for i, name in enumerate(PPO_TENSORS):
        assert tuple(v for v in shapes[2 * i:2 * i + 2] if v > 0) == ref[name], name
        assert sizes[i] == int(np.prod(ref[name])), name
        assert offs[i] % 64 == 0, name
        spans.append((offs[i], offs[i] + sizes[i]))
    assert all(a[1] <= b[0] for a, b in zip(spans, spans[1:]))      # creation order, no overlap
    assert total.value % 64 == 0 and spans[-1][1] <= total.value < spans[-1][1] + 64


@pytest.mark.parametrize("bad", [dict(A=0), dict(A=5), dict(S=0), dict(H1=0), dict(H2=0), dict(A=-1), dict(S=-3)],
                         ids=lambda d: "_".join("%s%d" % kv for kv in d.items()))
def test_layout_and_workspace_refuse_bad_shapes(lib, bad):
    from carla_ppo_b200 import _lib
    shape = dict(S=67, A=2, H1=500, H2=300)
    shape.update(bad)
    cfg = ppo_config(shape["S"], shape["A"], shape["H1"], shape["H2"])
    total = C.c_int64(-7)
    assert lib.cpb_ppo_layout(C.byref(cfg), None, None, None, C.byref(total)) == -1      # CPB_ERR_INVALID_ARGUMENT
    assert total.value == -7                                                             # nothing written
    assert lib.cpb_ppo_workspace_bytes(C.byref(cfg), 64, 0) == -1
    with pytest.raises(_lib.CpbError):
        _lib.check(lib.cpb_ppo_layout(C.byref(cfg), None, None, None, None), "cpb_ppo_layout")


def test_workspace_grows_with_batch_and_horizon(lib):
    for shape in (CASES["a4"], CASES["tiny"], CASES["wide"]):
        cfg = C.byref(ppo_config(*shape))
        # sizes are rounded up to an alignment, so neighbouring batch sizes may share one
        by_batch = [lib.cpb_ppo_workspace_bytes(cfg, b, 0) for b in (1, 2, 9, 256, 8192, 8200, 20000)]
        assert by_batch[0] > 0 and all(x <= y for x, y in zip(by_batch, by_batch[1:])), by_batch
        assert by_batch[0] < by_batch[3] < by_batch[4] < by_batch[5] < by_batch[6], by_batch
        base = lib.cpb_ppo_workspace_bytes(cfg, 64, 0)
        # the horizon (learn(): T rows of old-policy activations, returns, advantages) only counts beyond max_batch
        assert lib.cpb_ppo_workspace_bytes(cfg, 64, 64) == lib.cpb_ppo_workspace_bytes(cfg, 64, 10) == base
        by_horizon = [lib.cpb_ppo_workspace_bytes(cfg, 64, t) for t in (65, 300, 2500, 4097)]
        assert base <= by_horizon[0] and all(x <= y for x, y in zip(by_horizon, by_horizon[1:])), by_horizon
        assert base < by_horizon[1] < by_horizon[2] < by_horizon[3], by_horizon
        assert lib.cpb_ppo_workspace_bytes(cfg, 0, 0) == -1
        assert lib.cpb_ppo_workspace_bytes(cfg, 64, -1) == -1
    big = lib.cpb_ppo_workspace_bytes(C.byref(ppo_config(*CASES["wide"])), 8200, 8200)
    assert 0 < big < 1 << 30
