"""Categorical PPO heads without a GPU: the float64 restatement tests/ppo_restatement.py against torch autograd,
the cpb_ppo_cat_* layout and names, the refusal of every bad cpb_ppo_cat_spec by every twin before any launch, the
action-space duck typing, the replay environment's index -> control mapping and the checkpoint record."""
import ctypes as C

import numpy as np
import pytest

import ppo_restatement as pr
from harness import lib  # noqa: F401
from ppo_checks import SPEC_ENTRIES, ppo_call, torch_loss_and_grads

S = 67


@pytest.mark.parametrize("arch", [((1,), (1,)), ((3, 2), (1,))])
@pytest.mark.parametrize("nvec", [(2,), (7, 3), (2, 2, 2, 2), (31, 33)])
@pytest.mark.parametrize("case", ["full", "entropy_only", "policy_only"])
def test_restatement_matches_autograd(arch, nvec, case):
    rs = np.random.RandomState(len(nvec) + 7 * sum(nvec))
    B = 12
    p = {k: v.astype(np.float64) for k, v in pr.init_params(5, nvec, arch[0], arch[1], seed=3).items()}
    for k in p:
        p[k] = p[k] + 0.3 * rs.randn(*p[k].shape)          # nonzero biases, logits far from uniform
    old = {k: v + 0.2 * rs.randn(*v.shape) for k, v in p.items()}
    s = rs.randn(B, 5)
    a = np.stack([rs.randint(c, size=B) for c in nvec], axis=1)
    ret, adv = rs.randn(B), rs.randn(B)
    es = 0.01
    if case == "entropy_only":
        adv = np.zeros(B)
    elif case == "policy_only":
        es = 0.0
    r = pr.loss_and_grads(p, old, s, a, ret, adv, nvec, 0.2, 1.0, es)
    loss, grads = torch_loss_and_grads(p, old, s, a, ret, adv, nvec, 0.2, 1.0, es)
    assert abs(r["loss"] - loss) <= 1e-10 * max(1.0, abs(loss))
    for k, g in grads.items():
        assert np.abs(r["grads"][k] - g).max() <= 1e-10 * max(1.0, np.abs(g).max()), k


def _spec(cats, pol=(500, 300), val=(500, 300), state_dim=S):
    from carla_ppo_b200 import _lib
    base = _lib.PpoConfig()
    base.state_dim, base.epsilon, base.value_scale, base.entropy_scale = state_dim, 0.2, 1.0, 0.01
    return _lib.PpoCatSpec.of(base, pol, val, cats)


@pytest.mark.parametrize("cats,arch", [((2,), ((1,), (1,))), ((7, 3), ((500, 300), (500, 300))),
                                       ((31, 33), ((33, 7, 65), (31,))), ((2, 2, 2, 2), ((64,) * 8, (32,) * 8))])
def test_layout_and_names_equal_the_restatement(lib, cats, arch):
    sp = _spec(cats, *arch)
    n = lib.cpb_ppo_cat_num_tensors(C.byref(sp))
    shapes_ref = pr.param_shapes(S, cats, *arch)
    assert n == len(shapes_ref) == 2 * (len(arch[0]) + len(arch[1])) + 4
    offs = (C.c_int64 * n)(); sizes = (C.c_int64 * n)(); shapes = (C.c_int32 * (2 * n))(); total = C.c_int64()
    assert lib.cpb_ppo_cat_layout(C.byref(sp), offs, sizes, shapes, C.byref(total)) == 0
    names = [lib.cpb_ppo_cat_tensor_name(C.byref(sp), i).decode() for i in range(n)]
    assert names == list(shapes_ref)
    assert lib.cpb_ppo_cat_tensor_name(C.byref(sp), n) is None
    end = 0
    for i, (name, shape) in enumerate(shapes_ref.items()):
        got = tuple(v for v in shapes[2 * i:2 * i + 2] if v > 0)
        assert got == tuple(shape), name
        assert sizes[i] == int(np.prod(shape)) and offs[i] % 64 == 0 and offs[i] >= end
        end = offs[i] + sizes[i]
    assert total.value >= end
    assert lib.cpb_ppo_cat_workspace_bytes(C.byref(sp), 256, 2048) > 0


def _bad_specs():
    good = lambda: _spec((7, 3))
    out = {"null": None}
    s = good(); s.spec.base.num_actions = 0; out["K0"] = s
    s = good(); s.spec.base.num_actions = 5; out["K5"] = s
    s = good(); s.num_categories[1] = 1; out["n1"] = s
    s = good(); s.num_categories[0] = 65; out["n65"] = s
    s = _spec((40, 30)); out["N70"] = s
    s = good(); s.spec.base.action_low[0] = -1.0; out["low"] = s
    s = good(); s.spec.base.action_high[3] = 1.0; out["high"] = s
    s = good(); s.spec.num_policy = 0; out["depth0"] = s
    s = good(); s.spec.value_sizes[1] = 0; out["width0"] = s
    s = good(); s.spec.base.hidden1 = 500; out["hidden1"] = s
    s = good(); s.spec.base.state_dim = 0; out["state0"] = s
    return out


@pytest.mark.parametrize("bad", list(_bad_specs()))
def test_every_twin_refuses_a_bad_spec_before_any_launch(lib, bad):
    sp = _bad_specs()[bad]
    ref = None if sp is None else C.byref(sp)
    lib.cpb_reset_launch_count()
    for entry in SPEC_ENTRIES:
        assert ppo_call(lib, "cpb_ppo_cat_", entry, ref) == -1, entry
    assert lib.cpb_ppo_cat_tensor_name(ref, 0) is None
    assert lib.cpb_launch_count() == 0


def test_action_space_duck_typing():
    from carla_ppo_b200.ppo import PPO, action_categories
    from carla_ppo_b200.replay_env import Box, Discrete, MultiDiscrete
    assert action_categories(Box([-1.0, 0.0], [1.0, 1.0])) is None
    assert action_categories(Discrete(5)) == (5,)
    assert action_categories(MultiDiscrete([7, 3])) == (7, 3)
    for bad in (Discrete(1), Discrete(65), MultiDiscrete([40, 30]), MultiDiscrete([2] * 5)):
        with pytest.raises(ValueError):
            action_categories(bad)
    import tempfile
    with tempfile.TemporaryDirectory() as d:
        m = PPO((S,), MultiDiscrete([7, 3]), model_dir=d)
        assert m.num_actions == 2 and m.action_categories == (7, 3)


def test_replay_env_index_to_control():
    from carla_ppo_b200.replay_env import MultiDiscrete, ReplayEnv, discrete_controls
    frames = np.zeros((4, 80, 160, 3), np.uint8)
    env = ReplayEnv(frames, discrete_actions=(5, 3))
    assert isinstance(env.action_space, MultiDiscrete) and tuple(env.action_space.nvec) == (5, 3)
    steer, throttle = discrete_controls((5, 3))
    assert np.allclose(steer, [-1.0, -0.5, 0.0, 0.5, 1.0]) and np.allclose(throttle, [0.0, 0.5, 1.0])
    env.reset()
    env.step(np.array([4, 1]))
    assert env.vehicle.control.steer == 1.0 and env.vehicle.control.throttle == 0.5
    env.step(np.array([0, 2]))
    assert env.vehicle.control.steer == -1.0 and env.vehicle.control.throttle == 1.0


def test_checkpoint_record(tmp_path):
    from carla_ppo_b200.ppo import (CATEGORIES_KEY, blob_action_categories, blob_architecture,
                                    checkpoint_action_categories)
    from carla_ppo_b200.train import resolve_action_categories
    p = pr.init_params(S, (7, 3), (64,), (32,), seed=0)
    blob = {"policy/" + k: v for k, v in p.items()}
    blob[CATEGORIES_KEY] = np.array([7, 3], np.int32)
    assert blob_action_categories(blob) == (7, 3)
    assert blob_architecture(blob) == ((64,), (32,))
    bad = dict(blob); bad[CATEGORIES_KEY] = np.array([5, 3], np.int32)
    with pytest.raises(ValueError):
        blob_action_categories(bad)
    unrecorded = {k: v for k, v in blob.items() if k != CATEGORIES_KEY}
    with pytest.raises(ValueError):
        blob_action_categories(unrecorded)
    gauss = {"policy/action_mean/kernel": np.zeros((64, 2))}
    assert blob_action_categories(gauss) == ()
    assert checkpoint_action_categories(str(tmp_path)) is None
    # a resumed run takes the checkpoint's categories; a disagreeing flag is refused, and so is one on a Gaussian run
    assert resolve_action_categories(None, (7, 3)) == (7, 3)
    assert resolve_action_categories([7, 3], (7, 3)) == (7, 3)
    assert resolve_action_categories([7, 3], None) == (7, 3)
    assert resolve_action_categories(None, ()) is None
    for flag, ck in (([5, 3], (7, 3)), ([7, 3], ())):
        with pytest.raises(ValueError):
            resolve_action_categories(flag, ck)


def test_host_actions_are_validated():
    from carla_ppo_b200.ppo import PPO
    import tempfile
    from carla_ppo_b200.replay_env import MultiDiscrete
    with tempfile.TemporaryDirectory() as d:
        m = PPO((S,), MultiDiscrete([7, 3]), model_dir=d)
        import torch
        m._torch = torch
        for bad in ([[0.5, 1]], [[7, 0]], [[0, -1]], [[np.nan, 0]]):
            with pytest.raises(ValueError):
                m._actions(np.asarray(bad))
