"""Categorical PPO heads on the device (cpb_ppo_cat_*): every entry point against the float64 restatement
tests/ppo_restatement.py over Discrete / MultiDiscrete spaces from (2,) to (31, 33) and architectures from one
layer per trunk to eight, with the workspace filled with NaN before each call; determinism and launch counts equal to the
Gaussian head's; the fused actor; train.py with --discrete_actions; checkpoints."""
import os

import numpy as np
import pytest

import ppo_restatement as pr
from harness import lib  # noqa: F401
from helpers import committed_frames, rel_l2
from ppo_cases import (CAT_ARCHS as ARCHS, CLIP_HI, CLIP_LO, KINK_MARGIN, NVECS, S, cat_net, f64, gauss_net,
                       kink_free, learn_refs, learn_setup, make_batch, make_ppo, train_params)
from ppo_checks import (TOL, check_fused_actor, check_learn, check_learn_opts_clip_and_kl_stop, check_learn_segments,
                        check_loss, check_two_train_steps, five, fresh_process, nan_workspace)

pytestmark = pytest.mark.gpu


def _predict_states(net, n, seed):
    """n states on which every component's top two logits differ by more than 1e-3 (chosen from 4n candidates that the
    trunk biases were placed on), and the network"""
    state_dim, cats = net[:2]
    rs = np.random.RandomState(seed)
    cand = rs.randn(4 * n, state_dim).astype(np.float32)
    p = kink_free(net, cand, seed + 1)
    z, _ = pr.forward(f64(p), cand.astype(np.float64), cats)
    off = pr.offsets(cats)
    ok = np.ones(len(cand), bool)
    for k in range(len(cats)):
        zk = np.sort(z[:, off[k]:off[k + 1]], axis=1)
        ok &= zk[:, -1] - zk[:, -2] > 1e-3
    s = cand[ok][:n]
    assert len(s) == n
    return p, s


@pytest.mark.parametrize("state_dim", [67, 1027])
@pytest.mark.parametrize("nvec", list(NVECS))
@pytest.mark.parametrize("arch", list(ARCHS))
def test_predict_greedy_and_sampled(tmp_path, arch, nvec, state_dim):
    cats, net = NVECS[nvec], cat_net(ARCHS[arch], NVECS[nvec], state_dim)
    p, s = _predict_states(net, 37, 1)
    assert pr.relu_margin(p, s) > KINK_MARGIN and pr.logit_gap(f64(p), s, cats) > 1e-4
    m = make_ppo(tmp_path, net, p)
    # uniforms at least 1e-5 from every CDF boundary of the restatement
    rs = np.random.RandomState(2)
    bounds = pr.cdf_bounds(f64(p), s, cats)
    u = rs.rand(37, len(cats))
    for _ in range(100):
        near = np.stack([np.abs(bounds[k] - u[:, k:k + 1]).min(axis=1) < 1e-5 for k in range(len(cats))], axis=1)
        if not near.any():
            break
        u[near] = rs.rand(int(near.sum()))
    assert min(np.abs(bounds[k] - u[:, k:k + 1]).min() for k in range(len(cats))) >= 1e-5
    u = u.astype(np.float32)
    for nz in (None, u):
        nan_workspace(m, 37)
        act, val = m.predict(s, greedy=nz is None, noise=nz)
        ract, rval = pr.predict(f64(p), s, cats, noise=None if nz is None else nz.astype(np.float64))
        assert act.dtype == np.int64 and np.array_equal(act, ract), (nz is None, act, ract)
        assert rel_l2(val, rval) < TOL


@pytest.mark.parametrize("B", [1, 9, 256, 8200])
@pytest.mark.parametrize("nvec", list(NVECS))
def test_loss_and_gradients(tmp_path, nvec, B):
    net = cat_net(ARCHS["default"], NVECS[nvec])
    p, old, s, a, ret, adv = make_batch(net, B, 3 + B)
    assert pr.relu_margin(p, s) > KINK_MARGIN
    m = make_ppo(tmp_path, net, p, old)
    nan_workspace(m, B)
    r64 = check_loss(m, p, old, s, a, ret, adv, net[1])
    ratio = r64["ratio"]
    assert not (np.minimum(np.abs(ratio - CLIP_LO), np.abs(ratio - CLIP_HI)) < 1e-4).any()
    if B >= 256:
        for frac in ((ratio < CLIP_LO).mean(), (ratio > CLIP_HI).mean(), ((ratio >= CLIP_LO) & (ratio <= CLIP_HI)).mean()):
            assert frac >= 0.1, frac


@pytest.mark.parametrize("arch", list(ARCHS))
def test_loss_and_gradients_architectures(tmp_path, arch):
    net = cat_net(ARCHS[arch], NVECS["7x3"])
    p, old, s, a, ret, adv = make_batch(net, 256, 11)
    m = make_ppo(tmp_path, net, p, old)
    nan_workspace(m, 256)
    check_loss(m, p, old, s, a, ret, adv, net[1])


@pytest.mark.parametrize("case", ["entropy_only", "policy_only"])
def test_entropy_only_and_policy_only(tmp_path, case):
    net = cat_net(ARCHS["p64_v64"], NVECS["31x33"])
    p, old, s, a, ret, adv = make_batch(net, 256, 21)
    es = 0.01
    if case == "entropy_only":
        adv = np.zeros_like(adv)
    else:
        es = 0.0
    m = make_ppo(tmp_path, net, p, old, entropy_scale=es)
    nan_workspace(m, 256)
    check_loss(m, p, old, s, a, ret, adv, net[1], entropy_scale=es)


def test_two_train_steps(tmp_path):
    net = cat_net(ARCHS["odd"], NVECS["7x3"])
    check_two_train_steps(tmp_path, net, make_batch(net, 64, 17))


_LEARN_CASES = [("default", "7x3"), ("default", "64"), ("odd", "2x2x2x2"), ("deep", "31x33"), ("p64_v64", "2")]


def test_learn_both_paths(tmp_path):
    """T = 2048 in 4 epochs of 8 minibatches of 256: launch per kernel and the persistent kernel against float64, and
    the persistent kernel within 1e-6 of launch per kernel."""
    outs = fresh_process(tmp_path, [(arch + nvec, cat_net(ARCHS[arch], NVECS[nvec]), ("rollout", 2048, 4, 256, 40), {})
                                    for arch, nvec in _LEARN_CASES])
    for arch, nvec in _LEARN_CASES:
        net, tag = cat_net(ARCHS[arch], NVECS[nvec]), arch + nvec
        p, data, perms, adam = learn_setup(net, 2048, 4, 40)
        refs = five(learn_refs(net, p, data, perms, 256, adam))
        for o in outs:
            check_learn({k: o[tag + ":w:" + k] for k in p}, o[tag + ":metrics"], refs)
        for k in p:
            assert rel_l2(outs[1][tag + ":w:" + k], outs[0][tag + ":w:" + k]) < 1e-6, (tag, k)


def test_learn_segments(tmp_path):
    """16 segments x 128 rows."""
    check_learn_segments(tmp_path, cat_net(ARCHS["odd"], NVECS["7x3"]))


@pytest.mark.parametrize("nvec", ["7x3", "64"])
def test_learn_opts_clip_and_kl_stop(tmp_path, nvec):
    """Clipping binding on 25-75 % of the minibatches, then a KL stop at a minibatch k > 1 (steps_applied = k)."""
    check_learn_opts_clip_and_kl_stop(tmp_path, cat_net(ARCHS["p64_v64"], NVECS[nvec]))


# ------------------------------------------------------------------------------ determinism, launch counts
def _one_of_each(m, s, a, ret, adv, u, p, old, lib):
    """predict (greedy, sampled), loss_and_grads, train, learn: (results, launch counts)"""
    out, launches = {}, {}
    steps = [("greedy", lambda: m.predict(s, greedy=True)), ("sampled", lambda: m.predict(s, noise=u)),
             ("loss", lambda: m.loss_and_grads(s, a, ret, adv)), ("train", lambda: m.train(s, a, ret, adv)),
             ("learn", lambda: m.learn(s, a, ret, adv, np.zeros(len(s)), 0.3, num_epochs=2, batch_size=64,
                                       perms=np.stack([np.arange(len(s))[::-1], np.arange(len(s))]), return_metrics=True))]
    for name, f in steps:
        m.set_weights(p, old)
        m.adam_m.zero_(); m.adam_v.zero_()
        m.adam_powers.fill_(0.0).add_(m._torch.tensor([0.9, 0.999], device=m.adam_powers.device))
        lib.cpb_reset_launch_count()
        r = f()
        launches[name] = lib.cpb_launch_count()
        out[name] = r
        out[name + ":params"] = m.params.cpu().numpy()
    return out, launches


def test_deterministic_and_launch_counts_equal_gaussian(tmp_path, lib):
    import torch
    for arch in ("default", "odd"):
        net = cat_net(ARCHS[arch], NVECS["7x3"])
        p, old, s, a, ret, adv = make_batch(net, 256, 31)
        u = np.random.RandomState(3).rand(256, 2).astype(np.float32)
        m = make_ppo(tmp_path / arch, net, p, old)
        r1, l1 = _one_of_each(m, s, a, ret, adv, u, p, old, lib)
        r2, _ = _one_of_each(m, s, a, ret, adv, u, p, old, lib)
        for k in r1:
            x, y = r1[k], r2[k]
            flat = lambda t: [np.asarray(v.cpu() if isinstance(v, torch.Tensor) else v) for v in (t if isinstance(t, tuple) else (t,))]
            for xi, yi in zip(flat(x), flat(y)):
                if isinstance(xi, np.ndarray) and xi.dtype == object:
                    continue
                assert np.array_equal(xi, yi), (arch, k)
        g = make_ppo(tmp_path / ("g" + arch), gauss_net(ARCHS[arch]))
        _, lg = _one_of_each(g, s, np.zeros((256, 2), np.float32), ret, adv, np.random.RandomState(3).randn(256, 2)
                             .astype(np.float32), g.get_weights(), g.get_weights(), lib)
        assert l1 == lg, (arch, l1, lg)


# ----------------------------------------------------------------------------------------------------- fused actor
@pytest.mark.parametrize("kind", ["conv", "mlp"])
@pytest.mark.parametrize("n", [1, 4])
def test_fused_actor_equals_unfused(tmp_path, lib, kind, n):
    check_fused_actor(tmp_path, cat_net(ARCHS["odd"], NVECS["7x3"]), kind, n, greedy=(False, True))


# ----------------------------------------------------------------------------- train.py / run_eval.py over the replay env
def _run_training(tmp_path, tag, restart=False, env_cats=None, **over):
    from carla_ppo_b200.replay_env import ReplayEnv
    from carla_ppo_b200.train import train
    from ppo_cases import shipped_vae
    rgb, _ = committed_frames()
    cats = env_cats or over.get("discrete_actions")
    envs = [ReplayEnv(rgb, episode_length=24, seed=0, discrete_actions=cats) for _ in range(4)]
    vae = shipped_vae(tmp_path, tag)
    over.setdefault("num_envs", 4)
    model = train(train_params(tag, **over), restart=restart, env=envs, vae=vae, models_root=str(tmp_path / "models"),
                  interactive=False)
    return model


def test_train_discrete_fused_unfused_reference_loop_resume_and_eval(tmp_path):
    from carla_ppo_b200.ppo import checkpoint_action_categories
    from carla_ppo_b200.run_eval import load_model
    a = _run_training(tmp_path, "fused", discrete_actions=[7, 3])
    b = _run_training(tmp_path, "unfused", discrete_actions=[7, 3], unfused=True)
    c = _run_training(tmp_path, "reffused", discrete_actions=[7, 3], reference_loop=True)
    d = _run_training(tmp_path, "refunfused", discrete_actions=[7, 3], reference_loop=True, unfused=True)
    assert a.action_categories == (7, 3) and a.get_train_step_idx() > 0
    for x, y in ((a, b), (c, d)):
        wx, wy = x.get_weights(), y.get_weights()
        assert all(np.array_equal(wx[k], wy[k]) for k in wx)
        assert x.reward_history == y.reward_history
    assert checkpoint_action_categories(a.checkpoint_dir) == (7, 3)
    # resume: the checkpoint's categories without the flag; a disagreeing flag is refused before anything trains
    e = _run_training(tmp_path, "fused", env_cats=(7, 3), num_episodes=3)
    assert e.action_categories == (7, 3) and e.get_episode_idx() == 3
    with pytest.raises(ValueError, match="disagrees"):
        _run_training(tmp_path, "fused", discrete_actions=[5, 3], num_episodes=4)
    # run_eval's loader rebuilds the discrete agent from the record
    from carla_ppo_b200.replay_env import Box
    m = load_model(np.array([S]), Box([-1.0, 0.0], [1.0, 1.0]), os.path.dirname(a.checkpoint_dir.rstrip("/")))
    assert m.action_categories == (7, 3)
    assert m.get_episode_idx() == e.get_episode_idx() or m.get_episode_idx() >= 0


def test_checkpoint_refuses_gaussian_categorical_swap(tmp_path):
    net, gauss = cat_net(ARCHS["p64_v64"], NVECS["7x3"]), gauss_net(ARCHS["p64_v64"])
    c = make_ppo(tmp_path / "cat", net)
    c.save()
    g = make_ppo(tmp_path / "gauss", gauss)
    g.save()
    assert make_ppo(tmp_path / "cat", gauss).load_latest_checkpoint() is False
    assert make_ppo(tmp_path / "gauss", net).load_latest_checkpoint() is False
    assert make_ppo(tmp_path / "cat", cat_net(ARCHS["p64_v64"], (5, 5))).load_latest_checkpoint() is False
    back = make_ppo(tmp_path / "cat", net)
    assert back.load_latest_checkpoint() is True
    assert np.array_equal(back.params.cpu().numpy(), c.params.cpu().numpy())
