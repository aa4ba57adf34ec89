"""Categorical PPO heads on the device (cpb_ppo_cat_*): every entry point against the float64 restatement
tests/ppo_categorical_oracle.py over Discrete / MultiDiscrete spaces from (2,) to (31, 33) and architectures from one
layer per trunk to eight, with the workspace filled with NaN before each call; determinism and launch counts equal to the
Gaussian head's; the fused actor; train.py with --discrete_actions; checkpoints."""
import os
import subprocess
import sys

import numpy as np
import pytest

import ppo_categorical_oracle as pco
from harness import lib, make_conv_vae, make_mlp  # noqa: F401
from helpers import committed_frames, rel_l2, shipped_vae_weights
from ppo_cases import CLIP_HI, CLIP_LO, train_params, warm_adam
from ppo_categorical_cases import (ARCHS, LR, NVECS, S, f64, kink_free, learn_refs, learn_setup, make_batch, make_ppo,
                                   relu_margin)
from vae_checks import mlp_weights

pytestmark = pytest.mark.gpu

TOL = 1e-5
KINK_MARGIN = 1e-4


def _nan_workspace(m, *shape):
    ws = m._workspace(*shape)
    ws.fill_(0xFF)                  # every float of the workspace reads as NaN until written
    return ws


def _gate(got, r64, r32):
    """max(TOL, 2 x the float32 restatement's distance from float64)"""
    return rel_l2(got, r64) < max(TOL, 2 * rel_l2(r32, r64))


def _predict_states(arch, cats, n, seed, state_dim):
    """n states on which every component's top two logits differ by more than 1e-3 (chosen from 4n candidates that the
    trunk biases were placed on), and the network"""
    rs = np.random.RandomState(seed)
    cand = rs.randn(4 * n, state_dim).astype(np.float32)
    p = kink_free(arch, cats, cand, seed + 1, state_dim)
    z, _ = pco.forward(f64(p), cand.astype(np.float64))
    off = pco.offsets(cats)
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
    cats, net = NVECS[nvec], ARCHS[arch]
    p, s = _predict_states(net, cats, 37, 1, state_dim)
    assert relu_margin(p, s) > KINK_MARGIN and pco.logit_gap(f64(p), s, cats) > 1e-4
    m = make_ppo(tmp_path, net, cats, p, state_dim=state_dim)
    # uniforms at least 1e-5 from every CDF boundary of the restatement
    rs = np.random.RandomState(2)
    bounds = pco.cdf_bounds(f64(p), s, cats)
    u = rs.rand(37, len(cats))
    for _ in range(100):
        near = np.stack([np.abs(bounds[k] - u[:, k:k + 1]).min(axis=1) < 1e-5 for k in range(len(cats))], axis=1)
        if not near.any():
            break
        u[near] = rs.rand(int(near.sum()))
    assert min(np.abs(bounds[k] - u[:, k:k + 1]).min() for k in range(len(cats))) >= 1e-5
    u = u.astype(np.float32)
    for nz in (None, u):
        _nan_workspace(m, 37)
        act, val = m.predict(s, greedy=nz is None, noise=nz)
        ract, rval = pco.predict(f64(p), s, cats, noise=None if nz is None else nz.astype(np.float64))
        assert act.dtype == np.int64 and np.array_equal(act, ract), (nz is None, act, ract)
        assert rel_l2(val, rval) < TOL


def _check_loss(m, p, old, s, a, ret, adv, cats, entropy_scale=0.01):
    metrics, grads = m.loss_and_grads(s, a, ret, adv)
    r64 = pco.loss_and_grads(p, old, s, a, ret, adv, cats, 0.2, 1.0, entropy_scale)
    r32 = pco.loss_and_grads(p, old, s, a, ret, adv, cats, 0.2, 1.0, entropy_scale, dtype=np.float32)
    assert np.isfinite(metrics).all()
    for i, k in enumerate(("policy_loss", "value_loss", "entropy_loss", "loss", "mean_ratio")):
        if r64[k] == 0.0:
            assert metrics[i] == 0.0, k
            continue
        assert _gate(np.atleast_1d(metrics[i]), np.atleast_1d(r64[k]), np.atleast_1d(r32[k])), k
    assert set(grads) == set(r64["grads"])
    for k, g in grads.items():
        assert np.isfinite(g).all(), k
        assert _gate(g, r64["grads"][k], r32["grads"][k]), (k, rel_l2(g, r64["grads"][k]))
    return r64


@pytest.mark.parametrize("B", [1, 9, 256, 8200])
@pytest.mark.parametrize("nvec", list(NVECS))
def test_loss_and_gradients(tmp_path, nvec, B):
    cats, net = NVECS[nvec], ARCHS["default"]
    p, old, s, a, ret, adv = make_batch(net, cats, B, seed=3 + B)
    assert relu_margin(p, s) > KINK_MARGIN
    m = make_ppo(tmp_path, net, cats, p, old)
    _nan_workspace(m, B)
    r64 = _check_loss(m, p, old, s, a, ret, adv, cats)
    ratio = r64["ratio"]
    assert not (np.minimum(np.abs(ratio - CLIP_LO), np.abs(ratio - CLIP_HI)) < 1e-4).any()
    if B >= 256:
        for frac in ((ratio < CLIP_LO).mean(), (ratio > CLIP_HI).mean(), ((ratio >= CLIP_LO) & (ratio <= CLIP_HI)).mean()):
            assert frac >= 0.1, frac


@pytest.mark.parametrize("arch", list(ARCHS))
def test_loss_and_gradients_architectures(tmp_path, arch):
    cats = NVECS["7x3"]
    p, old, s, a, ret, adv = make_batch(ARCHS[arch], cats, 256, seed=11)
    m = make_ppo(tmp_path, ARCHS[arch], cats, p, old)
    _nan_workspace(m, 256)
    _check_loss(m, p, old, s, a, ret, adv, cats)


@pytest.mark.parametrize("case", ["entropy_only", "policy_only"])
def test_entropy_only_and_policy_only(tmp_path, case):
    cats = NVECS["31x33"]
    p, old, s, a, ret, adv = make_batch(ARCHS["p64_v64"], cats, 256, seed=21)
    es = 0.01
    if case == "entropy_only":
        adv = np.zeros_like(adv)
    else:
        es = 0.0
    m = make_ppo(tmp_path, ARCHS["p64_v64"], cats, p, old, entropy_scale=es)
    _nan_workspace(m, 256)
    _check_loss(m, p, old, s, a, ret, adv, cats, entropy_scale=es)


def test_two_train_steps(tmp_path):
    from oracle import vae_oracle as vo
    cats, net = NVECS["7x3"], ARCHS["odd"]
    p, old, s, a, ret, adv = make_batch(net, cats, 64, seed=17)
    m_, v_, powers = warm_adam(p, pco.loss_and_grads(p, old, s, a, ret, adv, cats, 0.2, 1.0, 0.01)["grads"], 19)
    m = make_ppo(tmp_path, net, cats, p, old)
    m.set_weights(p, old, m_, v_, powers)
    for _ in range(2):
        _nan_workspace(m, 64)
        m.train(s, a, ret, adv)

    def steps(dtype):
        q = {k: x.astype(dtype) for k, x in p.items()}
        st = dict(m={k: m_[k].astype(dtype) for k in p}, v={k: v_[k].astype(dtype) for k in p}, beta1_power=powers[0],
                  beta2_power=powers[1])
        for _ in range(2):
            vo.adam_apply(q, pco.loss_and_grads(q, old, s, a, ret, adv, cats, 0.2, 1.0, 0.01, dtype=dtype)["grads"], st, LR)
        return q
    p64, p32 = steps(np.float64), steps(np.float32)
    got = m.get_weights()
    for k in p64:
        assert _gate(got[k], p64[k], p32[k]), k


def _check_learn(got, metrics, refs, applied=None):
    (p64, rec64, n64), (p32, rec32, _) = refs
    for k in p64:
        assert np.isfinite(got[k]).all(), k
        assert _gate(got[k], p64[k], p32[k]), (k, rel_l2(got[k], p64[k]))
    ok = ~np.isnan(rec64[:, 0])
    assert np.array_equal(np.isnan(metrics[:, 0]), ~ok)
    for col in range(metrics.shape[1]):
        assert (_gate(metrics[ok, col], rec64[ok, col], rec32[ok, col])
                or (col == 5 and np.abs(metrics[ok, col] - rec64[ok, col]).max() < 1e-6)), col
    if applied is not None:
        assert applied == n64


def _five(refs):
    return (refs[0][0], refs[0][1][:, :5], refs[0][2]), (refs[1][0], refs[1][1][:, :5], 0)


_PERSISTENT_SNIPPET = r"""
import sys, numpy as np
sys.path[:0] = [%r, %r]
from pathlib import Path
import ppo_categorical_cases as t
out = {}
for arch, nvec in %r:
    w, metrics = t.persistent_learn(Path(%r) / (arch + nvec), arch, nvec, 2048, 256, 4)
    out.update({arch + nvec + ":" + k: x for k, x in w.items()})
    out[arch + nvec + ":metrics"] = metrics
np.savez(%r, **out)
"""
_LEARN_CASES = [("default", "7x3"), ("default", "64"), ("odd", "2x2x2x2"), ("deep", "31x33"), ("p64_v64", "2")]


def test_learn_both_paths(tmp_path):
    """T = 2048 in 4 epochs of 8 minibatches of 256: launch per kernel and the persistent kernel against float64, and
    the persistent kernel within 1e-6 of launch per kernel."""
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    outs = []
    for flag in ("0", "1"):
        path = str(tmp_path / ("w%s.npz" % flag))
        code = _PERSISTENT_SNIPPET % (root, os.path.join(root, "tests"), _LEARN_CASES, str(tmp_path / ("m" + flag)), path)
        res = subprocess.run([sys.executable, "-c", code], env=dict(os.environ, CPB_PPO_PERSISTENT=flag),
                             capture_output=True, text=True, timeout=1200)
        assert res.returncode == 0, res.stderr[-3000:]
        outs.append(dict(np.load(path)))
    for arch, nvec in _LEARN_CASES:
        cats, tag = NVECS[nvec], arch + nvec
        p, data, perms, adam = learn_setup(ARCHS[arch], cats, 2048, 4, seed=40)
        refs = learn_refs(p, cats, data, perms, 256, adam)
        for o in outs:
            _check_learn({k: o[tag + ":" + k] for k in p}, o[tag + ":metrics"], _five(refs))
        for k in p:
            assert rel_l2(outs[1][tag + ":" + k], outs[0][tag + ":" + k]) < 1e-6, (tag, k)


def test_learn_segments(tmp_path):
    """16 segments x 128 rows."""
    cats, net = NVECS["7x3"], ARCHS["odd"]
    p, data, perms, adam = learn_setup(net, cats, 2048, 2, seed=50)
    s, a, r, v, d = data
    lengths = [128] * 16
    boot = np.random.RandomState(51).randn(16)
    m = make_ppo(tmp_path, net, cats, p)
    m.set_weights(p, p, adam[0], adam[1], adam[2])
    _nan_workspace(m, 256, 2048)
    metrics = m.learn(s, a, v, r, d, boot, num_epochs=2, batch_size=256, perms=perms, return_metrics=True,
                      segment_lengths=lengths)
    refs = learn_refs(p, cats, data, perms, 256, adam, segment_lengths=lengths, bootstrap_values=boot)
    _check_learn(m.get_weights(), metrics, _five(refs))


@pytest.mark.parametrize("nvec", ["7x3", "64"])
def test_learn_opts_clip_and_kl_stop(tmp_path, nvec):
    """Clipping binding on 25-75 % of the minibatches, then a KL stop at a minibatch k > 1 (steps_applied = k)."""
    cats, net = NVECS[nvec], ARCHS["p64_v64"]
    lr = 3e-3
    p, data, perms, adam = learn_setup(net, cats, 2048, 4, seed=60)
    s, a, r, v, d = data
    (_, rec0, _), _ = learn_refs(p, cats, data, perms, 256, adam, lr=lr)
    for q in (0.375, 0.5, 0.625):
        max_norm = float(np.quantile(rec0[:, 6], q))
        (_, rec, _), _ = learn_refs(p, cats, data, perms, 256, adam, lr=lr, max_grad_norm=max_norm)
        clipped = (rec[:, 6] > max_norm).mean()
        if 0.25 <= clipped <= 0.75:
            break
    assert 0.25 <= clipped <= 0.75, clipped
    kl = rec[:, 5]
    k = next(i for i in range(2, len(kl)) if kl[i] > 1.2 * kl[:i].max() and kl[i] > 1e-5)
    target_kl = float((kl[:k].max() + kl[k]) / 2 / 1.5)
    refs = learn_refs(p, cats, data, perms, 256, adam, lr=lr, max_grad_norm=max_norm, target_kl=target_kl)
    assert refs[0][2] == k > 1, (refs[0][2], k)
    m = make_ppo(tmp_path, net, cats, p, learning_rate=lr)
    m.set_weights(p, p, adam[0], adam[1], adam[2])
    _nan_workspace(m, 256, 2048)
    metrics = m.learn(s, a, v, r, d, 0.3, num_epochs=4, batch_size=256, perms=perms, return_metrics=True,
                      max_grad_norm=max_norm, target_kl=target_kl)
    _check_learn(m.get_weights(), metrics, refs, applied=int(m.last_steps_applied.item()))


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
    from ppo_depth_cases import make_ppo as make_gauss_ppo
    for arch in ("default", "odd"):
        net = ARCHS[arch]
        cats = NVECS["7x3"]
        p, old, s, a, ret, adv = make_batch(net, cats, 256, seed=31)
        u = np.random.RandomState(3).rand(256, 2).astype(np.float32)
        m = make_ppo(tmp_path / arch, net, cats, p, old)
        r1, l1 = _one_of_each(m, s, a, ret, adv, u, p, old, lib)
        r2, _ = _one_of_each(m, s, a, ret, adv, u, p, old, lib)
        for k in r1:
            x, y = r1[k], r2[k]
            flat = lambda t: [np.asarray(v.cpu() if isinstance(v, torch.Tensor) else v) for v in (t if isinstance(t, tuple) else (t,))]
            for xi, yi in zip(flat(x), flat(y)):
                if isinstance(xi, np.ndarray) and xi.dtype == object:
                    continue
                assert np.array_equal(xi, yi), (arch, k)
        g = make_gauss_ppo(tmp_path / ("g" + arch), net)
        _, lg = _one_of_each(g, s, np.zeros((256, 2), np.float32), ret, adv, np.random.RandomState(3).randn(256, 2)
                             .astype(np.float32), g.get_weights(), g.get_weights(), lib)
        assert l1 == lg, (arch, l1, lg)


# ----------------------------------------------------------------------------------------------------- fused actor
def _vae(tmp_path, kind):
    if kind == "conv":
        return make_conv_vae(tmp_path, shipped_vae_weights()[0], loss="bce", tag="vae", training=False)
    enc, dec = (96, 256, 64), (160, 64)
    return make_mlp(tmp_path, mlp_weights(2, encoder_sizes=enc, decoder_sizes=dec), enc, dec, tag="vec", training=False)


def _fake_envs(n):
    import types
    rgb, _ = committed_frames()
    envs = []
    for i in range(n):
        v = types.SimpleNamespace(control=types.SimpleNamespace(steer=0.1 * (i % 7) - 0.3, throttle=0.05 * (i % 11)),
                                  get_speed=(lambda s=0.37 * i: s))
        envs.append(types.SimpleNamespace(observation=rgb[(5 * i) % len(rgb)], vehicle=v))
    return envs


@pytest.mark.parametrize("kind", ["conv", "mlp"])
@pytest.mark.parametrize("n", [1, 4])
def test_fused_actor_equals_unfused(tmp_path, lib, kind, n):
    from carla_ppo_b200.actor import FusedActor, UnfusedActor
    net, cats = ARCHS["odd"], NVECS["7x3"]
    vae = _vae(tmp_path, kind)
    meas = ("steer", "throttle", "speed")
    p = pco.init_params(S, cats, net[0], net[1], seed=90)
    p["action_logits/bias"] = np.random.RandomState(91).randn(10).astype(np.float32)      # a policy far from uniform
    models = [make_ppo(tmp_path / tag, net, cats, p) for tag in ("fused", "unfused")]
    envs = _fake_envs(n)
    for greedy in (False, True):
        fa_, ua_ = FusedActor(vae, models[0], meas), UnfusedActor(vae, models[1], meas)
        fa_.greedy = ua_.greedy = greedy
        fs, fa, fv = fa_.encode_predict(envs)
        us, ua, uv = ua_.encode_predict(envs)
        assert all(np.array_equal(x, y) for x, y in zip(fs, us))
        assert fa.dtype == ua.dtype == np.int64
        assert np.array_equal(fa, ua) and np.array_equal(fv, uv)
        assert (fa >= 0).all() and (fa < np.asarray(cats)).all()


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
    from ppo_depth_cases import make_ppo as make_gauss_ppo
    net, cats = ARCHS["p64_v64"], NVECS["7x3"]
    c = make_ppo(tmp_path / "cat", net, cats)
    c.save()
    g = make_gauss_ppo(tmp_path / "gauss", net)
    g.save()
    assert make_gauss_ppo(tmp_path / "cat", net).load_latest_checkpoint() is False
    assert make_ppo(tmp_path / "gauss", net, cats).load_latest_checkpoint() is False
    assert make_ppo(tmp_path / "cat", net, (5, 5)).load_latest_checkpoint() is False
    back = make_ppo(tmp_path / "cat", net, cats)
    assert back.load_latest_checkpoint() is True
    assert np.array_equal(back.params.cpu().numpy(), c.params.cpu().numpy())
