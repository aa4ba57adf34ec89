"""PPO policy / value trunks of any depth on the device (cpb_ppo_spec_*): every entry point against the float64
restatement tests/ppo_restatement.py at architectures from one unit per trunk to eight layers and 2048 wide, with the
workspace filled with NaN before each call; the default architecture through the spec bit for bit the legacy entry
points; the fused actor; checkpoints of a non-default architecture."""
import os

import numpy as np
import pytest

import ppo_restatement as pr
from harness import lib, library_state  # noqa: F401
from helpers import rel_l2
from ppo_cases import ARCHS, KINK_MARGIN, gauss_net, learn_refs, learn_setup, make_batch, make_ppo
from ppo_checks import (TOL, actor_vae, check_fused_actor, check_learn, check_learn_opts_clip_and_kl_stop,
                        check_learn_segments, check_loss, check_two_train_steps, five, fresh_process, nan_workspace)

pytestmark = pytest.mark.gpu

A, S = 2, 67


@pytest.mark.parametrize("arch", list(ARCHS))
def test_predict_greedy_and_sampled(tmp_path, arch):
    net = gauss_net(ARCHS[arch])
    low, high = net[1]
    p, _, s, _, _, _ = make_batch(net, 37, 1)
    assert pr.relu_margin(p, s) > KINK_MARGIN
    m = make_ppo(tmp_path, net, p)
    p64 = {k: v.astype(np.float64) for k, v in p.items()}
    noise = np.random.RandomState(2).randn(37, A).astype(np.float32) * 4.0        # clips at both bounds
    for nz in (None, noise):
        nan_workspace(m, 37)
        act, val = m.predict(s, greedy=nz is None, noise=nz)
        assert np.isfinite(act).all() and np.isfinite(val).all()
        ract, rval = pr.predict(p64, s.astype(np.float64), net[1], noise=nz)
        assert rel_l2(act, ract) < TOL and rel_l2(val, rval) < TOL, (rel_l2(act, ract), rel_l2(val, rval))
    assert (act == low).any() and (act == high).any()


@pytest.mark.parametrize("B", [1, 9, 256, 8200])
@pytest.mark.parametrize("arch", list(ARCHS))
def test_loss_and_gradients(tmp_path, arch, B):
    net = gauss_net(ARCHS[arch])
    p, old, s, a, ret, adv = make_batch(net, B, 3 + B)
    assert pr.relu_margin(p, s) > KINK_MARGIN
    m = make_ppo(tmp_path, net, p, old)
    nan_workspace(m, B)
    check_loss(m, p, old, s, a, ret, adv, net[1])


@pytest.mark.parametrize("arch", list(ARCHS))
def test_two_train_steps(tmp_path, arch):
    net = gauss_net(ARCHS[arch])
    check_two_train_steps(tmp_path, net, make_batch(net, 64, 17))


@pytest.mark.parametrize("arch", list(ARCHS))
def test_learn(tmp_path, arch):
    """T = 2048 in 4 epochs of 8 minibatches of 256, launch per kernel."""
    net = gauss_net(ARCHS[arch])
    p, data, perms, adam = learn_setup(net, 2048, 4, 40)
    assert pr.relu_margin(p, data[0]) > KINK_MARGIN
    m = make_ppo(tmp_path, net, p)
    m.set_weights(p, p, *adam)
    s, a, r, v, d = data
    nan_workspace(m, 256, 2048)
    metrics = m.learn(s, a, v, r, d, 0.3, num_epochs=4, batch_size=256, perms=perms, return_metrics=True)
    check_learn(m.get_weights(), metrics, five(learn_refs(net, p, data, perms, 256, adam)))


def test_persistent_learn_equals_launch_per_kernel(tmp_path):
    """The persistent kernel (CPB_PPO_PERSISTENT=1, read once per process) at every architecture: within 1e-6 of the
    launch-per-kernel path, and within the float32 gate of float64."""
    cases = [(name, gauss_net(arch), ("rollout", 2048, 4, 256, 40), {}) for name, arch in ARCHS.items()]
    outs = fresh_process(tmp_path, cases)
    for name, arch in ARCHS.items():
        net = gauss_net(arch)
        p, data, perms, adam = learn_setup(net, 2048, 4, 40)
        w1 = {k: outs[1][name + ":w:" + k] for k in p}
        check_learn(w1, outs[1][name + ":metrics"], five(learn_refs(net, p, data, perms, 256, adam)))
        for k in p:
            assert rel_l2(w1[k], outs[0][name + ":w:" + k]) < 1e-6, (name, k)


@pytest.mark.parametrize("arch", list(ARCHS))
def test_learn_segments(tmp_path, arch):
    """16 segments x 128 rows."""
    check_learn_segments(tmp_path, gauss_net(ARCHS[arch]))


@pytest.mark.parametrize("arch", list(ARCHS))
def test_learn_opts_clip_and_kl_stop(tmp_path, arch):
    """Clipping binding on 25-75 % of the minibatches, then a KL stop at a minibatch k > 1 (steps_applied = k).  The
    learning rate is 3e-3 so that the approximate KL of the later minibatches stands well above float32 rounding."""
    check_learn_opts_clip_and_kl_stop(tmp_path, gauss_net(ARCHS[arch]))


# ------------------------------------------------------------------------------ the default architecture: spec == legacy
def test_default_architecture_spec_equals_legacy(tmp_path):
    """learn, learn_opts, learn_segments and learn_segments_opts through the spec twins and through the legacy entry
    points: parameters, theta_old, Adam m / v, beta powers, metrics, steps_applied and launch counts identical, on the
    launch-per-kernel path and in the persistent kernel."""
    for flag, o in zip("01", fresh_process(tmp_path, 70, body="spec_vs_legacy", timeout=600)):
        legacy = {k[2:]: x for k, x in o.items() if k.startswith("0:")}
        spec = {k[2:]: x for k, x in o.items() if k.startswith("1:")}
        assert legacy.keys() == spec.keys() and len(legacy) > 0
        for k in legacy:
            assert np.array_equal(legacy[k], spec[k], equal_nan=True), (flag, k)


def test_default_architecture_predict_train_loss_equal_legacy(tmp_path, lib):
    import ctypes as C
    import torch
    from carla_ppo_b200 import _lib
    p, old, s, a, ret, adv = make_batch(gauss_net(ARCHS["default"]), 256, 80)
    m = make_ppo(tmp_path, gauss_net(ARCHS["default"]), p, old)
    ptr = _lib.ptr
    st, at = torch.from_numpy(s).cuda(), torch.from_numpy(a).cuda()
    rt, vt = torch.from_numpy(ret).cuda(), torch.from_numpy(adv).cuda()
    noise = torch.randn(256, A, device="cuda")
    results = []
    for name, cfg in (("cpb_ppo_", m._c), ("cpb_ppo_spec_", m._spec)):
        m.set_weights(p, old)
        m.adam_m.zero_(); m.adam_v.zero_()
        m.adam_powers.copy_(torch.tensor([0.9, 0.999]))
        ws = m._workspace(256)
        out = torch.empty(256 * (A + 1), device="cuda")
        met = torch.empty(5, device="cuda")
        met7 = torch.empty(7, device="cuda")
        lib.cpb_reset_launch_count()
        _lib.check(getattr(lib, name + "forward")(C.byref(cfg), ptr(m.params), ptr(st), 256, ptr(noise), ptr(out),
                                                  ptr(out[256 * A:]), ptr(ws), ws.numel(), None))
        _lib.check(getattr(lib, name + "loss_grad")(C.byref(cfg), ptr(m.params), ptr(m.params_old), ptr(st), ptr(at),
                                                    ptr(rt), ptr(vt), None, 256, ptr(m.grads), ptr(met), ptr(ws),
                                                    ws.numel(), None))
        g = m.grads.cpu().numpy()
        _lib.check(getattr(lib, name + "train_step")(C.byref(cfg), ptr(m.params), ptr(m.params_old), ptr(m.grads),
                                                     ptr(m.adam_m), ptr(m.adam_v), ptr(m.adam_powers), ptr(m._lr_dev),
                                                     ptr(st), ptr(at), ptr(rt), ptr(vt), None, 256, ptr(met), ptr(ws),
                                                     ws.numel(), None))
        opts = _lib.PpoLearnOptions(0.01, 0.0)
        applied = torch.zeros(1, dtype=torch.int32, device="cuda")
        _lib.check(getattr(lib, name + "train_step_opts")(C.byref(cfg), ptr(m.params), ptr(m.params_old), ptr(m.grads),
                                                          ptr(m.adam_m), ptr(m.adam_v), ptr(m.adam_powers),
                                                          ptr(m._lr_dev), ptr(st), ptr(at), ptr(rt), ptr(vt), None, 256,
                                                          ptr(met7), C.byref(opts), None, ptr(applied), ptr(ws),
                                                          ws.numel(), None))
        torch.cuda.synchronize()
        results.append(dict(out=out.cpu().numpy(), g=g, params=m.params.cpu().numpy(), m=m.adam_m.cpu().numpy(),
                            v=m.adam_v.cpu().numpy(), pw=m.adam_powers.cpu().numpy(), met=met.cpu().numpy(),
                            met7=met7.cpu().numpy(), applied=applied.cpu().numpy(), launches=lib.cpb_launch_count()))
    for k in results[0]:
        assert np.array_equal(results[0][k], results[1][k]), k


@pytest.mark.parametrize("kind", ["conv", "mlp"])
def test_default_architecture_actor_twins_equal_legacy(tmp_path, lib, kind):
    """cpb_vae_spec_ppo_spec_encode_predict = cpb_vae_spec_encode_predict and cpb_mlpvae_ppo_spec_encode_predict =
    cpb_mlpvae_encode_predict at the default PPO, bit for bit with equal launch counts, greedy and sampled."""
    import ctypes as C
    import torch
    from carla_ppo_b200 import _lib
    from helpers import committed_frames
    legacy = {"conv": "cpb_vae_spec_encode_predict", "mlp": "cpb_mlpvae_encode_predict"}[kind]
    vae = actor_vae(tmp_path, kind)
    net = gauss_net(ARCHS["default"])
    m = make_ppo(tmp_path / "ppo", net, pr.init_params(*net, seed=5))
    n = 4
    rgb, _ = committed_frames()
    frames = torch.from_numpy(np.ascontiguousarray(rgb[:n])).cuda()
    meas = torch.randn(n, 3, device="cuda")
    noise = torch.randn(n, A, device="cuda")
    cfg = vae._config(n, _lib.FRAME_U8)
    ws_v, ws_p = vae._workspace(n, _lib.WS_ENCODE), m._workspace(n)
    ptr = _lib.ptr
    for nz in (None, noise):
        res = []
        for name, ppo_arg in ((legacy, m._c), (vae._API["encode_predict"], m._spec)):
            lat, st = torch.empty(n, 64, device="cuda"), torch.empty(n, S, device="cuda")
            act, val = torch.empty(n, A, device="cuda"), torch.empty(n, device="cuda")
            ws_p.fill_(0xFF)
            lib.cpb_reset_launch_count()
            _lib.check(getattr(lib, name)(C.byref(cfg), ptr(vae.params), ptr(frames), ptr(meas), 3, C.byref(ppo_arg),
                                          ptr(m.params), ptr(nz), ptr(lat), ptr(st), ptr(act), ptr(val), ptr(vae._flags),
                                          ptr(ws_v), ws_v.numel(), ptr(ws_p), ws_p.numel(), None), name)
            torch.cuda.synchronize()
            res.append((lib.cpb_launch_count(), st.cpu().numpy(), act.cpu().numpy(), val.cpu().numpy()))
        assert res[0][0] == res[1][0]
        assert all(np.array_equal(x, y) for x, y in zip(res[0][1:], res[1][1:]))
        assert np.isfinite(res[1][2]).all()


# ----------------------------------------------------------------------------------------------------- fused actor
@pytest.mark.parametrize("kind", ["conv", "mlp"])
@pytest.mark.parametrize("n", [1, 4])
def test_fused_actor_equals_unfused(tmp_path, lib, kind, n):
    check_fused_actor(tmp_path, gauss_net(ARCHS["odd"]), kind, n, greedy=(False,))


# ------------------------------------------------------------------------------------------------------ checkpoints
@pytest.mark.parametrize("tf_format", [False, True])
def test_checkpoint_round_trip_and_architecture_refusal(tmp_path, tf_format):
    from carla_ppo_b200.ppo import checkpoint_architecture
    net = ARCHS["odd"]
    p, data, perms, adam = learn_setup(gauss_net(net), 512, 1, 100)
    a = make_ppo(tmp_path / "a", gauss_net(net), p)
    a.set_weights(p, p, *adam)
    s, act, r, v, d = data
    a.learn(s, act, v, r, d, 0.3, num_epochs=1, batch_size=128, perms=perms)
    a.episode_counter = 3
    a.save(tf_format=tf_format)
    assert checkpoint_architecture(a.checkpoint_dir) == net
    b = make_ppo(tmp_path / "a", gauss_net(net))
    assert b.load_latest_checkpoint() is True
    for x, y in ((a.params, b.params), (a.params_old, b.params_old), (a.adam_m, b.adam_m), (a.adam_v, b.adam_v),
                 (a.adam_powers, b.adam_powers)):
        assert np.array_equal(x.cpu().numpy(), y.cpu().numpy())
    assert b.get_episode_idx() == 3
    for other in (ARCHS["default"], ((33, 7, 65), (32,))):
        c = make_ppo(tmp_path / "a", gauss_net(other))
        before = c.params.cpu().numpy().copy()
        assert c.load_latest_checkpoint() is False
        assert np.array_equal(before, c.params.cpu().numpy())


def test_train_four_envs_fused_equals_unfused_and_resume(tmp_path):
    """train.train with 4 environments at (256, 256) / (256, 256, 256): fused == unfused bit for bit; the checkpoint
    carries the architecture; resuming takes it, and a size flag that disagrees with it is refused before training."""
    from carla_ppo_b200.ppo import checkpoint_architecture
    from carla_ppo_b200.replay_env import ReplayEnv
    from carla_ppo_b200.train import train
    from helpers import committed_frames
    from ppo_cases import shipped_vae, train_params
    rgb, _ = committed_frames()
    net = ((256, 256), (256, 256, 256))
    envs = lambda: [ReplayEnv(rgb, episode_length=24 + 5 * i, seed=0) for i in range(4)]
    models = []
    for tag, unfused in (("f4", False), ("u4", True)):
        params = train_params(tag, num_envs=4, eval_interval=1000, unfused=unfused, policy_hidden_sizes=[256, 256],
                              value_hidden_sizes=[256, 256, 256])
        models.append(train(params, restart=False, env=envs(), vae=shipped_vae(tmp_path, tag),
                            models_root=str(tmp_path / "models"), interactive=False))
    wa, wb = models[0].get_weights(), models[1].get_weights()
    assert models[0].architecture == net and models[0].get_train_step_idx() > 0
    assert all(np.array_equal(wa[k], wb[k]) for k in wa) and models[0].reward_history == models[1].reward_history
    models[0].save()
    assert checkpoint_architecture(os.path.join(str(tmp_path / "models"), "f4", "checkpoints")) == net
    resumed = train(train_params("f4", num_envs=4), restart=False, env=envs(),      # already at its 2 episodes
                    vae=shipped_vae(tmp_path, "r"), models_root=str(tmp_path / "models"), interactive=False)
    assert resumed.architecture == net
    assert np.array_equal(resumed.params.cpu().numpy(), models[0].params.cpu().numpy())
    # run_eval builds its PPO from the checkpoint (run_eval.main's load_model)
    from carla_ppo_b200.run_eval import load_model
    ev = load_model(np.array([S]), envs()[0].action_space, os.path.join(str(tmp_path / "models"), "f4"))
    assert ev.architecture == net
    for x, y in ((ev.params, models[0].params), (ev.params_old, models[0].params_old)):
        assert np.array_equal(x.cpu().numpy(), y.cpu().numpy())
    with pytest.raises(ValueError, match="disagrees"):
        train(train_params("f4", num_envs=4, value_hidden_sizes=[500, 300]), restart=False, env=envs(),
              vae=shipped_vae(tmp_path, "x"), models_root=str(tmp_path / "models"), interactive=False)
