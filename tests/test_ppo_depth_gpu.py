"""PPO policy / value trunks of any depth on the device (cpb_ppo_spec_*): every entry point against the float64
restatement tests/ppo_depth_oracle.py at architectures from one unit per trunk to eight layers and 2048 wide, with the
workspace filled with NaN before each call; the default architecture through the spec bit for bit the legacy entry
points; the fused actor; checkpoints of a non-default architecture."""
import os
import subprocess
import sys

import numpy as np
import pytest

import ppo_depth_oracle as pdo
from harness import lib, library_state, make_conv_vae, make_mlp  # noqa: F401
from helpers import rel_l2, shipped_vae_weights
from ppo_depth_cases import A, ARCHS, KINK_MARGIN, LR, S, learn_refs, learn_setup, make_batch, make_ppo
from ppo_cases import bounds
from vae_checks import mlp_weights

pytestmark = pytest.mark.gpu

TOL = 1e-5


def _nan_workspace(m, *shape):
    ws = m._workspace(*shape)
    ws.fill_(0xFF)                  # every float of the workspace reads as NaN until written
    return ws


def _gate(got, r64, r32):
    """max(TOL, 2 x the float32 restatement's distance from float64)"""
    return rel_l2(got, r64) < max(TOL, 2 * rel_l2(r32, r64))


@pytest.mark.parametrize("arch", list(ARCHS))
def test_predict_greedy_and_sampled(tmp_path, arch):
    net = ARCHS[arch]
    p, _, s, _, _, _ = make_batch(net, 37, seed=1)
    assert pdo.relu_margin(p, s) > KINK_MARGIN
    m = make_ppo(tmp_path, net, p)
    low, high = bounds(A)
    p64 = {k: v.astype(np.float64) for k, v in p.items()}
    noise = np.random.RandomState(2).randn(37, A).astype(np.float32) * 4.0        # clips at both bounds
    for nz in (None, noise):
        _nan_workspace(m, 37)
        act, val = m.predict(s, greedy=nz is None, noise=nz)
        assert np.isfinite(act).all() and np.isfinite(val).all()
        ract, rval = pdo.predict(p64, s.astype(np.float64), low, high, noise=nz)
        assert rel_l2(act, ract) < TOL and rel_l2(val, rval) < TOL, (rel_l2(act, ract), rel_l2(val, rval))
    assert (act == low).any() and (act == high).any()


@pytest.mark.parametrize("B", [1, 9, 256, 8200])
@pytest.mark.parametrize("arch", list(ARCHS))
def test_loss_and_gradients(tmp_path, arch, B):
    net = ARCHS[arch]
    low, high = bounds(A)
    p, old, s, a, ret, adv = make_batch(net, B, seed=3 + B)
    assert pdo.relu_margin(p, s) > KINK_MARGIN
    m = make_ppo(tmp_path, net, p, old)
    _nan_workspace(m, B)
    metrics, grads = m.loss_and_grads(s, a, ret, adv)
    r64 = pdo.loss_and_grads(p, old, s, a, ret, adv, low, high, 0.2, 1.0, 0.01)
    r32 = pdo.loss_and_grads(p, old, s, a, ret, adv, low, high, 0.2, 1.0, 0.01, dtype=np.float32)
    assert np.isfinite(metrics).all()
    for i, k in enumerate(("policy_loss", "value_loss", "entropy_loss", "loss", "mean_ratio")):
        assert _gate(np.atleast_1d(metrics[i]), np.atleast_1d(r64[k]), np.atleast_1d(r32[k])), k
    assert set(grads) == set(r64["grads"])
    for k, g in grads.items():
        assert np.isfinite(g).all(), k
        assert _gate(g, r64["grads"][k], r32["grads"][k]), (k, rel_l2(g, r64["grads"][k]))


@pytest.mark.parametrize("arch", list(ARCHS))
def test_two_train_steps(tmp_path, arch):
    from oracle import vae_oracle as vo
    from ppo_cases import warm_adam
    net = ARCHS[arch]
    low, high = bounds(A)
    p, old, s, a, ret, adv = make_batch(net, 64, seed=17)
    m_, v_, powers = warm_adam(p, pdo.loss_and_grads(p, old, s, a, ret, adv, low, high, 0.2, 1.0, 0.01)["grads"], 19)
    m = make_ppo(tmp_path, net, p, old)
    m.set_weights(p, old, m_, v_, powers)
    for _ in range(2):
        _nan_workspace(m, 64)
        m.train(s, a, ret, adv)

    def steps(dtype):
        q = {k: x.astype(dtype) for k, x in p.items()}
        st = dict(m={k: m_[k].astype(dtype) for k in p}, v={k: v_[k].astype(dtype) for k in p}, beta1_power=powers[0],
                  beta2_power=powers[1])
        for _ in range(2):
            vo.adam_apply(q, pdo.loss_and_grads(q, old, s, a, ret, adv, low, high, 0.2, 1.0, 0.01, dtype=dtype)["grads"],
                          st, LR)
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
    ncol = metrics.shape[1]
    ok = ~np.isnan(rec64[:, 0])
    assert np.array_equal(np.isnan(metrics[:, 0]), ~ok)
    for col in range(ncol):
        # approx_kl (column 5) is 0 at the first minibatch and ~1e-8 soon after: gated absolutely as well
        assert (_gate(metrics[ok, col], rec64[ok, col], rec32[ok, col])
                or (col == 5 and np.abs(metrics[ok, col] - rec64[ok, col]).max() < 1e-6)), col
    if applied is not None:
        assert applied == n64


@pytest.mark.parametrize("arch", list(ARCHS))
def test_learn(tmp_path, arch):
    """T = 2048 in 4 epochs of 8 minibatches of 256, launch per kernel."""
    net = ARCHS[arch]
    p, data, perms, adam = learn_setup(net, 2048, 256, 4, seed=40)
    assert pdo.relu_margin(p, data[0]) > KINK_MARGIN
    m = make_ppo(tmp_path, net, p)
    m.set_weights(p, p, adam[0], adam[1], adam[2])
    s, a, r, v, d = data
    _nan_workspace(m, 256, 2048)
    metrics = m.learn(s, a, v, r, d, 0.3, num_epochs=4, batch_size=256, perms=perms, return_metrics=True)
    refs = learn_refs(p, data, perms, 256, adam)
    _check_learn(m.get_weights(), metrics, ((refs[0][0], refs[0][1][:, :5], refs[0][2]), (refs[1][0], refs[1][1][:, :5], 0)))


def test_persistent_learn_equals_launch_per_kernel(tmp_path):
    """The persistent kernel (CPB_PPO_PERSISTENT=1, read once per process) at every architecture: within 1e-6 of the
    launch-per-kernel path, and within the float32 gate of float64."""
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    snippet = r"""
import sys, numpy as np
sys.path[:0] = [%r, %r]
from pathlib import Path
import ppo_depth_cases as t
out = {}
for name in t.ARCHS:
    w, metrics = t.persistent_learn(Path(%r) / name, name, 2048, 256, 4)
    out.update({name + ":" + k: x for k, x in w.items()})
    out[name + ":metrics"] = metrics
np.savez(%r, **out)
"""
    outs = []
    for flag in ("0", "1"):
        path = str(tmp_path / ("w%s.npz" % flag))
        code = snippet % (root, os.path.join(root, "tests"), str(tmp_path / ("m" + flag)), path)
        res = subprocess.run([sys.executable, "-c", code], env=dict(os.environ, CPB_PPO_PERSISTENT=flag),
                             capture_output=True, text=True, timeout=1200)
        assert res.returncode == 0, res.stderr[-3000:]
        outs.append(dict(np.load(path)))
    for name, net in ARCHS.items():
        p, data, perms, adam = learn_setup(net, 2048, 256, 4, seed=40)
        refs = learn_refs(p, data, perms, 256, adam)
        w1 = {k: outs[1][name + ":" + k] for k in p}
        _check_learn(w1, outs[1][name + ":metrics"],
                     ((refs[0][0], refs[0][1][:, :5], refs[0][2]), (refs[1][0], refs[1][1][:, :5], 0)))
        for k in p:
            assert rel_l2(w1[k], outs[0][name + ":" + k]) < 1e-6, (name, k)


@pytest.mark.parametrize("arch", list(ARCHS))
def test_learn_segments(tmp_path, arch):
    """16 segments x 128 rows."""
    net = ARCHS[arch]
    p, data, perms, adam = learn_setup(net, 2048, 256, 2, seed=50)
    s, a, r, v, d = data
    lengths = [128] * 16
    boot = np.random.RandomState(51).randn(16)
    m = make_ppo(tmp_path, net, p)
    m.set_weights(p, p, adam[0], adam[1], adam[2])
    _nan_workspace(m, 256, 2048)
    metrics = m.learn(s, a, v, r, d, boot, num_epochs=2, batch_size=256, perms=perms, return_metrics=True,
                      segment_lengths=lengths)
    refs = learn_refs(p, data, perms, 256, adam, segment_lengths=lengths, bootstrap_values=boot)
    _check_learn(m.get_weights(), metrics, ((refs[0][0], refs[0][1][:, :5], refs[0][2]), (refs[1][0], refs[1][1][:, :5], 0)))


@pytest.mark.parametrize("arch", list(ARCHS))
def test_learn_opts_clip_and_kl_stop(tmp_path, arch):
    """Clipping binding on 25-75 % of the minibatches, then a KL stop at a minibatch k > 1 (steps_applied = k).  The
    learning rate is 3e-3 so that the approximate KL of the later minibatches stands well above float32 rounding."""
    net = ARCHS[arch]
    lr = 3e-3
    p, data, perms, adam = learn_setup(net, 2048, 256, 4, seed=60)
    s, a, r, v, d = data
    # the pre-clip norms of the unguarded update set the clip; its KL values set the stop
    (_, rec0, _), _ = learn_refs(p, data, perms, 256, adam, lr=lr)
    for q in (0.375, 0.5, 0.625):          # the first quantile of the unclipped norms that clips 25-75 % of the steps
        max_norm = float(np.quantile(rec0[:, 6], q))
        (_, rec, _), _ = learn_refs(p, data, perms, 256, adam, lr=lr, max_grad_norm=max_norm)
        clipped = (rec[:, 6] > max_norm).mean()
        if 0.25 <= clipped <= 0.75:
            break
    assert 0.25 <= clipped <= 0.75, clipped
    kl = rec[:, 5]
    # the first minibatch from the third on whose KL exceeds every earlier one by 20 %, and is above float32 noise
    k = next(i for i in range(2, len(kl)) if kl[i] > 1.2 * kl[:i].max() and kl[i] > 1e-5)
    target_kl = float((kl[:k].max() + kl[k]) / 2 / 1.5)
    refs = learn_refs(p, data, perms, 256, adam, lr=lr, max_grad_norm=max_norm, target_kl=target_kl)
    stop = refs[0][2]
    assert stop == k > 1, (stop, k)
    m = make_ppo(tmp_path, net, p, learning_rate=lr)
    m.set_weights(p, p, adam[0], adam[1], adam[2])
    _nan_workspace(m, 256, 2048)
    metrics = m.learn(s, a, v, r, d, 0.3, num_epochs=4, batch_size=256, perms=perms, return_metrics=True,
                      max_grad_norm=max_norm, target_kl=target_kl)
    _check_learn(m.get_weights(), metrics, refs, applied=int(m.last_steps_applied.item()))


# ------------------------------------------------------------------------------ the default architecture: spec == legacy
_DEFAULT_SNIPPET = r"""
import sys, ctypes as C, numpy as np
sys.path[:0] = [%r, %r]
from pathlib import Path
import ppo_depth_cases as t
from carla_ppo_b200 import _lib
lib = _lib.load()
p, data, perms, adam = t.learn_setup(t.ARCHS["default"], 2048, 256, 2, seed=70)
s, a, r, v, d = data
out = {}
for use_spec in (0, 1):
    m = t.make_ppo(Path(%r) / str(use_spec), t.ARCHS["default"], p)
    if not use_spec:                  # the legacy entry points: the spec names mapped back
        real = m._call
        m._call = lambda name, *args, _r=real, _m=m: _r(name.replace("cpb_ppo_spec_", "cpb_ppo_"),
                                                        *((C.byref(_m._c),) + args[1:]))
    for opts in ({}, {"max_grad_norm": 0.05, "target_kl": 0.004}):
        for seg in (None, [1024, 1024]):
            m.set_weights(p, p, adam[0], adam[1], adam[2])
            lib.cpb_reset_launch_count()
            boot = 0.3 if seg is None else np.array([0.3, -0.1])
            met = m.learn(s, a, v, r, d, boot, num_epochs=2, batch_size=256, perms=perms, return_metrics=True,
                          segment_lengths=seg, **opts)
            tag = "%%d:%%d:%%d" %% (use_spec, bool(opts), seg is not None)
            out[tag + ":launches"] = np.int64(lib.cpb_launch_count())
            out[tag + ":metrics"] = met
            for k, w in m.get_weights().items():
                out[tag + ":" + k] = w
            out[tag + ":old"] = m.params_old.cpu().numpy()
            out[tag + ":m"] = m.adam_m.cpu().numpy(); out[tag + ":v"] = m.adam_v.cpu().numpy()
            out[tag + ":pw"] = m.adam_powers.cpu().numpy()
            if opts:
                out[tag + ":applied"] = m.last_steps_applied.cpu().numpy()
np.savez(%r, **out)
"""


def test_default_architecture_spec_equals_legacy(tmp_path):
    """learn, learn_opts, learn_segments and learn_segments_opts through the spec twins and through the legacy entry
    points: parameters, theta_old, Adam m / v, beta powers, metrics, steps_applied and launch counts identical, on the
    launch-per-kernel path and in the persistent kernel."""
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    for flag in ("0", "1"):
        path = str(tmp_path / ("d%s.npz" % flag))
        code = _DEFAULT_SNIPPET % (root, os.path.join(root, "tests"), str(tmp_path / ("m" + flag)), path)
        res = subprocess.run([sys.executable, "-c", code], env=dict(os.environ, CPB_PPO_PERSISTENT=flag),
                             capture_output=True, text=True, timeout=600)
        assert res.returncode == 0, res.stderr[-3000:]
        o = dict(np.load(path))
        legacy = {k[2:]: x for k, x in o.items() if k.startswith("0:")}
        spec = {k[2:]: x for k, x in o.items() if k.startswith("1:")}
        assert legacy.keys() == spec.keys() and len(legacy) > 0
        for k in legacy:
            assert np.array_equal(legacy[k], spec[k], equal_nan=True), (flag, k)


def test_default_architecture_predict_train_loss_equal_legacy(tmp_path, lib):
    import ctypes as C
    import torch
    from carla_ppo_b200 import _lib
    p, old, s, a, ret, adv = make_batch(ARCHS["default"], 256, seed=80)
    m = make_ppo(tmp_path, ARCHS["default"], p, old)
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
    vae = _vae(tmp_path, kind)
    m = make_ppo(tmp_path / "ppo", ARCHS["default"], pdo.init_params(S, A, *ARCHS["default"], seed=5))
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
def _vae(tmp_path, kind):
    if kind == "conv":
        return make_conv_vae(tmp_path, shipped_vae_weights()[0], loss="bce", tag="vae", training=False)
    enc, dec = (96, 256, 64), (160, 64)
    return make_mlp(tmp_path, mlp_weights(2, encoder_sizes=enc, decoder_sizes=dec), enc, dec, tag="vec", training=False)


def _fake_envs(n):
    import types
    from helpers import committed_frames
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
    net = ARCHS["odd"]
    vae = _vae(tmp_path, kind)
    meas = ("steer", "throttle", "speed")
    p = pdo.init_params(S, A, net[0], net[1], seed=90)
    models = [make_ppo(tmp_path / tag, net, p, initial_std=0.4) for tag in ("fused", "unfused")]
    envs = _fake_envs(n)
    fs, fa, fv = FusedActor(vae, models[0], meas).encode_predict(envs)
    us, ua, uv = UnfusedActor(vae, models[1], meas).encode_predict(envs)
    assert all(np.array_equal(x, y) for x, y in zip(fs, us))
    assert np.array_equal(fa, ua) and np.array_equal(fv, uv) and np.isfinite(fa).all()


# ------------------------------------------------------------------------------------------------------ checkpoints
@pytest.mark.parametrize("tf_format", [False, True])
def test_checkpoint_round_trip_and_architecture_refusal(tmp_path, tf_format):
    from carla_ppo_b200.ppo import checkpoint_architecture
    net = ARCHS["odd"]
    p, data, perms, adam = learn_setup(net, 512, 128, 1, seed=100)
    a = make_ppo(tmp_path / "a", net, p)
    a.set_weights(p, p, adam[0], adam[1], adam[2])
    s, act, r, v, d = data
    a.learn(s, act, v, r, d, 0.3, num_epochs=1, batch_size=128, perms=perms)
    a.episode_counter = 3
    a.save(tf_format=tf_format)
    assert checkpoint_architecture(a.checkpoint_dir) == net
    b = make_ppo(tmp_path / "a", net)
    assert b.load_latest_checkpoint() is True
    for x, y in ((a.params, b.params), (a.params_old, b.params_old), (a.adam_m, b.adam_m), (a.adam_v, b.adam_v),
                 (a.adam_powers, b.adam_powers)):
        assert np.array_equal(x.cpu().numpy(), y.cpu().numpy())
    assert b.get_episode_idx() == 3
    for other in (ARCHS["default"], ((33, 7, 65), (32,))):
        c = make_ppo(tmp_path / "a", other)
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
