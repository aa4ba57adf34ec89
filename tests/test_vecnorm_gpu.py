"""Running normalisation on the device (cpb_obs_normalize, cpb_reward_normalize, the *_encode_predict_norm twins)
against the float64 restatement tests/vecnorm_restatement.py, with every output filled with NaN before each call; the
fused actor bit for bit against the unfused one; checkpoints; train.py and run_eval.py."""
import ctypes as C
import os

import numpy as np
import pytest

import ppo_restatement as pr
import vecnorm_restatement as vr
from harness import lib  # noqa: F401
from helpers import committed_frames
from ppo_cases import ARCHS, CAT_ARCHS, NVECS, S, cat_net, gauss_net, make_ppo, train_params
from ppo_checks import actor_vae, fake_envs

pytestmark = pytest.mark.gpu


def _dev(x):
    import torch
    return torch.from_numpy(np.ascontiguousarray(x)).cuda()


def _nan(n):
    import torch
    return torch.full((n,), float("nan"), dtype=torch.float32, device="cuda")


def _stats_close(got, rms, D):
    mean, var = np.atleast_1d(rms.mean), np.atleast_1d(rms.var)
    assert np.all(np.abs(got[:D] - mean) <= 1e-12 * (np.abs(mean) + np.sqrt(var)))
    assert np.all(np.abs(got[D:2 * D] - var) <= 1e-12 * var)
    assert got[2 * D] == rms.count


def _within_one_ulp(got, ref64):
    ref32 = np.asarray(ref64, np.float64).astype(np.float32)
    assert np.all(np.abs(got.astype(np.float64) - ref32) <= np.spacing(np.abs(ref32)))


class ObsNorm:
    """cpb_obs_normalize on device statistics of width D"""

    def __init__(self, lib, D):
        import torch
        from carla_ppo_b200 import _lib
        self.lib, self.D, self.cfg = lib, D, _lib.RunningNorm(D, 10.0, 1e-8)
        self.stats = torch.full((2 * D + 1,), float("nan"), dtype=torch.float64, device="cuda")
        assert lib.cpb_running_norm_init(C.byref(self.cfg), self.stats.data_ptr(), None) == 0

    def __call__(self, x, update=True):
        x32 = _dev(np.asarray(x, np.float32))
        out = _nan(x32.numel())
        assert self.lib.cpb_obs_normalize(C.byref(self.cfg), self.stats.data_ptr(), x32.data_ptr(), x32.shape[0],
                                          int(update), out.data_ptr(), None) == 0
        return out.cpu().numpy().reshape(x32.shape)


BATCHES = (1, 2, 31, 32, 33, 1024, 8200)


def _obs_batch(rs, B, D, k):
    """Columns of mixed scale, with columns at offset 1e3 and standard deviation 1e-3; every other batch puts +-1e4
    outliers in column 0 (clipping at both ends)."""
    x = rs.randn(B, D) * rs.uniform(0.1, 3.0, D) + rs.uniform(-5, 5, D)
    x[:, 1::3] = 1e3 + 1e-3 * rs.randn(B, len(range(1, D, 3)))
    if k % 2 and B >= 2:
        x[0, 0], x[1, 0] = 1e4, -1e4
    return x.astype(np.float32)


def _run_obs_sequence(lib, D, seed):
    rs = np.random.RandomState(seed)
    dev, ref = ObsNorm(lib, D), vr.RunningMeanStd(shape=(D,))
    outs, hits = [], set()
    for k, B in enumerate(BATCHES):
        x = _obs_batch(rs, B, D, k)
        got = dev(x)
        want = vr.normalize_obs(ref, x.astype(np.float64))
        assert np.isfinite(got).all()
        _within_one_ulp(got, want)
        _stats_close(dev.stats.cpu().numpy(), ref, D)
        hits |= {float(v) for v in got[np.abs(got) == 10.0]}
        outs.append(got)
    return dev, ref, outs, hits


@pytest.mark.parametrize("D", [1, 7, 67, 1030])
def test_obs_kernel_sequences_match_the_restatement(lib, D):
    dev, ref, outs, hits = _run_obs_sequence(lib, D, seed=D)
    assert hits == {10.0, -10.0}
    # update = 0: the statistics stay bit for bit, the output uses them
    before = dev.stats.cpu().numpy()
    x = _obs_batch(np.random.RandomState(99), 33, D, 0)
    got = dev(x, update=False)
    assert np.array_equal(dev.stats.cpu().numpy(), before)
    _within_one_ulp(got, vr.normalize_obs(ref, x.astype(np.float64), update=False))
    # two identical sequences are bit-identical
    dev2, _, outs2, _ = _run_obs_sequence(lib, D, seed=D)
    assert all(np.array_equal(a, b) for a, b in zip(outs, outs2))
    assert np.array_equal(dev2.stats.cpu().numpy(), before)


def test_reward_kernel_matches_the_restatement(lib):
    import torch
    from carla_ppo_b200 import _lib
    rs = np.random.RandomState(7)
    N, gamma = 8, 0.99
    cfg = _lib.RunningNorm(1, 10.0, 1e-8)
    stats = torch.empty(3, dtype=torch.float64, device="cuda")
    assert lib.cpb_running_norm_init(C.byref(cfg), stats.data_ptr(), None) == 0
    ret = torch.zeros(N, dtype=torch.float64, device="cuda")
    ref = vr.RewardNormalizer(N, gamma)
    hits = set()
    for step in range(300):
        ids = rs.permutation(N)[:rs.randint(1, N + 1)].astype(np.int32)
        r = (0.1 * rs.randn(len(ids))).astype(np.float32)
        d = (rs.rand(len(ids)) < 0.1).astype(np.int32)
        if step % 50 == 3:          # a terminal reward far outside the running spread: clipped once the count has grown
            r[0], d[0] = 500.0 * (1 - 2 * ((step // 50) % 2)), 1
        out = _nan(len(ids))
        dr, dd, di = _dev(r), _dev(d), _dev(ids)
        assert lib.cpb_reward_normalize(C.byref(cfg), stats.data_ptr(), ret.data_ptr(), di.data_ptr(), dr.data_ptr(),
                                        dd.data_ptr(), len(ids), N, gamma, out.data_ptr(), None) == 0
        want = ref.step(r.astype(np.float64), d.astype(bool), ids)
        got = out.cpu().numpy()
        _within_one_ulp(got, want)
        _stats_close(stats.cpu().numpy(), ref.ret_rms, 1)
        g_ret = ret.cpu().numpy()
        assert np.all(np.abs(g_ret - ref.returns) <= 1e-12 * np.abs(ref.returns))
        hits |= {float(v) for v in got[np.abs(got) == 10.0]}
    assert hits == {10.0, -10.0}


# ------------------------------------------------------------------------------------------------------ fused actor
def _norm_ppos(tmp_path, net, **kw):
    p = pr.init_params(*net, seed=90)
    if pr.is_categorical(net[1]):
        p["action_logits/bias"] = np.random.RandomState(91).randn(sum(net[1])).astype(np.float32)
    return [make_ppo(tmp_path / tag, net, p, **kw) for tag in ("fused", "unfused")]


def _stats(m):
    v = m.vec_normalize
    return [v.obs_stats.cpu().numpy(), v.ret_stats.cpu().numpy(), v.returns.cpu().numpy()]


@pytest.mark.parametrize("kind", ["conv", "mlp"])
@pytest.mark.parametrize("head", ["gauss", "cat"])
@pytest.mark.parametrize("n", [1, 4, 33])
def test_fused_actor_equals_unfused(tmp_path, lib, kind, head, n):
    from carla_ppo_b200.actor import FusedActor, UnfusedActor
    net = gauss_net(ARCHS["odd"]) if head == "gauss" else cat_net(CAT_ARCHS["odd"], NVECS["7x3"])
    vae = actor_vae(tmp_path, kind)
    meas = ("steer", "throttle", "speed")
    fm, um = _norm_ppos(tmp_path, net, normalize_observations=True, normalize_rewards=True)
    fa, ua = FusedActor(vae, fm, meas), UnfusedActor(vae, um, meas)
    envs = fake_envs(n)
    rs = np.random.RandomState(n)
    for greedy in (False, True, False):
        fa.greedy = ua.greedy = greedy
        f, u = fa.encode_predict(envs), ua.encode_predict(envs)        # a reset: no rewards
        for step in range(3):
            ids = rs.permutation(n + 3)[:n]
            r, d = rs.randn(n) * 3, rs.rand(n) < 0.3
            f, u = fa.encode_predict(envs, r, d, ids), ua.encode_predict(envs, r, d, ids)
            assert len(f) == len(u) == 4
            assert all(x.dtype == np.float32 and np.array_equal(x, y) for x, y in zip(f[0], u[0]))
            for x, y in zip(f[1:], u[1:]):
                assert np.array_equal(x, y)
            assert all(np.array_equal(x, y) for x, y in zip(_stats(fm), _stats(um)))
            assert np.isfinite(f[3]).all() and not np.array_equal(f[3], r.astype(np.float32))


def test_launches_and_the_plain_path(tmp_path, lib):
    """Observation normalisation adds no launch and the reward path one; with normalisation off the actor calls the plain
    entry point and returns the plain float64 states."""
    from carla_ppo_b200.actor import FusedActor
    net = gauss_net(ARCHS["odd"])
    vae = actor_vae(tmp_path, "conv")
    meas = ("steer", "throttle", "speed")
    plain = make_ppo(tmp_path / "plain", net)
    obs_only = make_ppo(tmp_path / "obs", net, normalize_observations=True)
    both = make_ppo(tmp_path / "both", net, normalize_observations=True, normalize_rewards=True)
    envs = fake_envs(4)
    counts = {}
    for tag, m, with_r in (("plain", plain, False), ("obs", obs_only, False), ("both", both, True),
                           ("both_no_reward", both, False)):
        a = FusedActor(vae, m, meas)
        a.encode_predict(envs)                    # buffers and workspaces
        called = []
        real = vae._libh
        a.vae._libh = type("Spy", (), {"__getattr__": lambda s, k: (called.append(k), getattr(real, k))[1]})()
        lib.cpb_reset_launch_count()
        res = a.encode_predict(envs, [1.0] * 4, [0] * 4, [0, 1, 2, 3]) if with_r else a.encode_predict(envs)
        counts[tag] = lib.cpb_launch_count()
        a.vae._libh = real
        called = [k for k in called if "encode_predict" in k or "normalize" in k]
        assert called == [vae._API["encode_predict"] + ("" if tag == "plain" else "_norm")], (tag, called)
        assert (res[0][0].dtype == np.float64) == (tag == "plain")
    assert counts["obs"] == counts["plain"] == counts["both_no_reward"] and counts["both"] == counts["plain"] + 1


# ------------------------------------------------------------------------------------------------------- checkpoints
@pytest.mark.parametrize("tf_format", [False, True])
def test_checkpoints_restore_the_statistics(tmp_path, tf_format):
    net = gauss_net(ARCHS["p64_v64"])
    kw = dict(normalize_observations=True, normalize_rewards=True, clip_obs=5.0)
    m = make_ppo(tmp_path / "m", net, **kw)
    rs = np.random.RandomState(0)
    for _ in range(3):
        m.vec_normalize.normalize_obs(rs.randn(9, S) * 4 + 1)
        m.vec_normalize.normalize_rewards(rs.randn(3), [0, 1, 0], [2, 0, 1])
    m.save(tf_format=tf_format)
    back = make_ppo(tmp_path / "m", net, **kw)
    assert back.load_latest_checkpoint() is True
    for x, y in zip(_stats(m)[:2], _stats(back)[:2]):
        assert np.array_equal(x, y)
    assert np.array_equal(_stats(back)[2], [0.0])         # the returns are not checkpointed
    # a mismatched checkpoint is refused in both directions
    assert make_ppo(tmp_path / "m", net).load_latest_checkpoint() is False
    assert make_ppo(tmp_path / "m", net, normalize_observations=True).load_latest_checkpoint() is False
    plain = make_ppo(tmp_path / "plain", net)
    plain.save(tf_format=tf_format)
    assert make_ppo(tmp_path / "plain", net, **kw).load_latest_checkpoint() is False


# ----------------------------------------------------------------------------- train.py / run_eval.py over the replay env
def _run_training(tmp_path, tag, restart=False, **over):
    from carla_ppo_b200.replay_env import ReplayEnv
    from carla_ppo_b200.train import train
    from ppo_cases import shipped_vae
    rgb, _ = committed_frames()
    envs = [ReplayEnv(rgb, episode_length=24, seed=0) for _ in range(4)]
    over.setdefault("num_envs", 4)
    return train(train_params(tag, **over), restart=restart, env=envs, vae=shipped_vae(tmp_path, tag),
                 models_root=str(tmp_path / "models"), interactive=False)


def test_train_fused_unfused_reference_loop_resume_and_eval(tmp_path):
    from carla_ppo_b200.ppo import _latest_checkpoint_prefix, _read_blob
    from carla_ppo_b200.replay_env import Box, ReplayEnv
    from carla_ppo_b200.run_eval import load_model, run_eval
    from carla_ppo_b200.vae_common import create_encode_state_fn
    from ppo_cases import shipped_vae
    flags = dict(normalize_observations=True, normalize_rewards=True)
    a = _run_training(tmp_path, "fused", **flags)
    b = _run_training(tmp_path, "unfused", unfused=True, **flags)
    c = _run_training(tmp_path, "reffused", reference_loop=True, **flags)
    d = _run_training(tmp_path, "refunfused", reference_loop=True, unfused=True, **flags)
    assert a.get_train_step_idx() > 0 and a.vec_normalize.settings == (True, True, 10.0, 10.0)
    for x, y in ((a, b), (c, d)):
        wx, wy = x.get_weights(), y.get_weights()
        assert all(np.array_equal(wx[k], wy[k]) for k in wx)
        assert all(np.array_equal(s, t) for s, t in zip(_stats(x), _stats(y)))
        assert x.reward_history == y.reward_history
    # resume: the checkpoint's settings and statistics without the flags
    blob = _read_blob(_latest_checkpoint_prefix(a.checkpoint_dir))
    e = _run_training(tmp_path, "fused", num_episodes=3)
    assert e.vec_normalize.settings == (True, True, 10.0, 10.0) and e.get_episode_idx() == 3
    assert e.vec_normalize.obs_stats[-1].item() > float(blob["vec_normalize/obs_count"])
    # a flag the checkpoint does not have is refused before anything trains
    _run_training(tmp_path, "plain", num_episodes=1)
    with pytest.raises(ValueError, match="disagrees"):
        _run_training(tmp_path, "plain", num_episodes=2, normalize_rewards=True)
    # run_eval's loader restores the statistics and an evaluation episode leaves them unchanged
    model_dir = os.path.dirname(a.checkpoint_dir.rstrip("/"))
    blob = _read_blob(_latest_checkpoint_prefix(a.checkpoint_dir))
    m = load_model(np.array([S]), Box([-1.0, 0.0], [1.0, 1.0]), model_dir)
    assert m.vec_normalize.settings == (True, True, 10.0, 10.0) and m.vec_normalize.training is False
    before = m.vec_normalize.obs_stats.cpu().numpy()
    assert np.array_equal(before[:S], blob["vec_normalize/obs_mean"])
    assert np.array_equal(before[S:2 * S], blob["vec_normalize/obs_var"])
    vae = shipped_vae(tmp_path, "eval")
    env = ReplayEnv(committed_frames()[0], episode_length=24, seed=0,
                    encode_state_fn=create_encode_state_fn(vae, ("steer", "throttle", "speed"), m.vec_normalize))
    m.vec_normalize.training = True
    total = run_eval(env, m)
    assert np.isfinite(total) and m.vec_normalize.training is True
    assert np.array_equal(m.vec_normalize.obs_stats.cpu().numpy(), before)
