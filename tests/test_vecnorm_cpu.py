"""Running normalisation without a GPU: the float64 restatement tests/vecnorm_restatement.py against the closed form and
a direct loop, the refusal of every bad argument by every new entry point and actor twin before any launch, the
checkpoint record and the train.py flag-vs-checkpoint resolution."""
import ctypes as C
import math

import numpy as np
import pytest

import vecnorm_restatement as vr
from harness import lib  # noqa: F401
from ppo_checks import FAKE, WS_BYTES
from ppo_cases import LOW, HIGH, S


# ------------------------------------------------------------------------------------------------- the restatement
@pytest.mark.parametrize("sizes", [(1,), (5, 1, 7), (3, 64, 2, 200), (1, 1, 1, 1)])
def test_running_statistics_equal_the_closed_form(sizes):
    rs = np.random.RandomState(sum(sizes))
    rows = [rs.randn(n, 7) * rs.uniform(0.1, 5.0, 7) + rs.uniform(-3, 3, 7) for n in sizes]
    rms = vr.RunningMeanStd(shape=(7,))
    for x in rows:
        rms.update(x)
    closed = vr.RunningMeanStd(shape=(7,))
    allx = np.concatenate(rows)
    closed.update_from_moments(np.mean(allx, axis=0), np.var(allx, axis=0), allx.shape[0])
    assert np.all(np.abs(rms.mean - closed.mean) <= 1e-12 * (np.abs(closed.mean) + np.sqrt(closed.var)))
    assert np.all(np.abs(rms.var - closed.var) <= 1e-12 * closed.var)
    assert rms.count == closed.count == 1e-4 + sum(sizes)


def test_constant_column_is_finite():
    rms = vr.RunningMeanStd(shape=(3,))
    for _ in range(5):
        x = np.stack([np.full(8, 2.5), np.arange(8.0), np.zeros(8)], axis=1)
        y = vr.normalize_obs(rms, x)
        assert np.isfinite(y).all()
    assert np.all(y[:, 2] == 0.0) and np.all(np.abs(y) <= 10.0)


def test_reward_path_equals_a_per_environment_loop():
    rs = np.random.RandomState(4)
    num_envs, gamma = 5, 0.9
    norm = vr.RewardNormalizer(num_envs, gamma)
    ret = np.zeros(num_envs)
    count, mean, var = 1e-4, 0.0, 1.0
    for _ in range(60):
        ids = rs.permutation(num_envs)[:rs.randint(1, num_envs + 1)]
        r, d = rs.randn(len(ids)), rs.rand(len(ids)) < 0.2
        got = norm.step(r, d, ids)
        for j, e in enumerate(ids):
            ret[e] = ret[e] * gamma + r[j]
        b = np.array([ret[e] for e in ids])
        bm, bv, n = b.mean(), b.var(), len(b)
        delta, tot = bm - mean, count + n
        mean, var, count = mean + delta * n / tot, (var * count + bv * n + delta ** 2 * count * n / tot) / tot, tot
        want = np.clip(r / math.sqrt(var + 1e-8), -10, 10)
        for j, e in enumerate(ids):
            if d[j]:
                ret[e] = 0.0
        assert np.allclose(got, want, rtol=1e-12, atol=0) and np.allclose(norm.returns, ret, rtol=1e-12, atol=0)
    assert abs(norm.ret_rms.var - var) <= 1e-12 * var and norm.ret_rms.count == count


# ------------------------------------------------------------------------------------------------ refused calls
def _cfg(dim=S, clip=10.0, eps=1e-8):
    from carla_ppo_b200 import _lib
    return _lib.RunningNorm(dim, clip, eps)


BAD_CFGS = {"dim0": dict(dim=0), "dim_neg": dict(dim=-3), "clip0": dict(clip=0.0), "clip_neg": dict(clip=-1.0),
            "clip_nan": dict(clip=float("nan")), "clip_inf": dict(clip=float("inf")), "eps0": dict(eps=0.0),
            "eps_neg": dict(eps=-1e-8), "eps_nan": dict(eps=float("nan")), "eps_inf": dict(eps=float("inf"))}


def _entry_calls(lib):
    """Every standalone call with one bad argument: (tag, thunk)"""
    out = [("init:NULL cfg", lambda: lib.cpb_running_norm_init(None, FAKE, None)),
           ("init:NULL stats", lambda: lib.cpb_running_norm_init(C.byref(_cfg()), None, None))]
    obs = lambda cfg=None, **o: lib.cpb_obs_normalize(
        cfg, o.get("stats", FAKE), o.get("x", FAKE), o.get("batch", 4), 1, o.get("out", FAKE), None)
    rew = lambda cfg=None, **o: lib.cpb_reward_normalize(
        cfg, o.get("stats", FAKE), o.get("ret", FAKE), o.get("ids", FAKE), o.get("r", FAKE), o.get("d", FAKE),
        o.get("batch", 4), o.get("envs", 8), o.get("gamma", 0.99), o.get("out", FAKE), None)
    good1 = lambda: C.byref(_cfg(dim=1))
    out += [("obs:NULL cfg", lambda: obs(None))]
    out += [("obs:" + k, lambda v=v: obs(C.byref(_cfg(**v)))) for k, v in BAD_CFGS.items()]
    out += [("obs:" + k, lambda k=k: obs(C.byref(_cfg()), **{k: None})) for k in ("stats", "x", "out")]
    out += [("obs:batch0", lambda: obs(C.byref(_cfg()), batch=0))]
    out += [("rew:NULL cfg", lambda: rew(None)), ("rew:dim2", lambda: rew(C.byref(_cfg(dim=2))))]
    out += [("rew:" + k, lambda v=v: rew(C.byref(_cfg(**dict(v, dim=v.get("dim", 1)))))) for k, v in BAD_CFGS.items()]
    out += [("rew:" + k, lambda k=k: rew(good1(), **{k: None})) for k in ("stats", "ret", "ids", "r", "d", "out")]
    out += [("rew:" + k, lambda kw=kw: rew(good1(), **kw)) for k, kw in
            (("batch0", dict(batch=0)), ("envs0", dict(envs=0)), ("gamma_neg", dict(gamma=-0.01)),
             ("gamma_big", dict(gamma=1.01)), ("gamma_nan", dict(gamma=float("nan"))))]
    return out


def test_every_entry_point_refuses_bad_arguments_before_any_launch(lib):
    lib.cpb_reset_launch_count()
    for tag, call in _entry_calls(lib):
        assert call() == -1, tag
    assert lib.cpb_launch_count() == 0


def _good_norm(with_rewards):
    from carla_ppo_b200 import _lib
    n = _lib.ActorNorm()
    n.obs, n.obs_stats, n.update = _cfg(), FAKE, 1
    if with_rewards:
        n.reward, n.ret_stats, n.returns, n.env_ids, n.rewards, n.dones = _cfg(dim=1), FAKE, FAKE, FAKE, FAKE, FAKE
        n.num_envs, n.gamma, n.rewards_out = 8, 0.99, FAKE
    return n


def _bad_norms():
    """cpb_actor_norm values with one bad field each (None: a NULL cpb_actor_norm)"""
    out = {"NULL": None}

    def bad(tag, rewards, **fields):
        n = _good_norm(rewards)
        for k, v in fields.items():
            setattr(n, k, v)
        out[tag] = n
    for k, v in BAD_CFGS.items():
        bad("obs:" + k, False, obs=_cfg(**dict(v, dim=v.get("dim", S))))
        bad("reward:" + k, True, reward=_cfg(**dict(v, dim=v.get("dim", 1))))
    bad("obs:dim_not_state_dim", False, obs=_cfg(dim=S - 1))
    bad("obs:NULL stats", False, obs_stats=None)
    bad("reward:dim2", True, reward=_cfg(dim=2))
    for k in ("ret_stats", "returns", "env_ids", "dones", "rewards_out"):
        bad("reward:NULL " + k, True, **{k: None})
    bad("reward:envs0", True, num_envs=0)
    for tag, g in (("gamma_neg", -0.5), ("gamma_big", 1.5), ("gamma_nan", float("nan"))):
        bad("reward:" + tag, True, gamma=g)
    return out


@pytest.mark.parametrize("bad", list(_bad_norms()))
def test_every_actor_twin_refuses_a_bad_norm_before_any_launch(lib, bad):
    from carla_ppo_b200 import _lib
    from ppo_checks import ppo_args
    base = _lib.PpoConfig()
    base.state_dim, base.num_actions, base.epsilon, base.value_scale, base.entropy_scale = S, 2, 0.2, 1.0, 0.01
    for k in range(2):
        base.action_low[k], base.action_high[k] = LOW[k], HIGH[k]
    spec = _lib.PpoSpec.of(base, (500, 300), (500, 300))
    cat = _lib.PpoCatSpec.of(base, (500, 300), (500, 300), (7, 3))
    n = _bad_norms()[bad]
    ref = None if n is None else C.byref(n)
    lib.cpb_reset_launch_count()
    for desc, family in ((spec, "spec"), (cat, "cat")):
        for entry, vae in (("vae_actor", "cpb_vae_spec"), ("mlp_actor", "cpb_mlpvae")):
            name = "%s_ppo_%s_encode_predict_norm" % (vae, family)
            assert getattr(lib, name)(*ppo_args(entry, C.byref(desc), ws_bytes=WS_BYTES), ref) == -1, name
    assert lib.cpb_launch_count() == 0


def test_host_reward_inputs_are_validated():
    from carla_ppo_b200.vec_normalize import VecNormalize
    v = VecNormalize(S, True, True)
    with pytest.raises(ValueError):
        VecNormalize(S, True, False, clip_obs=0.0)
    with pytest.raises(ValueError):
        VecNormalize(S, False, True, gamma=1.5)
    for ids in ([0, 0], [-1, 2], [0.5, 1.0], [0]):
        with pytest.raises(ValueError):
            v.reward_inputs([1.0, 2.0], [0, 1], ids)


# ------------------------------------------------------------------------------------------------- checkpoints
def _record(obs=True, ret=True, clip=(10.0, 10.0), D=S):
    blob = {}
    if obs:
        blob.update({"vec_normalize/obs_mean": np.zeros(D), "vec_normalize/obs_var": np.ones(D),
                     "vec_normalize/obs_count": np.float64(5.0)})
    if ret:
        blob.update({"vec_normalize/ret_mean": np.float64(0.1), "vec_normalize/ret_var": np.float64(2.0),
                     "vec_normalize/ret_count": np.float64(5.0)})
    if obs or ret:
        blob["vec_normalize/clip"] = np.asarray(clip, np.float32)
    return blob


def test_checkpoint_reader_accepts_agreeing_and_refuses_disagreeing_records(tmp_path):
    import ppo_restatement as pr
    from carla_ppo_b200.ppo import PPO
    from carla_ppo_b200.replay_env import Box
    from carla_ppo_b200.vec_normalize import blob_normalization
    assert blob_normalization({}) is None
    assert blob_normalization(_record()) == (True, True, 10.0, 10.0)
    assert blob_normalization(_record(ret=False, clip=(5.0, 10.0))) == (True, False, 5.0, 10.0)
    assert blob_normalization(_record(obs=False)) == (False, True, 10.0, 10.0)
    incomplete = _record(); del incomplete["vec_normalize/obs_var"]
    no_clip = _record(); del no_clip["vec_normalize/clip"]
    for broken in (incomplete, no_clip, {"vec_normalize/clip": np.ones(2, np.float32)}):
        with pytest.raises(ValueError):
            blob_normalization(broken)
    weights = {"policy/" + k: v for k, v in pr.init_params(S, (LOW, HIGH), (64,), (32,), seed=0).items()}
    settings = [dict(), dict(normalize_observations=True), dict(normalize_rewards=True),
                dict(normalize_observations=True, normalize_rewards=True),
                dict(normalize_observations=True, normalize_rewards=True, clip_obs=5.0)]
    records = [{}, _record(ret=False), _record(obs=False), _record(), _record(clip=(5.0, 10.0))]
    for i, kw in enumerate(settings):
        m = PPO((S,), Box(LOW, HIGH), model_dir=str(tmp_path / str(i)), policy_hidden_sizes=(64,),
                value_hidden_sizes=(32,), **kw)
        for j, rec in enumerate(records):
            if i == j:
                assert blob_normalization(rec) == (None if m.vec_normalize is None else m.vec_normalize.settings)
            else:
                with pytest.raises(ValueError, match="checkpoint has"):
                    m.load_blob(dict(weights, **rec))


def test_train_flags_against_the_checkpoint():
    from carla_ppo_b200.train import resolve_normalization
    assert resolve_normalization(False, False, None) == (False, False)
    assert resolve_normalization(True, False, None) == (True, False)
    assert resolve_normalization(False, False, (True, True, 10.0, 10.0)) == (True, True)
    assert resolve_normalization(True, True, (True, True, 10.0, 10.0)) == (True, True)
    assert resolve_normalization(False, False, (False, False, None, None)) == (False, False)
    for obs, rew, ck in ((True, False, (False, False, None, None)), (False, True, (True, False, 10.0, 10.0)),
                         (True, True, (False, True, 10.0, 10.0))):
        with pytest.raises(ValueError, match="disagrees"):
            resolve_normalization(obs, rew, ck)
