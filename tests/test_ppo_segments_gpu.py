"""N environments on the device: the segmented GAE and PPO update against the float64 restatement
(tests/test_ppo_segments_cpu.py), bit-identity with the single-rollout entry points at one segment, the batched fused
encode + predict, and train.train with --num_envs."""
import numpy as np
import pytest

from harness import lib, library_state, math_mode  # noqa: F401
from helpers import committed_frames, rel_l2, shipped_ppo, shipped_vae_weights
from ppo_cases import (HIGH, LOW, REFERENCE, baseline_config3, make_ppo, model_state, restate, segment_inputs,
                       shipped_adam, shipped_vae, train_params)
from ppo_checks import TOL, actor_vae, fake_envs, fresh_process
from ppo_restatement import segmented_gae

pytestmark = pytest.mark.gpu

LENGTHS = (1, 31, 32, 33, 1023, 1024, 1025, 4097)


def _gae_segments(r, v, boot, d, lengths, gamma=0.99, lam=0.95):
    import torch
    from carla_ppo_b200 import _lib
    lib = _lib.load()
    dev = lambda x, t=torch.float64: torch.as_tensor(np.asarray(x), dtype=t, device="cuda").contiguous()
    rows = int(np.sum(lengths))
    offs = dev(np.concatenate([[0], np.cumsum(lengths)]), torch.int32)
    rt, vt, bt, dt = dev(r), dev(v), dev(boot), dev(d)
    out = [torch.empty(rows, dtype=torch.float64, device="cuda") for _ in range(3)]
    _lib.check(lib.cpb_gae_segments(rt.data_ptr(), vt.data_ptr(), bt.data_ptr(), dt.data_ptr(), offs.data_ptr(),
                                    len(lengths), rows, gamma, lam, out[0].data_ptr(), out[1].data_ptr(),
                                    out[2].data_ptr(), _lib.current_stream_handle()), "cpb_gae_segments")
    adv, ret, advn = (o.cpu().numpy() for o in out)
    return ret, advn, adv


@pytest.mark.parametrize("S", [1, 3, 64, 1000])
def test_gae_segments_match_float64(S):
    lengths = list(np.random.RandomState(S).choice(LENGTHS, S))
    r, v, boot, d = segment_inputs(lengths, seed=S)
    got = _gae_segments(r, v, boot, d, lengths)
    ref = segmented_gae(r, v, boot, d, lengths, 0.99, 0.95)
    for g, x, name in zip(got, ref, ("returns", "advantages_norm", "advantages")):
        assert rel_l2(g, x) < 1e-12, (name, rel_l2(g, x))


def test_one_segment_is_cpb_gae_bit_for_bit():
    import torch
    from carla_ppo_b200 import _lib
    lib = _lib.load()
    for T in (1, 1025, 4097):
        r, v, boot, d = segment_inputs([T], seed=T)
        got = _gae_segments(r, v, boot, d, [T])
        packed = torch.as_tensor(np.concatenate([r, v, d]), device="cuda")
        out = [torch.empty(T, dtype=torch.float64, device="cuda") for _ in range(3)]
        base = packed.data_ptr()
        _lib.check(lib.cpb_gae(base, base + 8 * T, float(boot[0]), base + 16 * T, T, 0.99, 0.95, out[0].data_ptr(),
                               out[1].data_ptr(), out[2].data_ptr(), _lib.current_stream_handle()), "cpb_gae")
        adv, ret, advn = (o.cpu().numpy() for o in out)
        assert np.array_equal(got[0], ret) and np.array_equal(got[1], advn) and np.array_equal(got[2], adv), T


# ------------------------------------------------------------------------------------------------ learn over segments
@pytest.mark.parametrize("persistent", ["0", "1"])
def test_one_segment_learn_is_cpb_ppo_learn_bit_for_bit(tmp_path, persistent):
    """cpb_ppo_learn_segments at S = 1 vs cpb_ppo_learn from ckpt-705 with warm Adam slots (2 epochs x 200, a short last
    minibatch): parameters, theta_old, Adam m / v, beta powers and every minibatch metric, launch-per-kernel and under
    CPB_PPO_PERSISTENT=1 (read once per process, hence the subprocess)."""
    ckpt = ("ckpt705", 2048, 2, 200, "policy_old", 1e-4, False)
    z, = fresh_process(tmp_path, [("one", REFERENCE, ckpt, {}), ("seg", REFERENCE, ckpt, dict(segment_lengths=[2048]))],
                       flags=(persistent,), timeout=300)
    for k in ("params", "old", "m", "v", "powers", "metrics"):
        assert np.array_equal(z["one:" + k], z["seg:" + k]), k


@pytest.mark.parametrize("lengths, E, B", [([128] * 16, 4, 256), ([1, 7, 128, 60, 3], 3, 64)], ids=["16x128", "ragged"])
def test_learn_segments_match_the_oracle(tmp_path, lengths, E, B):
    """configs[2]'s shapes (ckpt-705 with warm Adam slots, RandomState(0) permutations) over 16 segments of 128 rows, and
    ragged segments with a short last minibatch; gates as test_ppo_gpu's configs[2] test: max(1e-5, 2 x the float32
    restatement's error)."""
    pol, _ = shipped_ppo("policy")
    old, _ = shipped_ppo("policy_old")
    adam = shipped_adam()
    m = make_ppo(tmp_path, REFERENCE, pol, old)
    m.set_weights(pol, old, *adam)
    T = int(np.sum(lengths))
    s, a, r, v, _, perms = baseline_config3(T, E)
    d = np.zeros(T, bool)
    ends = np.cumsum(lengths) - 1
    d[ends[::2]] = True                                     # every other segment ends in a terminal
    d[np.random.RandomState(5).choice(T, 3)] = True         # and a few done flags inside segments
    boot = np.random.RandomState(6).randn(len(lengths)).astype(np.float32)
    metrics = m.learn(s, a, v, r, d, boot, num_epochs=E, batch_size=B, perms=perms, return_metrics=True,
                      segment_lengths=lengths)
    p64, _, rec64, _ = restate((LOW, HIGH), pol, adam, (s, a, r, v, d), perms, B, np.float64, segment_lengths=lengths,
                               bootstrap_values=boot)
    p32, _, rec32, _ = restate((LOW, HIGH), pol, adam, (s, a, r, v, d), perms, B, np.float32, segment_lengths=lengths,
                               bootstrap_values=boot)
    rec64, rec32 = rec64[:, :5], rec32[:, :5]
    got = m.get_weights()
    for name in p64:
        gate = max(TOL, 2 * rel_l2(p32[name], p64[name]))
        assert rel_l2(got[name], p64[name]) < gate, (name, rel_l2(got[name], p64[name]), gate)
    assert metrics.shape == rec64.shape == (E * -(-T // B), 5)
    for col in range(5):
        gate = max(TOL, 2 * rel_l2(rec32[:, col], rec64[:, col]))
        assert rel_l2(metrics[:, col], rec64[:, col]) < gate, (col, rel_l2(metrics[:, col], rec64[:, col]), gate)
    gold = m.get_old_weights()
    assert all(np.array_equal(gold[k], pol[k]) for k in pol)


# ------------------------------------------------------------------------------------------------ batched encode + predict
def _oracle_mean(vae, kind, frames):
    x = frames.astype(np.float64) / 255.0
    if kind == "conv":
        from oracle import vae_oracle as vo
        return vo.encode({k: w.astype(np.float64) for k, w in vae.get_weights().items()}, x)[0]
    import mlp_depth_oracle as mdo
    return mdo.loss_and_grads(vae.get_weights(), x, x, np.zeros((len(x), vae.z_dim)), "bce", want_grads=False)["mean"]


@pytest.mark.parametrize("mode", [1, 2])
@pytest.mark.parametrize("kind", ["conv", "mlp"])
@pytest.mark.parametrize("n", [2, 8, 33])
def test_batched_encode_predict(tmp_path, lib, n, kind, mode):
    """FusedActor.encode_predict at B = n: bit for bit the batched unfused calls (one vae.encode, one ppo.predict, the same
    noise), latents within max(1e-5, 2 x the single-frame calls' error) of float64, and actions / values within 1e-5 of
    the oracle's PPO on the device's states with the same noise."""
    from carla_ppo_b200.actor import FusedActor, UnfusedActor
    from carla_ppo_b200.ppo import PPO
    from oracle import ppo_oracle as po
    from helpers import Box
    with math_mode(lib, mode):
        vae = actor_vae(tmp_path, kind)
        meas = ("steer", "throttle", "speed")
        models = []
        for tag in ("fused", "unfused"):
            m = PPO((67,), Box(LOW, HIGH), initial_std=0.4, model_dir=str(tmp_path / tag), seed=0)
            m.init_session(init_logging=False)
            m.set_weights(shipped_ppo("policy")[0])
            models.append(m)
        envs = fake_envs(n)
        fs, fa, fv = FusedActor(vae, models[0], meas).encode_predict(envs)
        us, ua, uv = UnfusedActor(vae, models[1], meas).encode_predict(envs)
        assert len(fs) == n and fa.shape == (n, 2) and fv.shape == (n,)
        assert all(np.array_equal(a, b) for a, b in zip(fs, us))
        assert np.array_equal(fa, ua) and np.array_equal(fv, uv)
        frames = np.stack([e.observation for e in envs])
        ref = _oracle_mean(vae, kind, frames)
        single = np.concatenate([vae.encode(frames[i:i + 1]) for i in range(n)])
        lat = np.stack([s[:vae.z_dim] for s in fs])
        gate = max(1e-5, 2 * rel_l2(single, ref))
        assert rel_l2(lat, ref) < gate, (rel_l2(lat, ref), gate)
        noise = np.random.RandomState(0).randn(n, 2).astype(np.float32)      # PPO(seed=0)'s generator: the first draw
        p64 = {k: w.astype(np.float64) for k, w in shipped_ppo("policy")[0].items()}
        ract, rval = po.predict(p64, np.stack(fs).astype(np.float32), LOW, HIGH, noise=noise)
        assert rel_l2(fa, ract) < TOL and rel_l2(fv, rval) < TOL


# ------------------------------------------------------------------------------------------------ train.train --num_envs


def _train(tmp_path, tag, num_envs, fn=None, **over):
    from carla_ppo_b200.replay_env import ReplayEnv
    from carla_ppo_b200.train import train
    rgb, _ = committed_frames()
    envs = [ReplayEnv(rgb, episode_length=24 + 5 * i, seed=0) for i in range(num_envs)]
    vae = shipped_vae(tmp_path, tag)
    params = train_params(tag, num_envs=num_envs, **over)
    model = (fn or train)(params, restart=False, env=envs if fn is None else envs[0], vae=vae,
                          models_root=str(tmp_path / "models"), interactive=False)
    return model, envs


def test_one_environment_reproduces_the_loop_before_num_envs(tmp_path):
    """train.train(num_envs=1), fused, against the single-environment loop it replaced: bit-identical weights, Adam state,
    rewards and step counters; the same seeds give the same trajectory."""
    import single_env_train
    a, env_a = _train(tmp_path, "vec1", 1)
    b, env_b = _train(tmp_path, "old1", 1, fn=single_env_train.train_one_env)
    sa, sb = model_state(a), model_state(b)
    assert all(np.array_equal(sa[k], sb[k]) for k in sa)
    assert a.reward_history == b.reward_history and a.get_train_step_idx() == b.get_train_step_idx() > 0
    assert a.predict_step_counter == b.predict_step_counter and env_a[0].step_count == env_b[0].step_count
    c, _ = _train(tmp_path, "vec1_again", 1)
    assert all(np.array_equal(sa[k], x) for k, x in model_state(c).items()) and c.reward_history == a.reward_history


def test_four_environments(tmp_path):
    """num_envs = 4 over two rounds: fused == unfused bit for bit; PPO.learn over segments == the reference's Python loop
    (per-segment compute_gae, one normalisation, PPO.train minibatches) within 1e-6; and the trajectory and weights match
    the float64 oracle stepping the same four replays with the same noise and shuffle streams."""
    from carla_ppo_b200.ppo import PPO
    from carla_ppo_b200.replay_env import ReplayEnv
    from oracle import ppo_oracle as po, vae_oracle as vo
    a, _ = _train(tmp_path, "f4", 4, eval_interval=1000)
    b, _ = _train(tmp_path, "u4", 4, eval_interval=1000, unfused=True)
    c, _ = _train(tmp_path, "r4", 4, eval_interval=1000, unfused=True, reference_loop=True)
    wa, wb, wc = a.get_weights(), b.get_weights(), c.get_weights()
    assert a.get_episode_idx() == 2 and a.get_train_step_idx() == b.get_train_step_idx() == c.get_train_step_idx() > 0
    assert all(np.array_equal(wa[k], wb[k]) for k in wa) and a.reward_history == b.reward_history
    for k in wa:
        assert rel_l2(wb[k], wc[k]) < 1e-6, k

    # ---- the same lockstep loop on the oracle
    rgb, _ = committed_frames()
    envs = [ReplayEnv(rgb, episode_length=24 + 5 * i, seed=0) for i in range(4)]
    for i, e in enumerate(envs):
        e.seed(i)
    np.random.seed(0)
    probe = PPO((67,), envs[0].action_space, initial_std=0.4, model_dir=str(tmp_path / "probe"), seed=0)
    probe.init_session(init_logging=False)
    p = {k: x.astype(np.float64) for k, x in probe.get_weights().items()}
    st = vo.adam_init_state(p)
    noise_rng = np.random.RandomState(0)
    vw = {k: x.astype(np.float64) for k, x in shipped_vae_weights()[0].items()}
    low, high = envs[0].action_space.low.astype(np.float64), envs[0].action_space.high.astype(np.float64)

    def encode_predict(es):
        mu, _ = vo.encode(vw, np.stack([e.observation for e in es]).astype(np.float64) / 255.0)
        states = [np.append(mu[j], [e.vehicle.control.steer, e.vehicle.control.throttle, e.vehicle.get_speed()])
                  for j, e in enumerate(es)]
        return states, *predict(states)

    def predict(states):
        act, val = po.predict(p, np.stack(states), low, high, noise=noise_rng.randn(len(states), 2).astype(np.float32))
        return list(np.reshape(act, (len(states), 2))), list(np.float32(np.reshape(val, (len(states),))))

    for e in envs:
        e.encode_state_fn = lambda env: None
    history = []
    for episode in range(2):
        for e in envs:
            e.reset()
        state, action, value = encode_predict(envs)
        totals, active, first = [0.0] * 4, [0, 1, 2, 3], True
        while active:
            if not first:
                acts, vals = predict([state[i] for i in active])
                for j, i in enumerate(active):
                    action[i], value[i] = acts[j], vals[j]
            first = False
            ro = {i: ([], [], [], [], []) for i in active}
            for _ in range(16):
                stepped, term = list(active), {}
                for i in stepped:
                    _, rwd, term[i], _ = envs[i].step(action[i])
                    totals[i] += rwd
                    for buf, x in zip(ro[i], (state[i], action[i], value[i], rwd, term[i])):
                        buf.append(x)
                ns, na, nv = encode_predict([envs[i] for i in stepped])
                for j, i in enumerate(stepped):
                    state[i], action[i], value[i] = ns[j], na[j], nv[j]
                active = [i for i in stepped if not term[i]]
                if not active:
                    break
            segs = [i for i in sorted(ro) if ro[i][3]]
            S_, A_, V_, R_, D_ = ([x for i in segs for x in ro[i][k]] for k in range(5))
            perms = []
            for _ in range(2):
                idx = np.arange(len(R_)); np.random.shuffle(idx); perms.append(idx)
            returns, adv_n, _ = segmented_gae(R_, V_, [value[i] for i in segs], D_, [len(ro[i][3]) for i in segs], 0.99, 0.95)
            ret32, adv32 = returns.astype(np.float32).astype(np.float64), adv_n.astype(np.float32).astype(np.float64)
            old = {k: x.copy() for k, x in p.items()}
            s_arr, a_arr = np.array(S_, np.float32).astype(np.float64), np.array(A_, np.float32).astype(np.float64)
            for e_ in range(2):
                for i in range(int(np.ceil(len(R_) / 8))):
                    mb = perms[e_][i * 8:(i + 1) * 8]
                    out = po.loss_and_grads(p, old, s_arr[mb], a_arr[mb], ret32[mb], adv32[mb], low, high, 0.2, 1.0, 0.01)
                    vo.adam_apply(p, out["grads"], st, 1e-4)
        history.append(float(np.mean(totals)))
    assert np.allclose(a.reward_history, history, rtol=1e-5, atol=1e-7), (a.reward_history, history)
    for k in p:
        assert rel_l2(wa[k], p[k]) < 2e-5, (k, rel_l2(wa[k], p[k]))
