"""PPO over several trajectory segments without a GPU: the float64 restatement of the segmented GAE, the C ABI's refusals
of cpb_gae_segments / cpb_ppo_learn_segments (no launch), PPO.learn's checks of segment_lengths, and the bookkeeping of
train.train(num_envs=N) on scripted environments with recording fakes of the VAE and the PPO."""
import ctypes as C
import os
import types

import numpy as np
import pytest

import single_env_train
from harness import lib, library_state  # noqa: F401
from helpers import Box
from ppo_cases import ppo_config, segment_inputs
from ppo_checks import SEGMENTS_POINTERS, ppo_args
from ppo_restatement import segmented_gae


# ------------------------------------------------------------------------------------------------ float64 restatement


def test_one_segment_is_the_single_rollout_computation_bit_for_bit():
    from oracle import ppo_oracle as po
    for T in (1, 33, 1025):
        r, v, boot, d = segment_inputs([T], seed=T)
        got = segmented_gae(r, v, boot, d, [T], 0.99, 0.95)
        ref = po.returns_and_normalised_advantages(r, v, boot[0], d, 0.99, 0.95)
        for g, x in zip(got, ref):
            assert np.array_equal(g, x)


def test_segments_do_not_leak_into_each_other():
    """A segment's advantages depend only on its own rows and bootstrap value."""
    from oracle import ppo_oracle as po
    lengths = [5, 1, 9]
    r, v, boot, d = segment_inputs(lengths, seed=3)
    adv = segmented_gae(r, v, boot, d, lengths, 0.99, 0.95)[2]
    assert np.array_equal(adv[6:], po.compute_gae(r[6:], v[6:], boot[2], d[6:], 0.99, 0.95))
    r2 = r.copy(); r2[6:] += 1.0
    adv2 = segmented_gae(r2, v, boot, d, lengths, 0.99, 0.95)[2]
    assert np.array_equal(adv2[:6], adv[:6])


# ------------------------------------------------------------------------------------------------ C ABI refusals
FAKE = 0x1000          # never dereferenced: every call below must be refused before it touches memory


def _gae_args(**over):
    a = dict(rewards=FAKE, values=FAKE, bootstrap=FAKE, dones=FAKE, offsets=FAKE, S=2, rows=8, adv=FAKE)
    a.update(over)
    return (a["rewards"], a["values"], a["bootstrap"], a["dones"], a["offsets"], a["S"], a["rows"], 0.99, 0.95, a["adv"],
            None, None, None)


@pytest.mark.parametrize("over", [dict(S=0), dict(S=-1), dict(S=9, rows=8), dict(rows=0), dict(rewards=None),
                                  dict(values=None), dict(bootstrap=None), dict(dones=None), dict(offsets=None),
                                  dict(adv=None)], ids=lambda d: "_".join("%s%s" % kv for kv in d.items()))
def test_gae_segments_refuses_bad_arguments_without_a_launch(lib, over):
    before = lib.cpb_launch_count()
    assert lib.cpb_gae_segments(*_gae_args(**over)) == -1
    assert lib.cpb_launch_count() == before
    assert b"gae_segments" in lib.cpb_last_error()


@pytest.mark.parametrize("over", [dict(S=0), dict(S=-2), dict(S=41), dict(rows=2), dict(batch=0), dict(epochs=-1)]
                         + [{k: None} for k in SEGMENTS_POINTERS],
                         ids=lambda d: "_".join("%s%s" % kv for kv in d.items()))
def test_learn_segments_refuses_bad_arguments_without_a_launch(lib, over):
    cfg = ppo_config(67, 2, 500, 300)
    before = lib.cpb_launch_count()
    assert lib.cpb_ppo_learn_segments(*ppo_args("learn_segments", C.byref(cfg), **over)) == -1
    assert lib.cpb_launch_count() == before


def test_learn_segments_refuses_a_small_workspace(lib):
    cfg = ppo_config(67, 2, 500, 300)
    need = lib.cpb_ppo_workspace_bytes(C.byref(cfg), 16, 40)
    args = ppo_args("learn_segments", C.byref(cfg), ws_bytes=need - 1)
    assert lib.cpb_ppo_learn_segments(*args) == -3          # CPB_ERR_WORKSPACE_TOO_SMALL


# ------------------------------------------------------------------------------------------------ PPO.learn checks
@pytest.mark.parametrize("lengths, boot", [([], []), ([0, 10], [0.0, 0.0]), ([4, 5], [0.0, 0.0]), ([11], [0.0]),
                                           ([-1, 11], [0.0, 0.0]), ([5, 5], [0.0]), ([5, 5], [0.0, 0.0, 0.0])])
def test_ppo_learn_refuses_bad_segment_lengths(tmp_path, lengths, boot):
    from carla_ppo_b200.ppo import PPO
    m = PPO((67,), Box([-1.0, 0.0], [1.0, 1.0]), model_dir=str(tmp_path / "ppo"), seed=0)
    s = np.zeros((10, 67), np.float32)
    with pytest.raises(ValueError):
        m.learn(s, np.zeros((10, 2), np.float32), np.zeros(10), np.zeros(10), np.zeros(10), boot, segment_lengths=lengths)


# ------------------------------------------------------------------------------------------------ --num_envs bookkeeping
class ScriptedEnv:
    """Replay-environment surface with scripted training-episode lengths (one per training reset); evaluation episodes
    last 2 steps.  Reward of step t: t + tag / 10, so every row says which environment and step produced it."""

    def __init__(self, lengths, tag):
        self.lengths, self.tag = list(lengths), tag
        self.action_space = Box([-1.0, 0.0], [1.0, 1.0])
        self.encode_state_fn = None
        self.extra_info = []
        self.actions = []
        self.seeded = None
        self._reset_counters()

    def _reset_counters(self):
        self.t = 0
        self.distance_traveled = self.speed_accum = self.center_lane_deviation = 0.0
        self.step_count = 0
        self.vehicle = types.SimpleNamespace(control=types.SimpleNamespace(steer=0.0, throttle=0.0), get_speed=lambda: 1.5)
        self.observation = np.full((2, 2, 3), self.tag, np.uint8)

    def seed(self, seed):
        self.seeded = seed

    def reset(self, is_training=True):
        self._reset_counters()
        self.T = self.lengths.pop(0) if is_training else 2
        return self.encode_state_fn(self)

    def step(self, action):
        self.actions.append(np.array(action))
        self.t += 1
        self.step_count += 1
        self.vehicle.control.steer, self.vehicle.control.throttle = float(action[0]), float(action[1])
        self.observation = np.full((2, 2, 3), (self.tag * 16 + self.t) % 256, np.uint8)
        return self.encode_state_fn(self), self.t + self.tag / 10, self.t >= self.T, {"closed": False}

    def render(self, mode="human"):
        return None


class FakeVAE:
    z_dim = 2

    def __init__(self, log):
        self.log = log

    def encode(self, frames):
        x = np.asarray(frames, np.float32)
        self.log.append(("encode", len(x)))
        return x.reshape(len(x), -1)[:, :2] / 255


def fake_ppo_class(log):
    class FakePPO:
        """The PPO surface train.train touches; records predict / learn / train calls.  predict draws its noise from its
        own generator like PPO.predict (randn(B, A), none when greedy)."""

        def __init__(self, input_shape, action_space, model_dir="./", seed=None, **kw):
            self.state_dim, self.num_actions = int(np.atleast_1d(input_shape)[0]), 2
            self.low, self.high = action_space.low, action_space.high
            self.model_dir = model_dir
            self.checkpoint_dir, self.log_dir, self.video_dir = (os.path.join(model_dir, d) for d in ("c", "l", "v"))
            self.dirs = [self.checkpoint_dir, self.log_dir, self.video_dir]
            self.train_writer, self.predict_step_counter, self.episode, self.steps = None, 0, 0, 0

        def init_session(self, init_logging=True):
            self._rng = np.random.RandomState(0)

        def load_latest_checkpoint(self):
            return None

        def predict(self, x, greedy=False, write_to_summary=False):
            x = np.asarray(x, np.float32)
            x = x if x.ndim == 2 else x[None]
            noise = np.zeros((len(x), 2)) if greedy else self._rng.randn(len(x), 2)
            act = np.clip(np.tanh(x.sum(1))[:, None] * 0.5 + 0.3 * noise, self.low, self.high).astype(np.float32)
            val = (x.sum(1) + 0.25).astype(np.float32)
            log.append(("predict", x.copy(), bool(greedy)))
            if write_to_summary:
                self.predict_step_counter += 1
            return (act[0], val[0]) if len(x) == 1 else (act, val)

        def learn(self, states, actions, values, rewards, dones, last_value, gamma=0.99, lam=0.95, num_epochs=3,
                  batch_size=32, perms=None, return_metrics=False, segment_lengths=None):
            log.append(("learn", np.array(states), np.array(actions), np.array(values), np.array(rewards), np.array(dones),
                        np.array(last_value), np.array(perms), segment_lengths))
            self.steps += num_epochs * -(-len(rewards) // batch_size)

        def save(self):
            log.append(("save",))

        def get_episode_idx(self):
            return self.episode

        def get_train_step_idx(self):
            return self.steps

        def write_dict_to_summary(self, *a):
            pass

        def write_value_to_summary(self, name, value, step):
            log.append(("summary", name, float(value), step))

        def write_episodic_summaries(self):
            self.episode += 1

    return FakePPO


def _params(**over):
    p = dict(learning_rate=1e-4, lr_decay=1.0, discount_factor=0.99, gae_lambda=0.95, ppo_epsilon=0.2, initial_std=0.4,
             value_scale=1.0, entropy_scale=0.01, horizon=4, num_epochs=2, num_episodes=2, batch_size=3,
             vae_model="unused", vae_model_type=None, vae_z_dim=None, synchronous=True, fps=30, action_smoothing=0.0,
             model_name="fake", reward_fn="reward_speed_centering_angle_multiply", seed=0, eval_interval=1000,
             record_eval=False, logging=False, unfused=True)
    p.update(over)
    return p


def _run(monkeypatch, tmp_path, module, train_fn, envs, **over):
    log = []
    monkeypatch.setattr(module, "PPO", fake_ppo_class(log))
    model = train_fn(_params(**over), restart=False, env=envs, vae=FakeVAE(log), models_root=str(tmp_path), interactive=False)
    return model, log


def _same(a, b):
    if isinstance(a, np.ndarray) or isinstance(b, np.ndarray):
        return np.array_equal(np.asarray(a), np.asarray(b))
    if isinstance(a, (tuple, list)) and isinstance(b, (tuple, list)):
        return len(a) == len(b) and all(_same(x, y) for x, y in zip(a, b))
    return a == b


def test_one_environment_makes_the_calls_of_the_loop_before_num_envs(monkeypatch, tmp_path):
    """num_envs = 1: the same encode / predict / learn calls in the same order, the same noise and shuffle streams, the
    same actions and summaries as the single-environment loop it replaces."""
    from carla_ppo_b200 import train as train_mod
    script = [9, 3, 4]               # an episode longer than two horizons, one shorter than one, one exactly one
    env_a, env_b = ScriptedEnv(script, 0), ScriptedEnv(script, 0)
    a, log_a = _run(monkeypatch, tmp_path, train_mod, train_mod.train, env_a, num_episodes=3, eval_interval=2)
    b, log_b = _run(monkeypatch, tmp_path, single_env_train, single_env_train.train_one_env, env_b, num_episodes=3,
                    eval_interval=2)
    assert sum(1 for e in log_b if e[0] == "learn") == 3 + 1 + 1
    assert len(log_a) == len(log_b)
    for x, y in zip(log_a, log_b):
        assert _same(x, y), (x, y)
    assert _same(env_a.actions, env_b.actions) and env_a.seeded == env_b.seeded == 0
    assert a.reward_history == b.reward_history and a.predict_step_counter == b.predict_step_counter


def test_segments_follow_the_scripted_terminals(monkeypatch, tmp_path):
    """Three environments, horizon 4.  Round 1 (episodes of 5, 12 and 3 steps): rollouts of 4 + 4 + 3 rows, then 1 + 4
    (env 2 has finished), then 4 (env 0 too).  Round 2 (2, 3, 1 steps): one rollout of 2 + 3 + 1.  One learn call per
    rollout, segments in environment order, one bootstrap value each, permutations over all rows from np.random."""
    from carla_ppo_b200 import train as train_mod
    envs = [ScriptedEnv([5, 2], 0), ScriptedEnv([12, 3], 1), ScriptedEnv([3, 1], 2)]
    model, log = _run(monkeypatch, tmp_path, train_mod, train_mod.train, envs, num_envs=3)
    learns = [e for e in log if e[0] == "learn"]
    assert [e[8] for e in learns] == [[4, 4, 3], [1, 4], [4], [2, 3, 1]]
    assert [e[6].shape for e in learns] == [(3,), (2,), (1,), (3,)]
    assert [e.seeded for e in envs] == [0, 1, 2]
    # rows: env order within a rollout, step order within a segment
    tags_steps = [(round(r % 1 * 10), int(r)) for r in learns[0][4]]
    assert tags_steps == [(0, 1), (0, 2), (0, 3), (0, 4), (1, 1), (1, 2), (1, 3), (1, 4), (2, 1), (2, 2), (2, 3)]
    assert list(learns[0][5]) == [0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 1]
    assert list(learns[1][4]) == [5.0, 5.1, 6.1, 7.1, 8.1] and list(learns[1][5]) == [1, 0, 0, 0, 0]
    assert list(learns[2][5]) == [0, 0, 0, 1]
    # the permutation stream: np.random.seed(seed), then num_epochs shuffles of arange(rows) per update
    np.random.seed(0)
    for e in learns:
        rows = len(e[4])
        ref = []
        for _ in range(2):
            idx = np.arange(rows); np.random.shuffle(idx); ref.append(idx)
        assert np.array_equal(e[7], np.stack(ref))
    # one batched predict per lockstep step over the environments stepped, plus one on reset and one per later rollout
    sizes = [len(e[1]) for e in log if e[0] == "predict" and not e[2]]
    assert sizes[:6] == [3, 3, 3, 3, 2, 2]       # reset, steps 1-3 (env 2 ends at step 3), step 4, next rollout
    encodes = [e[1] for e in log if e[0] == "encode"]
    assert encodes[:8] == [1, 1, 1, 3, 3, 3, 3, 2]   # the evaluation episode on env 0, then reset and steps 1-4
    # means over the environments
    rewards = [e for e in log if e[0] == "summary" and e[1] == "train/reward"]
    assert rewards[0][2] == pytest.approx(np.mean([sum(t for t in range(1, 6)), sum(t + 0.1 for t in range(1, 13)),
                                                   sum(t + 0.2 for t in range(1, 4))]))
    assert model.reward_history[0] == rewards[0][2] and model.get_episode_idx() == 2


def test_num_envs_must_match_the_environments_given(monkeypatch, tmp_path):
    from carla_ppo_b200 import train as train_mod
    with pytest.raises(ValueError):
        _run(monkeypatch, tmp_path, train_mod, train_mod.train, [ScriptedEnv([2], 0)], num_envs=2)
