"""Offline replay environment: stands in for the reference's ``CarlaEnv.carla_lap_env.CarlaLapEnv`` so that the re-authored
``train.py`` / ``run_eval.py`` loops (reference train.py:139-216, run_eval.py:30-73) run without the CARLA simulator.

Only the surface the training / evaluation loops and ``vae_common.create_encode_state_fn`` touch is provided
(SURVEY.md section 8f-3); the simulator itself (sensors, HUD, planner, reward shaping on real waypoints) is out of scope:

  * ``action_space`` with ``.shape / .low / .high``          (steer in [-1, 1], throttle in [0, 1], carla_lap_env.py), or
    with ``discrete_actions=(n_steer, n_throttle)`` a MultiDiscrete whose index i of a control is linspace(low, high, n)[i]
  * ``observation``                                           uint8 [80, 160, 3] camera frame (served from a recorded dataset)
  * ``vehicle.control.steer / .throttle``, ``vehicle.get_speed()``, ``vehicle.get_forward_vector()``
  * ``reset(is_training=True) -> state``, ``step(action) -> (state, reward, terminal, info)`` with ``info["closed"]``
  * ``render(mode)``, ``seed(seed)``, ``close()``, ``extra_info``, and the episodic counters the loops log
    (``distance_traveled``, ``speed_accum``, ``step_count``, ``center_lane_deviation``, ``average_fps``)

Dynamics (deterministic given the seed; NOT a driving simulator): frames are replayed in recorded order starting at a
seeded offset; the vehicle is a first-order longitudinal model driven by the throttle, the "lane deviation" integrates the
steering error against a slowly varying recorded-road curvature.  The reward is any callable of the environment
(``reward_fn(env)``), like the reference's reward_functions table.
"""
from __future__ import annotations

import types

import numpy as np


class Box:
    """The three attributes of gym.spaces.Box the PPO class reads (ppo.py:38); gym itself is not a dependency."""

    def __init__(self, low, high):
        self.low = np.asarray(low, np.float32)
        self.high = np.asarray(high, np.float32)
        self.shape = self.low.shape

    def sample(self, rng=np.random):
        return rng.uniform(self.low, self.high).astype(np.float32)


class Discrete:
    """gym.spaces.Discrete(n): the ``.n`` the PPO class reads."""

    def __init__(self, n):
        self.n = int(n)
        self.shape = ()

    def sample(self, rng=np.random):
        return int(rng.randint(self.n))


class MultiDiscrete:
    """gym.spaces.MultiDiscrete(nvec): the ``.nvec`` the PPO class reads."""

    def __init__(self, nvec):
        self.nvec = np.asarray(nvec, np.int64).reshape(-1)
        self.shape = self.nvec.shape

    def sample(self, rng=np.random):
        return np.array([rng.randint(n) for n in self.nvec], np.int64)


def discrete_controls(nvec, low=(-1.0, 0.0), high=(1.0, 1.0)):
    """Index -> control tables of a discretised (steer, throttle): component k's index i is linspace(low_k, high_k, n_k)[i]."""
    return [np.linspace(lo, hi, int(n)) for n, lo, hi in zip(nvec, low, high)]


class _Vehicle:
    def __init__(self):
        self.control = types.SimpleNamespace(steer=0.0, throttle=0.0)
        self.speed = 0.0          # m/s
        self.heading = 0.0

    def get_speed(self):
        return self.speed

    def get_forward_vector(self):
        return types.SimpleNamespace(x=float(np.cos(self.heading)), y=float(np.sin(self.heading)), z=0.0)


def reward_speed_centering(env, target_kmh=20.0):
    """Offline counterpart of the reference's speed x centering rewards (reward_functions.py): 1 at the target speed on
    the centre line, falling linearly with the speed error and the lane deviation."""
    kmh = 3.6 * env.vehicle.get_speed()
    speed_term = max(0.0, 1.0 - abs(kmh - target_kmh) / target_kmh)
    centre_term = max(0.0, 1.0 - abs(env.lane_offset) / env.max_lane_offset)
    return speed_term * centre_term


reward_functions = {"reward_speed_centering_angle_multiply": reward_speed_centering,
                    "reward_speed_centering": reward_speed_centering}


class ReplayEnv:
    action_space_box_low, action_space_box_high = (-1.0, 0.0), (1.0, 1.0)     # steer, throttle
    def __init__(self, frames, obs_res=(160, 80), action_smoothing=0.0, encode_state_fn=None, reward_fn=None,
                 synchronous=True, fps=30, start_carla=False, episode_length=256, seed=0, discrete_actions=None):
        frames = np.asarray(frames)
        if frames.dtype != np.uint8 or frames.ndim != 4 or tuple(frames.shape[1:]) != (obs_res[1], obs_res[0], 3):
            raise ValueError("frames must be uint8 [N, %d, %d, 3]" % (obs_res[1], obs_res[0]))
        self.frames = frames
        self.action_space = Box(self.action_space_box_low, self.action_space_box_high)
        # discrete_actions = (n_steer, n_throttle): the agent picks one of n_k evenly spaced values of each control
        self._controls = None
        if discrete_actions is not None:
            self.action_space = MultiDiscrete(discrete_actions)
            self._controls = discrete_controls(self.action_space.nvec, self.action_space_box_low, self.action_space_box_high)
        self.action_smoothing = float(action_smoothing)
        self.encode_state_fn = encode_state_fn if encode_state_fn is not None else (lambda env: env.observation)
        self.reward_fn = reward_fn if reward_fn is not None else reward_speed_centering
        self.fps = self.average_fps = float(fps)
        self.episode_length = int(episode_length)
        self.max_lane_offset = 3.0
        self.vehicle = _Vehicle()
        self.extra_info = []
        self.closed = False
        self._rng = np.random.RandomState(seed)
        self._cursor = 0
        self.observation = frames[0]
        self._reset_counters()

    # ------------------------------------------------------------------ reference surface
    def seed(self, seed):
        self._rng = np.random.RandomState(seed)

    def _reset_counters(self):
        self.step_count = 0
        self.total_reward = 0.0
        self.distance_traveled = 0.0
        self.speed_accum = 0.0
        self.center_lane_deviation = 0.0
        self.lane_offset = 0.0
        self.terminal_state = False

    def reset(self, is_training=True):
        self.is_training = bool(is_training)
        self._reset_counters()
        self.vehicle = _Vehicle()
        # training episodes start at a seeded offset of the recording; evaluation always replays from frame 0
        self._cursor = int(self._rng.randint(0, len(self.frames))) if is_training else 0
        self._phase = float(self._rng.uniform(0, 2 * np.pi)) if is_training else 0.0
        self.observation = self.frames[self._cursor]
        self.extra_info = []
        return self.encode_state_fn(self)

    def step(self, action):
        if action is not None:
            if self._controls is not None:
                steer, throttle = [float(t[int(i)]) for t, i in zip(self._controls, np.asarray(action).reshape(-1)[:2])]
            else:
                steer, throttle = [float(a) for a in np.asarray(action, np.float64).reshape(-1)[:2]]
            c = self.vehicle.control
            c.steer = c.steer * self.action_smoothing + steer * (1.0 - self.action_smoothing)
            c.throttle = c.throttle * self.action_smoothing + throttle * (1.0 - self.action_smoothing)
        dt = 1.0 / self.fps
        v = self.vehicle
        # first-order longitudinal model: 8 m/s^2 at full throttle, linear drag that tops out at 20 m/s
        v.speed = max(0.0, v.speed + (8.0 * v.control.throttle - 0.4 * v.speed) * dt)
        curvature = 0.3 * np.sin(self._phase + 0.05 * self.step_count)      # what the recorded road "asks" for
        v.heading += (v.control.steer - curvature) * v.speed * dt * 0.1
        self.lane_offset += np.sin(v.heading) * v.speed * dt
        self.distance_traveled += v.speed * dt
        self.speed_accum += v.speed
        self.center_lane_deviation += abs(self.lane_offset)
        self.step_count += 1
        self._cursor = (self._cursor + 1) % len(self.frames)
        self.observation = self.frames[self._cursor]
        if abs(self.lane_offset) > self.max_lane_offset or self.step_count >= self.episode_length:
            self.terminal_state = True
        self.last_reward = float(self.reward_fn(self))
        self.total_reward += self.last_reward
        self.extra_info = []
        return self.encode_state_fn(self), self.last_reward, self.terminal_state, {"closed": self.closed}

    def render(self, mode="human"):
        if mode == "rgb_array":
            return self.observation
        return None

    def close(self):
        self.closed = True
