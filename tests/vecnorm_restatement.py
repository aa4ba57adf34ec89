"""A float64 NumPy restatement of Stable-Baselines3's VecNormalize, the semantics of the running normalisation
(include/carla_ppo_b200.h, "Running normalisation").  SB3 is not a dependency; this restates, line for line:

  * stable_baselines3/common/running_mean_std.py: RunningMeanStd(epsilon=1e-4) -- ``update`` (batch mean and np.var,
    then ``update_from_moments``, Chan's parallel formula);
  * stable_baselines3/common/vec_env/vec_normalize.py: ``normalize_obs`` (clip((obs - mean) / sqrt(var + epsilon),
    +-clip_obs)), ``_update_reward`` (returns = returns * gamma + reward; ret_rms.update(returns)),
    ``normalize_reward`` (clip(reward / sqrt(ret_var + epsilon), +-clip_reward)) and the ``returns[dones] = 0`` of
    ``step_wait``.

The reward path takes a subset of the environments (env_ids) per step, as the lockstep loop steps only the active ones.
"""
import numpy as np

EPSILON = 1e-8


class RunningMeanStd:
    def __init__(self, shape=(), epsilon=1e-4):
        self.mean = np.zeros(shape, np.float64)
        self.var = np.ones(shape, np.float64)
        self.count = epsilon

    def update(self, arr):
        arr = np.asarray(arr, np.float64)
        batch_mean = np.mean(arr, axis=0)
        batch_var = np.var(arr, axis=0)
        batch_count = arr.shape[0]
        self.update_from_moments(batch_mean, batch_var, batch_count)

    def update_from_moments(self, batch_mean, batch_var, batch_count):
        delta = batch_mean - self.mean
        tot_count = self.count + batch_count
        new_mean = self.mean + delta * batch_count / tot_count
        m_a = self.var * self.count
        m_b = batch_var * batch_count
        m_2 = m_a + m_b + np.square(delta) * self.count * batch_count / tot_count
        new_var = m_2 / tot_count
        new_count = batch_count + self.count
        self.mean, self.var, self.count = new_mean, new_var, new_count

    def stats(self):
        """[mean | var | count], the device layout"""
        return np.concatenate([np.atleast_1d(self.mean), np.atleast_1d(self.var), [self.count]])


def normalize_obs(rms, obs, clip_obs=10.0, epsilon=EPSILON, update=True):
    """VecNormalize's observation path: update (when training), then normalise with the updated statistics."""
    obs = np.asarray(obs, np.float64)
    if update:
        rms.update(obs)
    return np.clip((obs - rms.mean) / np.sqrt(rms.var + epsilon), -clip_obs, clip_obs)


class RewardNormalizer:
    def __init__(self, num_envs, gamma=0.99, clip_reward=10.0, epsilon=EPSILON):
        self.ret_rms = RunningMeanStd(shape=())
        self.returns = np.zeros(num_envs, np.float64)
        self.gamma, self.clip_reward, self.epsilon = gamma, clip_reward, epsilon

    def _update_reward(self, reward, env_ids):
        self.returns[env_ids] = self.returns[env_ids] * self.gamma + reward
        self.ret_rms.update(self.returns[env_ids])

    def normalize_reward(self, reward):
        return np.clip(reward / np.sqrt(self.ret_rms.var + self.epsilon), -self.clip_reward, self.clip_reward)

    def step(self, rewards, dones, env_ids):
        rewards = np.asarray(rewards, np.float64)
        env_ids = np.asarray(env_ids)
        self._update_reward(rewards, env_ids)
        out = self.normalize_reward(rewards)
        self.returns[env_ids[np.asarray(dones, bool)]] = 0
        return out
