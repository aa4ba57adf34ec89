"""Running normalisation of the PPO's observations and rewards: Stable-Baselines3's ``VecNormalize`` on the device
(include/carla_ppo_b200.h, "Running normalisation").

Normalisation wraps the environment: the agent sees, stores and learns from the normalised states and rewards, while
``PPO.learn`` / ``train`` / ``predict`` stay as they are.  ``VecNormalize`` owns the device statistics (RunningMeanStd in
float64) and the discounted returns of the reward path, and is the only code that knows their format:

  * ``normalize_obs(states, update)``: states [B, D] -> normalised fp32 [B, D]; the statistics are first updated with the
    batch when ``update`` (default: ``training``).
  * ``normalize_rewards(rewards, dones, env_ids)``: the stepped environments' raw rewards -> normalised fp32 rewards
    (unchanged when reward normalisation is off or ``training`` is False).
  * ``actor_norm(...)``: the cpb_actor_norm of one FusedActor call, which does both inside the actor's C call.
  * ``state_dict()`` / ``load_state_dict(blob)``: the ``vec_normalize/*`` checkpoint variables.

The returns vector is not checkpointed (SB3 does not pickle it either); it starts at 0 and grows with the largest
environment index seen.
"""
from __future__ import annotations

import ctypes as C

import numpy as np

from . import _lib

EPSILON = 1e-8          # SB3's VecNormalize epsilon, added to the variance under the square root
KEYS_OBS = ("vec_normalize/obs_mean", "vec_normalize/obs_var", "vec_normalize/obs_count")
KEYS_RET = ("vec_normalize/ret_mean", "vec_normalize/ret_var", "vec_normalize/ret_count")
KEY_CLIP = "vec_normalize/clip"


def blob_normalization(blob):
    """(normalize_observations, normalize_rewards, clip_obs, clip_reward) a checkpoint blob records, or None for one
    without normalisation (the reference's).  Raises ValueError for an incomplete record."""
    obs, ret = (all(k in blob for k in keys) for keys in (KEYS_OBS, KEYS_RET))
    partial = [k for k in KEYS_OBS + KEYS_RET if k in blob and not (obs if k in KEYS_OBS else ret)]
    if partial or ((obs or ret) != (KEY_CLIP in blob)):
        raise ValueError("the checkpoint's vec_normalize record is incomplete")
    if not (obs or ret):
        return None
    clip = np.asarray(blob[KEY_CLIP], np.float32).reshape(-1)
    if clip.shape != (2,):
        raise ValueError("the checkpoint's %s must hold [clip_obs, clip_reward]" % KEY_CLIP)
    return obs, ret, float(clip[0]), float(clip[1])


class VecNormalize:
    def __init__(self, state_dim, normalize_observations=False, normalize_rewards=False, clip_obs=10.0, clip_reward=10.0,
                 gamma=0.99):
        self.state_dim = int(state_dim)
        self.norm_obs, self.norm_reward = bool(normalize_observations), bool(normalize_rewards)     # SB3's names
        self.clip_obs, self.clip_reward = float(np.float32(clip_obs)), float(np.float32(clip_reward))
        self.gamma = float(gamma)
        for name, v in (("clip_obs", self.clip_obs), ("clip_reward", self.clip_reward)):
            if not (np.isfinite(v) and v > 0):
                raise ValueError("%s must be finite and > 0, got %r" % (name, v))
        if not 0.0 <= self.gamma <= 1.0:
            raise ValueError("reward_gamma must lie in [0, 1], got %r" % (gamma,))
        self.training = True          # False: the statistics are frozen and rewards stay raw (evaluation)
        self._obs_cfg = _lib.RunningNorm(self.state_dim, self.clip_obs, EPSILON)
        self._ret_cfg = _lib.RunningNorm(1, self.clip_reward, EPSILON)
        self._torch = None

    @property
    def settings(self):
        """(normalize_observations, normalize_rewards, clip_obs, clip_reward), as blob_normalization reads them back"""
        return self.norm_obs, self.norm_reward, self.clip_obs, self.clip_reward

    def init_session(self, torch, lib, device, stream):
        """Device statistics at their initial values (mean 0, var 1, count 1e-4) and zero returns."""
        self._torch, self._libh, self._device, self._stream = torch, lib, device, stream
        f64 = dict(dtype=torch.float64, device=device)
        self.obs_stats = torch.empty(2 * self.state_dim + 1, **f64)
        self.ret_stats = torch.empty(3, **f64)
        self.returns = torch.zeros(1, **f64)
        with torch.cuda.device(device):
            for cfg, stats in ((self._obs_cfg, self.obs_stats), (self._ret_cfg, self.ret_stats)):
                _lib.check(lib.cpb_running_norm_init(C.byref(cfg), _lib.ptr(stats), stream()), "cpb_running_norm_init")

    # ------------------------------------------------------------------ inputs from the host
    def _env_ids(self, env_ids, n):
        """int32 env_ids after the host checks (distinct integers >= 0, one per reward); the returns grow to cover them."""
        ids = np.asarray(env_ids).reshape(-1)
        if ids.shape[0] != n or n < 1:
            raise ValueError("normalize_rewards: %d rewards need as many environment indices, got %d" % (n, ids.shape[0]))
        if not np.issubdtype(ids.dtype, np.integer) or np.any(ids < 0) or np.any(ids >= 2 ** 31 - 1):
            raise ValueError("environment indices must be integers >= 0, got %r" % (ids,))
        if len(np.unique(ids)) != n:
            raise ValueError("environment indices must be distinct, got %r" % (ids,))
        need = int(ids.max()) + 1
        if need > self.returns.shape[0]:
            grown = self._torch.zeros(need, dtype=self._torch.float64, device=self._device)
            grown[:self.returns.shape[0]].copy_(self.returns)
            self.returns = grown
        return ids.astype(np.int32)

    def reward_inputs(self, rewards, dones, env_ids):
        """(float32 rewards, int32 dones, int32 env_ids) of one reward batch, checked on the host."""
        r = np.asarray(rewards, np.float32).reshape(-1)
        d = np.asarray(dones).reshape(-1).astype(bool).astype(np.int32)
        if d.shape != r.shape:
            raise ValueError("normalize_rewards: %d rewards but %d terminal flags" % (r.shape[0], d.shape[0]))
        return r, d, self._env_ids(env_ids, r.shape[0])

    @property
    def reward_active(self):
        """True when rewards are normalised now (reward normalisation on and training)"""
        return self.norm_reward and self.training

    # ------------------------------------------------------------------ the entry points
    def normalize_obs(self, states, update=None):
        """states [B, D] -> fp32 [B, D], normalised with the running statistics (updated with the batch first when
        ``update``, default ``training``).  Returned unchanged (as fp32) when observation normalisation is off."""
        x = np.ascontiguousarray(np.asarray(states, np.float32).reshape(-1, self.state_dim))
        if not self.norm_obs:
            return x
        torch = self._torch
        update = self.training if update is None else bool(update)
        dev_x = torch.from_numpy(x).to(self._device)
        out = torch.empty_like(dev_x)
        with torch.cuda.device(self._device):
            _lib.check(self._libh.cpb_obs_normalize(C.byref(self._obs_cfg), _lib.ptr(self.obs_stats), _lib.ptr(dev_x),
                                                    x.shape[0], int(update), _lib.ptr(out), self._stream()),
                       "cpb_obs_normalize")
        return out.cpu().numpy()

    def normalize_rewards(self, rewards, dones, env_ids):
        """The stepped environments' raw rewards -> normalised fp32 rewards, updating their returns and the return
        statistics; the raw rewards as fp32 when reward normalisation is off or not training."""
        r, d, ids = self.reward_inputs(rewards, dones, env_ids)
        if not self.reward_active:
            return r
        torch = self._torch
        n = r.shape[0]
        packed = torch.from_numpy(np.concatenate([r.view(np.int32), d, ids])).to(self._device)
        out = torch.empty(n, dtype=torch.float32, device=self._device)
        with torch.cuda.device(self._device):
            self.normalize_rewards_on_device(_lib.ptr(packed[2 * n:]), _lib.ptr(packed), _lib.ptr(packed[n:]), n,
                                             _lib.ptr(out))
        return out.cpu().numpy()

    def normalize_rewards_on_device(self, env_ids, rewards, dones, n, out):
        """cpb_reward_normalize on device pointers of [n] inputs that reward_inputs checked, on the current stream."""
        _lib.check(self._libh.cpb_reward_normalize(
            C.byref(self._ret_cfg), _lib.ptr(self.ret_stats), _lib.ptr(self.returns), env_ids, rewards, dones, n,
            self.returns.shape[0], self.gamma, out, self._stream()), "cpb_reward_normalize")

    def actor_norm(self, update, env_ids=0, rewards=0, dones=0, rewards_out=0):
        """The cpb_actor_norm of one actor call: device pointers of the [B] reward inputs and output (rewards = 0: no
        reward path this call)."""
        n = _lib.ActorNorm()
        n.obs, n.obs_stats, n.update = self._obs_cfg, _lib.ptr(self.obs_stats), int(update)
        if rewards:
            n.reward, n.ret_stats, n.returns = self._ret_cfg, _lib.ptr(self.ret_stats), _lib.ptr(self.returns)
            n.env_ids, n.rewards, n.dones, n.rewards_out = env_ids, rewards, dones, rewards_out
            n.num_envs, n.gamma = self.returns.shape[0], self.gamma
        return n

    # ------------------------------------------------------------------ checkpoints
    def state_dict(self):
        """The vec_normalize/* checkpoint variables of the parts that are on."""
        out = {}
        if self.norm_obs:
            s = self.obs_stats.cpu().numpy()
            D = self.state_dim
            out.update(zip(KEYS_OBS, (s[:D].copy(), s[D:2 * D].copy(), np.float64(s[2 * D]))))
        if self.norm_reward:
            out.update(zip(KEYS_RET, (np.float64(v) for v in self.ret_stats.cpu().numpy())))
        if out:
            out[KEY_CLIP] = np.asarray([self.clip_obs, self.clip_reward], np.float32)
        return out

    def load_state_dict(self, blob):
        """Restore the statistics from a checkpoint blob whose settings (blob_normalization) are this object's."""
        torch = self._torch
        if self.norm_obs:
            s = np.concatenate([np.asarray(blob[KEYS_OBS[0]], np.float64).reshape(-1),
                                np.asarray(blob[KEYS_OBS[1]], np.float64).reshape(-1),
                                np.asarray(blob[KEYS_OBS[2]], np.float64).reshape(-1)])
            if s.shape[0] != 2 * self.state_dim + 1:
                raise ValueError("the checkpoint's observation statistics are not %d wide" % self.state_dim)
            self.obs_stats.copy_(torch.from_numpy(s))
        if self.norm_reward:
            s = np.array([float(np.asarray(blob[k], np.float64).reshape(-1)[0]) for k in KEYS_RET], np.float64)
            self.ret_stats.copy_(torch.from_numpy(s))
