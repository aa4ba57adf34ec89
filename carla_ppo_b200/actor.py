"""Fused per-step inference of the RL loop: camera frames -> VAE mean -> [latent | measurements] -> PPO action / value in
ONE C call (cpb_vae_spec_ppo_spec_encode_predict; cpb_mlpvae_ppo_spec_encode_predict for an MlpVAE), one pinned H2D (frames + measurements + noise)
and one D2H (states + actions + values), for one environment or for N environments stepped in lockstep (B = N).

In the reference every environment step costs two TensorFlow session runs with a host round trip in between:
``encode_state_fn(env)`` (vae_common.py:45-61: sess.run(vae.mean)) inside ``env.step`` and then ``model.predict(state)``
(train.py:143, ppo.py:231-251).  ``FusedActor`` keeps that loop shape -- it hands the environment an ``encode_state_fn`` and
the loop a ``predict`` -- but computes both at ``encode_state_fn`` time and serves ``predict(state)`` from the cached result
when it is asked about the very state it just produced.  ``encode_predict(envs)`` does the same for several environments
at once.  Noise is drawn from the PPO object's generator exactly once per sampled action, in call order, so the fused and
the unfused loop (``UnfusedActor`` for several environments) produce identical trajectories.  A categorical PPO
(discrete action space) runs through the cpb_*_ppo_cat_encode_predict twins with uniform noise.

With running normalisation on (``PPO(normalize_observations=..., normalize_rewards=...)``, vec_normalize.py) the call
goes through the *_encode_predict_norm twins: the states come back normalised, and ``encode_predict`` takes the stepped
environments' raw rewards, terminal flags and indices and returns their normalised rewards from the same H2D, call and
D2H.  With normalisation off it makes exactly the calls it makes without it.
"""
from __future__ import annotations

import ctypes as C

import numpy as np

from . import _lib
from .vae_common import _vector


class FusedActor:
    def __init__(self, vae, ppo, measurements_to_include=("steer", "throttle", "speed")):
        self.vae, self.ppo = vae, ppo
        ppo._require_session(); vae._require_session()
        self._flags_m = ["steer" in measurements_to_include, "throttle" in measurements_to_include,
                         "speed" in measurements_to_include, "orientation" in measurements_to_include]
        self._m = sum(self._flags_m[:3]) + (3 if self._flags_m[3] else 0)
        if vae.z_dim + self._m != ppo.state_dim:
            raise ValueError("PPO state_dim %d != z_dim %d + %d measurements" % (ppo.state_dim, vae.z_dim, self._m))
        if str(vae._device) != str(ppo._device):
            raise ValueError("VAE and PPO must live on the same device")
        self._torch = vae._torch
        self._frame_bytes = int(np.prod(vae.source_shape))     # one uint8 frame at the VAE's frame size
        self._capacity = 0           # environments the pinned / device buffers hold
        self.greedy = False          # run_eval sets this: no sampling noise (ppo.py:244-247, run_eval.py:51)
        self._cached = None
        self.calls = 0

    def _buffers(self, n):
        """Pinned host / device buffers for n environments: in = uint8 frames [n, H, W, 3] | float32 measurements [n, M] |
        float32 noise [n, A] (| float32 rewards [n] | int32 dones [n] | int32 env_ids [n]); out = float32 states
        [n, state_dim] | actions [n, A] | values [n] (| normalised rewards [n])."""
        if n > self._capacity:
            torch, dev, ppo = self._torch, self.vae._device, self.ppo
            n_in = n * (self._frame_bytes + 4 * (self._m + ppo.num_actions + 3))
            n_out = n * (ppo.state_dim + ppo.num_actions + 2)
            self._in_host = torch.empty(n_in, dtype=torch.uint8).pin_memory()
            self._in_dev = torch.empty(n_in, dtype=torch.uint8, device=dev)
            self._out_dev = torch.empty(n_out, dtype=torch.float32, device=dev)
            self._out_host = torch.empty(n_out, dtype=torch.float32).pin_memory()
            self._latent = torch.empty(n * self.vae.z_dim, dtype=torch.float32, device=dev)
            self._flags = torch.zeros(1, dtype=torch.int32, device=dev)
            self._capacity = n

    def _measurements(self, env):
        meas = []
        if self._flags_m[0]: meas.append(env.vehicle.control.steer)
        if self._flags_m[1]: meas.append(env.vehicle.control.throttle)
        if self._flags_m[2]: meas.append(env.vehicle.get_speed())
        if self._flags_m[3]: meas.extend(_vector(env.vehicle.get_forward_vector()))
        return meas

    def encode_predict(self, envs, rewards=None, dones=None, env_ids=None):
        """The current frames of `envs` -> (states, actions [n, A], values [n]) in ONE cpb_encode_predict call at B = n:
        one H2D copy of the packed frames, measurements and noise, one D2H copy of the results.  states[i] is what
        encode_state_fn(envs[i]) returns.  The noise is ppo._rng.randn(n, A), rows in environment order (none when
        greedy); for a categorical PPO it is ppo._rng.rand(n, K) and the actions are int64 indices.

        ``rewards`` / ``dones`` / ``env_ids`` ([n] each: the raw rewards and terminal flags of the step that produced
        these frames, and the environments' indices) add a fourth result: the rewards as the agent sees them, normalised
        when the PPO normalises rewards and is training, else as given (float32).  With observation normalisation on,
        states[i] is the normalised float32 state."""
        vae, ppo, torch = self.vae, self.ppo, self._torch
        n, a, sd, nf = len(envs), ppo.num_actions, ppo.state_dim, self._frame_bytes
        norm = getattr(ppo, "vec_normalize", None)
        if rewards is not None:
            r_in = (norm.reward_inputs(rewards, dones, env_ids) if norm is not None
                    else (np.asarray(rewards, np.float32).reshape(-1),))
            if r_in[0].shape[0] != n:
                raise ValueError("encode_predict: %d environments but %d rewards" % (n, r_in[0].shape[0]))
        with_rewards = rewards is not None and norm is not None and norm.reward_active
        with_obs = norm is not None and norm.norm_obs
        self._buffers(n)
        host = self._in_host.numpy()
        n_in = n * (nf + 4 * (self._m + a + (3 if with_rewards else 0)))
        fview = host[n * nf:n_in].view(np.float32)
        meas = []
        for i, env in enumerate(envs):
            obs = np.asarray(env.observation)
            if obs.dtype != np.uint8:
                raise TypeError("FusedActor expects the uint8 camera frame the environment produces")
            host[i * nf:(i + 1) * nf] = obs.reshape(-1)
            meas.append(self._measurements(env))
        if self._m:
            fview[:n * self._m] = np.asarray(meas, np.float32).reshape(-1)
        if not self.greedy:
            draw = ppo._rng.randn if ppo.action_categories is None else ppo._rng.rand
            fview[n * self._m:n * (self._m + a)] = draw(n, a).astype(np.float32).reshape(-1)   # the draw PPO.predict would make
        if with_rewards:
            fview[n * (self._m + a):] = np.concatenate([r_in[0], r_in[1].view(np.float32), r_in[2].view(np.float32)])
        with torch.cuda.device(vae._device):
            self._in_dev[:n_in].copy_(self._in_host[:n_in], non_blocking=True)
            base = self._in_dev.data_ptr()
            cfg = vae._config(n, _lib.FRAME_U8)
            ws_v = vae._workspace(n, _lib.WS_ENCODE)
            ws_p = ppo._workspace(n)
            out = self._out_dev.data_ptr()
            name = vae._API["encode_predict" if ppo.action_categories is None else "encode_predict_cat"]
            rw = base + n * (nf + 4 * (self._m + a))                  # rewards | dones | env_ids on the device
            r_out = out + 4 * n * (sd + a + 1)
            args = (C.byref(cfg), _lib.ptr(vae.params), base, base + n * nf, self._m, C.byref(ppo._spec), _lib.ptr(ppo.params),
                    None if self.greedy else base + n * (nf + 4 * self._m), _lib.ptr(self._latent), out, out + 4 * n * sd,
                    out + 4 * n * (sd + a), _lib.ptr(self._flags), _lib.ptr(ws_v), ws_v.numel(), _lib.ptr(ws_p), ws_p.numel(),
                    vae._stream())
            if with_obs:
                an = (norm.actor_norm(norm.training, rw + 8 * n, rw, rw + 4 * n, r_out) if with_rewards
                      else norm.actor_norm(norm.training))
                _lib.check(getattr(vae._libh, name + "_norm")(*args, C.byref(an)), name + "_norm")
            else:
                _lib.check(getattr(vae._libh, name)(*args), name)
                if with_rewards:
                    norm.normalize_rewards_on_device(rw + 8 * n, rw, rw + 4 * n, n, r_out)
            n_out = n * (sd + a + (2 if with_rewards else 1))
            self._out_host[:n_out].copy_(self._out_dev[:n_out], non_blocking=True)
            torch.cuda.current_stream(vae._device).synchronize()
        res = self._out_host.numpy()
        st = res[:n * sd].reshape(n, sd)
        if with_obs:
            states = [st[i].copy() for i in range(n)]
        else:
            # vae_common.py:61: np.append(float32 latent, python floats) -> float64 state vector
            states = [np.append(st[i, :vae.z_dim].copy(), meas[i]) for i in range(n)]
        self.calls += 1
        actions = res[n * sd:n * (sd + a)].reshape(n, a).copy()
        if ppo.action_categories is not None:
            actions = actions.astype(np.int64)
        values = res[n * (sd + a):n * (sd + a + 1)].copy()
        if rewards is None:
            return states, actions, values
        return states, actions, values, (res[n * (sd + a + 1):n_out].copy() if with_rewards else r_in[0])

    # -- the callback CarlaEnv / ReplayEnv invokes from reset() / step()
    def encode_state_fn(self, env):
        states, actions, values = self.encode_predict([env])
        self._cached = (states[0], actions[0], np.float32(values[0]), self.greedy)
        return states[0]

    # -- drop-in for model.predict(state, greedy=..., write_to_summary=...)
    def predict(self, state, greedy=False, write_to_summary=False):
        c = self._cached
        if c is not None and c[0] is state and c[3] == bool(greedy):
            self._cached = None
            if write_to_summary:
                if self.ppo.train_writer is not None:
                    for i in range(self.ppo.num_actions):
                        self.ppo.train_writer.add_scalar("predict_actor/action_%d/sampled_action" % i, float(c[1][i]), self.ppo.predict_step_counter)
                self.ppo.predict_step_counter += 1
            return c[1], c[2]
        return self.ppo.predict(state, greedy=greedy, write_to_summary=write_to_summary)


class UnfusedActor:
    """FusedActor.encode_predict as the reference's two separate steps: one ``vae.encode`` on all frames (through
    vae_common.create_encode_states_fn), then one ``ppo.predict`` on all states, which draws ppo._rng.randn(n, A)
    (rand(n, K) for a categorical PPO) -- the noise FusedActor draws, so both produce the same trajectories.  With
    running normalisation the states go through cpb_obs_normalize between the two, and the rewards through
    cpb_reward_normalize."""

    def __init__(self, vae, ppo, measurements_to_include=("steer", "throttle", "speed")):
        from .vae_common import create_encode_states_fn
        self.ppo = ppo
        self._encode_states = create_encode_states_fn(vae, measurements_to_include, getattr(ppo, "vec_normalize", None))
        self.greedy = False

    def encode_predict(self, envs, rewards=None, dones=None, env_ids=None):
        states = self._encode_states(envs)
        actions, values = self.ppo.predict(np.stack(states), greedy=self.greedy)
        res = states, np.reshape(actions, (len(envs), self.ppo.num_actions)), np.reshape(values, (len(envs),))
        if rewards is None:
            return res
        norm = getattr(self.ppo, "vec_normalize", None)
        return res + (np.asarray(rewards, np.float32).reshape(-1) if norm is None
                      else norm.normalize_rewards(rewards, dones, env_ids),)
