"""Fused per-step inference of the RL loop: camera frames -> VAE mean -> [latent | measurements] -> PPO action / value in
ONE C call (cpb_encode_predict; cpb_mlpvae_encode_predict for an MlpVAE), one pinned H2D (frames + measurements + noise)
and one D2H (states + actions + values), for one environment or for N environments stepped in lockstep (B = N).

In the reference every environment step costs two TensorFlow session runs with a host round trip in between:
``encode_state_fn(env)`` (vae_common.py:45-61: sess.run(vae.mean)) inside ``env.step`` and then ``model.predict(state)``
(train.py:143, ppo.py:231-251).  ``FusedActor`` keeps that loop shape -- it hands the environment an ``encode_state_fn`` and
the loop a ``predict`` -- but computes both at ``encode_state_fn`` time and serves ``predict(state)`` from the cached result
when it is asked about the very state it just produced.  ``encode_predict(envs)`` does the same for several environments
at once.  Noise is drawn from the PPO object's generator exactly once per sampled action, in call order, so the fused and
the unfused loop (``UnfusedActor`` for several environments) produce identical trajectories.
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
        float32 noise [n, A]; out = float32 states [n, state_dim] | actions [n, A] | values [n]."""
        if n > self._capacity:
            torch, dev, ppo = self._torch, self.vae._device, self.ppo
            n_in = n * (self._frame_bytes + 4 * (self._m + ppo.num_actions))
            n_out = n * (ppo.state_dim + ppo.num_actions + 1)
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

    def encode_predict(self, envs):
        """The current frames of `envs` -> (states, actions [n, A], values [n]) in ONE cpb_encode_predict call at B = n:
        one H2D copy of the packed frames, measurements and noise, one D2H copy of the results.  states[i] is what
        encode_state_fn(envs[i]) returns.  The noise is ppo._rng.randn(n, A), rows in environment order (none when
        greedy)."""
        vae, ppo, torch = self.vae, self.ppo, self._torch
        n, a, sd, nf = len(envs), ppo.num_actions, ppo.state_dim, self._frame_bytes
        self._buffers(n)
        host = self._in_host.numpy()
        fview = host[n * nf:n * (nf + 4 * (self._m + a))].view(np.float32)
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
            fview[n * self._m:] = ppo._rng.randn(n, a).astype(np.float32).reshape(-1)   # the draw PPO.predict would make
        with torch.cuda.device(vae._device):
            n_in = n * (nf + 4 * (self._m + a))
            self._in_dev[:n_in].copy_(self._in_host[:n_in], non_blocking=True)
            base = self._in_dev.data_ptr()
            cfg = vae._config(n, _lib.FRAME_U8)
            ws_v = vae._workspace(n, _lib.WS_ENCODE)
            ws_p = ppo._workspace(n)
            out = self._out_dev.data_ptr()
            name = vae._API["encode_predict"]
            _lib.check(getattr(vae._libh, name)(
                C.byref(cfg), _lib.ptr(vae.params), base, base + n * nf, self._m, C.byref(ppo._c), _lib.ptr(ppo.params),
                None if self.greedy else base + n * (nf + 4 * self._m), _lib.ptr(self._latent), out, out + 4 * n * sd,
                out + 4 * n * (sd + a), _lib.ptr(self._flags), _lib.ptr(ws_v), ws_v.numel(), _lib.ptr(ws_p), ws_p.numel(),
                vae._stream()), name)
            n_out = n * (sd + a + 1)
            self._out_host[:n_out].copy_(self._out_dev[:n_out], non_blocking=True)
            torch.cuda.current_stream(vae._device).synchronize()
        res = self._out_host.numpy()
        st = res[:n * sd].reshape(n, sd)
        # vae_common.py:61: np.append(float32 latent, python floats) -> float64 state vector
        states = [np.append(st[i, :vae.z_dim].copy(), meas[i]) for i in range(n)]
        self.calls += 1
        return states, res[n * sd:n * (sd + a)].reshape(n, a).copy(), res[n * (sd + a):n_out].copy()

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
    vae_common.create_encode_states_fn), then one ``ppo.predict`` on all states, which draws ppo._rng.randn(n, A) --
    the noise FusedActor draws, so both produce the same trajectories."""

    def __init__(self, vae, ppo, measurements_to_include=("steer", "throttle", "speed")):
        from .vae_common import create_encode_states_fn
        self.ppo = ppo
        self._encode_states = create_encode_states_fn(vae, measurements_to_include)
        self.greedy = False

    def encode_predict(self, envs):
        states = self._encode_states(envs)
        actions, values = self.ppo.predict(np.stack(states), greedy=self.greedy)
        return states, np.reshape(actions, (len(envs), self.ppo.num_actions)), np.reshape(values, (len(envs),))
