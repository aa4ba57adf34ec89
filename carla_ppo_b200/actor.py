"""Fused per-step inference of the RL loop: camera frame -> VAE mean -> [latent | measurements] -> PPO action / value in
ONE C call (cpb_encode_predict; cpb_mlpvae_encode_predict for an MlpVAE), one pinned H2D (frame + measurements + noise) and one D2H (state + action + value).

In the reference every environment step costs two TensorFlow session runs with a host round trip in between:
``encode_state_fn(env)`` (vae_common.py:45-61: sess.run(vae.mean)) inside ``env.step`` and then ``model.predict(state)``
(train.py:143, ppo.py:231-251).  ``FusedActor`` keeps that loop shape -- it hands the environment an ``encode_state_fn`` and
the loop a ``predict`` -- but computes both at ``encode_state_fn`` time and serves ``predict(state)`` from the cached result
when it is asked about the very state it just produced.  Noise is drawn from the PPO object's generator exactly once per
sampled action, in call order, so the fused and the unfused loop produce identical trajectories.
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
        torch = vae._torch
        self._torch = torch
        dev = vae._device
        a = ppo.num_actions
        self._nin = 80 * 160 * 3 + 4 * (self._m + a)                 # bytes: uint8 frame | float32 measurements | float32 noise
        self._in_host = torch.empty(self._nin, dtype=torch.uint8).pin_memory()
        self._in_dev = torch.empty(self._nin, dtype=torch.uint8, device=dev)
        self._out_dev = torch.empty(ppo.state_dim + a + 1, dtype=torch.float32, device=dev)
        self._out_host = torch.empty(ppo.state_dim + a + 1, dtype=torch.float32).pin_memory()
        self._latent = torch.empty(vae.z_dim, dtype=torch.float32, device=dev)
        self._flags = torch.zeros(1, dtype=torch.int32, device=dev)
        self.greedy = False          # run_eval sets this: no sampling noise (ppo.py:244-247, run_eval.py:51)
        self._cached = None
        self.calls = 0

    # -- the callback CarlaEnv / ReplayEnv invokes from reset() / step()
    def encode_state_fn(self, env):
        vae, ppo, torch = self.vae, self.ppo, self._torch
        obs = np.asarray(env.observation)
        if obs.dtype != np.uint8:
            raise TypeError("FusedActor expects the uint8 camera frame the environment produces")
        meas = []
        if self._flags_m[0]: meas.append(env.vehicle.control.steer)
        if self._flags_m[1]: meas.append(env.vehicle.control.throttle)
        if self._flags_m[2]: meas.append(env.vehicle.get_speed())
        if self._flags_m[3]: meas.extend(_vector(env.vehicle.get_forward_vector()))
        a = ppo.num_actions
        host = self._in_host.numpy()
        nf = 80 * 160 * 3
        host[:nf] = obs.reshape(-1)
        fview = host[nf:].view(np.float32)
        fview[:self._m] = np.asarray(meas, np.float32)
        noise = None
        if not self.greedy:
            noise = ppo._rng.randn(1, a).astype(np.float32)          # the same draw PPO.predict would make
            fview[self._m:] = noise.reshape(-1)
        with torch.cuda.device(vae._device):
            self._in_dev.copy_(self._in_host, non_blocking=True)
            base = self._in_dev.data_ptr()
            cfg = vae._config(1, _lib.FRAME_U8)
            ws_v = vae._workspace(1, _lib.WS_ENCODE)
            ws_p = ppo._workspace(1)
            sd = ppo.state_dim
            out = self._out_dev.data_ptr()
            name = vae._API["encode_predict"]
            _lib.check(getattr(vae._libh, name)(
                C.byref(cfg), _lib.ptr(vae.params), base, base + nf, self._m, C.byref(ppo._c), _lib.ptr(ppo.params),
                None if self.greedy else base + nf + 4 * self._m, _lib.ptr(self._latent), out, out + 4 * sd, out + 4 * (sd + a),
                _lib.ptr(self._flags), _lib.ptr(ws_v), ws_v.numel(), _lib.ptr(ws_p), ws_p.numel(), vae._stream()), name)
            self._out_host.copy_(self._out_dev, non_blocking=True)
            torch.cuda.current_stream(vae._device).synchronize()
        res = self._out_host.numpy()
        # vae_common.py:61: np.append(float32 latent, python floats) -> float64 state vector
        state = np.append(res[:vae.z_dim].copy(), meas)
        self._cached = (state, res[sd:sd + a].copy(), np.float32(res[sd + a]), self.greedy)
        self.calls += 1
        return state

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
