"""Drop-in for the reference's ``vae_common.py``: ``load_vae``, ``preprocess_frame`` and
``create_encode_state_fn`` with the same signatures (vae_common.py:6-62), without importing ``carla``
at module import time (the reference does, through CarlaEnv.wrappers).
"""
from __future__ import annotations

import re

import numpy as np

from .vae.models import ConvVAE, MlpVAE, recorded_source_shape


def load_vae(model_dir, z_dim=None, model_type=None, source_shape=None):
    """Loads a pretrained VAE; z_dim / model type / target depth are parsed from the directory name when
    not given (vae_common.py:12-15).  The frame size is ``source_shape`` when given, else the one the checkpoint
    recorded (ConvVAE.save writes it), else the reference's 80x160x3.  Raises Exception("Failed to load VAE") like the
    reference."""
    if z_dim is None:
        z_dim = int(re.findall(r"zdim(\d+)", model_dir)[0])
    if model_type is None:
        model_type = "mlp" if "mlp" in model_dir else "cnn"
    vae_class = MlpVAE if model_type == "mlp" else ConvVAE
    target_depth = 1 if "seg_" in model_dir else 3
    if source_shape is None:
        source_shape = recorded_source_shape("{}/checkpoints/".format(model_dir)) or (80, 160, 3)
    h, w = int(source_shape[0]), int(source_shape[1])
    vae = vae_class(source_shape=np.array([h, w, 3]), target_shape=np.array([h, w, target_depth]),
                    z_dim=z_dim, models_dir="vae", model_dir=model_dir, training=False)
    vae.init_session(init_logging=False)
    if not vae.load_latest_checkpoint():
        raise Exception("Failed to load VAE")
    return vae


def preprocess_frame(frame):
    return frame.astype(np.float32) / 255.0


def _vector(v):
    """CarlaEnv.wrappers.vector: carla.Vector3D / Location / Rotation -> np.array."""
    if hasattr(v, "x"):
        return np.array([v.x, v.y, v.z])
    if hasattr(v, "pitch"):
        return np.array([v.pitch, v.yaw, v.roll])
    return np.asarray(v)


def create_encode_state_fn(vae, measurements_to_include):
    """Returns fn(env) -> np.float64[z_dim + M]: VAE mean of the current camera frame with the selected
    measurements appended (vae_common.py:33-62).  A uint8 observation is uploaded as uint8 and scaled by
    1/255 inside the conv1 loader -- numerically the same as preprocess_frame followed by a float feed."""
    encode_states = create_encode_states_fn(vae, measurements_to_include)
    return lambda env: encode_states([env])[0]


def create_encode_states_fn(vae, measurements_to_include):
    """create_encode_state_fn for several environments: fn(envs) -> [state of envs[i]], with ONE vae.encode on all their
    frames."""
    measure_flags = ["steer" in measurements_to_include, "throttle" in measurements_to_include,
                     "speed" in measurements_to_include, "orientation" in measurements_to_include]

    def encode_states(envs):
        frames = [env.observation for env in envs]
        if any(getattr(obs, "dtype", None) != np.uint8 for obs in frames):
            frames = [preprocess_frame(np.asarray(obs)) for obs in frames]
        encoded_states = vae.encode(frames)
        states = []
        for env, encoded_state in zip(envs, encoded_states):
            measurements = []
            if measure_flags[0]: measurements.append(env.vehicle.control.steer)
            if measure_flags[1]: measurements.append(env.vehicle.control.throttle)
            if measure_flags[2]: measurements.append(env.vehicle.get_speed())
            if measure_flags[3]: measurements.extend(_vector(env.vehicle.get_forward_vector()))
            states.append(np.append(encoded_state, measurements))
        return states

    return encode_states
