"""ctypes binding of libcarla_ppo_b200.so (the C ABI declared in include/carla_ppo_b200.h).

There is NO fallback: if the shared library is missing or a call fails, this raises.  PyTorch is used
only as the owner of device memory and CUDA streams (tensor.data_ptr(), current stream handle).
"""
from __future__ import annotations

import ctypes as C
import os
from typing import Optional

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(_HERE, "libcarla_ppo_b200.so")

LOSS_MSE, LOSS_BCE, LOSS_BCE_V2 = 0, 1, 2
FRAME_F32, FRAME_U8 = 0, 1
WS_ENCODE, WS_FORWARD, WS_TRAIN = 0, 1, 2
# cpb_set_math_mode: fp32 SIMT, 3xTF32 wgmma (default, fp32-accurate), one TF32 wgmma pass (not fp32-accurate)
MATH_SIMT, MATH_3XTF32, MATH_TF32 = 0, 1, 2


class CpbError(RuntimeError):
    pass


class VaeConfig(C.Structure):
    _fields_ = [("batch", C.c_int32), ("target_channels", C.c_int32), ("z_dim", C.c_int32),
                ("loss_type", C.c_int32), ("source_dtype", C.c_int32), ("target_dtype", C.c_int32),
                ("target_u8_scale", C.c_float), ("beta", C.c_float), ("kl_tolerance", C.c_float),
                ("loss_scale", C.c_float)]


class VaeSpec(C.Structure):
    """A ConvVAE at frame size height x width (each a multiple of 16 in [48, 512])."""
    _fields_ = [("base", VaeConfig), ("height", C.c_int32), ("width", C.c_int32)]


class MlpVaeConfig(C.Structure):
    _fields_ = [("base", VaeConfig), ("enc1", C.c_int32), ("enc2", C.c_int32), ("dec1", C.c_int32), ("dec2", C.c_int32)]


MLP_MAX_LAYERS = 8


class MlpVaeSpec(C.Structure):
    _fields_ = [("base", VaeConfig), ("num_encoder", C.c_int32), ("encoder_sizes", C.c_int32 * MLP_MAX_LAYERS),
                ("num_decoder", C.c_int32), ("decoder_sizes", C.c_int32 * MLP_MAX_LAYERS)]

    @classmethod
    def of(cls, base, encoder_sizes, decoder_sizes):
        """The spec of an MlpVAE with these hidden-layer sizes (at most MLP_MAX_LAYERS per side)."""
        return cls(base, len(encoder_sizes), (C.c_int32 * MLP_MAX_LAYERS)(*encoder_sizes), len(decoder_sizes),
                   (C.c_int32 * MLP_MAX_LAYERS)(*decoder_sizes))


class PpoConfig(C.Structure):
    _fields_ = [("state_dim", C.c_int32), ("num_actions", C.c_int32), ("hidden1", C.c_int32),
                ("hidden2", C.c_int32), ("action_low", C.c_float * 4), ("action_high", C.c_float * 4),
                ("epsilon", C.c_float), ("value_scale", C.c_float), ("entropy_scale", C.c_float)]


PPO_MAX_LAYERS = 8
PPO_DEFAULT_HIDDEN = (500, 300)       # the reference's policy and value trunks (ppo.py:17)


class PpoSpec(C.Structure):
    """cpb_ppo_spec: the policy and value trunks' hidden-layer sizes (1..PPO_MAX_LAYERS each, every width >= 1).
    base.hidden1 / base.hidden2 stay 0."""
    _fields_ = [("base", PpoConfig), ("num_policy", C.c_int32), ("policy_sizes", C.c_int32 * PPO_MAX_LAYERS),
                ("num_value", C.c_int32), ("value_sizes", C.c_int32 * PPO_MAX_LAYERS)]

    @classmethod
    def of(cls, base, policy_sizes, value_sizes):
        """The spec of the PPO on `base` (a PpoConfig; its hidden1 / hidden2 are dropped) with these trunks.  Lists longer
        than PPO_MAX_LAYERS raise here; every other bound is checked by the library."""
        if len(policy_sizes) > PPO_MAX_LAYERS or len(value_sizes) > PPO_MAX_LAYERS:
            raise ValueError("at most %d hidden layers per trunk, got %d and %d"
                             % (PPO_MAX_LAYERS, len(policy_sizes), len(value_sizes)))
        b = PpoConfig.from_buffer_copy(base)
        b.hidden1 = b.hidden2 = 0
        return cls(b, len(policy_sizes), (C.c_int32 * PPO_MAX_LAYERS)(*policy_sizes), len(value_sizes),
                   (C.c_int32 * PPO_MAX_LAYERS)(*value_sizes))


PPO_MAX_LOGITS = 64


class PpoCatSpec(C.Structure):
    """cpb_ppo_cat_spec: a cpb_ppo_spec with a categorical policy head.  spec.base.num_actions = K components (1..4),
    num_categories[k] = n_k (2..64 each, 64 in all); spec.base.action_low / action_high stay 0."""
    _fields_ = [("spec", PpoSpec), ("num_categories", C.c_int32 * 4)]

    @classmethod
    def of(cls, base, policy_sizes, value_sizes, categories):
        """The spec of the categorical PPO on `base` (its num_actions and action bounds are replaced) with these trunks
        and components.  Every bound is checked by the library."""
        b = PpoConfig.from_buffer_copy(base)
        b.num_actions = len(categories)
        for k in range(4):
            b.action_low[k] = b.action_high[k] = 0.0
        cats = list(categories)[:4] + [0] * max(0, 4 - len(categories))
        return cls(PpoSpec.of(b, policy_sizes, value_sizes), (C.c_int32 * 4)(*cats))


class PpoLearnOptions(C.Structure):
    """cpb_ppo_learn_options: 0 turns a guard off."""
    _fields_ = [("max_grad_norm", C.c_float), ("target_kl", C.c_float)]


class RunningNorm(C.Structure):
    """cpb_running_norm: the statistics' width, the clip and the epsilon under the square root."""
    _fields_ = [("dim", C.c_int32), ("clip", C.c_float), ("epsilon", C.c_double)]


class ActorNorm(C.Structure):
    """cpb_actor_norm: the normalisation of one actor call (rewards = None: no rewards this step)."""
    _fields_ = [("obs", RunningNorm), ("obs_stats", C.c_void_p), ("update", C.c_int32), ("reward", RunningNorm),
                ("ret_stats", C.c_void_p), ("returns", C.c_void_p), ("env_ids", C.c_void_p), ("rewards", C.c_void_p),
                ("dones", C.c_void_p), ("num_envs", C.c_int32), ("gamma", C.c_double), ("rewards_out", C.c_void_p)]


_P = C.c_void_p
_i32, _i64, _f32, _f64 = C.c_int32, C.c_int64, C.c_float, C.c_double
_RN = C.POINTER(RunningNorm)
_AN = C.POINTER(ActorNorm)
_VC = C.POINTER(VaeConfig)
_VS = C.POINTER(VaeSpec)
_MC = C.POINTER(MlpVaeConfig)
_MS = C.POINTER(MlpVaeSpec)
_PC = C.POINTER(PpoConfig)
_PO = C.POINTER(PpoLearnOptions)
_PS = C.POINTER(PpoSpec)
_PK = C.POINTER(PpoCatSpec)

# name -> (restype, argtypes); must list every symbol of include/carla_ppo_b200.h
PROTOTYPES = {
    "cpb_last_error": (C.c_char_p, []),
    "cpb_build_info": (C.c_char_p, []),
    "cpb_vae_num_tensors": (_i32, []),
    "cpb_vae_tensor_name": (C.c_char_p, [_i32]),
    "cpb_vae_layout": (_i32, [_i32, _i32, _P, _P, _P, _P]),
    "cpb_vae_workspace_bytes": (_i64, [_i32, _i32, _i32, _i32]),
    "cpb_vae_encode": (_i32, [_VC, _P, _P, _P, _P, _P, _P, _i64, _P]),
    "cpb_vae_decode": (_i32, [_VC, _P, _P, _P, _P, _i64, _P]),
    "cpb_vae_forward": (_i32, [_VC, _P, _P, _P, _P, _P, _P, _P, _P, _P, _P, _P, _i64, _P]),
    "cpb_vae_loss_grad": (_i32, [_VC, _P, _P, _P, _P, _P, _P, _P, _P, _i64, _P]),
    "cpb_adam_apply": (_i32, [_P, _P, _P, _P, _i64, _P, _f32, _P, _f32, _f32, _f32, _P]),
    "cpb_adam_apply_guarded": (_i32, [_P, _P, _P, _P, _i64, _P, _f32, _P, _f32, _f32, _f32, _P, _P]),
    "cpb_vae_train_step": (_i32, [_VC, _P, _P, _P, _P, _P, _f32, _P, _P, _P, _P, _P, _P, _i64, _P]),
    "cpb_vae_staging_bytes": (_i64, [_VC]),
    "cpb_vae_train_step_host": (_i32, [_VC, _P, _P, _P, _P, _P, _f32, _P, _P, _P, _P, _P, _P, _i64, _P, _i64, _P]),
    "cpb_vae_spec_layout": (_i32, [_VS, _P, _P, _P, _P]),
    "cpb_vae_spec_workspace_bytes": (_i64, [_VS, _i32]),
    "cpb_vae_spec_encode": (_i32, [_VS, _P, _P, _P, _P, _P, _P, _i64, _P]),
    "cpb_vae_spec_decode": (_i32, [_VS, _P, _P, _P, _P, _i64, _P]),
    "cpb_vae_spec_forward": (_i32, [_VS, _P, _P, _P, _P, _P, _P, _P, _P, _P, _P, _P, _i64, _P]),
    "cpb_vae_spec_loss_grad": (_i32, [_VS, _P, _P, _P, _P, _P, _P, _P, _P, _i64, _P]),
    "cpb_vae_spec_train_step": (_i32, [_VS, _P, _P, _P, _P, _P, _f32, _P, _P, _P, _P, _P, _P, _i64, _P]),
    "cpb_vae_spec_staging_bytes": (_i64, [_VS]),
    "cpb_vae_spec_train_step_host": (_i32, [_VS, _P, _P, _P, _P, _P, _f32, _P, _P, _P, _P, _P, _P, _i64, _P, _i64, _P]),
    "cpb_vae_spec_encode_predict": (_i32, [_VS, _P, _P, _P, _i32, _PC, _P, _P, _P, _P, _P, _P, _P, _P, _i64, _P, _i64, _P]),
    "cpb_mlpvae_num_tensors": (_i32, []),
    "cpb_mlpvae_tensor_name": (C.c_char_p, [_i32]),
    "cpb_mlpvae_layout": (_i32, [_MC, _P, _P, _P, _P]),
    "cpb_mlpvae_workspace_bytes": (_i64, [_MC, _i32]),
    "cpb_mlpvae_encode": (_i32, [_MC, _P, _P, _P, _P, _P, _P, _i64, _P]),
    "cpb_mlpvae_decode": (_i32, [_MC, _P, _P, _P, _P, _i64, _P]),
    "cpb_mlpvae_forward": (_i32, [_MC, _P, _P, _P, _P, _P, _P, _P, _P, _P, _P, _P, _i64, _P]),
    "cpb_mlpvae_loss_grad": (_i32, [_MC, _P, _P, _P, _P, _P, _P, _P, _P, _i64, _P]),
    "cpb_mlpvae_spec_num_tensors": (_i32, [_MS]),
    "cpb_mlpvae_spec_tensor_name": (C.c_char_p, [_MS, _i32]),
    "cpb_mlpvae_spec_layout": (_i32, [_MS, _P, _P, _P, _P]),
    "cpb_mlpvae_spec_workspace_bytes": (_i64, [_MS, _i32]),
    "cpb_mlpvae_spec_encode": (_i32, [_MS, _P, _P, _P, _P, _P, _P, _i64, _P]),
    "cpb_mlpvae_spec_decode": (_i32, [_MS, _P, _P, _P, _P, _i64, _P]),
    "cpb_mlpvae_spec_forward": (_i32, [_MS, _P, _P, _P, _P, _P, _P, _P, _P, _P, _P, _P, _i64, _P]),
    "cpb_mlpvae_spec_loss_grad": (_i32, [_MS, _P, _P, _P, _P, _P, _P, _P, _P, _i64, _P]),
    "cpb_mlpvae_encode_predict": (_i32, [_MS, _P, _P, _P, _i32, _PC, _P, _P, _P, _P, _P, _P, _P, _P, _i64, _P, _i64, _P]),
    "cpb_ppo_num_tensors": (_i32, []),
    "cpb_ppo_tensor_name": (C.c_char_p, [_i32]),
    "cpb_ppo_layout": (_i32, [_PC, _P, _P, _P, _P]),
    "cpb_ppo_workspace_bytes": (_i64, [_PC, _i32, _i32]),
    "cpb_ppo_forward": (_i32, [_PC, _P, _P, _i32, _P, _P, _P, _P, _i64, _P]),
    "cpb_ppo_loss_grad": (_i32, [_PC, _P, _P, _P, _P, _P, _P, _P, _i32, _P, _P, _P, _i64, _P]),
    "cpb_ppo_train_step": (_i32, [_PC, _P, _P, _P, _P, _P, _P, _P, _P, _P, _P, _P, _P, _i32, _P, _P, _i64, _P]),
    "cpb_encode_predict": (_i32, [_VC, _P, _P, _P, _i32, _PC, _P, _P, _P, _P, _P, _P, _P, _P, _i64, _P, _i64, _P]),
    "cpb_gae": (_i32, [_P, _P, _f64, _P, _i32, _f64, _f64, _P, _P, _P, _P]),
    "cpb_ppo_learn": (_i32, [_PC, _P, _P, _P, _P, _P, _P, _P, _P, _P, _P, _P, _f64, _P, _i32, _f64, _f64,
                             _i32, _i32, _P, _P, _P, _i64, _P]),
    "cpb_gae_segments": (_i32, [_P, _P, _P, _P, _P, _i32, _i32, _f64, _f64, _P, _P, _P, _P]),
    "cpb_ppo_learn_segments": (_i32, [_PC, _P, _P, _P, _P, _P, _P, _P, _P, _P, _P, _P, _P, _P, _P, _i32, _i32, _f64, _f64,
                                      _i32, _i32, _P, _P, _P, _i64, _P]),
    "cpb_ppo_learn_opts": (_i32, [_PC, _P, _P, _P, _P, _P, _P, _P, _P, _P, _P, _P, _f64, _P, _i32, _f64, _f64,
                                  _i32, _i32, _P, _P, _PO, _P, _P, _i64, _P]),
    "cpb_ppo_learn_segments_opts": (_i32, [_PC, _P, _P, _P, _P, _P, _P, _P, _P, _P, _P, _P, _P, _P, _P, _i32, _i32, _f64,
                                           _f64, _i32, _i32, _P, _P, _PO, _P, _P, _i64, _P]),
    "cpb_ppo_train_step_opts": (_i32, [_PC, _P, _P, _P, _P, _P, _P, _P, _P, _P, _P, _P, _P, _i32, _P, _PO, _P, _P, _P,
                                       _i64, _P]),
    "cpb_ppo_spec_num_tensors": (_i32, [_PS]),
    "cpb_ppo_spec_tensor_name": (C.c_char_p, [_PS, _i32]),
    "cpb_ppo_spec_layout": (_i32, [_PS, _P, _P, _P, _P]),
    "cpb_ppo_spec_workspace_bytes": (_i64, [_PS, _i32, _i32]),
    "cpb_ppo_spec_forward": (_i32, [_PS, _P, _P, _i32, _P, _P, _P, _P, _i64, _P]),
    "cpb_ppo_spec_loss_grad": (_i32, [_PS, _P, _P, _P, _P, _P, _P, _P, _i32, _P, _P, _P, _i64, _P]),
    "cpb_ppo_spec_train_step": (_i32, [_PS, _P, _P, _P, _P, _P, _P, _P, _P, _P, _P, _P, _P, _i32, _P, _P, _i64, _P]),
    "cpb_ppo_spec_train_step_opts": (_i32, [_PS, _P, _P, _P, _P, _P, _P, _P, _P, _P, _P, _P, _P, _i32, _P, _PO, _P, _P,
                                            _P, _i64, _P]),
    "cpb_ppo_spec_learn": (_i32, [_PS, _P, _P, _P, _P, _P, _P, _P, _P, _P, _P, _P, _f64, _P, _i32, _f64, _f64,
                                  _i32, _i32, _P, _P, _P, _i64, _P]),
    "cpb_ppo_spec_learn_opts": (_i32, [_PS, _P, _P, _P, _P, _P, _P, _P, _P, _P, _P, _P, _f64, _P, _i32, _f64, _f64,
                                       _i32, _i32, _P, _P, _PO, _P, _P, _i64, _P]),
    "cpb_ppo_spec_learn_segments": (_i32, [_PS, _P, _P, _P, _P, _P, _P, _P, _P, _P, _P, _P, _P, _P, _P, _i32, _i32, _f64,
                                           _f64, _i32, _i32, _P, _P, _P, _i64, _P]),
    "cpb_ppo_spec_learn_segments_opts": (_i32, [_PS, _P, _P, _P, _P, _P, _P, _P, _P, _P, _P, _P, _P, _P, _P, _i32, _i32,
                                                _f64, _f64, _i32, _i32, _P, _P, _PO, _P, _P, _i64, _P]),
    "cpb_vae_spec_ppo_spec_encode_predict": (_i32, [_VS, _P, _P, _P, _i32, _PS, _P, _P, _P, _P, _P, _P, _P, _P, _i64, _P,
                                                    _i64, _P]),
    "cpb_mlpvae_ppo_spec_encode_predict": (_i32, [_MS, _P, _P, _P, _i32, _PS, _P, _P, _P, _P, _P, _P, _P, _P, _i64, _P,
                                                  _i64, _P]),
    "cpb_ppo_cat_num_tensors": (_i32, [_PK]),
    "cpb_ppo_cat_tensor_name": (C.c_char_p, [_PK, _i32]),
    "cpb_ppo_cat_layout": (_i32, [_PK, _P, _P, _P, _P]),
    "cpb_ppo_cat_workspace_bytes": (_i64, [_PK, _i32, _i32]),
    "cpb_ppo_cat_forward": (_i32, [_PK, _P, _P, _i32, _P, _P, _P, _P, _i64, _P]),
    "cpb_ppo_cat_loss_grad": (_i32, [_PK, _P, _P, _P, _P, _P, _P, _P, _i32, _P, _P, _P, _i64, _P]),
    "cpb_ppo_cat_train_step": (_i32, [_PK, _P, _P, _P, _P, _P, _P, _P, _P, _P, _P, _P, _P, _i32, _P, _P, _i64, _P]),
    "cpb_ppo_cat_train_step_opts": (_i32, [_PK, _P, _P, _P, _P, _P, _P, _P, _P, _P, _P, _P, _P, _i32, _P, _PO, _P, _P,
                                           _P, _i64, _P]),
    "cpb_ppo_cat_learn": (_i32, [_PK, _P, _P, _P, _P, _P, _P, _P, _P, _P, _P, _P, _f64, _P, _i32, _f64, _f64,
                                 _i32, _i32, _P, _P, _P, _i64, _P]),
    "cpb_ppo_cat_learn_opts": (_i32, [_PK, _P, _P, _P, _P, _P, _P, _P, _P, _P, _P, _P, _f64, _P, _i32, _f64, _f64,
                                      _i32, _i32, _P, _P, _PO, _P, _P, _i64, _P]),
    "cpb_ppo_cat_learn_segments": (_i32, [_PK, _P, _P, _P, _P, _P, _P, _P, _P, _P, _P, _P, _P, _P, _P, _i32, _i32, _f64,
                                          _f64, _i32, _i32, _P, _P, _P, _i64, _P]),
    "cpb_ppo_cat_learn_segments_opts": (_i32, [_PK, _P, _P, _P, _P, _P, _P, _P, _P, _P, _P, _P, _P, _P, _P, _i32, _i32,
                                               _f64, _f64, _i32, _i32, _P, _P, _PO, _P, _P, _i64, _P]),
    "cpb_vae_spec_ppo_cat_encode_predict": (_i32, [_VS, _P, _P, _P, _i32, _PK, _P, _P, _P, _P, _P, _P, _P, _P, _i64, _P,
                                                   _i64, _P]),
    "cpb_mlpvae_ppo_cat_encode_predict": (_i32, [_MS, _P, _P, _P, _i32, _PK, _P, _P, _P, _P, _P, _P, _P, _P, _i64, _P,
                                                 _i64, _P]),
    "cpb_running_norm_init": (_i32, [_RN, _P, _P]),
    "cpb_obs_normalize": (_i32, [_RN, _P, _P, _i32, _i32, _P, _P]),
    "cpb_reward_normalize": (_i32, [_RN, _P, _P, _P, _P, _P, _i32, _i32, _f64, _P, _P]),
    "cpb_vae_spec_ppo_spec_encode_predict_norm": (_i32, [_VS, _P, _P, _P, _i32, _PS, _P, _P, _P, _P, _P, _P, _P, _P, _i64,
                                                         _P, _i64, _P, _AN]),
    "cpb_mlpvae_ppo_spec_encode_predict_norm": (_i32, [_MS, _P, _P, _P, _i32, _PS, _P, _P, _P, _P, _P, _P, _P, _P, _i64,
                                                       _P, _i64, _P, _AN]),
    "cpb_vae_spec_ppo_cat_encode_predict_norm": (_i32, [_VS, _P, _P, _P, _i32, _PK, _P, _P, _P, _P, _P, _P, _P, _P, _i64,
                                                        _P, _i64, _P, _AN]),
    "cpb_mlpvae_ppo_cat_encode_predict_norm": (_i32, [_MS, _P, _P, _P, _i32, _PK, _P, _P, _P, _P, _P, _P, _P, _P, _i64,
                                                      _P, _i64, _P, _AN]),
    "cpb_set_math_mode": (_i32, [_i32]),
    "cpb_debug_vae_buffer_offsets": (_i32, [_i32, _i32, _i32, _i32, _P, _i32]),
    "cpb_debug_vae_spec_buffer_offsets": (_i32, [_VS, _i32, _P, _i32]),
    "cpb_debug_vae_backward_stop": (_i32, [C.c_char_p]),
    "cpb_debug_mlpvae_buffer_offsets": (_i32, [_MC, _i32, _P, _i32]),
    "cpb_debug_mlpvae_spec_buffer_offsets": (_i32, [_MS, _i32, _P, _i32]),
    "cpb_debug_tc_wgrad": (_i32, [_P, _P, _P, _i32, _i32, _i32, _i32, _P, _P]),
    "cpb_debug_tc_gemm": (_i32, [_P, _P, _P, _i32, _i32, _i32, _P, _P]),
    "cpb_get_math_mode": (_i32, []),
    "cpb_launch_count": (_i64, []),
    "cpb_reset_launch_count": (None, []),
    "cpb_profile_enable": (None, [_i32]),
    "cpb_profile_reset": (None, []),
    "cpb_profile_report": (_i64, [C.c_char_p, _i64]),
}

_lib: Optional[C.CDLL] = None


def load() -> C.CDLL:
    """Load the shared library (once).  Raises CpbError when it has not been built."""
    global _lib
    if _lib is not None:
        return _lib
    if not os.path.isfile(LIB_PATH):
        raise CpbError(
            "%s not found: the CUDA extension has not been built (run `python -c 'import __graft_entry__ as g; "
            "g.build()'` or carla_ppo_b200/csrc/build.sh).  There is no CPU fallback." % LIB_PATH)
    lib = C.CDLL(LIB_PATH)
    for name, (res, args) in PROTOTYPES.items():
        fn = getattr(lib, name)          # AttributeError if the symbol is missing
        fn.restype = res
        fn.argtypes = args
    _lib = lib
    return lib


def check(status: int, what: str = "") -> int:
    if status is not None and status < 0:
        msg = load().cpb_last_error().decode(errors="replace")
        raise CpbError("%s failed (status %d): %s" % (what or "libcarla_ppo_b200 call", status, msg))
    return status


def ptr(t) -> Optional[int]:
    """Device (or pinned-host) pointer of a torch tensor / numpy array, or None."""
    if t is None:
        return None
    if hasattr(t, "data_ptr"):
        return t.data_ptr()
    if hasattr(t, "ctypes"):
        return t.ctypes.data
    raise TypeError(type(t))


def current_stream_handle(device=None) -> int:
    """cudaStream_t of torch's current stream ON `device` (default: the current device).  The library launches on the
    CUDA device that is current at call time, so callers holding a device wrap the call in ``torch.cuda.device(dev)``
    and pass the same device here."""
    import torch
    return torch.cuda.current_stream(device).cuda_stream


def require_cuda():
    import torch
    if not torch.cuda.is_available():
        raise CpbError("no CUDA device: carla_ppo_b200 runs on H100 (sm_90a) only and has no CPU fallback")
    return torch
