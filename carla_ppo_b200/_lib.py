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


_P = C.c_void_p
_i32, _i64, _f32, _f64 = C.c_int32, C.c_int64, C.c_float, C.c_double
_VC = C.POINTER(VaeConfig)
_VS = C.POINTER(VaeSpec)
_MC = C.POINTER(MlpVaeConfig)
_MS = C.POINTER(MlpVaeSpec)
_PC = C.POINTER(PpoConfig)

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
