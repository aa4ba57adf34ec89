"""carla_ppo_b200 -- H100-native (sm_90a) implementation of the neural hot path of bitsauce/Carla-ppo:
the ConvVAE training step and the PPO update that consumes its latents.

Layout (only what the path needs):
  csrc/            hand-written CUDA kernels + the C ABI (include/carla_ppo_b200.h) -> libcarla_ppo_b200.so
  _lib.py          ctypes binding (no fallback: raises when the library is missing)
  vae/models.py    drop-in for the reference's vae/models.py   (ConvVAE, loss selectors)
  ppo.py           drop-in for the reference's ppo.py          (PPO)
  utils.py         drop-in for utils.compute_gae
  vae_common.py    drop-in for vae_common.py                   (load_vae, create_encode_state_fn)
  tf_bundle.py     TF-V2 checkpoint reader so the reference's shipped checkpoints load
"""
__version__ = "0.1.0"
