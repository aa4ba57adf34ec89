"""Throughput of train.train with N replay environments in lockstep, and the cost of one PPO update over segments.

On the committed frames (tests/golden/frames_u8.npz), the shipped checkpoint-232 rgb ConvVAE and the checkpoint-705 agent,
TensorBoard logging off:
  * environment steps/s of train.train for N in {1, 4, 16, 64} at the reference's defaults (horizon 128, 3 epochs,
    minibatch 32, fused encode + predict); training steps over the wall time of the training rounds, the evaluation
    episode excluded; one untimed warm-up run per N first;
  * PPO.learn over 16 segments x 128 rows against one 2048-row call, both 4 epochs x 256 (BASELINE configs[2]),
    alternated, host clock around each call after a device synchronise.
The card's name, power limit and max SM clock are read in the same run.

    python scripts/vec_rollout_bench.py [--envs 1 4 16 64] [--rounds 2] [--learn_reps 20]
"""
import argparse
import json
import os
import subprocess
import sys
import tempfile
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))


def card():
    import torch
    out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                         capture_output=True, text=True).stdout.strip().splitlines()
    return dict(torch_name=torch.cuda.get_device_name(), nvidia_smi=out[torch.cuda.current_device()] if out else "not available")


def write_agent_checkpoint(model_dir):
    """The checkpoint-705 agent (policy, policy_old, Adam slots, beta powers) where train.train restores it from."""
    from helpers import shipped_ppo
    pol, z = shipped_ppo("policy")
    old, _ = shipped_ppo("policy_old")
    blob = {"policy/" + k: v for k, v in pol.items()}
    blob.update({"policy_old/" + k: v for k, v in old.items()})
    blob.update({"policy/%s/Adam" % k: z["adam_m/" + k] for k in pol})
    blob.update({"policy/%s/Adam_1" % k: z["adam_v/" + k] for k in pol})
    blob["beta1_power"], blob["beta2_power"] = z["beta1_power"], z["beta2_power"]
    ck = os.path.join(model_dir, "checkpoints")
    os.makedirs(ck, exist_ok=True)
    np.savez(os.path.join(ck, "model.ckpt-705.npz"), **blob)
    with open(os.path.join(ck, "checkpoint"), "w") as f:
        f.write('model_checkpoint_path: "model.ckpt-705"\nall_model_checkpoint_paths: "model.ckpt-705"\n')


def train_rate(n, rounds, workdir, vae, frames):
    from carla_ppo_b200 import train as train_mod
    from carla_ppo_b200.replay_env import ReplayEnv

    class CountingEnv(ReplayEnv):
        training_steps = 0

        def step(self, action):
            if self.is_training:
                CountingEnv.training_steps += 1
            return super().step(action)

    eval_time = [0.0]
    run_eval = train_mod.run_eval

    def timed_eval(*a, **kw):
        t0 = time.perf_counter()
        try:
            return run_eval(*a, **kw)
        finally:
            eval_time[0] += time.perf_counter() - t0

    train_mod.run_eval = timed_eval
    try:
        out = None
        for tag, num_rounds in (("warmup", 1), ("timed", rounds)):
            name = "n%d_%s" % (n, tag)
            write_agent_checkpoint(os.path.join(workdir, name))
            envs = [CountingEnv(frames, episode_length=256, seed=0) for _ in range(n)]
            params = dict(learning_rate=1e-4, lr_decay=1.0, discount_factor=0.99, gae_lambda=0.95, ppo_epsilon=0.2,
                          initial_std=1.0, value_scale=1.0, entropy_scale=0.01, horizon=128, num_epochs=3,
                          num_episodes=num_rounds, batch_size=32, vae_model="unused", vae_model_type=None, vae_z_dim=None,
                          synchronous=True, fps=30, action_smoothing=0.0, model_name=name,
                          reward_fn="reward_speed_centering_angle_multiply", seed=0, eval_interval=10 ** 9,
                          record_eval=False, logging=False, num_envs=n)
            CountingEnv.training_steps, eval_time[0] = 0, 0.0
            import torch
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            model = train_mod.train(params, restart=False, env=envs, vae=vae, models_root=workdir, interactive=False)
            torch.cuda.synchronize()
            wall = time.perf_counter() - t0 - eval_time[0]
            out = dict(num_envs=n, rounds=num_rounds, env_steps=CountingEnv.training_steps, seconds=wall,
                       env_steps_per_s=CountingEnv.training_steps / wall, updates_minibatches=model.get_train_step_idx())
        return out
    finally:
        train_mod.run_eval = run_eval


def learn_times(reps, workdir):
    import torch
    from helpers import Box, shipped_ppo
    from carla_ppo_b200.ppo import PPO
    pol, z = shipped_ppo("policy")
    old, _ = shipped_ppo("policy_old")
    m = PPO((67,), Box([-1.0, 0.0], [1.0, 1.0]), model_dir=os.path.join(workdir, "learn"), seed=0)
    m.init_session(init_logging=False)
    m.set_weights(pol, old, {k: z["adam_m/" + k] for k in pol}, {k: z["adam_v/" + k] for k in pol},
                  (float(z["beta1_power"]), float(z["beta2_power"])))
    T, E, B = 2048, 4, 256
    rs = np.random.RandomState(0)
    s = rs.randn(T, 67).astype(np.float32)
    a = np.clip(rs.randn(T, 2), [-1.0, 0.0], [1.0, 1.0]).astype(np.float32)
    r, v = rs.rand(T), rs.randn(T).astype(np.float32)
    d = np.zeros(T, bool)
    d[127::256] = True
    perms = np.stack([np.random.RandomState(0).permutation(T) for _ in range(E)])
    boot = rs.randn(16).astype(np.float32)
    calls = {"one_2048": lambda: m.learn(s, a, v, r, d, float(boot[-1]), num_epochs=E, batch_size=B, perms=perms),
             "segments_16x128": lambda: m.learn(s, a, v, r, d, boot, num_epochs=E, batch_size=B, perms=perms,
                                                segment_lengths=[128] * 16)}
    for f in calls.values():
        for _ in range(3):
            f()
    times = {k: [] for k in calls}
    for _ in range(reps):
        for k, f in calls.items():
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            f()
            torch.cuda.synchronize()
            times[k].append((time.perf_counter() - t0) * 1e3)
    m._pending_metrics = []
    return {k: dict(median_ms=float(np.median(x)), min_ms=float(np.min(x)), max_ms=float(np.max(x)), reps=reps)
            for k, x in times.items()}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--envs", type=int, nargs="+", default=[1, 4, 16, 64])
    ap.add_argument("--rounds", type=int, default=2)
    ap.add_argument("--learn_reps", type=int, default=20)
    args = ap.parse_args()
    from carla_ppo_b200 import _lib
    _lib.require_cuda()
    from helpers import committed_frames, shipped_vae_weights
    from carla_ppo_b200.vae.models import ConvVAE
    print(json.dumps(dict(card=card())), flush=True)
    with tempfile.TemporaryDirectory() as workdir:
        vae = ConvVAE(source_shape=(80, 160, 3), z_dim=64, model_dir=os.path.join(workdir, "vae"), training=False, seed=0)
        vae.init_session(init_logging=False)
        vae.set_weights(shipped_vae_weights()[0])
        frames = committed_frames()[0]
        for n in args.envs:
            print(json.dumps(dict(train=train_rate(n, args.rounds, workdir, vae, frames))), flush=True)
        print(json.dumps(dict(learn=learn_times(args.learn_reps, workdir))), flush=True)
    print(json.dumps(dict(card=card())), flush=True)


if __name__ == "__main__":
    main()
