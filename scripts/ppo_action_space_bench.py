"""PPO.learn and FusedActor.encode_predict with a Gaussian and with categorical policy heads (README "PPO action spaces").

PPO.learn at BASELINE configs[2]'s shapes (T = 2048, 4 epochs x 8 minibatches of 256, state 67, default trunks 500, 300;
seeded weights, the same seeded rollout with Box actions for the Gaussian head and index actions for the categorical
ones): the Gaussian head over 2 actions, categorical (7, 3) and categorical (64,), one PPO object per head, calls
alternated across the heads so that drift on the host or the card hits every row alike; median and min-max of the
per-call times.  The persistent kernel (CPB_PPO_PERSISTENT=1) is read once per process, so each learn path runs in its
own process.  FusedActor.encode_predict at 64 environments for the same three heads (sampled actions).

    python scripts/ppo_action_space_bench.py [--calls 20] [--out DIR]
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
sys.path[:0] = [ROOT, os.path.join(ROOT, "tests")]

HEADS = {"gaussian, 2 actions": None, "categorical (7, 3)": (7, 3), "categorical (64,)": (64,)}


def _space(cats):
    from carla_ppo_b200.replay_env import Box, MultiDiscrete
    return Box([-1.0, 0.0], [1.0, 1.0]) if cats is None else MultiDiscrete(cats)


def _ppo(cats):
    from carla_ppo_b200.ppo import PPO
    m = PPO((67,), _space(cats), learning_rate=1e-4, value_scale=1.0, entropy_scale=0.01, model_dir=tempfile.mkdtemp(),
            seed=0)
    m.init_session(init_logging=False)
    return m


def learn_times(calls):
    import torch
    T = 2048
    rs = np.random.RandomState(0)
    s = rs.randn(T, 67).astype(np.float32)
    r, v = rs.rand(T), rs.randn(T)
    d = np.zeros(T)
    d[T // 2] = 1.0
    perms = np.stack([rs.permutation(T) for _ in range(4)]).astype(np.int32)
    to_dev = lambda x: torch.from_numpy(np.ascontiguousarray(x)).cuda()
    models, acts = {}, {}
    for name, cats in HEADS.items():
        models[name] = _ppo(cats)
        if cats is None:
            a = np.clip(rs.randn(T, 2), [-1.0, 0.0], [1.0, 1.0]).astype(np.float32)
        else:
            a = np.stack([rs.randint(c, size=T) for c in cats], axis=1).astype(np.float32)
        acts[name] = to_dev(a)
    dev = {k: to_dev(x) for k, x in dict(s=s, r=r, v=v, d=d, p=perms).items()}
    run = lambda name: models[name].learn(dev["s"], acts[name], dev["v"], dev["r"], dev["d"], 0.3, num_epochs=4,
                                          batch_size=256, perms=dev["p"])
    for name in models:           # warm-up
        run(name)
        run(name)
    torch.cuda.synchronize()
    times = {k: [] for k in models}
    for _ in range(calls):
        for name in models:
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            run(name)
            torch.cuda.synchronize()
            times[name].append((time.perf_counter() - t0) * 1e3)
    return times


def actor_times(calls):
    import torch
    import types
    from pathlib import Path
    from helpers import committed_frames, shipped_vae_weights
    from harness import make_conv_vae
    from carla_ppo_b200.actor import FusedActor
    rgb, _ = committed_frames()
    vae = make_conv_vae(Path(tempfile.mkdtemp()), shipped_vae_weights()[0], loss="bce", tag="vae", training=False)
    envs = []
    for i in range(64):
        veh = types.SimpleNamespace(control=types.SimpleNamespace(steer=0.0, throttle=0.1), get_speed=lambda: 1.0)
        envs.append(types.SimpleNamespace(observation=rgb[i % len(rgb)], vehicle=veh))
    actors = {name: FusedActor(vae, _ppo(cats), ("steer", "throttle", "speed")) for name, cats in HEADS.items()}
    for a in actors.values():
        a.encode_predict(envs)
    times = {k: [] for k in actors}
    for _ in range(calls):
        for name, a in actors.items():
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            a.encode_predict(envs)          # ends in a device synchronise (results copied to the host)
            times[name].append((time.perf_counter() - t0) * 1e3)
    return times


def summary(times):
    return {k: {"median_ms": float(np.median(t)), "min_ms": float(np.min(t)), "max_ms": float(np.max(t)), "n": len(t)}
            for k, t in times.items()}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--calls", type=int, default=20)
    ap.add_argument("--out", default=None)
    ap.add_argument("--child", choices=["learn", "actor"], default=None)
    args = ap.parse_args()
    if args.child:
        t = learn_times(args.calls) if args.child == "learn" else actor_times(args.calls)
        print(json.dumps(summary(t)))
        return
    out = {}
    try:
        out["gpu"] = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                                    capture_output=True, text=True).stdout.strip()
    except OSError:
        out["gpu"] = "unknown"
    for label, child, flag in (("learn, launch per kernel", "learn", "0"), ("learn, persistent kernel", "learn", "1"),
                               ("FusedActor.encode_predict, 64 envs", "actor", "0")):
        res = subprocess.run([sys.executable, __file__, "--child", child, "--calls", str(args.calls)],
                             env=dict(os.environ, CPB_PPO_PERSISTENT=flag), capture_output=True, text=True, check=True)
        out[label] = json.loads(res.stdout.strip().splitlines()[-1])
    text = json.dumps(out, indent=1)
    print(text)
    if args.out:
        os.makedirs(args.out, exist_ok=True)
        with open(os.path.join(args.out, "ppo_action_space_bench.json"), "w") as f:
            f.write(text)


if __name__ == "__main__":
    main()
