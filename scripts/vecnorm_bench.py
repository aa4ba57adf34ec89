"""The cost of running normalisation (README "PPO observation and reward normalisation").

FusedActor.encode_predict at 1, 16, 64 and 256 environments (ConvVAE 80x160, z 64, default PPO, sampled actions) with
normalisation off, observations only, and observations + rewards; cpb_obs_normalize alone at B = 64 and 2048 with
D = 67, and at B = 64 with D = 1030.  The variants of one size are alternated call by call in one process, so that drift
on the host or the card hits them alike; median and min-max of the per-call times (host clock around calls that end in
a device synchronise for the actor, CUDA events for the kernel).  The card's name, power limit and max SM clock are
printed first.

    python scripts/vecnorm_bench.py [--calls 30] [--out DIR]
"""
import argparse
import ctypes as C
import json
import os
import subprocess
import sys
import tempfile
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [ROOT, os.path.join(ROOT, "tests")]

VARIANTS = {"off": {}, "obs": dict(normalize_observations=True),
            "obs+rewards": dict(normalize_observations=True, normalize_rewards=True)}


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True)
    return q.stdout.strip()


def summary(ts):
    ts = np.asarray(ts) * 1e3
    return {"median_ms": float(np.median(ts)), "min_ms": float(ts.min()), "max_ms": float(ts.max()), "calls": len(ts)}


def actor_times(calls):
    from carla_ppo_b200.actor import FusedActor
    from carla_ppo_b200.ppo import PPO
    from carla_ppo_b200.replay_env import Box
    from carla_ppo_b200.vae.models import ConvVAE
    from ppo_checks import fake_envs
    vae = ConvVAE((80, 160, 3), z_dim=64, loss_fn="bce", model_dir=tempfile.mkdtemp(), seed=0, training=False)
    vae.init_session(init_logging=False)
    actors = {}
    for name, kw in VARIANTS.items():
        m = PPO((67,), Box([-1.0, 0.0], [1.0, 1.0]), model_dir=tempfile.mkdtemp(), seed=0, **kw)
        m.init_session(init_logging=False)
        actors[name] = FusedActor(vae, m)
    out = {}
    for n in (1, 16, 64, 256):
        envs = fake_envs(n)
        r, d, ids = np.linspace(-1, 1, n), np.zeros(n, bool), np.arange(n)
        call = {"off": lambda: actors["off"].encode_predict(envs),
                "obs": lambda: actors["obs"].encode_predict(envs),
                "obs+rewards": lambda: actors["obs+rewards"].encode_predict(envs, r, d, ids)}
        ts = {k: [] for k in call}
        for k in call:                      # warm-up: buffers, workspaces, modules
            for _ in range(3):
                call[k]()
        for _ in range(calls):
            for k, f in call.items():
                t0 = time.perf_counter()
                f()                         # ends in a stream synchronise
                ts[k].append(time.perf_counter() - t0)
        out["encode_predict n=%d" % n] = {k: summary(v) for k, v in ts.items()}
    return out


def kernel_times(calls):
    import torch
    from carla_ppo_b200 import _lib
    lib = _lib.load()
    out = {}
    for B, D in ((64, 67), (2048, 67), (64, 1030)):
        cfg = _lib.RunningNorm(D, 10.0, 1e-8)
        stats = torch.empty(2 * D + 1, dtype=torch.float64, device="cuda")
        _lib.check(lib.cpb_running_norm_init(C.byref(cfg), stats.data_ptr(), None))
        x = torch.randn(B, D, device="cuda")
        y = torch.empty_like(x)
        stream = torch.cuda.current_stream().cuda_stream
        run = lambda: _lib.check(lib.cpb_obs_normalize(C.byref(cfg), stats.data_ptr(), x.data_ptr(), B, 1, y.data_ptr(),
                                                       stream))
        for _ in range(10):
            run()
        ts = []
        for _ in range(calls):
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            for _ in range(100):
                run()
            e1.record()
            e1.synchronize()
            ts.append(e0.elapsed_time(e1) / 100 / 1e3)
        out["cpb_obs_normalize B=%d D=%d (per call, 100 back to back)" % (B, D)] = summary(ts)
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--calls", type=int, default=30)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    import torch
    assert torch.cuda.is_available(), "vecnorm_bench needs a GPU"
    res = {"card": card()}
    print("card (name, power limit, max SM clock):", res["card"], flush=True)
    res.update(actor_times(args.calls))
    res.update(kernel_times(args.calls))
    for k, v in res.items():
        print(k, json.dumps(v))
    if args.out:
        os.makedirs(args.out, exist_ok=True)
        with open(os.path.join(args.out, "vecnorm_bench.json"), "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
