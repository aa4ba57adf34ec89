"""PPO.learn and FusedActor.encode_predict at several policy / value architectures (README "PPO network size").

PPO.learn at BASELINE configs[2] (T = 2048, 4 epochs x 8 minibatches of 256; the reference agent's checkpoint-705 weights
at the default architecture, seeded glorot weights elsewhere, the same seeded rollout), one PPO object per architecture
and learn path, calls alternated across the architectures so that drift on the host or the card hits every row alike;
median and min-max of the per-call times.  The default architecture runs twice: through the legacy cpb_ppo_config entry
points and through the cpb_ppo_spec twins.  The persistent kernel (CPB_PPO_PERSISTENT=1) is read once per process, so
each learn path runs in its own process.  FusedActor.encode_predict at 64 environments, default vs (256, 256).

    python scripts/ppo_arch_bench.py [--calls 20] [--out DIR]
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

ARCHS = {"default (legacy)": ((500, 300), (500, 300)), "default (spec)": ((500, 300), (500, 300)),
         "64x2 / 64x2": ((64, 64), (64, 64)), "256x2 / 256x2": ((256, 256), (256, 256)),
         "256x3 / 256x3": ((256, 256, 256), (256, 256, 256))}


def _legacy(m):
    """Route m's calls through the cpb_ppo_config entry points (the spec twins' legacy callers)."""
    real = m._call
    m._call = lambda name, *args: real(name.replace("cpb_ppo_spec_", "cpb_ppo_"), *((C.byref(m._c),) + args[1:]))


def learn_times(calls):
    import torch
    from helpers import Box
    from carla_ppo_b200.ppo import PPO
    from bench import ppo_config3_inputs, shipped_agent
    from ppo_restatement import init_params
    pol, old, am, av, pw = shipped_agent()
    s, a, r, v, d, perms = ppo_config3_inputs()
    models = {}
    for name, (ps, vs) in ARCHS.items():
        m = PPO((67,), Box(np.array([-1.0, 0.0]), np.array([1.0, 1.0])), learning_rate=1e-4, value_scale=1.0,
                entropy_scale=0.01, model_dir=tempfile.mkdtemp(), seed=0, policy_hidden_sizes=ps, value_hidden_sizes=vs)
        m.init_session(init_logging=False)
        if ps == (500, 300) and vs == (500, 300):
            m.set_weights(pol, old, am, av, pw)
        else:
            w = init_params(67, (np.array([-1.0, 0.0]), np.array([1.0, 1.0])), ps, vs, seed=1)
            m.set_weights(w, w)
        if "legacy" in name:
            _legacy(m)
        models[name] = m
    dev = {k: torch.from_numpy(np.ascontiguousarray(x)).cuda() for k, x in
           dict(s=s, a=a, r=r.astype(np.float64), v=v.astype(np.float64), d=d.astype(np.float64),
                p=perms.astype(np.int32)).items()}
    run = lambda m: m.learn(dev["s"], dev["a"], dev["v"], dev["r"], dev["d"], 0.3, num_epochs=4, batch_size=256,
                            perms=dev["p"])
    for m in models.values():       # warm-up
        run(m)
        run(m)
    torch.cuda.synchronize()
    times = {k: [] for k in models}
    for _ in range(calls):
        for name, m in models.items():
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            run(m)
            torch.cuda.synchronize()
            times[name].append((time.perf_counter() - t0) * 1e3)
    return times


def actor_times(calls):
    import torch
    import types
    from helpers import Box, committed_frames, shipped_vae_weights
    from harness import make_conv_vae
    from carla_ppo_b200.actor import FusedActor
    from carla_ppo_b200.ppo import PPO
    from pathlib import Path
    rgb, _ = committed_frames()
    vae = make_conv_vae(Path(tempfile.mkdtemp()), shipped_vae_weights()[0], loss="bce", tag="vae", training=False)
    envs = []
    for i in range(64):
        veh = types.SimpleNamespace(control=types.SimpleNamespace(steer=0.0, throttle=0.1), get_speed=lambda: 1.0)
        envs.append(types.SimpleNamespace(observation=rgb[i % len(rgb)], vehicle=veh))
    actors = {}
    for name, arch in (("default", ((500, 300), (500, 300))), ("256x2 / 256x2", ((256, 256), (256, 256)))):
        m = PPO((67,), Box(np.array([-1.0, 0.0]), np.array([1.0, 1.0])), model_dir=tempfile.mkdtemp(), seed=0,
                policy_hidden_sizes=arch[0], value_hidden_sizes=arch[1])
        m.init_session(init_logging=False)
        actors[name] = FusedActor(vae, m, ("steer", "throttle", "speed"))
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
        with open(os.path.join(args.out, "ppo_arch_bench.json"), "w") as f:
            f.write(text)


if __name__ == "__main__":
    main()
