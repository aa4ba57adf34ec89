"""Cost of the latent padding: the ConvVAE train step at batch 4096 for z_dim 32, 64, 100 and 128, in one process.

    python scripts/zdim_bench.py [--rounds 5] [--steps 10] [--out DIR]

The library runs a latent of z columns at z_pad = 64 * ceil(z / 64) columns, so z = 32 should cost what z = 64 costs
and z = 100 what z = 128 costs: only the heads, dense1, sampling / KL and the boundary copies see z, under 1 % of the
forward work.  For math modes 1 (3xTF32) and 2 (one TF32 pass): every z is warmed, then blocks of --steps train steps
(glorot init, seeded uniform frames, device-resident inputs as in bench.py) alternate over the z values for --rounds
rounds, the order reversed every round; each block is timed with CUDA events.  Reported per mode and z: median ms/step
and spread (max - min over the rounds), and the per-group profile (cpb_profile_*) of the z-dependent groups (heads.*,
dense1.*) plus the step's total.  The card (name, power limit, max SM clock) is read with a read-only nvidia-smi query.
Writes DIR/zdim_bench.json.
"""
import argparse
import ctypes as C
import json
import os
import statistics
import subprocess
import sys
import tempfile

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

MODES = {"3xtf32": 1, "tf32": 2}
ZS = (32, 64, 100, 128)
B = 4096


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True)
    return q.stdout.strip()


def timed_block(vae, x, eps, steps):
    import torch
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    torch.cuda.synchronize()
    e0.record()
    for _ in range(steps):
        vae.train_step_device(x, x, eps)
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / steps


def profile(lib, vae, x, eps, steps=5):
    import torch
    lib.cpb_profile_reset(); lib.cpb_profile_enable(1)
    for _ in range(steps):
        vae.train_step_device(x, x, eps)
    torch.cuda.synchronize()
    lib.cpb_profile_enable(0)
    buf = C.create_string_buffer(1 << 16)
    n = lib.cpb_profile_report(buf, len(buf))
    lib.cpb_profile_reset()
    groups = {}
    for line in buf.raw[:n].decode().splitlines():
        label, _, ms = line.split()
        groups[label] = float(ms) / steps
    out = {k: round(v, 4) for k, v in sorted(groups.items()) if k.startswith(("heads.", "dense1."))}
    out["z_groups_total"] = round(sum(out.values()), 4)
    out["all_groups_total"] = round(sum(groups.values()), 4)
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--steps", type=int, default=10, help="train steps per timed block")
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    import torch
    from carla_ppo_b200 import _lib
    from carla_ppo_b200.vae.models import ConvVAE
    if not torch.cuda.is_available():
        raise SystemExit("zdim_bench.py measures on a CUDA device; none is present")
    lib = _lib.load()
    result = {"card": card(), "batch": B, "rounds": args.rounds, "steps_per_block": args.steps}
    g = torch.Generator(device="cuda"); g.manual_seed(1234)
    x = torch.rand(B, 80, 160, 3, generator=g, device="cuda")
    vaes, eps = {}, {}
    for z in ZS:
        vaes[z] = ConvVAE((80, 160, 3), z_dim=z, beta=1.0, learning_rate=1e-4, loss_fn="mse", model_dir=tempfile.mkdtemp(),
                          seed=0)
        vaes[z].init_session(init_logging=False)
        eps[z] = torch.randn(B, z, generator=g, device="cuda")
    for name, mode in MODES.items():
        _lib.check(lib.cpb_set_math_mode(mode), "cpb_set_math_mode")
        times = {z: [] for z in ZS}
        for z in ZS:
            for _ in range(3):
                vaes[z].train_step_device(x, x, eps[z])
        torch.cuda.synchronize()
        for r in range(args.rounds):
            order = ZS if r % 2 == 0 else tuple(reversed(ZS))
            for z in order:
                times[z].append(timed_block(vaes[z], x, eps[z], args.steps))
            print("%s round %d: " % (name, r) + "  ".join("z=%d %.2f ms" % (z, times[z][-1]) for z in ZS), flush=True)
        result[name] = {str(z): {"median_ms": round(statistics.median(v), 3), "spread_ms": round(max(v) - min(v), 3),
                                 "all_ms": [round(t, 3) for t in v], "profile_ms_per_step": profile(lib, vaes[z], x, eps[z])}
                        for z, v in times.items()}
    _lib.check(lib.cpb_set_math_mode(1), "cpb_set_math_mode")
    result["card_after"] = card()
    print(json.dumps(result, indent=1))
    if args.out:
        os.makedirs(args.out, exist_ok=True)
        with open(os.path.join(args.out, "zdim_bench.json"), "w") as f:
            json.dump(result, f, indent=1)


if __name__ == "__main__":
    main()
