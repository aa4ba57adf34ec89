"""Math mode 1 (3xTF32, the default) against math mode 2 (one TF32 pass) on the ConvVAE train step, in one process.

    python scripts/tf32_bench.py [--rounds 5] [--train-steps 300] [--out DIR]

1. Step time.  Both modes are warmed at both batch sizes, then blocks of train steps (glorot init, seeded uniform
   frames, device-resident inputs as in bench.py) alternate between the modes at batch 4096 and 512 for --rounds
   rounds, the order of the two modes swapped every round; each block is timed with CUDA events.  Reported per mode:
   median ms/step and spread (max - min over the rounds), and the per-group profile (cpb_profile_*) at batch 4096.
2. Difference.  One loss_grad per mode from the same weights on the same seeded batch-4096 inputs: relative
   difference of the two losses and of the flat gradient.
3. Training.  --train-steps Adam steps from the same glorot init on the 128 committed frames (batch 32, BCE, seeded
   minibatches and noise) in each mode; both loss curves are printed.  Evidence that training behaves alike, not a gate.
The card (name, power limit, max SM clock) is read with a read-only nvidia-smi query.  Writes DIR/tf32_bench.json.
"""
import argparse
import ctypes as C
import json
import os
import statistics
import subprocess
import sys
import tempfile

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

MODES = {"3xtf32": 1, "tf32": 2}


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True)
    return q.stdout.strip()


def make_vae(loss="mse", seed=0):
    from carla_ppo_b200.vae.models import ConvVAE
    vae = ConvVAE((80, 160, 3), z_dim=64, beta=1.0, learning_rate=1e-4, loss_fn=loss, model_dir=tempfile.mkdtemp(),
                  seed=seed)
    vae.init_session(init_logging=False)          # glorot-uniform init (seed 0), as bench.py
    return vae


def set_mode(lib, mode):
    from carla_ppo_b200 import _lib
    _lib.check(lib.cpb_set_math_mode(mode), "cpb_set_math_mode")


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
        groups[label] = round(float(ms) / steps, 4)
    return dict(sorted(groups.items(), key=lambda kv: -kv[1]))


def rel(a, b):
    a = np.asarray(a, np.float64).ravel(); b = np.asarray(b, np.float64).ravel()
    return float(np.linalg.norm(a - b) / np.linalg.norm(b))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--steps-4096", type=int, default=10, help="train steps per timed block at batch 4096")
    ap.add_argument("--steps-512", type=int, default=40, help="train steps per timed block at batch 512")
    ap.add_argument("--train-steps", type=int, default=300)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    import torch
    from carla_ppo_b200 import _lib
    if not torch.cuda.is_available():
        raise SystemExit("tf32_bench.py measures on a CUDA device; none is present")
    lib = _lib.load()
    result = {"card": card(), "rounds": args.rounds}

    # ---- 1. step time
    vae = make_vae()
    g = torch.Generator(device="cuda"); g.manual_seed(1234)
    x = torch.rand(4096, 80, 160, 3, generator=g, device="cuda")
    eps = torch.randn(4096, 64, generator=g, device="cuda")
    batches = {4096: (x, eps, args.steps_4096), 512: (x[:512], eps[:512], args.steps_512)}
    for mode in MODES.values():
        set_mode(lib, mode)
        for b, (xb, eb, _) in batches.items():
            for _ in range(3):
                vae.train_step_device(xb, xb, eb)
    torch.cuda.synchronize()
    times = {b: {m: [] for m in MODES} for b in batches}
    for r in range(args.rounds):
        order = list(MODES) if r % 2 == 0 else list(reversed(list(MODES)))
        for b, (xb, eb, steps) in batches.items():
            for name in order:
                set_mode(lib, MODES[name])
                times[b][name].append(timed_block(vae, xb, eb, steps))
        print("round %d: " % r + "  ".join("B=%d %s %.2f ms" % (b, m, times[b][m][-1]) for b in batches for m in MODES),
              flush=True)
    result["ms_per_step"] = {str(b): {m: {"median": round(statistics.median(v), 3), "spread": round(max(v) - min(v), 3),
                                          "all": [round(t, 3) for t in v]} for m, v in tm.items()} for b, tm in times.items()}
    for b in batches:
        med = result["ms_per_step"][str(b)]
        result["ms_per_step"][str(b)]["speedup"] = round(med["3xtf32"]["median"] / med["tf32"]["median"], 3)
    result["profile_ms_per_step_B4096"] = {}
    for name, mode in MODES.items():
        set_mode(lib, mode)
        result["profile_ms_per_step_B4096"][name] = profile(lib, vae, x, eps)

    # ---- 2. what mode 2 changes, same weights and inputs
    diff = {}
    vae2 = make_vae()
    for name, mode in MODES.items():
        set_mode(lib, mode)
        vae2.loss_grad_device(x, x, eps)
        torch.cuda.synchronize()
        diff[name] = (vae2._losses.cpu().numpy().astype(np.float64), vae2.grads.cpu().numpy())
    l1, g1 = diff["3xtf32"]; l2, g2 = diff["tf32"]
    result["tf32_vs_3xtf32_B4096"] = {"recon_rel": float(abs(l2[0] - l1[0]) / abs(l1[0])),
                                      "kl_rel": float(abs(l2[1] - l1[1]) / abs(l1[1])), "grad_rel_l2": rel(g2, g1)}
    del vae, vae2, x, eps, batches
    torch.cuda.empty_cache()

    # ---- 3. training curves on the committed frames
    frames = torch.as_tensor(np.load(os.path.join(ROOT, "tests", "golden", "frames_u8.npz"))["rgb"], device="cuda")
    curves = {}
    for name, mode in MODES.items():
        set_mode(lib, mode)
        v = make_vae(loss="bce")
        rs = np.random.RandomState(0)
        out = []
        for _ in range(args.train_steps):
            idx = torch.as_tensor(rs.choice(frames.shape[0], 32, replace=False), device="cuda")
            xb = frames[idx]
            e = torch.as_tensor(rs.randn(32, 64).astype(np.float32), device="cuda")
            out.append(v.train_step_device(xb, xb, e).clone())
        curves[name] = torch.stack(out).cpu().numpy().astype(np.float64)
    set_mode(lib, 1)
    every = max(1, args.train_steps // 12)
    print("training on the committed frames (batch 32, bce): step, recon + kl per mode")
    for s in list(range(0, args.train_steps, every)) + [args.train_steps - 1]:
        print("  %4d  " % s + "  ".join("%s %10.2f" % (m, curves[m][s].sum()) for m in MODES))
    tail = max(1, args.train_steps // 6)
    result["training"] = {m: {"recon_kl_every_%d" % every: [round(float(c[s].sum()), 3) for s in range(0, len(c), every)],
                              "mean_last_%d" % tail: round(float(c[-tail:].sum(axis=1).mean()), 3)} for m, c in curves.items()}
    result["card_after"] = card()
    print(json.dumps({k: v for k, v in result.items() if k != "training"}, indent=1))
    if args.out:
        os.makedirs(args.out, exist_ok=True)
        with open(os.path.join(args.out, "tf32_bench.json"), "w") as f:
            json.dump(result, f, indent=1)


if __name__ == "__main__":
    main()
