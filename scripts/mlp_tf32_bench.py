"""Math mode 1 (fp32 SIMT for the MlpVAE) against math mode 2 (its five frame-wide products as one TF32 pass) on the
MlpVAE train step (by default encoder 512/256, decoder 256/512, z = 64, rgb target), in one process.

    python scripts/mlp_tf32_bench.py [--encoder_sizes 512 256] [--decoder_sizes 256 512] [--rounds 5] [--train-steps 300]
                                     [--out DIR] [--dump DIR [--dump-only]]

1. Step time.  Both modes are warmed at both batch sizes, then blocks of train steps (glorot init, seeded uniform
   frames, device-resident inputs) alternate between the modes at batch 4096 and 512 for --rounds rounds, the order of
   the two modes swapped every round; each block is timed with CUDA events.  Reported per mode: median ms/step and
   spread (max - min over the rounds).
2. Profile.  The per-group device time (cpb_profile_*) of each mode at both batch sizes, and for the five frame-wide
   groups the achieved TFLOP/s computed from the layer shapes (2 x multiply-adds / group time).  The labels name the
   first encoder layer "enc" and the output layer "dec2" at every depth.
3. Training (skipped with --train-steps 0).  --train-steps Adam steps from the same glorot init on the 128 committed frames (batch 32, BCE, seeded
   minibatches and noise) in each mode; both loss curves are printed.  Evidence that training behaves alike, not a gate.
--dump DIR writes DIR/mlp_mode1_loss_grad.npz: the losses and the flat gradient of one mode-1 loss_grad (glorot seed 0,
seeded batch of 64, the default sizes): running it against two builds shows whether mode 1 changed.  --package-root loads the package
(and its library) from another tree, e.g. a checkout of the other build.
The card (name, power limit, max SM clock) is read with a read-only nvidia-smi query.  Writes DIR/mlp_tf32_bench.json.
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
MODES = {"3xtf32": 1, "tf32": 2}
ENC, DEC, Z, IN, OUT = (512, 256), (256, 512), 64, 38400, 38400


def group_macs(enc, dec):
    """Multiply-adds per frame of the five frame-wide products (profile labels of the MlpVAE loss_grad): the first
    encoder layer and the output layer."""
    return {"mlp.enc.fwd": IN * enc[0], "mlp.enc.wgrad": IN * enc[0], "mlp.dec2.fwd": dec[-1] * OUT,
            "mlp.dec2.dgrad": dec[-1] * OUT, "mlp.dec2.wgrad": dec[-1] * OUT}


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True)
    return q.stdout.strip()


def make_vae(loss="mse", seed=0, enc=ENC, dec=DEC):
    from carla_ppo_b200.vae.models import MlpVAE
    vae = MlpVAE((80, 160, 3), z_dim=Z, encoder_sizes=enc, decoder_sizes=dec, beta=1.0, learning_rate=1e-4, loss_fn=loss,
                 model_dir=tempfile.mkdtemp(), seed=seed)
    vae.init_session(init_logging=False)          # glorot-uniform init
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


def dump(lib, out_dir):
    import torch
    set_mode(lib, 1)
    vae = make_vae()
    g = torch.Generator(device="cuda"); g.manual_seed(4321)
    x = torch.rand(64, 80, 160, 3, generator=g, device="cuda")
    eps = torch.randn(64, Z, generator=g, device="cuda")
    vae.loss_grad_device(x, x, eps)
    torch.cuda.synchronize()
    os.makedirs(out_dir, exist_ok=True)
    path = os.path.join(out_dir, "mlp_mode1_loss_grad.npz")
    np.savez(path, losses=vae._losses.cpu().numpy(), grads=vae.grads.cpu().numpy())
    print("wrote", path)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--steps-4096", type=int, default=5, help="train steps per timed block at batch 4096")
    ap.add_argument("--steps-512", type=int, default=20, help="train steps per timed block at batch 512")
    ap.add_argument("--train-steps", type=int, default=300)
    ap.add_argument("--out", default=None)
    ap.add_argument("--dump", default=None, help="write one mode-1 loss_grad's losses and gradient to this directory")
    ap.add_argument("--dump-only", action="store_true")
    ap.add_argument("--package-root", default=ROOT, help="tree to import carla_ppo_b200 from")
    ap.add_argument("--encoder_sizes", type=int, nargs="+", default=list(ENC))
    ap.add_argument("--decoder_sizes", type=int, nargs="+", default=list(DEC))
    args = ap.parse_args()
    enc, dec = tuple(args.encoder_sizes), tuple(args.decoder_sizes)
    sys.path.insert(0, ROOT)
    sys.path.insert(0, os.path.abspath(args.package_root))
    import torch
    from carla_ppo_b200 import _lib
    if not torch.cuda.is_available():
        raise SystemExit("mlp_tf32_bench.py measures on a CUDA device; none is present")
    lib = _lib.load()
    if args.dump:
        dump(lib, args.dump)
        if args.dump_only:
            return
    result = {"card": card(), "rounds": args.rounds, "model": {"encoder": enc, "decoder": dec, "z": Z}}

    # ---- 1. step time
    vae = make_vae(enc=enc, dec=dec)
    g = torch.Generator(device="cuda"); g.manual_seed(1234)
    x = torch.rand(4096, 80, 160, 3, generator=g, device="cuda")
    eps = torch.randn(4096, Z, generator=g, device="cuda")
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
        med["speedup"] = round(med["3xtf32"]["median"] / med["tf32"]["median"], 3)

    # ---- 2. per-group profile and achieved rates of the five frame-wide products
    result["profile_ms_per_step"], result["tflops"] = {}, {}
    for b, (xb, eb, _) in batches.items():
        for name, mode in MODES.items():
            set_mode(lib, mode)
            prof = profile(lib, vae, xb, eb)
            result["profile_ms_per_step"]["B%d_%s" % (b, name)] = prof
            result["tflops"]["B%d_%s" % (b, name)] = {
                k: round(2.0 * macs * b / (prof[k] * 1e-3) / 1e12, 1) for k, macs in group_macs(enc, dec).items() if prof.get(k)}
    del vae, x, eps, batches
    torch.cuda.empty_cache()

    # ---- 3. training curves on the committed frames
    if args.train_steps == 0:
        finish(result, args.out)
        return
    frames = torch.as_tensor(np.load(os.path.join(ROOT, "tests", "golden", "frames_u8.npz"))["rgb"], device="cuda")
    curves = {}
    for name, mode in MODES.items():
        set_mode(lib, mode)
        v = make_vae(loss="bce", enc=enc, dec=dec)
        rs = np.random.RandomState(0)
        out = []
        for _ in range(args.train_steps):
            idx = torch.as_tensor(rs.choice(frames.shape[0], 32, replace=False), device="cuda")
            xb = frames[idx]
            e = torch.as_tensor(rs.randn(32, Z).astype(np.float32), device="cuda")
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
    finish(result, args.out)


def finish(result, out):
    result["card_after"] = card()
    print(json.dumps({k: v for k, v in result.items() if k != "training"}, indent=1))
    if out:
        os.makedirs(out, exist_ok=True)
        with open(os.path.join(out, "mlp_tf32_bench.json"), "w") as f:
            json.dump(result, f, indent=1)


if __name__ == "__main__":
    main()
