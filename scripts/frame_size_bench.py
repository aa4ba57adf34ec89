"""ConvVAE throughput by frame size: the train step at B = 2048 and encode at B = 4096, in math modes 1 (3xTF32) and 2
(one TF32 pass), at 64x128, 80x160, 128x256 and 160x320, all through the cpb_vae_spec_* entry points.

    python scripts/frame_size_bench.py --out DIR [--rounds 5] [--steps 10]

One process; every round visits every (geometry, mode) pair in turn, so drift of the shared machine hits all of them
alike.  Each measurement is `steps` calls after two warm-up calls, timed with CUDA events around the whole window; the
figure reported is the median over the rounds, with the spread (max - min).  Frames are float32 uniform [0, 1),
resident on the device; the rgb target is the source; loss mse, z_dim 64.  A separate profiled call per pair gives the
per-group breakdown (cpb_profile_*: CUDA events around each labelled kernel group).  The card's name, power limit and
max SM clock are read in the same run.  Writes DIR/frame_size.json and prints a table.

Algorithmic FLOP per frame (flop_per_frame): 2 x the multiply-accumulates of every layer, from the geometry.  A layer
with output [Ho, Wo, Co] and kernel [k, k, Ci] does Ho*Wo*Co * k*k*Ci MACs per pass; a transposed convolution is
counted on its small side (Hs*Ws*Cs * k*k*Cb).  The train step runs the forward pass, the data gradient of every layer
but conv1 and every weight gradient; encode runs conv1-4 and the mean head.  At 80x160 the train step is 776 494 080
FLOP/frame and encode 117 992 448 (SURVEY section 8(d))."""
import argparse
import json
import os
import statistics
import subprocess
import sys
import tempfile

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

GEOMETRIES = [(64, 128), (80, 160), (128, 256), (160, 320)]
MODES = [1, 2]
TRAIN_B, ENCODE_B, Z = 2048, 4096, 64


def layer_macs(h, w, z=Z, ct=3):
    """MACs per frame of each layer's forward pass at frame h x w."""
    s = [(h, w, 3)]
    for c in (32, 64, 128, 256):
        s.append(((s[-1][0] - 4) // 2 + 1, (s[-1][1] - 4) // 2 + 1, c))
    conv = lambda i: s[i][0] * s[i][1] * s[i][2] * 16 * s[i - 1][2]      # conv i: output side i, input side i - 1
    feat = s[4][0] * s[4][1] * 256
    return {"conv1": conv(1), "conv2": conv(2), "conv3": conv(3), "conv4": conv(4), "mean": feat * z, "logstd_sqare": feat * z,
            "dense1": z * feat, "deconv1": conv(4), "deconv2": conv(3),
            "deconv3": s[2][0] * s[2][1] * 64 * 25 * 32,                  # 5x5 kernel, small side [H2, W2, 64] -> 32
            "deconv4": s[1][0] * s[1][1] * 32 * 16 * ct}


def flop_per_frame(h, w, what):
    m = layer_macs(h, w)
    fwd = sum(m.values())
    if what == "train":
        return 2 * (fwd + (fwd - m["conv1"]) + fwd)
    return 2 * (m["conv1"] + m["conv2"] + m["conv3"] + m["conv4"] + m["mean"])


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True)
    return q.stdout.strip()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", required=True)
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--steps", type=int, default=10)
    args = ap.parse_args()
    assert flop_per_frame(80, 160, "train") == 776_494_080 and flop_per_frame(80, 160, "encode") == 117_992_448
    os.makedirs(args.out, exist_ok=True)

    import torch
    from carla_ppo_b200 import _lib
    from carla_ppo_b200.vae.models import ConvVAE
    lib = _lib.load()
    result = {"card": card(), "train_batch": TRAIN_B, "encode_batch": ENCODE_B, "rounds": args.rounds, "steps": args.steps,
              "flop_per_frame": {"%dx%d" % g: {"train": flop_per_frame(*g, "train"), "encode": flop_per_frame(*g, "encode")}
                                 for g in GEOMETRIES}}
    gen = torch.Generator(device="cuda")
    gen.manual_seed(0)
    models, data = {}, {}
    for h, w in GEOMETRIES:
        vae = ConvVAE((h, w, 3), target_shape=(h, w, 3), z_dim=Z, loss_fn="mse", model_dir=tempfile.mkdtemp(), seed=0)
        vae.init_session(init_logging=False)
        models[(h, w)] = vae
        x = torch.rand(ENCODE_B, h, w, 3, generator=gen, device="cuda")
        data[(h, w)] = (x, torch.randn(TRAIN_B, Z, generator=gen, device="cuda"))

    def window(vae, geo, what, steps):
        x, eps = data[geo]
        xt = x[:TRAIN_B]
        if what == "train":
            call = lambda: vae.train_step_device(xt, xt, eps)
        else:
            call = lambda: vae.encode_device(x, check=False)
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        for _ in range(steps):
            call()
        b.record()
        torch.cuda.synchronize()
        return a.elapsed_time(b) / steps

    times = {}
    for r in range(args.rounds):
        for geo in GEOMETRIES:
            vae = models[geo]
            for mode in MODES:
                _lib.check(lib.cpb_set_math_mode(mode))
                for what in ("train", "encode"):
                    window(vae, geo, what, 2)                       # warm-up: workspace, first launches
                    ms = window(vae, geo, what, args.steps)
                    times.setdefault((geo, mode, what), []).append(ms)
                    print("round %d %dx%d mode %d %s: %.3f ms" % (r, geo[0], geo[1], mode, what, ms), flush=True)
            vae._ws.clear()                                         # one geometry's workspaces at a time
            torch.cuda.empty_cache()

    rows = []
    for (geo, mode, what), ms in sorted(times.items()):
        med = statistics.median(ms)
        b = TRAIN_B if what == "train" else ENCODE_B
        rows.append({"frame": "%dx%d" % geo, "math_mode": mode, "work": what, "batch": b, "ms_median": round(med, 4),
                     "ms_spread": round(max(ms) - min(ms), 4), "ms_all": [round(v, 4) for v in ms],
                     "frames_per_s": round(b / (med * 1e-3)), "tflops": round(flop_per_frame(*geo, what) * b / (med * 1e-3) / 1e12, 2)})
    result["timings"] = rows

    # separate profiled pass: the per-group breakdown of one call per pair
    prof = {}
    buf = __import__("ctypes").create_string_buffer(1 << 16)
    for geo in GEOMETRIES:
        vae = models[geo]
        for mode in MODES:
            _lib.check(lib.cpb_set_math_mode(mode))
            for what in ("train", "encode"):
                window(vae, geo, what, 1)
                lib.cpb_profile_reset()
                lib.cpb_profile_enable(1)
                window(vae, geo, what, 1)
                lib.cpb_profile_enable(0)
                n = lib.cpb_profile_report(buf, len(buf))
                groups = {}
                for line in buf.raw[:n].decode().splitlines():
                    label, _, ms = line.split()
                    groups[label] = round(float(ms), 4)
                prof["%dx%d mode %d %s" % (geo[0], geo[1], mode, what)] = dict(sorted(groups.items(), key=lambda kv: -kv[1]))
                lib.cpb_profile_reset()
        vae._ws.clear()
        torch.cuda.empty_cache()
    _lib.check(lib.cpb_set_math_mode(1))
    result["profile_ms"] = prof
    result["card_after"] = card()
    with open(os.path.join(args.out, "frame_size.json"), "w") as f:
        json.dump(result, f, indent=1)
    print(result["card"])
    print("%-8s %4s %-6s %6s %10s %9s %12s %8s" % ("frame", "mode", "work", "batch", "ms", "spread", "frames/s", "TFLOP/s"))
    for r in rows:
        print("%-8s %4d %-6s %6d %10.3f %9.3f %12d %8.2f" % (r["frame"], r["math_mode"], r["work"], r["batch"], r["ms_median"],
                                                          r["ms_spread"], r["frames_per_s"], r["tflops"]))


if __name__ == "__main__":
    main()
