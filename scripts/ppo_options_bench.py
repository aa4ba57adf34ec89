"""Cost of the bounded-update guards: PPO.learn at BASELINE configs[2] (T = 2048, 4 epochs x 256, ckpt-705) and over 16
segments x 128 rows, with the guards off (cpb_ppo_learn / _segments), clipping only, and clipping + a KL target that
never triggers (so every variant applies the same 32 Adam steps).  Each path (launch-per-kernel, CPB_PPO_PERSISTENT=1)
runs in its own child process, since the library reads the variable once; within one, the variants alternate call by
call and each time is CUDA events around one learn() call on device-resident inputs.  Prints one JSON object (median and
spread of `--reps` calls per variant, the card's name and power limit) and writes it to --out when given.

    python scripts/ppo_options_bench.py --reps 20 --out /tmp/ppo_options_bench.json
"""
import argparse
import json
import os
import subprocess
import sys
import tempfile
from pathlib import Path

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
VARIANTS = {"off": {}, "clip": dict(max_grad_norm=0.5), "clip+kl": dict(max_grad_norm=0.5, target_kl=1e3)}
WORKLOADS = {"config3": None, "16x128": [128] * 16}


def child(reps):
    sys.path.insert(0, ROOT)
    sys.path.insert(0, os.path.join(ROOT, "tests"))
    import numpy as np
    import torch
    import ppo_cases as oc
    dev = torch.device("cuda")
    tmp = Path(tempfile.mkdtemp())
    out = {}
    for wname, lengths in WORKLOADS.items():
        if lengths is None:
            s, a, r, v, d, perms = oc.baseline_config3(oc.T3, oc.E3)
            last = 0.3
        else:
            s, a, r, v, d, last, perms = oc.segment_rollout(lengths)
        on = lambda x, dt: torch.as_tensor(np.asarray(x), dtype=dt, device=dev)
        args = (on(s, torch.float32), on(a, torch.float32), on(v, torch.float64), on(r, torch.float64),
                on(np.asarray(d, np.float64), torch.float64), last)
        p = on(perms, torch.int32)
        models = {k: oc.shipped_model(tmp / wname / k) for k in VARIANTS}
        for k, m in models.items():          # warm-up: workspace, modules, the first launches
            m.learn(*args, num_epochs=oc.E3, batch_size=oc.B3, perms=p, segment_lengths=lengths, **VARIANTS[k])
        times = {k: [] for k in VARIANTS}
        for _ in range(reps):
            for k, m in models.items():
                e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                torch.cuda.synchronize()
                e0.record()
                m.learn(*args, num_epochs=oc.E3, batch_size=oc.B3, perms=p, segment_lengths=lengths, **VARIANTS[k])
                e1.record()
                torch.cuda.synchronize()
                times[k].append(e0.elapsed_time(e1))
        for k in VARIANTS:
            applied = int(models[k].last_steps_applied.item()) if VARIANTS[k] else oc.E3 * (oc.T3 // oc.B3)
            t = np.asarray(times[k])
            out["%s/%s" % (wname, k)] = dict(median_ms=float(np.median(t)), min_ms=float(t.min()), max_ms=float(t.max()),
                                             steps_applied=applied)
    print(json.dumps(out))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=20)
    ap.add_argument("--out", default=None)
    ap.add_argument("--child", action="store_true")
    a = ap.parse_args()
    if a.child:
        return child(a.reps)
    import torch
    res = dict(device=torch.cuda.get_device_name(0), reps=a.reps)
    q = subprocess.run(["nvidia-smi", "--query-gpu=power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True)
    res["power_limit_and_max_sm_clock"] = q.stdout.strip().splitlines()[0] if q.returncode == 0 else "unavailable"
    for path, flag in (("launch", "0"), ("persistent", "1")):
        r = subprocess.run([sys.executable, __file__, "--child", "--reps", str(a.reps)], capture_output=True, text=True,
                           env=dict(os.environ, CPB_PPO_PERSISTENT=flag))
        if r.returncode != 0:
            sys.stderr.write(r.stderr[-3000:])
            raise SystemExit("%s child failed" % path)
        res[path] = json.loads(r.stdout.strip().splitlines()[-1])
    text = json.dumps(res, indent=1)
    print(text)
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as f:
            f.write(text)


if __name__ == "__main__":
    main()
