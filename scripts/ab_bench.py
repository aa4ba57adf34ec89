"""A/B timing of two builds of libcarla_ppo_b200.so on the flagship workload (bench.py, ConvVAE train step at batch 4096).

    python scripts/ab_bench.py --a OLD.so --b NEW.so --runs 3 --out DIR

The library path is fixed (carla_ppo_b200/libcarla_ppo_b200.so), so each run copies its build there first; runs
alternate a, b, a, b, ... so that drift of the shared machine hits both sides alike.  Each run is one
`bench.py --gpus 1 --steps S --warmup 3 --no-cpu-baseline --dump-outputs` process.  Writes DIR/ab.json: the card
(name, power limit, max SM clock), every run's ms_per_step, e2e, kernel launch count and per-group profile, the
median and spread per side, and the largest differences between the two sides' dumped outputs (losses, parameters, gradient).
With --b omitted only --a is timed (a "before" measurement).  The library at the fixed path is restored at the end.
"""
import argparse
import json
import os
import shutil
import statistics
import subprocess
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
LIB = os.path.join(ROOT, "carla_ppo_b200", "libcarla_ppo_b200.so")


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True)
    return q.stdout.strip()


def run_bench(lib, steps, dump):
    shutil.copyfile(lib, LIB)
    r = subprocess.run([sys.executable, os.path.join(ROOT, "bench.py"), "--gpus", "1", "--steps", str(steps), "--warmup", "3",
                        "--no-cpu-baseline", "--dump-outputs", dump], cwd=ROOT, capture_output=True, text=True)
    if r.returncode != 0:
        sys.stderr.write(r.stderr[-4000:])
        raise SystemExit("bench.py failed with %s" % lib)
    line = [l for l in r.stdout.splitlines() if l.startswith("{")][-1]
    out = json.loads(line)
    return {"ms_per_step": out["ms_per_step"], "e2e_ms_per_step": out["e2e"]["ms_per_step"], "clocks": out.get("clocks"),
            "gpu_launches": out.get("gpu_launches"),
            "groups_ms_per_step": out.get("roofline", {}).get("groups_ms_per_step")}


def compare(da, db):
    res = {}
    for name in ("losses", "params", "grads"):
        a = np.load(os.path.join(da, name + ".npy")).astype(np.float64)
        b = np.load(os.path.join(db, name + ".npy")).astype(np.float64)
        res[name] = {"bit_identical": bool(np.array_equal(a, b)),
                     "rel_l2": float(np.linalg.norm(a - b) / max(np.linalg.norm(a), 1e-300)),
                     "max_abs": float(np.abs(a - b).max())}
    return res


def summary(runs):
    ms = [r["ms_per_step"] for r in runs]
    e2e = [r["e2e_ms_per_step"] for r in runs]
    groups = {}
    for r in runs:
        for k, v in (r["groups_ms_per_step"] or {}).items():
            groups.setdefault(k, []).append(v)
    return {"ms_per_step": ms, "median_ms": statistics.median(ms), "spread_ms": max(ms) - min(ms),
            "gpu_launches": sorted(set(r["gpu_launches"] for r in runs)),
            "e2e_median_ms": statistics.median(e2e),
            "groups_median_ms": {k: round(statistics.median(v), 4) for k, v in sorted(groups.items(), key=lambda kv: -statistics.median(kv[1]))}}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--a", required=True, help="first build (e.g. the parent commit's library)")
    ap.add_argument("--b", default=None, help="second build")
    ap.add_argument("--runs", type=int, default=3, help="bench.py runs per build")
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--out", required=True)
    args = ap.parse_args()
    os.makedirs(args.out, exist_ok=True)
    sides = {"a": args.a} if args.b is None else {"a": args.a, "b": args.b}
    saved = LIB + ".ab_saved"
    shutil.copyfile(LIB, saved)
    result = {"card": card(), "libs": sides, "runs": {k: [] for k in sides}}
    try:
        for i in range(args.runs):
            for side, lib in sides.items():
                r = run_bench(lib, args.steps, os.path.join(args.out, "dump_%s" % side))
                print("run %d %s: %.2f ms/step" % (i, side, r["ms_per_step"]), flush=True)
                result["runs"][side].append(r)
    finally:
        shutil.move(saved, LIB)
    result["summary"] = {k: summary(v) for k, v in result["runs"].items()}
    if args.b is not None:
        result["outputs_a_vs_b"] = compare(os.path.join(args.out, "dump_a"), os.path.join(args.out, "dump_b"))
        sa, sb = result["summary"]["a"], result["summary"]["b"]
        result["speedup"] = sa["median_ms"] / sb["median_ms"]
    result["card_after"] = card()
    with open(os.path.join(args.out, "ab.json"), "w") as f:
        json.dump(result, f, indent=1)
    print(json.dumps({k: result[k] for k in result if k != "runs"}, indent=1))


if __name__ == "__main__":
    main()
