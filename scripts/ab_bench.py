"""A/B timing of two builds of libcarla_ppo_b200.so on the flagship workload (bench.py, ConvVAE train step at batch 4096).

    python scripts/ab_bench.py --a OLD.so --b NEW.so --runs 3 --out DIR [--math-mode 2]

The library path is fixed (carla_ppo_b200/libcarla_ppo_b200.so), so each run copies its build there first; runs
alternate a, b, a, b, ... so that drift of the shared machine hits both sides alike.  Each run is one
`bench.py --gpus 1 --steps S --warmup 3 --no-cpu-baseline --dump-outputs` process.  Writes DIR/ab.json: the card
(name, power limit, max SM clock), every run's ms_per_step, e2e, kernel launch count and per-group profile, the
median and spread per side, and the largest differences between the two sides' dumped outputs (losses, parameters, gradient).
With --b omitted only --a is timed (a "before" measurement).  --a-root runs side a from another checkout (its own
bench.py and Python package, e.g. the parent commit's, whose bindings match its library).  --math-mode sets cpb_set_math_mode before bench.py runs
(bench.py itself runs the library's default, mode 1).  The library at the fixed path is restored at the end.
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
LIB_REL = os.path.join("carla_ppo_b200", "libcarla_ppo_b200.so")
LIB = os.path.join(ROOT, LIB_REL)


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True)
    return q.stdout.strip()


# bench.py of the checkout in the working directory, in this process after cpb_set_math_mode(mode): argv[1] is the mode,
# the rest bench.py's arguments
WITH_MODE = ("import os, runpy, sys; sys.path.insert(0, os.getcwd()); from carla_ppo_b200 import _lib; "
             "_lib.check(_lib.load().cpb_set_math_mode(int(sys.argv[1]))); sys.argv = ['bench.py'] + sys.argv[2:]; "
             "runpy.run_path('bench.py', run_name='__main__')")


def run_bench(lib, steps, dump, math_mode=None, root=ROOT):
    shutil.copyfile(lib, os.path.join(root, LIB_REL))
    args = ["--gpus", "1", "--steps", str(steps), "--warmup", "3", "--no-cpu-baseline", "--dump-outputs", dump]
    cmd = [sys.executable, "bench.py"] if math_mode is None else [sys.executable, "-c", WITH_MODE, str(math_mode)]
    r = subprocess.run(cmd + args, cwd=root, capture_output=True, text=True)
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
    ap.add_argument("--a-root", default=ROOT, help="checkout whose bench.py and package run side a (default: this one)")
    ap.add_argument("--math-mode", type=int, default=None, choices=[0, 1, 2], help="cpb_set_math_mode before bench.py runs")
    args = ap.parse_args()
    os.makedirs(args.out, exist_ok=True)
    sides = {"a": args.a} if args.b is None else {"a": args.a, "b": args.b}
    saved = LIB + ".ab_saved"
    shutil.copyfile(LIB, saved)
    roots = {"a": os.path.abspath(args.a_root), "b": ROOT}
    saved_a = os.path.join(roots["a"], LIB_REL) + ".ab_saved"
    if roots["a"] != ROOT:
        shutil.copyfile(os.path.join(roots["a"], LIB_REL), saved_a)
    result = {"card": card(), "libs": sides, "roots": roots, "math_mode": args.math_mode, "runs": {k: [] for k in sides}}
    try:
        for i in range(args.runs):
            for side, lib in sides.items():
                r = run_bench(lib, args.steps, os.path.abspath(os.path.join(args.out, "dump_%s" % side)), args.math_mode, roots[side])
                print("run %d %s: %.2f ms/step" % (i, side, r["ms_per_step"]), flush=True)
                result["runs"][side].append(r)
    finally:
        shutil.move(saved, LIB)
        if roots["a"] != ROOT:
            shutil.move(saved_a, os.path.join(roots["a"], LIB_REL))
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
