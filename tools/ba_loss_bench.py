"""Cost of the robust losses in the bundle-adjustment solve, one JSON line.

C3 (400 x 4096, SIMPLE_RADIAL, shared camera, 10 % of the observations displaced by 20-80 px): LM iterations per second
of device time for TRIVIAL, SOFT_L1 and CAUCHY (scale 1 px), alternating in one process `--reps` times, for both linear
solvers (DENSE_SCHUR, ITERATIVE_SCHUR).  Every solve runs exactly `--iters` LM iterations (tolerances 0), from the same
start.  A separate pass under torch.profiler gives each kernel's device time per LM iteration, per loss and solver.
The card's name, power limit and SM clock are sampled before and after."""
import argparse
import json
import os
import subprocess
import sys

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from vggsfm_b200 import bundle_adjustment as ba  # noqa: E402
from vggsfm_b200.synthetic import make_scene, perturb  # noqa: E402

LOSSES = ("TRIVIAL", "SOFT_L1", "CAUCHY")
SOLVERS = ("DENSE_SCHUR", "ITERATIVE_SCHUR")


def gpu_state():
    try:
        return subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.sm,clocks.max.sm", "--format=csv,noheader"],
                              capture_output=True, text=True, timeout=30).stdout.strip()
    except Exception as e:                       # noqa: BLE001
        return f"unavailable: {e}"


def c3_problem(dev, seed=0):
    """lm_solve's arrays of C3 with outliers: uv, mask, poses, intr, points (the last three are copied per solve)"""
    sc = make_scene(400, 4096, "SIMPLE_RADIAL", seed=seed)
    extr, K, extra, pts = perturb(sc)
    rng = np.random.default_rng(seed + 1)
    uv = sc.tracks.astype(np.float64)
    pick = sc.mask & (rng.uniform(size=sc.mask.shape) < 0.1)
    ang = rng.uniform(0.0, 2.0 * np.pi, size=sc.mask.shape)
    mag = rng.uniform(20.0, 80.0, size=sc.mask.shape)
    uv = np.where(pick[..., None], uv + np.stack([np.cos(ang), np.sin(ang)], -1) * mag[..., None], uv)
    intr = np.zeros((400, 4))
    intr[:] = [K[0, 0, 0], K[0, 0, 2], K[0, 1, 2], extra[0, 0]]
    t = lambda a, dt=None: torch.from_numpy(np.ascontiguousarray(a if dt is None else a.astype(dt))).to(dev)
    return t(uv, np.float32), t(sc.mask, np.uint8), t(extr), t(intr), t(pts)


def solve(prob, solver, loss, iters):
    uv, mask, poses, intr, pts = prob
    o = ba.default_options()
    o.max_num_iterations = iters
    o.function_tolerance = o.gradient_tolerance = o.parameter_tolerance = 0.0
    return ba.lm_solve(uv, mask, poses.clone(), intr.clone(), pts.clone(), ba.SIMPLE_RADIAL, ba.INTR_SHARED, options=o,
                       linear_solver_type=solver, max_linear_solver_iterations=200, loss_function_type=loss)


def timed(prob, iters, reps):
    out = {s: {l: {"lm_it_per_s": [], "iterations": [], "final_cost": []} for l in LOSSES} for s in SOLVERS}
    for solver in SOLVERS:
        for loss in LOSSES:                                                     # warm-up of every instantiation
            solve(prob, solver, loss, 1)
    for _ in range(reps):
        for solver in SOLVERS:
            for loss in LOSSES:
                s = solve(prob, solver, loss, iters)
                o = out[solver][loss]
                o["lm_it_per_s"].append(s.iterations / (s.device_ms * 1e-3))
                o["iterations"].append(s.iterations)
                o["final_cost"].append(s.final_cost)
    for solver in SOLVERS:
        for loss in LOSSES:
            v = out[solver][loss]["lm_it_per_s"]
            out[solver][loss]["median_lm_it_per_s"] = float(np.median(v))
        t = out[solver]["TRIVIAL"]["median_lm_it_per_s"]
        for loss in LOSSES[1:]:
            out[solver][loss]["relative_to_trivial"] = out[solver][loss]["median_lm_it_per_s"] / t
    return out


def profiled(prob, iters):
    """device time per LM iteration of each kernel (microseconds), one solve per (solver, loss) under the profiler"""
    from torch.profiler import ProfilerActivity, profile
    res = {}
    for solver in SOLVERS:
        for loss in LOSSES:
            torch.cuda.synchronize()
            with profile(activities=[ProfilerActivity.CUDA]) as prof:
                s = solve(prob, solver, loss, iters)
                torch.cuda.synchronize()
            per = {}
            for e in prof.key_averages():
                t = getattr(e, "device_time_total", None)
                if t is None:
                    t = e.cuda_time_total
                if t > 0:
                    per[e.key.split("<")[0].replace("void ", "").replace("vgg::", "")] = per.get(
                        e.key.split("<")[0].replace("void ", "").replace("vgg::", ""), 0.0) + t / max(1, s.iterations)
            top = dict(sorted(per.items(), key=lambda kv: -kv[1])[:12])
            res.setdefault(solver, {})[loss] = {k: round(v, 1) for k, v in top.items()}
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--iters", type=int, default=10)
    ap.add_argument("--json", default=None)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("ba_loss_bench needs a GPU")
    dev = torch.device("cuda:0")
    prob = c3_problem(dev)
    res = {"gpu_before": gpu_state(), "shape": "C3 400x4096 SIMPLE_RADIAL shared, 10% outliers, scale 1 px",
           "iters": a.iters, "timed": timed(prob, a.iters, a.reps), "kernel_us_per_lm_iteration": profiled(prob, a.iters),
           "gpu_after": gpu_state()}
    line = json.dumps(res)
    print(line)
    if a.json:
        with open(a.json, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
