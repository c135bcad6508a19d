"""Direct (DENSE_SCHUR) against iterative (ITERATIVE_SCHUR) bundle-adjustment solves, one JSON line.

C3 (400 x 4096, SIMPLE_RADIAL, shared camera, the configuration bench.py times): LM iterations per second of device
time, CG iterations and kernel launches per LM iteration, workspace bytes; the two solvers alternate `--reps` times.
Long sequence (the final joint BA of a tools/video_c5.py sequence, default 2500 frames x 2048 new points per window):
the direct workspace vgg_ba_workspace_bytes would need, and the iterative joint BA's LM iterations per second, peak
torch.cuda.max_memory_allocated, termination and final cost.  The card's name, power limit and SM clock are sampled
before and after."""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from tools.video_c5 import final_problem_arrays  # noqa: E402
from vggsfm_b200 import bundle_adjustment as ba  # noqa: E402
from vggsfm_b200.synthetic import make_scene, perturb  # noqa: E402


def gpu_state():
    try:
        return subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.sm,clocks.max.sm", "--format=csv,noheader"],
                              capture_output=True, text=True, timeout=30).stdout.strip()
    except Exception as e:                       # noqa: BLE001
        return f"unavailable: {e}"


def c3_problem(dev):
    sc = make_scene(400, 4096, "SIMPLE_RADIAL", seed=0)
    extr, K, extra, pts = perturb(sc)
    t = lambda a: torch.from_numpy(np.ascontiguousarray(a)).to(dev)
    return t(pts), t(extr), t(K), t(extra), t(sc.tracks), t(sc.mask)


def run_c3(dev, reps):
    pts, extr, K, extra, tracks, masks = c3_problem(dev)
    out = {}
    for r in range(reps):
        for kind in ("DENSE_SCHUR", "ITERATIVE_SCHUR"):
            *_, s = ba.bundle_adjustment(pts, extr, K, extra, tracks, masks, shared_camera=True, camera_type="SIMPLE_RADIAL",
                                         options=ba.prepare_ba_options(), linear_solver_type=kind,
                                         max_linear_solver_iterations=200)
            o = out.setdefault(kind, {"lm_it_per_s": [], "iterations": [], "final_cost": [], "cg_per_lm": [],
                                      "launches_per_lm": []})
            o["lm_it_per_s"].append(s.iterations / (s.device_ms * 1e-3))
            o["iterations"].append(s.iterations)
            o["final_cost"].append(s.final_cost)
            o["cg_per_lm"].append(s.cg_iterations / max(1, s.iterations))
            o["launches_per_lm"].append(s.kernel_launches / max(1, s.iterations))
    S, P = masks.shape
    Pp = ba.pad_tracks(P)
    out["DENSE_SCHUR"]["workspace_bytes"] = ba.workspace_bytes(S, Pp, ba.SIMPLE_RADIAL, ba.INTR_SHARED)
    out["ITERATIVE_SCHUR"]["workspace_bytes"] = ba.workspace_bytes(S, Pp, ba.SIMPLE_RADIAL, ba.INTR_SHARED, True)
    return out


def run_long(dev, frames, new):
    t0 = time.perf_counter()
    tracks, masks, xyz, extr, K = final_problem_arrays(frames, new, dev=dev)
    build_s = time.perf_counter() - t0
    S, P = masks.shape
    direct = ba.workspace_bytes(S, ba.pad_tracks(P), ba.SIMPLE_PINHOLE, ba.INTR_SHARED)
    torch.cuda.synchronize()
    torch.cuda.reset_peak_memory_stats(dev)
    t0 = time.perf_counter()
    *_, s = ba.bundle_adjustment(xyz, extr, K.expand(S, -1, -1), None, tracks, masks, shared_camera=True,
                                 options=ba.default_options(), filter_reconstruction=False,
                                 linear_solver_type="ITERATIVE_SCHUR")
    torch.cuda.synchronize()
    wall = time.perf_counter() - t0
    return {"frames": S, "points": P, "observations": int(masks.sum().item()), "problem_build_s": build_s,
            "direct_workspace_bytes": direct,
            "iterative_workspace_bytes": ba.workspace_bytes(S, ba.pad_tracks(P), ba.SIMPLE_PINHOLE, ba.INTR_SHARED, True),
            "lm_iterations": s.iterations, "lm_it_per_s": s.iterations / (s.device_ms * 1e-3), "wall_s": wall,
            "cg_iterations": s.cg_iterations, "launches": s.kernel_launches,
            "peak_bytes": torch.cuda.max_memory_allocated(dev), "termination": s.termination,
            "initial_cost": s.initial_cost, "final_cost": s.final_cost}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--frames", type=int, default=2500)
    ap.add_argument("--new", type=int, default=2048)
    ap.add_argument("--skip-long", action="store_true")
    ap.add_argument("--json", default=None)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("ba_iterative_bench needs a GPU")
    dev = torch.device("cuda:0")
    res = {"gpu_before": gpu_state(), "c3": run_c3(dev, a.reps)}
    if not a.skip_long:
        res["long"] = run_long(dev, a.frames, a.new)
    res["gpu_after"] = gpu_state()
    line = json.dumps(res)
    print(line)
    if a.json:
        with open(a.json, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
