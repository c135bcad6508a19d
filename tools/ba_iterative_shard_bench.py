"""ITERATIVE_SCHUR on one GPU and over emulated track shards, one JSON line.

single: the single-GPU iterative solve at C3 (400 x 4096, SIMPLE_RADIAL, shared camera, prepare_ba_options, at most 200
CG iterations per step) and on the final joint BA of a tools/video_c5.py sequence (default 2500 frames x 2048 new points
per window, `--long-iters` LM iterations): LM iterations per second of device time, CG iterations, kernel launches per
LM iteration and the final cost, `--reps` times.  `--root DIR` imports vggsfm_b200 from DIR instead of this tree, so two
builds can be alternated by running the script once per build.

ranks: the per-rank device time of one LM iteration's kernels on the long sequence at K = 1, 2, 4 ranks emulated on
this GPU (tests/emulated_ranks.py: one rank at a time has work in flight), from torch.profiler: the sum of all kernel,
copy and memset time over the ranks, divided by K.  It is kernel time per rank, not a multi-GPU wall time: the NCCL
latency of the per-CG-iteration reduction is not part of it.  The card's name and power limit are read before and
after."""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np

HERE = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def gpu_state():
    try:
        return subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.sm,clocks.max.sm", "--format=csv,noheader"],
                              capture_output=True, text=True, timeout=30).stdout.strip()
    except Exception as e:                       # noqa: BLE001
        return f"unavailable: {e}"


def summary_row(s):
    return {"lm_it_per_s": s.iterations / (s.device_ms * 1e-3), "iterations": s.iterations,
            "cg_iterations": s.cg_iterations, "launches_per_lm": s.kernel_launches / max(1, s.iterations),
            "final_cost": s.final_cost, "termination": s.termination}


def run_single(ba, dev, reps, frames, new, long_iters):
    import torch
    from tools.video_c5 import final_problem_arrays
    from vggsfm_b200.synthetic import make_scene, perturb
    sc = make_scene(400, 4096, "SIMPLE_RADIAL", seed=0)
    extr, K, extra, pts = perturb(sc)
    t = lambda a: torch.from_numpy(np.ascontiguousarray(a)).to(dev)
    c3 = (t(pts), t(extr), t(K), t(extra), t(sc.tracks), t(sc.mask))
    tracks, masks, xyz, lextr, LK = final_problem_arrays(frames, new, dev=dev)
    S = masks.shape[0]
    o = ba.default_options()
    o.max_num_iterations = long_iters
    out = {"c3": [], "long": []}
    for _ in range(reps):
        *_, s = ba.bundle_adjustment(*c3[:4], c3[4], c3[5], shared_camera=True, camera_type="SIMPLE_RADIAL",
                                     options=ba.prepare_ba_options(), linear_solver_type="ITERATIVE_SCHUR",
                                     max_linear_solver_iterations=200)
        out["c3"].append(summary_row(s))
        *_, s = ba.bundle_adjustment(xyz, lextr, LK.expand(S, -1, -1), None, tracks, masks, shared_camera=True,
                                     options=o, filter_reconstruction=False, linear_solver_type="ITERATIVE_SCHUR")
        out["long"].append(dict(summary_row(s), cg_trace=s.cg_trace.tolist()))
    return out


def run_ranks(ba, dev, frames, new, ks, max_cg):
    import torch
    from torch.profiler import ProfilerActivity, profile
    from tests.emulated_ranks import DeviceAllReduce, RankGroup
    from tools.video_c5 import final_problem_arrays
    from vggsfm_b200.dist import shard_range
    tracks, masks, xyz, extr, LK = final_problem_arrays(frames, new, dev=dev)
    S, P = masks.shape
    o = ba.default_options()
    o.max_num_iterations = 1

    def solve(lo, hi, hook):
        *_, s = ba.bundle_adjustment(xyz[lo:hi], extr, LK.expand(S, -1, -1), None, tracks[:, lo:hi], masks[:, lo:hi],
                                     shared_camera=True, options=o, filter_reconstruction=False,
                                     linear_solver_type="ITERATIVE_SCHUR", max_linear_solver_iterations=max_cg,
                                     allreduce=hook)
        torch.cuda.current_stream().synchronize()
        return s

    def sharded(K):
        if K == 1:
            return [solve(0, P, None)]
        group = RankGroup(K)

        def rank(r):
            lo, hi = shard_range(P, r, K)
            st = torch.cuda.Stream(device=dev)
            with torch.cuda.stream(st):
                return solve(lo, hi, DeviceAllReduce(group, r))
        return group.run(rank)

    # one workspace per rank thread: the process-wide cache is keyed by shape, and ranks with equal shards would share
    import ctypes
    import threading
    from vggsfm_b200 import _lib
    local = threading.local()

    def workspace(S_, N_, model, mode, device, iterative=False):
        cache = local.__dict__.setdefault("cache", {})
        key = (S_, N_, model, mode, str(device), iterative)
        if key not in cache:
            nbytes = ctypes.c_size_t()
            fn = _lib.lib().vgg_ba_workspace_bytes_iterative if iterative else _lib.lib().vgg_ba_workspace_bytes
            _lib.check(fn(S_, N_, model, mode, ctypes.byref(nbytes)), "workspace")
            cache[key] = torch.empty(nbytes.value, dtype=torch.uint8, device=device)
        return cache[key]

    ba.workspace = workspace
    out = {"frames": S, "points": P, "max_cg": max_cg}
    for K in ks:
        sharded(K)                                    # warm-up: workspaces, modules
        torch.cuda.synchronize()
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            res = sharded(K)
            torch.cuda.synchronize()
        dev_us = sum(e.self_device_time_total for e in prof.key_averages())
        out[f"K{K}"] = {"device_ms_per_rank": dev_us / 1e3 / K, "device_ms_all_ranks": dev_us / 1e3,
                        "cg_iterations": [s.cg_iterations for s in res], "final_cost": res[0].final_cost}
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--mode", choices=("single", "ranks"), default="single")
    ap.add_argument("--root", default=HERE, help="directory vggsfm_b200 is imported from")
    ap.add_argument("--reps", type=int, default=2)
    ap.add_argument("--frames", type=int, default=2500)
    ap.add_argument("--new", type=int, default=2048)
    ap.add_argument("--long-iters", type=int, default=10)
    ap.add_argument("--ranks", default="1,2,4")
    ap.add_argument("--max-cg", type=int, default=100)
    ap.add_argument("--json", default=None)
    a = ap.parse_args()
    sys.path.insert(0, HERE)
    sys.path.insert(0, os.path.abspath(a.root))
    import torch
    from vggsfm_b200 import bundle_adjustment as ba
    if not torch.cuda.is_available():
        sys.exit("ba_iterative_shard_bench needs a GPU")
    dev = torch.device("cuda:0")
    res = {"gpu_before": gpu_state(), "root": os.path.abspath(a.root), "mode": a.mode}
    t0 = time.perf_counter()
    if a.mode == "single":
        res.update(run_single(ba, dev, a.reps, a.frames, a.new, a.long_iters))
    else:
        res["ranks"] = run_ranks(ba, dev, a.frames, a.new, [int(k) for k in a.ranks.split(",")], a.max_cg)
    res["wall_s"] = time.perf_counter() - t0
    res["gpu_after"] = gpu_state()
    line = json.dumps(res)
    print(line)
    if a.json:
        with open(a.json, "a") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
