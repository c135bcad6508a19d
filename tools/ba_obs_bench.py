"""The joint BA with ITERATIVE_SCHUR through the [S,P] grid (video.joint_BA) and through the observation list
(video.joint_BA_obs), one JSON line per measurement and a summary line.

  * 2500-frame joint BA (tools/video_c5.py final_problem_arrays(2500, 2048)): grid and list alternated three times, LM
    it/s and peak device memory; the grid's peak as a multiple of its 9 S P bytes (video.GRID_PEAK_MULTIPLE comes from
    it); per CG iteration the time of the matvec's Schur part (pcg_schur_kernel, or list_point_w + list_schur) from
    torch.profiler in a separate pass;
  * C3 (400 x 4096, every cell an observation): both paths, where the grid has no padding;
  * the 8000-frame problem at 2048 new points per window, built as a list window by window (its grid would be > 70 GB):
    the list only, through SceneStore.joint_bundle_adjustment.

The card's name and power limit are read in the same call.  Usage: python tools/ba_obs_bench.py [--out DIR]"""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

from vggsfm_b200 import bundle_adjustment as ba            # noqa: E402
from vggsfm_b200 import video                              # noqa: E402
from vggsfm_b200.synthetic import _exp_so3, make_video_scene   # noqa: E402


def final_problem_obs(frames, new_per_window, seed=0, dev=None):
    """final_problem_arrays (tools/video_c5.py) as an observation list, built window by window so that no [S,P] grid is
    ever formed: (obs_uv [M,2] f32, obs_frame [M], obs_point [M], points [P,3], extrinsics [S,3,4], K [1,3,3]), points
    seen in >= 3 frames, the same ground truth + noise."""
    dev = dev or torch.device("cuda:0")
    sc = make_video_scene(F=frames, new_per_window=new_per_window, seed=seed)
    rng = np.random.default_rng(seed + 2)
    uvs, frs, pts_ = [], [], []
    for w in range(sc.num_windows()):
        ids = np.nonzero(sc.birth == w)[0]
        f0, f1 = int(sc.first_frame[ids[0]]), int(sc.last_frame[ids[0]])
        u, o = sc.observe(ids, f0, f1)
        f, n = np.nonzero(o)
        uvs.append(torch.from_numpy(np.ascontiguousarray(u[f, n], dtype=np.float32)).to(dev))
        frs.append(torch.from_numpy((f + f0).astype(np.int32)).to(dev))
        pts_.append(torch.from_numpy(ids[n].astype(np.int64)).to(dev))
    obs_uv, obs_frame, obs_point = torch.cat(uvs), torch.cat(frs), torch.cat(pts_)
    del uvs, frs, pts_
    P = sc.points3d.shape[0]
    keep = (torch.bincount(obs_point, minlength=P) >= 3).cpu().numpy()
    w = rng.normal(size=(frames, 3))
    w = w / np.linalg.norm(w, axis=1, keepdims=True) * np.deg2rad(0.2)
    extr = sc.extrinsics.copy()
    extr[:, :, :3] = _exp_so3(w) @ extr[:, :, :3]
    extr[:, :, 3] += rng.normal(size=(frames, 3)) * 0.005
    pts = sc.points3d[keep] + rng.normal(size=(int(keep.sum()), 3)) * 0.01
    K = torch.tensor([[[sc.focal, 0.0, sc.pp[0]], [0.0, sc.focal, sc.pp[1]], [0.0, 0.0, 1.0]]], dtype=torch.float64,
                     device=dev)
    kt = torch.from_numpy(keep).to(dev)
    new_id = torch.cumsum(kt.long(), 0) - 1
    sel = kt[obs_point]
    T = lambda a: torch.from_numpy(np.ascontiguousarray(a)).to(dev)
    return obs_uv[sel], obs_frame[sel], new_id[obs_point[sel]], T(pts), T(extr), K


def store_of(obs_uv, obs_frame, obs_point, pts, extr, dev):
    """a SceneStore holding the problem (frames 0..S-1)"""
    st = video.SceneStore(dev)
    st.xyz = pts.float()
    st.rgb = torch.zeros_like(st.xyz)
    st.obs_uv, st.obs_frame, st.obs_point = obs_uv.float(), obs_frame.long(), obs_point.long()
    st.obs_vis = torch.ones(obs_uv.shape[0], dtype=torch.float32, device=dev)
    st.set_extrinsics(0, extr)
    return st


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                       text=True).stdout.strip().splitlines()
    return q[0] if q else "unknown"


def _opts(iters):
    o = ba.default_options()
    o.max_num_iterations = iters
    return o


def run_grid(tracks, masks, pts, extr, K, iters, max_cg):
    torch.cuda.synchronize()
    base = torch.cuda.memory_allocated()
    torch.cuda.reset_peak_memory_stats()
    t0 = time.perf_counter()
    video.joint_BA(pts, extr, K, None, tracks, masks, linear_solver_type="ITERATIVE_SCHUR",
                   max_linear_solver_iterations=max_cg, options=_opts(iters))
    torch.cuda.synchronize()
    dt = time.perf_counter() - t0
    s = video.last_joint_summary
    return dict(seconds=dt, lm_it=s.iterations, lm_it_per_s=s.iterations / dt, cg_it=s.cg_iterations,
                peak_gb=torch.cuda.max_memory_allocated() / 1e9, added_gb=(torch.cuda.max_memory_allocated() - base) / 1e9,
                final_cost=s.final_cost, initial_cost=s.initial_cost, termination=s.termination)


def run_list(uv, fr, pt, pts, extr, K, iters, max_cg):
    torch.cuda.synchronize()
    base = torch.cuda.memory_allocated()
    torch.cuda.reset_peak_memory_stats()
    t0 = time.perf_counter()
    video.joint_BA_obs(pts, extr, K, None, uv, fr, pt, max_linear_solver_iterations=max_cg, options=_opts(iters))
    torch.cuda.synchronize()
    dt = time.perf_counter() - t0
    s = video.last_joint_summary
    return dict(seconds=dt, lm_it=s.iterations, lm_it_per_s=s.iterations / dt, cg_it=s.cg_iterations,
                peak_gb=torch.cuda.max_memory_allocated() / 1e9, added_gb=(torch.cuda.max_memory_allocated() - base) / 1e9,
                final_cost=s.final_cost, initial_cost=s.initial_cost, termination=s.termination)


def schur_us_per_cg(fn, names):
    """time of the matvec's Schur-part kernels per CG iteration, torch.profiler pass of its own"""
    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        fn()
        torch.cuda.synchronize()
    us = sum(e.device_time_total for e in prof.key_averages() if any(n in e.key for n in names))
    cg = video.last_joint_summary.cg_iterations
    return us / max(1, cg)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", default=None)
    ap.add_argument("--iters", type=int, default=5)
    ap.add_argument("--max-cg", type=int, default=100)
    ap.add_argument("--skip-8000", action="store_true")
    a = ap.parse_args()
    dev = torch.device("cuda:0")
    from tools.video_c5 import final_problem_arrays
    res = dict(card=card())
    emit = lambda d: print(json.dumps(d), flush=True)
    emit(res)

    # ---- 2500 frames: grid vs list, alternated
    tracks, masks, pts, extr, K = final_problem_arrays(2500, 2048, dev=dev)
    S, P = masks.shape
    f, n = torch.nonzero(masks, as_tuple=True)
    uv = tracks[f, n]
    rows = []
    for rep in range(3):
        g = run_grid(tracks, masks, pts, extr, K, a.iters, a.max_cg)
        lst = run_list(uv, f, n, pts, extr, K, a.iters, a.max_cg)
        rows.append(dict(rep=rep, grid=g, list=lst))
        emit(dict(workload="joint2500", S=S, P=P, M=int(f.numel()), **rows[-1]))
    grid_multiple = max(r["grid"]["added_gb"] for r in rows) * 1e9 / (9.0 * S * P) + 1.0
    sg = schur_us_per_cg(lambda: run_grid(tracks, masks, pts, extr, K, a.iters, a.max_cg), ["pcg_schur_kernel"])
    sl = schur_us_per_cg(lambda: run_list(uv, f, n, pts, extr, K, a.iters, a.max_cg),
                         ["list_point_w_kernel", "list_schur_kernel"])
    res["joint2500"] = dict(S=S, P=P, M=int(f.numel()), grid_bytes_9SP=9.0 * S * P, grid_peak_multiple=grid_multiple,
                            schur_us_per_cg_grid=sg, schur_us_per_cg_list=sl, runs=rows)
    emit(dict(workload="joint2500", grid_peak_multiple=grid_multiple, schur_us_per_cg_grid=sg, schur_us_per_cg_list=sl))
    del tracks, masks, uv, f, n
    torch.cuda.empty_cache()

    # ---- C3: every cell observed
    from tests.helpers import ba_case
    from oracle import ba_oracle as bo
    c = ba_case(400, 4096, "SIMPLE_RADIAL", bo.INTR_SHARED, seed=0, invisible_frac=0.0)
    T = lambda x, dt=None: torch.from_numpy(np.ascontiguousarray(x)).to(dev, dt) if dt else \
        torch.from_numpy(np.ascontiguousarray(x)).to(dev)
    uvg, mk = T(c["uv"], torch.float32), T(c["mask"].astype(np.uint8))
    fc, nc = torch.nonzero(mk, as_tuple=True)
    o = ba.prepare_ba_options()
    o.max_num_iterations = 10
    c3 = []
    for rep in range(3):
        for name in ("grid", "list"):
            poses, intr, X = T(c["poses"]), T(c["intr"]), T(c["points"])
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            if name == "grid":
                s = ba.lm_solve(uvg, mk, poses, intr, X, c["model"], c["mode"], options=o,
                                linear_solver_type="ITERATIVE_SCHUR", max_linear_solver_iterations=200)
            else:
                s = ba.lm_solve_obs(uvg[fc, nc], fc, nc, poses, intr, X, c["model"], c["mode"], options=o,
                                    max_linear_solver_iterations=200)
            torch.cuda.synchronize()
            dt = time.perf_counter() - t0
            c3.append(dict(rep=rep, path=name, lm_it=s.iterations, cg_it=s.cg_iterations, lm_it_per_s=s.iterations / dt,
                           device_ms=s.device_ms, final_cost=s.final_cost))
            emit(dict(workload="C3", **c3[-1]))
    res["C3"] = c3

    # ---- 8000 frames, list only, through SceneStore (the size rule picks the list)
    if not a.skip_8000:
        t0 = time.perf_counter()
        uv8, f8, n8, p8, e8, K8 = final_problem_obs(8000, 2048, dev=dev)
        build_s = time.perf_counter() - t0
        S8, P8, M8 = e8.shape[0], p8.shape[0], int(f8.numel())
        store = store_of(uv8, f8, n8, p8, e8, dev)
        del uv8, f8, n8
        torch.cuda.synchronize()
        torch.cuda.reset_peak_memory_stats()
        t0 = time.perf_counter()
        store.joint_bundle_adjustment(0, S8, K8, None, linear_solver_type="ITERATIVE_SCHUR",
                                      max_linear_solver_iterations=a.max_cg, options=_opts(10))
        torch.cuda.synchronize()
        dt = time.perf_counter() - t0
        s = video.last_joint_summary
        res["frames8000"] = dict(S=S8, P=P8, M=M8, grid_bytes_9SP=9.0 * S8 * P8, grid_fits=video.grid_fits(S8, P8, dev),
                                 build_seconds=build_s, seconds=dt, lm_it=s.iterations, cg_it=s.cg_iterations,
                                 lm_it_per_s=s.iterations / dt, initial_cost=s.initial_cost, final_cost=s.final_cost,
                                 termination=s.termination, peak_gb=torch.cuda.max_memory_allocated() / 1e9,
                                 points_after=store.num_points)
        emit(dict(workload="frames8000", **res["frames8000"]))
    emit(dict(summary=True, **{k: v for k, v in res.items() if k != "C3"}))
    if a.out:
        os.makedirs(a.out, exist_ok=True)
        with open(os.path.join(a.out, "ba_obs_bench.json"), "w") as fh:
            json.dump(res, fh, indent=1)


if __name__ == "__main__":
    main()
