"""Timing of the dense depth stage (align_dense_depth_maps and the sparse extraction) on one GPU.

Workload: F frames of H x W with ~4096 sparse samples each, at two inlier ratios, without and with
visual_dense_point_cloud (the visual run uses fewer frames: its host output is ~48 bytes per valid pixel).  Prints one
JSON line per configuration with the whole-call time, the per-kernel CUDA time from torch.profiler, the apply kernel's
bytes per pixel and share of 3.35 TB/s, the host<->device copy time, the oracle's time per frame on the host cores, and
the card's name and power limit read in the same run.
"""
import argparse
import json
import os
import re
import subprocess
import sys
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from vggsfm_b200 import dense_depth  # noqa: E402
from vggsfm_b200.reconstruction import Camera, Image, Reconstruction, Rigid3d, Rotation3d  # noqa: E402


def scene(F, H, W, n, ratio, seed=0):
    rng = np.random.default_rng(seed)
    rec = Reconstruction()
    sparse, disp, rgb = {}, {}, {}
    yy, xx = np.mgrid[0:H, 0:W]
    base = 2.0 + 1.5 * np.sin(xx / W * 3) + yy / H
    for f in range(F):
        nm = f"frame_{f:04d}.png"
        rec.add_camera(Camera("SIMPLE_PINHOLE", W, H, np.array([1.2 * W, W / 2, H / 2]), f))
        rec.add_image(Image(id=f, name=nm, camera_id=f, cam_from_world=Rigid3d(Rotation3d(), rng.normal(0, 1, 3))))
        a, b = rng.uniform(0.5, 2), rng.uniform(-0.05, 0.05)
        disp[nm] = (a / base + b).astype(np.float32)
        u, v = rng.uniform(0, W - 1, n), rng.uniform(0, H - 1, n)
        d = base[np.round(v).astype(int), np.round(u).astype(int)] * (1 + rng.normal(0, 1e-3, n))
        out = rng.uniform(size=n) > ratio
        d[out] = rng.uniform(0.5, 6, out.sum())
        sparse[nm] = np.column_stack([u, v, d])
        rgb[nm] = np.zeros((H, W, 3), dtype=np.uint8)
    return rec, sparse, disp, rgb


def gpu_info():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                           capture_output=True, text=True, timeout=30).stdout.strip()
    except Exception as e:  # noqa: BLE001
        q = f"nvidia-smi unavailable: {e}"
    return q or torch.cuda.get_device_name(0)


def run(F, H, W, n, ratio, visual, oracle_frames):
    rec, sparse, disp, rgb = scene(F, H, W, n, ratio)
    seeds = np.arange(F)
    fresh = {k: v.copy() for k, v in disp.items()}
    dense_depth.align_dense_depth_maps(rec, {k: sparse[k] for k in list(sparse)[:2]},
                                       {k: fresh[k] for k in list(sparse)[:2]}, rgb, visual, seeds=seeds[:2])
    torch.cuda.synchronize()
    fresh = {k: v.copy() for k, v in disp.items()}
    t0 = time.perf_counter()
    out = dense_depth.align_dense_depth_maps(rec, sparse, fresh, rgb, visual, seeds=seeds, return_debug=True)
    torch.cuda.synchronize()
    total = time.perf_counter() - t0
    dbg = out[2]
    fresh = {k: v.copy() for k, v in disp.items()}
    acts = [torch.profiler.ProfilerActivity.CPU, torch.profiler.ProfilerActivity.CUDA]
    with torch.profiler.profile(activities=acts, acc_events=True) as prof:
        dense_depth.align_dense_depth_maps(rec, sparse, fresh, rgb, visual, seeds=seeds)
        torch.cuda.synchronize()
    kern, copies = {}, {"HtoD": 0.0, "DtoH": 0.0}
    for e in prof.events():
        if e.device_type == torch.autograd.DeviceType.CUDA:
            name = e.name
            us = e.device_time if hasattr(e, "device_time") else e.cuda_time
            if "Memcpy HtoD" in name:
                copies["HtoD"] += us
            elif "Memcpy DtoH" in name:
                copies["DtoH"] += us
            else:
                m = re.search(r"(dd_\w+_kernel)", name)
                if m:
                    kern[m.group(1)] = kern.get(m.group(1), 0.0) + us
    npix = F * H * W
    apply_ms = kern.get("dd_apply_kernel", float("nan")) / 1e3
    bpp = 4 + 4 + 4                     # read disparity, write disparity and depth
    # sparse extraction on a Reconstruction of the same size (every frame observes n points)
    P = n
    ext = np.zeros((F, 3, 4)); ext[:, :, :3] = np.eye(3); ext[:, 2, 3] = 5.0
    K = np.tile(np.array([[1.2 * W, 0, W / 2], [0, 1.2 * W, H / 2], [0, 0, 1]]), (F, 1, 1))
    pts = np.random.default_rng(1).normal(0, 1, (P, 3))
    r2 = Reconstruction.from_batch_matrix(pts, ext, K, np.zeros((F, P, 2)), np.ones((F, P), bool), np.array([W, H]))
    t1 = time.perf_counter()
    dense_depth.extract_sparse_depth_and_point_from_reconstruction(None, {"reconstruction": r2})
    extract_s = time.perf_counter() - t1
    from oracle import dense_depth_oracle as O
    t2 = time.perf_counter()
    names = list(sparse)[:oracle_frames]
    for f, nm in enumerate(names):
        O.align_frame(disp[nm], sparse[nm], int(seeds[f]))
    oracle_s = (time.perf_counter() - t2) / max(1, len(names))
    return dict(frames=F, H=H, W=W, samples=n, inlier_ratio=ratio, visual=visual, call_s=round(total, 4),
                n_trials_mean=float(np.mean(dbg["n_trials"])), n_trials_max=int(np.max(dbg["n_trials"])),
                kernel_ms={k: round(v / 1e3, 3) for k, v in kern.items()},
                copy_ms={k: round(v / 1e3, 3) for k, v in copies.items()},
                apply_bytes_per_pixel=bpp, apply_share_of_3p35TBps=round(npix * bpp / (apply_ms * 1e-3) / 3.35e12, 3),
                sparse_extraction_s=round(extract_s, 4), oracle_s_per_frame=round(oracle_s, 4),
                oracle_cores=os.cpu_count(), gpu=gpu_info())


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--frames", type=int, default=400)
    ap.add_argument("--visual-frames", type=int, default=40)
    ap.add_argument("--height", type=int, default=1080)
    ap.add_argument("--width", type=int, default=1920)
    ap.add_argument("--samples", type=int, default=4096)
    ap.add_argument("--oracle-frames", type=int, default=2)
    a = ap.parse_args()
    assert torch.cuda.is_available(), "the dense depth bench needs a GPU"
    for ratio in (0.8, 0.3):
        for visual in (False, True):
            F = a.visual_frames if visual else a.frames
            print(json.dumps(run(F, a.height, a.width, a.samples, ratio, visual, a.oracle_frames)), flush=True)


if __name__ == "__main__":
    main()
