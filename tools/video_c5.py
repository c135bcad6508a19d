"""C5 (BASELINE.json configs[4]): the sequential video pipeline's geometry path on a synthetic 1000-frame sequence.

Control flow of VideoRunner (vggsfm/runners/video_runner.py) with the learned stages replaced by synthetic inputs: an
init window of 32 frames (global BA), then windows of 16 frames -- pose alignment of the new frames against the carried
points (`align_next_window`), LORANSAC triangulation of the window's new tracks (`triangulate_window_points`), window
BA with the anchor frame and the carried points fixed (`window_bundle_adjustment`), the scene tables (`SceneStore`) --
and a joint BA over everything so far after every 6th window (`joint_BA`).  The BA runs on the DENSE [frames, points]
grid (a point lives for 3 windows, so ~95 % of the grid is masked out at 1000 frames): this measures what the current
kernels do on that shape, not a band-aware solver (DESIGN section 8).

    python tools/video_c5.py [--frames 1000] [--new 512] [--json out.json]
prints one JSON line: frames/s of the whole sequence, the time split, the final joint-BA problem and its LM it/s.
"""
import argparse
import json
import os
import sys
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from vggsfm_b200 import bundle_adjustment as ba            # noqa: E402
from vggsfm_b200 import video                              # noqa: E402
from vggsfm_b200.synthetic import make_video_scene, _exp_so3   # noqa: E402


def run(frames=1000, new_per_window=512, joint_every=6, seed=0, dev=None, verbose=False):
    dev = dev or torch.device("cuda:0")
    sc = make_video_scene(F=frames, new_per_window=new_per_window, seed=seed)
    rng = np.random.default_rng(seed + 1)
    T = lambda a, dt=None: (torch.from_numpy(np.ascontiguousarray(a)).to(dt) if dt else torch.from_numpy(np.ascontiguousarray(a))).to(dev)
    K = torch.tensor([[[sc.focal, 0.0, sc.pp[0]], [0.0, sc.focal, sc.pp[1]], [0.0, 0.0, 1.0]]], dtype=torch.float64, device=dev)
    ex = None
    cam = "SIMPLE_PINHOLE"
    store = video.SceneStore(dev)
    scene_id = np.zeros(0, dtype=np.int64)          # scene point of every store row
    split = {"align": 0.0, "triangulate": 0.0, "window_ba": 0.0, "joint_ba": 0.0, "tables": 0.0}
    stats = {"windows": 0, "joint_bas": 0, "joint_iterations": 0, "window_iterations": 0}

    def tick():
        torch.cuda.synchronize()
        return time.perf_counter()

    def noisy(extr, rot_deg, trans):
        w = rng.normal(size=(extr.shape[0], 3))
        w = w / np.linalg.norm(w, axis=1, keepdims=True) * np.deg2rad(rot_deg)
        out = extr.copy()
        out[:, :, :3] = _exp_so3(w) @ out[:, :, :3]
        out[:, :, 3] += rng.normal(size=(extr.shape[0], 3)) * trans
        return out

    t_start = tick()
    # ---- init window: noisy cameras, triangulation of its tracks, global BA (gauge fixed by the controller rules)
    s0, e0 = sc.window_range(0)
    ids0 = np.nonzero(sc.birth == 0)[0]
    uv, ok = sc.observe(ids0, s0, e0)
    extr0 = T(noisy(sc.extrinsics[s0:e0], 0.3, 0.01))
    t0 = tick()
    pts, inl, valid = video.triangulate_window_points(extr0, K, ex, T(uv), T(ok.astype(np.float32)), torch.ones(uv.shape[:2], device=dev))
    split["triangulate"] += tick() - t0
    t0 = tick()
    pts_o, extr_o, K_o, _, vidx, summ = ba.bundle_adjustment(pts[valid], extr0, K.expand(e0 - s0, -1, -1), None, T(uv)[:, valid], inl[:, valid],
                                                             shared_camera=True, camera_type=cam, refine_focal_length=False,
                                                             refine_extra_params=False)
    split["window_ba"] += tick() - t0
    stats["window_iterations"] += int(summ.iterations)
    t0 = tick()
    keep = torch.nonzero(valid).flatten()[vidx]
    store.set_extrinsics(0, extr_o)
    store.add_points(pts_o, None, T(uv)[:, keep], T(ok.astype(np.float32))[:, keep], inl[:, keep], 0)
    scene_id = ids0[keep.cpu().numpy()]
    split["tables"] += tick() - t0

    final_problem = None
    for w in range(1, sc.num_windows()):
        s, e = sc.window_range(w)
        a = s - 1                                            # anchor = last frame of the previous window
        S = e - a
        # cameras of the new frames as a camera predictor would hand them over: previous pose composed with the true
        # relative motion, plus noise
        anchor = store.extri[a].cpu().numpy()
        rel_R = sc.extrinsics[a:e, :, :3] @ sc.extrinsics[a, :, :3].T
        rel_t = sc.extrinsics[a:e, :, 3] - np.einsum("sij,j->si", rel_R, sc.extrinsics[a, :, 3])
        # the store's gauge drifts from the ground truth's by a similarity (the joint BA normalises the scene): scale the
        # predicted relative translation by the ratio of the last window's baseline in both gauges
        b = max(0, a - sc.window)
        prev = store.extri[b].cpu().numpy()
        c_s = lambda p: -p[:, :3].T @ p[:, 3]
        base_gt = np.linalg.norm(c_s(sc.extrinsics[a]) - c_s(sc.extrinsics[b]))
        gauge_scale = np.linalg.norm(c_s(anchor) - c_s(prev)) / max(base_gt, 1e-12)
        init = np.concatenate([rel_R @ anchor[:, :3], (np.einsum("sij,j->si", rel_R, anchor[:, 3]) + gauge_scale * rel_t)[:, :, None]], axis=2)
        init[1:] = noisy(init[1:], 0.3, 0.01)
        extr_w = T(init)
        # carried points that are still alive in this window
        alive = np.nonzero(sc.last_frame[scene_id] > s)[0]
        uv_c, ok_c = sc.observe(scene_id[alive], a, e)
        P_c = alive.size
        xyz_c = store.xyz[T(alive)].double()
        t0 = tick()
        if P_c:
            extr_w = video.align_next_window(extr_w, T(uv_c), T(ok_c), xyz_c, K, ex, camera_type=cam)
        split["align"] += tick() - t0
        # new tracks of this window
        ids_n = np.nonzero(sc.birth == w)[0]
        uv_n, ok_n = sc.observe(ids_n, a, e)
        t0 = tick()
        pts_n, inl_n, valid_n = video.triangulate_window_points(extr_w, K, ex, T(uv_n), T(ok_n.astype(np.float32)),
                                                                torch.ones(uv_n.shape[:2], device=dev))
        split["triangulate"] += tick() - t0
        vn = valid_n.cpu().numpy()
        # window BA: carried points first (constant), then the new ones
        pts_all = torch.cat([xyz_c, pts_n[valid_n]])
        tr_all = torch.cat([T(uv_c), T(uv_n)[:, valid_n]], dim=1)
        m_all = torch.cat([T(ok_c), inl_n[:, valid_n]], dim=1)
        t0 = tick()
        pts_w, extr_b, summ, okba = video.window_bundle_adjustment(pts_all, extr_w, K, ex, tr_all, m_all, P_c, camera_type=cam)
        split["window_ba"] += tick() - t0
        stats["window_iterations"] += int(summ.iterations)
        t0 = tick()
        store.set_extrinsics(a, extr_b)
        if P_c:
            store.extend_tracks(T(alive), T(uv_c)[1:], T(ok_c.astype(np.float32))[1:], T(ok_c)[1:], s)
        if vn.any():
            store.add_points(pts_w[P_c:], None, T(uv_n)[:, valid_n], T(ok_n.astype(np.float32))[:, valid_n], inl_n[:, valid_n], a)
            scene_id = np.concatenate([scene_id, ids_n[vn]])
        split["tables"] += tick() - t0
        stats["windows"] += 1
        if w % joint_every == 0 or w == sc.num_windows() - 1:
            t0 = tick()
            xyz, tracks, masks, extr = store.dense(0, e)
            split["tables"] += tick() - t0
            t0 = tick()
            pts_j, extr_j, K_j, ex_j, new_masks, valid_p = video.joint_BA(xyz, extr, K, ex, tracks, masks, camera_type=cam)
            dt = tick() - t0
            split["joint_ba"] += dt
            it = int(video.last_joint_summary.iterations) if video.last_joint_summary is not None else -1
            stats["joint_bas"] += 1
            stats["joint_iterations"] += max(it, 0)
            final_problem = {"frames": int(e), "points": int(xyz.shape[0]), "observations": int(masks.sum()),
                             "grid_fill": float(masks.float().mean()), "seconds": dt, "lm_iterations": it,
                             "lm_it_per_s": (it / dt if it > 0 else None), "kept_points": int(valid_p.sum())}
            t0 = tick()
            store.replace_from_ba(0, pts_j, extr_j, tracks, new_masks, valid_p)
            scene_id = scene_id[valid_p.cpu().numpy()]
            K = K_j[:1].double()
            split["tables"] += tick() - t0
            if verbose:
                print(f"[c5] window {w}: joint BA over {e} frames x {xyz.shape[0]} points: {dt * 1e3:.0f} ms, {it} iterations", file=sys.stderr)
    total = tick() - t_start
    # accuracy against the ground truth after a similarity alignment of the camera centres
    est = store.extri[:frames].cpu().numpy()
    Ce = -np.einsum("fji,fj->fi", est[:, :, :3], est[:, :, 3])
    Cg = -np.einsum("fji,fj->fi", sc.extrinsics[:, :, :3], sc.extrinsics[:, :, 3])
    mu_e, mu_g = Ce.mean(0), Cg.mean(0)
    U, sv, Vt = np.linalg.svd((Cg - mu_g).T @ (Ce - mu_e))
    D = np.diag([1, 1, np.sign(np.linalg.det(U @ Vt))])
    Rm = U @ D @ Vt
    sc_ = np.trace(np.diag(sv) @ D) / ((Ce - mu_e) ** 2).sum()
    err = np.linalg.norm((sc_ * (Rm @ (Ce - mu_e).T).T + mu_g) - Cg, axis=1)
    return {"workload": f"C5: {frames} frames, window 16 / init 32, {new_per_window} new tracks per window (lifetime 3 windows), "
                        f"joint BA every {joint_every} windows, SIMPLE_PINHOLE shared camera, dense [frames, points] grid",
            "frames": frames, "seconds": total, "frames_per_s": frames / total, "split_seconds": split, **stats,
            "final_joint_ba": final_problem, "camera_centre_rmse_vs_gt": float(np.sqrt((err ** 2).mean())),
            "trajectory_length": float(np.linalg.norm(Cg[-1] - Cg[0])), "store_points": store.num_points}


def final_problem_arrays(frames=1000, new_per_window=512, seed=0, dev=None):
    """The last joint BA of the sequence as device tensors (tracks [S,P,2] float32, masks [S,P] bool, points [P,3],
    extrinsics [S,3,4], K [1,3,3]), ground truth + noise, points seen in >= 3 frames.  The [S,P] grid is filled on the
    device window by window, so the host never holds it (a 2500-frame sequence at 2048 new points per window is 6 GB)."""
    dev = dev or torch.device("cuda:0")
    sc = make_video_scene(F=frames, new_per_window=new_per_window, seed=seed)
    rng = np.random.default_rng(seed + 2)
    P = sc.points3d.shape[0]
    uv = torch.zeros(frames, P, 2, dtype=torch.float32, device=dev)
    ok = torch.zeros(frames, P, dtype=torch.bool, device=dev)
    for w in range(sc.num_windows()):
        ids = np.nonzero(sc.birth == w)[0]
        f0, f1 = int(sc.first_frame[ids[0]]), int(sc.last_frame[ids[0]])
        u, o = sc.observe(ids, f0, f1)
        it = torch.from_numpy(ids).to(dev)
        uv[f0:f1, it] = torch.from_numpy(np.ascontiguousarray(u, dtype=np.float32)).to(dev)
        ok[f0:f1, it] = torch.from_numpy(np.ascontiguousarray(o)).to(dev)
    keep = (ok.sum(0) >= 3).cpu().numpy()
    w = rng.normal(size=(frames, 3))
    w = w / np.linalg.norm(w, axis=1, keepdims=True) * np.deg2rad(0.2)
    extr = sc.extrinsics.copy()
    extr[:, :, :3] = _exp_so3(w) @ extr[:, :, :3]
    extr[:, :, 3] += rng.normal(size=(frames, 3)) * 0.005
    pts = sc.points3d[keep] + rng.normal(size=(int(keep.sum()), 3)) * 0.01
    K = torch.tensor([[[sc.focal, 0.0, sc.pp[0]], [0.0, sc.focal, sc.pp[1]], [0.0, 0.0, 1.0]]], dtype=torch.float64, device=dev)
    kt = torch.from_numpy(keep).to(dev)
    tracks, masks = uv[:, kt].contiguous(), ok[:, kt].contiguous()
    del uv, ok
    T = lambda a: torch.from_numpy(np.ascontiguousarray(a)).to(dev)
    return tracks, masks, T(pts), T(extr), K


def final_problem(frames=1000, new_per_window=512, seed=0, dev=None, reps=1, shuffle=False):
    """Only the LAST joint BA of the sequence, built directly from the synthetic scene (ground truth + noise instead of
    the sequential estimates): the problem the launch lists and the multi-GPU leg look at."""
    dev = dev or torch.device("cuda:0")
    sc = make_video_scene(F=frames, new_per_window=new_per_window, seed=seed)
    rng = np.random.default_rng(seed + 2)
    T = lambda a: torch.from_numpy(np.ascontiguousarray(a)).to(dev)
    P = sc.points3d.shape[0]
    uv = np.zeros((frames, P, 2), np.float32)
    ok = np.zeros((frames, P), bool)
    for w in range(sc.num_windows()):                       # window by window: observe() works on [frames, points] blocks
        ids = np.nonzero(sc.birth == w)[0]
        f0, f1 = int(sc.first_frame[ids[0]]), int(sc.last_frame[ids[0]])
        u, o = sc.observe(ids, f0, f1)
        uv[f0:f1, ids] = u
        ok[f0:f1, ids] = o
    keep = ok.sum(0) >= 3
    w = rng.normal(size=(frames, 3))
    w = w / np.linalg.norm(w, axis=1, keepdims=True) * np.deg2rad(0.2)
    extr = sc.extrinsics.copy()
    extr[:, :, :3] = _exp_so3(w) @ extr[:, :, :3]
    extr[:, :, 3] += rng.normal(size=(frames, 3)) * 0.005
    pts = sc.points3d[keep] + rng.normal(size=(int(keep.sum()), 3)) * 0.01
    K = torch.tensor([[[sc.focal, 0.0, sc.pp[0]], [0.0, sc.focal, sc.pp[1]], [0.0, 0.0, 1.0]]], dtype=torch.float64, device=dev)
    uvk, okk = uv[:, keep], ok[:, keep]
    if shuffle:                                              # points in random order: the band detection finds nothing to skip
        perm = rng.permutation(pts.shape[0])
        uvk, okk, pts = uvk[:, perm], okk[:, perm], pts[perm]
    tracks, masks = T(uvk), T(okk)
    xyz, ex0 = T(pts), T(extr)
    times, its = [], []
    for _ in range(reps):
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        video.joint_BA(xyz, ex0, K, None, tracks, masks, camera_type="SIMPLE_PINHOLE")
        torch.cuda.synchronize()
        times.append(time.perf_counter() - t0)
        its.append(int(video.last_joint_summary.iterations))
    return {"workload": f"C5 final joint BA: {frames} frames x {int(keep.sum())} points, dense grid fill {float(ok[:, keep].mean()):.3f}",
            "seconds": times, "lm_iterations": its, "lm_it_per_s": [i / t for i, t in zip(its, times)]}


if __name__ == "__main__":
    ap = argparse.ArgumentParser()
    ap.add_argument("--frames", type=int, default=1000)
    ap.add_argument("--new", type=int, default=512)
    ap.add_argument("--json", default=None)
    ap.add_argument("-v", action="store_true")
    ap.add_argument("--final-only", type=int, default=0, help="time only the last joint BA, this many repetitions")
    a = ap.parse_args()
    out = final_problem(a.frames, a.new, reps=a.final_only) if a.final_only else run(a.frames, a.new, verbose=a.v)
    line = json.dumps(out)
    print(line)
    if a.json:
        open(a.json, "w").write(line + "\n")
