"""Sliding-window pieces of the video pipeline that sit on the geometry hot path, on device tensors.

Tensor-level mirrors of the bundle-adjustment / pose-alignment blocks of ``VideoRunner``
(vggsfm/runners/video_runner.py); the runner's dict bookkeeping (point_dict / frame_dict,
dicts_to_reconstruction, reconstruction_to_dicts) is what these calls replace, so they take and return the
dense [S,P] tensors the runner already holds at those points.  Everything numeric goes through
libvggsfm_b200.so; there is no fallback.
"""
from __future__ import annotations

import torch

from . import bundle_adjustment as ba
from . import pose_refinement as pr
from . import triangulation as tri


last_joint_summary = None       # Summary of the most recent joint_BA solve (iterations, costs), for drivers and benches


def filter_points_and_compute_masks(points, tracks, extrinsics, intrinsics, extra_params, min_valid_track_length=3,
                                    max_reproj_error=4):
    """video_runner.py:907-939.  intrinsics [1,3,3] / extra_params [1,1] are the runner's shared camera.
    Returns (filtered_points, filtered_tracks, filtered_inlier_masks, valid_tracks_mask)."""
    S = extrinsics.shape[0]
    _, inlier_mask = tri.filter_all_points3D(points, tracks, extrinsics, intrinsics.expand(S, -1, -1),
                                             extra_params=extra_params.expand(S, -1) if extra_params is not None else None,
                                             max_reproj_error=max_reproj_error, return_detail=True, hard_max=-1)
    valid = inlier_mask.sum(dim=0) >= min_valid_track_length
    return points[valid], tracks[:, valid], inlier_mask[:, valid], valid


def align_next_window(extrinsics, tracks, inlier, points3D, intrinsics, extra_params=None, camera_type="SIMPLE_PINHOLE",
                      min_vis_num=50, use_pnp=False):
    """video_runner.py:941-1017: every frame but the first is refined against the carried 3D points with the shared
    camera held constant; a frame with <= min_vis_num inliers uses all points.  ``use_pnp`` first re-estimates each of
    those frames by P3P LO-RANSAC at 12 px on its inlier points (:985-998, default estimation options: no focal
    ladder); a frame without a model keeps its incoming pose.  Returns refined_extrinsics [S,3,4] f64."""
    model = ba.camera_model_id(camera_type)
    S = extrinsics.shape[0]
    dev = extrinsics.device
    inl = inlier.bool().clone()
    few = inl.sum(dim=1) <= min_vis_num
    inl[few] = True                                                      # :973-977
    poses = extrinsics.double().contiguous().clone()
    K = intrinsics.expand(S, -1, -1)
    ex = extra_params.expand(S, -1) if extra_params is not None else None
    intr4 = pr._intr4(K, ex, model)
    flags = torch.full((S,), pr.FLAG_ACTIVE, dtype=torch.uint8, device=dev)
    flags[0] = 0
    if use_pnp:
        p_est, _, n_est, _ = pr.absolute_pose_estimation_batched(tracks, points3D, inl, intr4, model, frames=flags.bool(),
                                                                 estimate_focal_length=False, max_error=12.0)
        ok = n_est > 0
        poses[ok] = p_est[ok]
    pr.last_report = pr.pose_refinement_batched(poses, intr4, points3D, tracks, inl, flags, model, pr.default_pose_options())
    return poses


def window_bundle_adjustment(window_points_all, extrinsics, intrinsics, extra_params, window_tracks_all,
                             window_inlier_masks_all, exist_points_3D_num, shared_camera=True,
                             camera_type="SIMPLE_PINHOLE"):
    """The BA block of VideoRunner.move_window (video_runner.py:800-853) + solve_bundle_adjustment (:1321-1331):
    window_size+1 frames, frame 0 (the last frame of the previous window) fixed, the first
    ``exist_points_3D_num`` points (carried over) constant, the rest variable, intrinsics constant, default
    Ceres options, no Normalize (the runner drives pycolmap.BundleAdjuster directly, not the controller).

    Returns (window_points3D_opt [P,3], extrinsics [S,3,4], summary, ba_success) where ba_success is the
    runner's ``num_residuals_reduced > 0`` test."""
    S, P = window_inlier_masks_all.shape
    dev = window_tracks_all.device
    K = intrinsics.expand(S, -1, -1)
    ex = extra_params.expand(S, -1) if extra_params is not None else None
    const_pose = torch.zeros(S, dtype=torch.bool, device=dev)
    const_pose[0] = True                                                 # :817-818
    const_points = torch.arange(P, device=dev) < exist_points_3D_num     # :820-825
    pts, extr, _, _, valid_idx, summary = ba.bundle_adjustment(
        window_points_all, extrinsics, K, ex, window_tracks_all, window_inlier_masks_all, shared_camera=shared_camera,
        camera_type=camera_type, options=ba.default_options(), refine_focal_length=False, refine_extra_params=False,
        const_pose=const_pose, const_points=const_points, gauge=False, do_normalize=False, drop_negative_depth=False)
    out = window_points_all.double().clone()
    out[valid_idx] = pts
    # residuals that touch at least one free parameter block: observations of free frames, or of free points
    free_obs = window_inlier_masks_all.bool()[:, valid_idx]
    reduced = int(free_obs[1:].sum()) + int((free_obs[:1] & ~const_points[valid_idx][None]).sum())
    return out, extr, summary, reduced > 0


def joint_BA(points3D, extrinsics, intrinsics, extra_params, tracks, masks, camera_type="SIMPLE_PINHOLE", reproj_error=2.0,
             tri_angle=1.5, normalize=True, linear_solver_type="DENSE_SCHUR", min_linear_solver_iterations=0,
             max_linear_solver_iterations=500, eta=0.1, allreduce=None, options=None):
    """Tensor form of VideoRunner.joint_BA (video_runner.py:494-541): all frames so far, all points, ONE shared
    camera, default Ceres options through the COLMAP controller (gauge + negative-depth filter + Normalize), then the
    2 px / 1.5 degree point filter and a second normalisation.  The runner keeps this state in its point_dict /
    frame_dict; here it is the dense [S,P] form those dicts unroll to.

    points3D [P,3], extrinsics [S,3,4], intrinsics [1,3,3], extra_params [1,1]|None, tracks [S,P,2], masks [S,P].
    Returns (points3D [P,3], extrinsics [S,3,4], intrinsics [1,3,3], extra_params [1,1]|None, masks [S,P],
    valid_points [P]) -- filtered observations are cleared in `masks`, deleted points are False in `valid_points`.
    The observation filter is the reference's own filter_all_points3D rule (reprojection <= reproj_error and positive
    depth per observation, >= 2 survivors, one camera pair with >= tri_angle), which is what COLMAP's
    ObservationManager.filter_all_points3D + filter_observations_with_negative_depth compute [3P-memory].
    linear_solver_type="ITERATIVE_SCHUR" (and the CG options of bundle_adjustment.lm_solve) solves long sequences whose
    dense reduced camera system does not fit in memory.  `allreduce` (vggsfm_b200.dist.AllReduceHook) runs the BA over
    track shards with either linear solver: every rank passes all frames and its own slice of the points (normalize
    reads the cameras only, and the point filter is per point, so the rest of the call is the rank's own).  options: the
    BA's BAOptions (default: bundle_adjustment.default_options())."""
    S, P = masks.shape
    K = intrinsics.expand(S, -1, -1)
    ex = extra_params.expand(S, -1) if extra_params is not None else None
    poses, pts = extrinsics.double(), points3D.double()
    if normalize:
        poses, pts = ba.normalize(poses, pts, 5.0, 0.1, 0.9)                             # :503-504
    global last_joint_summary
    pts_o, extr, K_o, ex_o, valid_idx, summary = ba.bundle_adjustment(
        pts, poses, K, ex, tracks, masks, shared_camera=True, camera_type=camera_type,
        options=options or ba.default_options(), filter_reconstruction=False, linear_solver_type=linear_solver_type,
        min_linear_solver_iterations=min_linear_solver_iterations,
        max_linear_solver_iterations=max_linear_solver_iterations, eta=eta, allreduce=allreduce)
    last_joint_summary = summary
    out = pts.clone()
    out[valid_idx] = pts_o
    _, detail = tri.filter_all_points3D(out, tracks, extr, K_o, extra_params=ex_o, max_reproj_error=reproj_error,
                                        min_tri_angle=tri_angle, check_triangle=False, return_detail=True, hard_max=-1)
    in_problem = torch.zeros(P, dtype=torch.bool, device=masks.device)
    in_problem[valid_idx] = True
    new_masks = masks.bool() & detail & in_problem[None]
    ok_tri, _ = tri.filter_all_points3D(out, tracks, extr, K_o, extra_params=ex_o, max_reproj_error=reproj_error,
                                        min_tri_angle=tri_angle, check_triangle=True, hard_max=-1)
    valid_points = (new_masks.sum(dim=0) >= 2) & ok_tri
    new_masks = new_masks & valid_points[None]
    if normalize:
        extr, out = ba.normalize(extr, out, 5.0, 0.1, 0.9, valid_points)                 # :513-514
    return out, extr, K_o[:1].clone(), (ex_o[:1].clone() if ex_o is not None else None), new_masks, valid_points


def joint_BA_obs(points3D, extrinsics, intrinsics, extra_params, obs_uv, obs_frame, obs_point,
                 camera_type="SIMPLE_PINHOLE", reproj_error=2.0, tri_angle=1.5, normalize=True,
                 min_linear_solver_iterations=0, max_linear_solver_iterations=500, eta=0.1, allreduce=None, options=None):
    """joint_BA with ITERATIVE_SCHUR on the observations as a list -- the form VideoRunner.joint_BA hands COLMAP, each
    point carrying its track (video_runner.py:494-541) -- instead of the [S,P] grid: COO obs_uv [M,2], obs_frame [M],
    obs_point [M] into points3D [P,3].  bundle_adjustment_obs, then the point filter on the list
    (triangulation.filter_observations: reprojection <= reproj_error at positive depth per observation, >= 2 survivors,
    one surviving pair with >= tri_angle) and the second normalisation.  Returns (points3D [P,3], extrinsics [S,3,4],
    intrinsics [1,3,3], extra_params [1,1]|None, keep [M] bool, valid_points [P]) -- keep is the list form of
    joint_BA's masks.  options: the BA's BAOptions (default: bundle_adjustment.default_options())."""
    S, P = extrinsics.shape[0], points3D.shape[0]
    K = intrinsics.expand(S, -1, -1)
    ex = extra_params.expand(S, -1) if extra_params is not None else None
    poses, pts = extrinsics.double(), points3D.double()
    if normalize:
        poses, pts = ba.normalize(poses, pts, 5.0, 0.1, 0.9)                             # :503-504
    global last_joint_summary
    pts_o, extr, K_o, ex_o, valid_idx, summary = ba.bundle_adjustment_obs(
        pts, poses, K, ex, obs_uv, obs_frame, obs_point, shared_camera=True, camera_type=camera_type,
        options=options or ba.default_options(), filter_reconstruction=False,
        min_linear_solver_iterations=min_linear_solver_iterations,
        max_linear_solver_iterations=max_linear_solver_iterations, eta=eta, allreduce=allreduce)
    last_joint_summary = summary
    out = pts.clone()
    out[valid_idx] = pts_o
    keep, ok_tri = tri.filter_observations(out, obs_uv, obs_frame, obs_point, extr, K_o, extra_params=ex_o,
                                           max_reproj_error=reproj_error, min_tri_angle=tri_angle)
    in_problem = torch.zeros(P, dtype=torch.bool, device=out.device)
    in_problem[valid_idx] = True
    op = obs_point.to(out.device, torch.int64)
    keep = keep & in_problem[op]
    valid_points = (torch.bincount(op[keep], minlength=P) >= 2) & ok_tri
    keep = keep & valid_points[op]
    if normalize:
        extr, out = ba.normalize(extr, out, 5.0, 0.1, 0.9, valid_points)                 # :513-514
    return out, extr, K_o[:1].clone(), (ex_o[:1].clone() if ex_o is not None else None), keep, valid_points


# The grid path's peak device memory in SceneStore.joint_bundle_adjustment, as a multiple of the 9 S P bytes of its
# [S,P] grid (uv 8 B + mask 1 B per cell): 3.01 measured on an H100 80GB HBM3 (700 W) by tools/ba_obs_bench.py on the
# 2500-frame joint BA (tools/video_c5.py final_problem_arrays(2500, 2048): the grid's 7.2 GB plus 14.5 GB the call
# allocates beside it), rounded up; see DESIGN 4.10.
GRID_PEAK_MULTIPLE = 3.1


def grid_fits(S, P, device) -> bool:
    """whether the grid path of a joint BA over S frames and P points fits on `device`: GRID_PEAK_MULTIPLE x 9 S P
    bytes within the device's total memory"""
    return GRID_PEAK_MULTIPLE * 9.0 * S * P <= torch.cuda.get_device_properties(device).total_memory


class SceneStore:
    """GPU-resident scene tables of the sliding-window pipeline -- what ``VideoRunner`` keeps in ``point_dict`` /
    ``frame_dict`` (vggsfm/runners/video_runner.py:354-492, :543-638) and walks with O(points x frames) Python loops
    before and after every bundle adjustment.

    Points: ``xyz [P,3] float32`` (the runner stores ``.float()``, :620), ``rgb [P,3]``; point ids are row numbers, new
    points are appended (``exist_max_point + index``, :395-399).  Observations: coordinate list ``(obs_point, obs_frame,
    obs_uv, obs_vis)``.  Frames: ``extri [F,3,4] float64``.  ``dense(start, end)`` unrolls the tables into the [S,P]
    grid the BA kernels take (the tensor form of ``dicts_to_reconstruction``, :543-604); ``replace_from_ba`` is
    ``reconstruction_to_dicts`` (:606-638: surviving points renumbered 0..P'-1 in id order, visibilities reset to 1)."""

    def __init__(self, device):
        self.device = device
        self.xyz = torch.zeros(0, 3, dtype=torch.float32, device=device)
        self.rgb = torch.zeros(0, 3, dtype=torch.float32, device=device)
        self.obs_point = torch.zeros(0, dtype=torch.int64, device=device)
        self.obs_frame = torch.zeros(0, dtype=torch.int64, device=device)
        self.obs_uv = torch.zeros(0, 2, dtype=torch.float32, device=device)
        self.obs_vis = torch.zeros(0, dtype=torch.float32, device=device)
        self.extri = torch.zeros(0, 3, 4, dtype=torch.float64, device=device)
        self.has_extri = torch.zeros(0, dtype=torch.bool, device=device)

    @property
    def num_points(self):
        return int(self.xyz.shape[0])

    def set_extrinsics(self, start_idx, extrinsics):
        end = start_idx + extrinsics.shape[0]
        if end > self.extri.shape[0]:
            grow = end - self.extri.shape[0]
            self.extri = torch.cat([self.extri, torch.zeros(grow, 3, 4, dtype=torch.float64, device=self.device)])
            self.has_extri = torch.cat([self.has_extri, torch.zeros(grow, dtype=torch.bool, device=self.device)])
        self.extri[start_idx:end] = extrinsics.to(torch.float64)
        self.has_extri[start_idx:end] = True

    def _append_obs(self, point_ids, tracks, vis, valid, start_idx):
        """tracks [S,P,2], vis/valid [S,P] for the points `point_ids` [P] in frames start_idx.."""
        s_idx, p_idx = torch.nonzero(valid, as_tuple=True)
        self.obs_point = torch.cat([self.obs_point, point_ids[p_idx]])
        self.obs_frame = torch.cat([self.obs_frame, s_idx + start_idx])
        self.obs_uv = torch.cat([self.obs_uv, tracks[s_idx, p_idx].float()])
        self.obs_vis = torch.cat([self.obs_vis, vis[s_idx, p_idx].float()])

    def add_points(self, points3D, points3D_rgb, tracks, vis, valid_2D_mask, start_idx):
        """New points of a window (convert_pred_to_point_frame_dict + _update_points_to_dict, :354-470, for points not
        yet in the store): appended, ids returned."""
        P = points3D.shape[0]
        ids = torch.arange(self.num_points, self.num_points + P, device=self.device)
        self.xyz = torch.cat([self.xyz, points3D.float()])
        rgb = points3D_rgb.float() if points3D_rgb is not None else torch.full((P, 3), float("nan"), device=self.device)
        self.rgb = torch.cat([self.rgb, rgb])
        self._append_obs(ids, tracks, vis, valid_2D_mask.bool(), start_idx)
        return ids

    def extend_tracks(self, point_ids, tracks, vis, valid_2D_mask, start_idx):
        """Observations of EXISTING points in new frames (_update_points_to_dict with ids already in the dict)."""
        self._append_obs(point_ids, tracks, vis, valid_2D_mask.bool(), start_idx)

    def visible_points(self, frame_idx):
        """frame_dict[frame]["visible_points"], ascending ids."""
        return torch.sort(self.obs_point[self.obs_frame == frame_idx]).values

    def dense(self, start_idx, end_idx):
        """All points x frames [start, end): (xyz [P,3] f64, tracks [S,P,2] f32, masks [S,P] bool, extrinsics [S,3,4])."""
        S, P = end_idx - start_idx, self.num_points
        tracks = torch.zeros(S, P, 2, dtype=torch.float32, device=self.device)
        masks = torch.zeros(S, P, dtype=torch.bool, device=self.device)
        sel = (self.obs_frame >= start_idx) & (self.obs_frame < end_idx)
        f, p = self.obs_frame[sel] - start_idx, self.obs_point[sel]
        tracks[f, p] = self.obs_uv[sel]
        masks[f, p] = True
        return self.xyz.double(), tracks, masks, self.extri[start_idx:end_idx].clone()

    def replace_from_ba(self, start_idx, points3D, extrinsics, tracks, masks, keep):
        """reconstruction_to_dicts after a normalising joint BA (:532-536, :606-638): the store is rebuilt from the BA's
        result -- points `keep` [P] bool survive and are renumbered in id order, their observations are the surviving
        `masks` [S,P] of frames start_idx.., visibilities become 1, xyz is stored as float32."""
        new_id = torch.cumsum(keep.long(), 0) - 1
        self.xyz = points3D[keep].float()
        self.rgb = self.rgb[keep]
        m = masks & keep[None]
        s_idx, p_idx = torch.nonzero(m, as_tuple=True)
        self.obs_point = new_id[p_idx]
        self.obs_frame = s_idx + start_idx
        self.obs_uv = tracks[s_idx, p_idx].float()
        self.obs_vis = torch.ones(s_idx.numel(), dtype=torch.float32, device=self.device)
        self.has_extri[:] = False
        self.set_extrinsics(start_idx, extrinsics)

    def observations(self, start_idx, end_idx):
        """The observations of frames [start, end) as a list: (xyz [P,3] f64, obs_uv [M,2] f32, obs_frame [M] (relative
        to start), obs_point [M], extrinsics [S,3,4])."""
        sel = (self.obs_frame >= start_idx) & (self.obs_frame < end_idx)
        return (self.xyz.double(), self.obs_uv[sel], self.obs_frame[sel] - start_idx, self.obs_point[sel],
                self.extri[start_idx:end_idx].clone())

    def replace_from_obs(self, start_idx, points3D, extrinsics, obs_uv, obs_frame, obs_point, keep_obs, keep):
        """replace_from_ba on the list form of the BA's result: points `keep` [P] survive and are renumbered in id
        order, their observations are the list entries `keep_obs` [M] (obs_frame relative to start_idx), stored in the
        (frame, point) order replace_from_ba gives them; visibilities become 1, xyz is stored as float32."""
        new_id = torch.cumsum(keep.long(), 0) - 1
        self.xyz = points3D[keep].float()
        self.rgb = self.rgb[keep]
        op = obs_point.to(torch.int64)
        sel = keep_obs & keep[op]
        f, p, uv = obs_frame[sel].to(torch.int64), new_id[op[sel]], obs_uv[sel]
        order = torch.sort(f * max(1, self.num_points) + p).indices
        self.obs_point = p[order]
        self.obs_frame = f[order] + start_idx
        self.obs_uv = uv[order].float()
        self.obs_vis = torch.ones(order.numel(), dtype=torch.float32, device=self.device)
        self.has_extri[:] = False
        self.set_extrinsics(start_idx, extrinsics)

    def joint_bundle_adjustment(self, start_idx, end_idx, intrinsics, extra_params, camera_type="SIMPLE_PINHOLE",
                                reproj_error=2.0, tri_angle=1.5, normalize=True, linear_solver_type="DENSE_SCHUR",
                                min_linear_solver_iterations=0, max_linear_solver_iterations=500, eta=0.1,
                                options=None):
        """VideoRunner.joint_BA (:494-541) on the store: dense view -> joint_BA (CUDA) -> store rebuilt from the result.
        Returns the refined shared (intrinsics [1,3,3], extra_params [1,1]|None).  Linear-solver options as joint_BA.
        With ITERATIVE_SCHUR a problem whose grid does not fit on the device (grid_fits) takes the observation list
        instead (joint_BA_obs, replace_from_obs); every problem that fits runs the grid path.  options: the BA's
        BAOptions (default: bundle_adjustment.default_options())."""
        S, P = end_idx - start_idx, self.num_points
        if linear_solver_type == "ITERATIVE_SCHUR" and not grid_fits(S, P, self.device):
            xyz, uv, fr, pt, extr = self.observations(start_idx, end_idx)
            pts, extr, K, ex, keep_obs, valid = joint_BA_obs(
                xyz, extr, intrinsics, extra_params, uv, fr, pt, camera_type=camera_type, reproj_error=reproj_error,
                tri_angle=tri_angle, normalize=normalize, min_linear_solver_iterations=min_linear_solver_iterations,
                max_linear_solver_iterations=max_linear_solver_iterations, eta=eta, options=options)
            self.replace_from_obs(start_idx, pts, extr, uv, fr, pt, keep_obs, valid)
            return K.float(), (ex.float() if ex is not None else None)
        xyz, tracks, masks, extr = self.dense(start_idx, end_idx)
        pts, extr, K, ex, new_masks, valid = joint_BA(xyz, extr, intrinsics, extra_params, tracks, masks, camera_type=camera_type,
                                                      reproj_error=reproj_error, tri_angle=tri_angle, normalize=normalize,
                                                      linear_solver_type=linear_solver_type,
                                                      min_linear_solver_iterations=min_linear_solver_iterations,
                                                      max_linear_solver_iterations=max_linear_solver_iterations, eta=eta,
                                                      options=options)
        self.replace_from_ba(start_idx, pts, extr, tracks, new_masks, valid)
        return K.float(), (ex.float() if ex is not None else None)


def triangulate_window_points(extrinsics, intrinsics, extra_params, tracks, vis, score, max_reproj_error=4.0, min_inlier_num=3):
    """VideoRunner.triangulate_window_points (video_runner.py:1189-1262) on tensors: LORANSAC triangulation of the
    window's new tracks with the window's (already aligned) cameras, keep tracks with more than ``min_inlier_num`` inliers
    (:1241 ``inlier_num > 3``-style test is the caller's), then the reprojection / cheirality filter.
    extrinsics [S,3,4], intrinsics [1,3,3] shared, tracks [S,N,2].  Returns (points3D [N,3], inlier_mask [S,N], valid [N])."""
    S = extrinsics.shape[0]
    K = intrinsics.expand(S, -1, -1)
    ex = extra_params.expand(S, -1) if extra_params is not None else None
    tn = tri.cam_from_img(tracks, K, ex)
    pts, num, mask = tri.triangulate_tracks(extrinsics, tn, track_vis=vis, track_score=score)
    valid = num > min_inlier_num
    ok, detail = tri.filter_all_points3D(pts, tracks, extrinsics, K, extra_params=ex, max_reproj_error=max_reproj_error,
                                        return_detail=True, hard_max=-1)
    valid = valid & ok
    return pts, detail & valid[None], valid
