"""``Triangulator`` -- the reference's triangulation + bundle-adjustment stage on the CUDA kernels.

Drop-in for ``vggsfm.models.triangulator.Triangulator`` (hydra ``cfg.MODEL.TRIANGULAE._target_``,
cfgs/demo.yaml:105-106): same ``forward`` arguments and the same 9-tuple back
(vggsfm/models/triangulator.py:44-61, :353-363).  Every stage runs through libvggsfm_b200.so:

  get_EFP -> cam_from_img -> triangulate_by_pair -> find_best_initial_pair -> init_BA -> init_refine_pose
  -> triangulate_tracks_and_BA -> robust_refine x (refine_pose -> triangulate_tracks_and_BA)
  -> BA_iters x iterative_global_BA -> validity masks (-> colours)

The returned ``reconstruction`` is the pycolmap-shaped object of vggsfm_b200/reconstruction.py (same ``.images /
.cameras / .points3D / .add_point3D / .deregister_image / .write`` surface the runner touches, runner.py:555-631),
not a ``pycolmap.Reconstruction`` (pycolmap is not a dependency of this path).

``get_EFP``, ``find_best_initial_pair`` and ``create_intri_matrix`` below are close transcriptions of the reference's
dozen tensor statements each (models/utils.py:38-72, models/triangulator.py:442-476): host glue whose semantics must
match statement for statement; they are pinned to goldens produced by the reference (tests/test_host_mirrors.py).
"""
from __future__ import annotations

import torch

from . import bundle_adjustment as ba
from . import pose_refinement as pr
from . import triangulation as tri
from .corr import sample_features4d


def create_intri_matrix(focal_length, principal_point):
    """vggsfm/utils/triangulation_helpers.py:590-623."""
    K = torch.zeros(focal_length.shape[:-1] + (3, 3), dtype=focal_length.dtype, device=focal_length.device)
    K[..., 0, 0] = focal_length[..., 0]
    K[..., 1, 1] = focal_length[..., 1]
    K[..., 2, 2] = 1.0
    K[..., 0, 2] = principal_point[..., 0]
    K[..., 1, 2] = principal_point[..., 1]
    return K


def get_EFP(pred_cameras, image_size, B, S, default_focal=False):
    """vggsfm/models/utils.py:38-72: camera object (``.focal_length [B*S,2]`` in NDC, ``.R [B*S,3,3]``,
    ``.T [B*S,3]``) -> extrinsics [B,S,3,4], intrinsics [B,S,3,3]; one focal per frame = mean(fx,fy) * min(W,H)/2
    clamped to [0.2, 5] * scale, principal point at the image centre."""
    scale = image_size.min()
    focal_length = pred_cameras.focal_length
    principal_point = torch.zeros_like(focal_length)
    focal_length = focal_length * scale / 2
    principal_point = (image_size[None] - principal_point * scale) / 2
    extrinsics = torch.cat([pred_cameras.R.clone(), pred_cameras.T.clone()[..., None]], dim=-1).reshape(B, S, 3, 4)
    focal_length = focal_length.reshape(B, S, 2)
    principal_point = principal_point.reshape(B, S, 2)
    if default_focal:
        focal_length = torch.full_like(focal_length, float(scale))
    else:
        focal_length = focal_length.mean(dim=-1, keepdim=True).expand(-1, -1, 2)
        focal_length = focal_length.clamp(0.2 * scale, 5 * scale)
    return extrinsics, create_intri_matrix(focal_length, principal_point)


def find_best_initial_pair(inlier_geo_vis, cheirality_mask_pair, triangle_value_pair, init_tri_angle_thres):
    """vggsfm/models/triangulator.py:442-476: halve the triangulation-angle threshold (at most 5 times, not below
    2) until the best frame has >= 100 inliers and >= 25 % of the tracks."""
    trial_count = 0
    N = inlier_geo_vis.shape[-1]
    base = torch.logical_and(inlier_geo_vis, cheirality_mask_pair)
    while trial_count < 5:
        inlier_total = torch.logical_and(base, triangle_value_pair >= init_tri_angle_thres)
        max_num_inlier = int(inlier_total.sum(dim=-1).max())
        if max_num_inlier >= 100 and max_num_inlier / N >= 0.25:
            break
        if init_tri_angle_thres < 2:
            break
        init_tri_angle_thres = init_tri_angle_thres // 2
        trial_count += 1
    return inlier_total, init_tri_angle_thres


def _hist(termination):
    """{termination name: frames} of a pose report, for the stage log."""
    v, c = torch.unique(termination, return_counts=True)
    return {pr.TERMINATION.get(int(a), "?"): int(b) for a, b in zip(v, c)}


class Triangulator(torch.nn.Module):
    def __init__(self, cfg=None):
        super().__init__()
        self.cfg = cfg
        self.verbose = False

    def _log(self, stage, extrinsics, intrinsics, extra_params, extra=""):
        if self.verbose:
            k = "" if extra_params is None else f" k[0]={float(extra_params[0, 0]):.5f}"
            print(f"[Triangulator] {stage}: f[0]={float(intrinsics[0, 0, 0]):.3f} f[-1]={float(intrinsics[-1, 0, 0]):.3f}{k} {extra}")

    @torch.no_grad()
    def forward(self, pred_cameras, pred_tracks, pred_vis, images, preliminary_dict, pred_score=None,
                init_max_reproj_error=0.5, BA_iters=2, shared_camera=False, max_reproj_error=4,
                init_tri_angle_thres=16, min_valid_track_length=3, robust_refine=2, extract_color=True,
                camera_type="SIMPLE_PINHOLE"):
        """vggsfm/models/triangulator.py:44-363.  pred_tracks [1,S,N,2] pixels, pred_vis/pred_score [1,S,N],
        images [1,S,3,H,W], preliminary_dict["fmat_inlier_mask"] [1,S-1,N]."""
        device = pred_tracks.device
        B, S, _, H, W = images.shape
        assert B == 1
        image_size = torch.tensor([W, H], dtype=pred_tracks.dtype, device=device)
        extrinsics, intrinsics = get_EFP(pred_cameras, image_size, B, S)
        extrinsics = extrinsics.double()[0]
        intrinsics = intrinsics[0]
        inlier_fmat = preliminary_dict["fmat_inlier_mask"][0]
        pred_tracks = pred_tracks[0]
        pred_vis = pred_vis[0]
        pred_score = pred_score[0] if pred_score is not None else None
        if shared_camera:
            intrinsics[:, 0, 0] = intrinsics[:, 0, 0].mean()
            intrinsics[:, 1, 1] = intrinsics[:, 1, 1].mean()
        extra_params = None
        if camera_type == "SIMPLE_RADIAL":
            extra_params = torch.zeros_like(extrinsics[:, 0, 0:1])

        tracks_normalized = tri.cam_from_img(pred_tracks, intrinsics)
        inlier_geo_vis = torch.logical_and(inlier_fmat, (pred_vis > 0.05)[1:])
        points_3d_pair, cheirality_mask_pair, triangle_value_pair = tri.triangulate_by_pair(
            extrinsics[None], tracks_normalized[None])
        inlier_total, _ = find_best_initial_pair(inlier_geo_vis, cheirality_mask_pair, triangle_value_pair,
                                                 init_tri_angle_thres)
        points3D_init, extrinsics, intrinsics, extra_params, track_init_mask, reconstruction, init_idx = ba.init_BA(
            extrinsics, intrinsics, extra_params, pred_tracks, points_3d_pair, inlier_total, image_size,
            shared_camera=shared_camera, init_max_reproj_error=init_max_reproj_error, camera_type=camera_type)
        self._log("init_BA", extrinsics, intrinsics, extra_params,
                  f"init_idx={init_idx} inliers={int(inlier_total[init_idx].sum())} kept={int(track_init_mask.sum())} "
                  f"its={reconstruction.summary.iterations} {reconstruction.summary.termination}")
        extrinsics, intrinsics, extra_params, _ = pr.init_refine_pose(
            extrinsics, intrinsics, extra_params, inlier_geo_vis, points3D_init, pred_tracks, track_init_mask, image_size,
            init_idx, shared_camera=shared_camera, camera_type=camera_type)
        self._log("init_refine_pose", extrinsics, intrinsics, extra_params,
                  f"term={_hist(pr.last_report.termination)} its<={int(pr.last_report.iterations.max())}")
        points3D, extrinsics, intrinsics, extra_params, valid_tracks, reconstruction = self.triangulate_tracks_and_BA(
            pred_tracks, intrinsics, extrinsics, extra_params, pred_vis, pred_score, image_size, min_valid_track_length,
            max_reproj_error, shared_camera=shared_camera, camera_type=camera_type)
        self._log("triangulate_tracks_and_BA", extrinsics, intrinsics, extra_params,
                  f"valid={int(valid_tracks.sum())} its={reconstruction.summary.iterations} {reconstruction.summary.termination}")

        for refine_idx in range(robust_refine):
            inlier_vis_all = pred_vis > 0.05
            extrinsics, intrinsics, extra_params, _ = pr.refine_pose(
                extrinsics, intrinsics, extra_params, inlier_vis_all, points3D, pred_tracks, valid_tracks, image_size,
                force_estimate=(refine_idx == robust_refine - 1), shared_camera=shared_camera, camera_type=camera_type)
            self._log(f"refine_pose {refine_idx}", extrinsics, intrinsics, extra_params,
                      f"term={_hist(pr.last_report.termination)} inliers>={int(pr.last_report.num_inliers.min())}")
            points3D, extrinsics, intrinsics, extra_params, valid_tracks, reconstruction = self.triangulate_tracks_and_BA(
                pred_tracks, intrinsics, extrinsics, extra_params, pred_vis, pred_score, image_size,
                min_valid_track_length, max_reproj_error, shared_camera=shared_camera, camera_type=camera_type)
            self._log(f"robust refine {refine_idx}", extrinsics, intrinsics, extra_params,
                      f"valid={int(valid_tracks.sum())} its={reconstruction.summary.iterations} {reconstruction.summary.termination}")

        ba_options = ba.default_options()                       # pycolmap.BundleAdjustmentOptions(), :254
        BA_inlier_masks = None
        for BA_iter in range(BA_iters):
            (points3D, extrinsics, intrinsics, extra_params, valid_tracks, BA_inlier_masks,
             reconstruction) = ba.iterative_global_BA(
                pred_tracks, intrinsics, extrinsics, pred_vis, pred_score, valid_tracks, points3D, image_size,
                lastBA=(BA_iter == BA_iters - 1), extra_params=extra_params, shared_camera=shared_camera,
                min_valid_track_length=min_valid_track_length, max_reproj_error=max_reproj_error, ba_options=ba_options,
                camera_type=camera_type)
            self._log(f"iterative BA {BA_iter}", extrinsics, intrinsics, extra_params, f"valid={int(valid_tracks.sum())}")
            max_reproj_error = max(max_reproj_error // 2, 1)     # :293-295

        scale = image_size.max()
        valid_frame_mask = ba.get_valid_frame_mask(intrinsics, extrinsics, extra_params, scale)
        valid_2D_mask = torch.ones_like(pred_tracks[..., 0]).bool()
        valid_2D_mask[:, ~valid_tracks] = False
        if BA_inlier_masks is not None:
            valid_2D_mask[:, valid_tracks] = BA_inlier_masks

        points3D_rgb = None
        if extract_color and BA_inlier_masks is not None:
            pred_track_rgb = sample_features4d(images[0], pred_tracks)             # [S,N,3]
            valid_track_rgb = pred_track_rgb[:, valid_tracks]
            sum_rgb = (BA_inlier_masks.float()[..., None] * valid_track_rgb).sum(dim=0)
            points3D_rgb = sum_rgb / BA_inlier_masks.sum(dim=0)[:, None]
            if points3D_rgb.shape[0] == max(reconstruction.point3D_ids()):           # :333-340
                reconstruction.set_point_colors(points3D_rgb)
            else:
                print("Cannot save point rgb colors to colmap reconstruction object.")
        return (extrinsics, intrinsics, extra_params, points3D, points3D_rgb, reconstruction, valid_frame_mask,
                valid_2D_mask, valid_tracks)

    def triangulate_tracks_and_BA(self, pred_tracks, intrinsics, extrinsics, extra_params, pred_vis, pred_score,
                                  image_size, min_valid_track_length, max_reproj_error=4, shared_camera=False,
                                  camera_type="SIMPLE_PINHOLE"):
        """vggsfm/models/triangulator.py:365-439: LORANSAC over all frames -> tracks with enough inliers ->
        global BA -> reprojection filter."""
        tn = tri.cam_from_img(pred_tracks, intrinsics, extra_params)
        best_points, best_inlier_num, best_inlier_mask = tri.triangulate_tracks(
            extrinsics, tn, track_vis=pred_vis, track_score=pred_score)
        valid_tracks = best_inlier_num >= min_valid_track_length
        points3D, extrinsics, intrinsics, extra_params, reconstruction = ba.global_BA(
            best_points, valid_tracks, pred_tracks, best_inlier_mask, extrinsics, intrinsics, extra_params, image_size,
            shared_camera=shared_camera, camera_type=camera_type)
        valid_points3D_mask, _ = tri.filter_all_points3D(
            points3D, pred_tracks[:, valid_tracks], extrinsics, intrinsics, extra_params, check_triangle=False,
            max_reproj_error=max_reproj_error)
        points3D = points3D[valid_points3D_mask]
        valid_tracks_tmp = valid_tracks.clone()
        valid_tracks_tmp[valid_tracks] = valid_points3D_mask
        return points3D, extrinsics, intrinsics, extra_params, valid_tracks_tmp, reconstruction
