"""Absolute-pose refinement on device tensors -- host-side mirror of ``refine_pose`` / ``init_refine_pose``.

The reference walks the frames in Python and calls ``pycolmap.pose_refinement`` once per frame
(vggsfm/utils/triangulation.py:341-441 and :542-608): S sequential CPU Ceres solves, each preceded by
``.cpu()`` copies.  Here every frame is one CTA of a single launch (``vgg_pose_refinement``,
csrc/pose_refine.cu) and nothing leaves the GPU.  PyTorch is used for device memory and index
compaction only; there is no fallback path.

``pycolmap.absolute_pose_estimation`` -- the ``force_estimate`` fall-back of refine_pose (triangulation.py:404-433)
and the video runner's PnP alignment -- is ``absolute_pose_estimation_batched`` below: P3P + LO-RANSAC for all the
frames that need it and all 31 focal-length factors in one launch (csrc/pnp.cu), followed by the same refinement
kernel.  COLMAP draws its minimal samples from an internal generator no caller can seed; here they come from
torch's CPU generator (``draw_pnp_samples``), like the triangulation pairs.
"""
from __future__ import annotations

import ctypes
import dataclasses
from typing import Optional

import torch

from . import _lib
from ._lib import PoseOptions
from .bundle_adjustment import SIMPLE_RADIAL, camera_model_id, get_valid_frame_mask

FLAG_ACTIVE, FLAG_FOCAL, FLAG_EXTRA = 1, 2, 4
TERMINATION = {0: "NO_CONVERGENCE", 1: "CONVERGENCE_GRADIENT", 2: "CONVERGENCE_FUNCTION", 3: "CONVERGENCE_PARAMETER",
               4: "MIN_TRUST_REGION_RADIUS", 5: "FAILURE", 6: "SKIPPED", 7: "FEW_INLIERS"}


def default_pose_options() -> PoseOptions:
    """pycolmap.AbsolutePoseRefinementOptions() as the reference builds it (triangulation.py:328-331)."""
    o = PoseOptions()
    _lib.lib().vgg_pose_default_options(ctypes.byref(o))
    return o


@dataclasses.dataclass
class PoseReport:
    iterations: torch.Tensor            # [S] int32
    successful: torch.Tensor            # [S] int32
    termination: torch.Tensor           # [S] int32 (TERMINATION)
    initial_cost: torch.Tensor          # [S] f64
    final_cost: torch.Tensor            # [S] f64
    final_radius: torch.Tensor          # [S] f64 trust-region radius at the end (0 for frames that were not refined)
    num_inliers: torch.Tensor           # [S] int64 effective inliers per frame
    inlier_used: torch.Tensor           # [S,P] bool
    needs_absolute_pose: Optional[torch.Tensor] = None   # [S] bool (refine_pose only)
    absolute_pose_ok: Optional[torch.Tensor] = None      # [S] bool: frames re-estimated by P3P LO-RANSAC
    kernel_launches: int = 0


def pose_refinement_batched(poses, intr4, points3D, tracks2D, inlier, frame_flags, model: int,
                            options: Optional[PoseOptions] = None):
    """One ``vgg_pose_refinement`` launch.  poses [S,3,4] f64 and intr4 [S,4] f64 are updated IN PLACE.

    points3D [P,3] f64, tracks2D [S,P,2] f32, inlier [S,P] uint8/bool, frame_flags [S] uint8."""
    if not poses.is_cuda:
        raise RuntimeError("vggsfm_b200.pose_refinement needs CUDA tensors (no CPU fallback)")
    L = _lib.lib()
    dev = poses.device
    S, P = inlier.shape
    if S == 0 or P == 0:                     # nothing to refine: every frame is reported as having too few inliers
        z = torch.zeros(S, dtype=torch.float64, device=dev)
        return PoseReport(torch.zeros(S, dtype=torch.int32, device=dev), torch.zeros(S, dtype=torch.int32, device=dev),
                          torch.full((S,), 7, dtype=torch.int32, device=dev), z, z.clone(), z.clone(),
                          torch.zeros(S, dtype=torch.int64, device=dev), torch.zeros(S, P, dtype=torch.bool, device=dev))
    assert poses.dtype == torch.float64 and poses.is_contiguous() and intr4.dtype == torch.float64 and intr4.is_contiguous()
    pts = points3D.double().contiguous()
    uv = tracks2D.float().contiguous()
    inl = inlier.to(torch.uint8).contiguous()
    flags = frame_flags.to(torch.uint8).contiguous()
    used = torch.empty(S, P, dtype=torch.uint8, device=dev)
    sd = torch.zeros(S, 4, dtype=torch.float64, device=dev)
    si = torch.zeros(S, 4, dtype=torch.int32, device=dev)
    opt = options or default_pose_options()
    with torch.cuda.device(dev):
        stream = torch.cuda.current_stream(dev).cuda_stream
        _lib.check(L.vgg_pose_refinement(S, P, model, uv.data_ptr(), inl.data_ptr(), flags.data_ptr(), pts.data_ptr(),
                                     poses.data_ptr(), intr4.data_ptr(), ctypes.byref(opt), used.data_ptr(),
                                     sd.data_ptr(), si.data_ptr(), stream), "vgg_pose_refinement")
    return PoseReport(si[:, 0], si[:, 1], si[:, 2], sd[:, 0], sd[:, 1], sd[:, 2], sd[:, 3].round().long(), used.bool(),
                      kernel_launches=1 if S > 0 else 0)


def draw_pnp_samples(num_trials: int = 128) -> torch.Tensor:
    """Minimal-sample draws of the absolute-pose RANSAC: [num_trials,3] uniform numbers from torch's CPU generator
    (``torch.manual_seed`` makes a run reproducible); the kernel maps them to the frame's usable points."""
    return torch.rand(num_trials, 3, dtype=torch.float64)


def absolute_pose_estimation_batched(tracks2D, points3D, masks, intr4, model: int, frames=None, estimate_focal_length=False,
                                     max_error=12.0, u_samples=None, num_trials=128):
    """``pycolmap.absolute_pose_estimation`` (estimation part) for many frames at once: ``vgg_absolute_pose_estimation``.

    tracks2D [S,P,2], points3D [P,3], masks [S,P] usable observations, intr4 [S,4] f64 (f,cx,cy,k), frames [S] bool
    (default: all).  Returns (poses [S,3,4] f64 -- rows of failed / skipped frames are zero, focal [S] f64,
    num_inliers [S] int32 -- 0 where the reference would get ``None``, inliers [S,P] bool)."""
    if not tracks2D.is_cuda:
        raise RuntimeError("vggsfm_b200.absolute_pose_estimation needs CUDA tensors (no CPU fallback)")
    L = _lib.lib()
    dev = tracks2D.device
    S, P = masks.shape
    poses = torch.zeros(S, 3, 4, dtype=torch.float64, device=dev)
    focal = intr4[:, 0].clone().double()
    ninl = torch.zeros(S, dtype=torch.int32, device=dev)
    inl = torch.zeros(S, P, dtype=torch.uint8, device=dev)
    if S == 0 or P < 3:
        return poses, focal, ninl, inl.bool()
    uv = tracks2D.float().contiguous()
    mk = masks.to(torch.uint8).contiguous()
    fl = (torch.ones(S, dtype=torch.uint8, device=dev) if frames is None else frames.to(torch.uint8)).contiguous()
    pts = points3D.double().contiguous()
    it4 = intr4.double().contiguous()
    us = (draw_pnp_samples(num_trials) if u_samples is None else u_samples).to(torch.float64).to(dev).contiguous()
    nb = ctypes.c_size_t()
    _lib.check(L.vgg_pnp_workspace_bytes(S, 1 if estimate_focal_length else 0, ctypes.byref(nb)), "vgg_pnp_workspace_bytes")
    ws = torch.empty(max(nb.value, 256), dtype=torch.uint8, device=dev)
    with torch.cuda.device(dev):
        stream = torch.cuda.current_stream(dev).cuda_stream
        _lib.check(L.vgg_absolute_pose_estimation(S, P, model, uv.data_ptr(), mk.data_ptr(), fl.data_ptr(), pts.data_ptr(),
                                                  it4.data_ptr(), us.data_ptr(), us.shape[0], 1 if estimate_focal_length else 0,
                                                  float(max_error), poses.data_ptr(), focal.data_ptr(), ninl.data_ptr(),
                                                  inl.data_ptr(), ws.data_ptr(), ws.numel(), stream),
                   "vgg_absolute_pose_estimation")
    return poses, focal, ninl, inl.bool()


def _intr4(intrinsics, extra_params, model):
    S = intrinsics.shape[0]
    a = torch.zeros(S, 4, dtype=torch.float64, device=intrinsics.device)
    a[:, 0] = intrinsics[:, 0, 0]
    a[:, 1] = intrinsics[:, 0, 2]
    a[:, 2] = intrinsics[:, 1, 2]
    if model == SIMPLE_RADIAL:
        a[:, 3] = extra_params.reshape(S, -1)[:, 0]
    return a


def _calibration_matrix(intr4):
    S = intr4.shape[0]
    K = torch.zeros(S, 3, 3, dtype=torch.float64, device=intr4.device)
    K[:, 0, 0] = intr4[:, 0]
    K[:, 1, 1] = intr4[:, 0]
    K[:, 0, 2] = intr4[:, 1]
    K[:, 1, 2] = intr4[:, 2]
    K[:, 2, 2] = 1.0
    return K


def _merge(dst: PoseReport, src: PoseReport, rows):
    for f in ("iterations", "successful", "termination", "initial_cost", "final_cost", "final_radius", "num_inliers",
              "inlier_used"):
        getattr(dst, f)[rows] = getattr(src, f)
    dst.kernel_launches += src.kernel_launches


def _run_frames(poses, intr4, points3D, tracks2D, inlier, active, model, shared_camera, opt):
    """The frame loop of both mirrors.  Per-frame cameras: one launch.  Shared camera
    (triangulation.py:373-375, :564-566): the single pycolmap.Camera is refined by frame 0 only and every later
    frame sees the updated, now constant, intrinsics -- frame 0 is launched first, then the rest."""
    S = poses.shape[0]
    dev = poses.device
    flags = active.to(torch.uint8) * FLAG_ACTIVE
    if not shared_camera:
        flags = flags | (FLAG_FOCAL | FLAG_EXTRA)
        return pose_refinement_batched(poses, intr4, points3D, tracks2D, inlier, flags, model, opt)
    # effective masks at the INPUT cameras for every frame (the reference filters before its loop, :298-315)
    rep = pose_refinement_batched(poses, intr4, points3D, tracks2D, inlier, torch.zeros(S, dtype=torch.uint8, device=dev),
                                  model, opt)
    saved = opt.max_reproj_error
    opt.max_reproj_error = 0.0
    try:
        intr4[:] = intr4[0].clone()
        f0 = flags[:1] | (FLAG_FOCAL | FLAG_EXTRA)
        r0 = pose_refinement_batched(poses[:1], intr4[:1], points3D, tracks2D[:1], rep.inlier_used[:1], f0, model, opt)
        _merge(rep, r0, slice(0, 1))
        if S > 1:
            intr4[1:] = intr4[0].clone()
            r1 = pose_refinement_batched(poses[1:], intr4[1:], points3D, tracks2D[1:], rep.inlier_used[1:], flags[1:],
                                         model, opt)
            _merge(rep, r1, slice(1, S))
    finally:
        opt.max_reproj_error = saved
    return rep


def _finish(poses, intr4, extrinsics, intrinsics, extra_params, model, scale):
    """Read-back + validity revert shared by both mirrors (triangulation.py:443-472, :611-640)."""
    refined_extrinsics = poses
    refined_intrinsics = _calibration_matrix(intr4)
    refined_extra = intr4[:, 3:4].clone() if extra_params is not None else None
    valid = get_valid_frame_mask(refined_intrinsics, refined_extrinsics, refined_extra, scale)
    bad = ~valid
    if bad.any():
        refined_extrinsics[bad] = extrinsics[bad].to(refined_extrinsics.dtype)
        refined_intrinsics[bad] = intrinsics[bad].to(refined_extrinsics.dtype)
        if extra_params is not None:
            refined_extra[bad] = extra_params[bad].reshape(-1, 1).to(refined_extrinsics.dtype)
    return refined_extrinsics, refined_intrinsics, refined_extra, valid


last_report: Optional[PoseReport] = None


def refine_pose(extrinsics, intrinsics, extra_params, inlier, points3D, tracks, valid_track_mask, image_size,
                shared_camera=False, max_reproj_error=12, camera_type="SIMPLE_PINHOLE", force_estimate=False):
    """vggsfm/utils/triangulation.py:260-479, same arguments and return tuple
    (refined_extrinsics [S,3,4] f64, refined_intrinsics [S,3,3] f64, refined_extra_params [S,1]|None,
    valid_frame_mask [S]).  The solver report of the call is left in ``pose_refinement.last_report``."""
    global last_report
    model = camera_model_id(camera_type)
    S, P = tracks.shape[0], tracks.shape[1]
    assert len(intrinsics) == S and inlier.shape[0] == S and inlier.shape[1] == P and len(valid_track_mask) == P
    empty = points3D.abs().sum(-1) <= 0                                           # :289-295
    if empty.any():
        tmp = valid_track_mask.clone()
        tmp[valid_track_mask] = ~empty
        valid_track_mask = tmp
        points3D = points3D[~empty]
    tracks2D = tracks[:, valid_track_mask]
    inl = inlier[:, valid_track_mask]
    poses = extrinsics.double().contiguous().clone()
    intr4 = _intr4(intrinsics, extra_params, model)
    opt = default_pose_options()
    opt.max_reproj_error = float(max_reproj_error)
    opt.min_inliers = 100                                                          # :386
    active = torch.ones(S, dtype=torch.bool, device=poses.device)
    rep = _run_frames(poses, intr4, points3D, tracks2D, inl, active, model, shared_camera, opt)
    scale = image_size.max()
    focal = intr4[:, 0]
    refined = rep.termination < 6
    rep.needs_absolute_pose = (~refined) | (focal < 0.1 * scale) | (focal > 30 * scale)   # :396-402
    if force_estimate and bool(rep.needs_absolute_pose.any()):
        _estimate_absolute_poses(rep.needs_absolute_pose, poses, intr4, points3D, tracks2D, inl, model, shared_camera,
                                 float(max_reproj_error), rep)
    last_report = rep
    return _finish(poses, intr4, extrinsics, intrinsics, extra_params, model, scale)


def _estimate_absolute_poses(need, poses, intr4, points3D, tracks2D, inl_nongeo, model, shared_camera, max_error, rep):
    """triangulation.py:404-433 for the frames in ``need`` (in place on poses / intr4): P3P LO-RANSAC with the focal
    ladder on the visible matches when a frame has more than 50 of them (retried on all matches when that fails), on
    all matches otherwise; a found model replaces the pose and is refined with the RANSAC inliers, like
    pycolmap.absolute_pose_estimation's own refinement step.  With a shared camera the estimated focal length is used
    for the pose only (COLMAP would write it into the single shared Camera in the middle of the frame loop)."""
    S, P = inl_nongeo.shape
    dev = poses.device
    vis = inl_nongeo.bool()
    enough = vis.sum(dim=1) > 50
    all_pts = torch.ones_like(vis)
    first = torch.where(enough[:, None], vis, all_pts)
    us = draw_pnp_samples()
    p1, f1, n1, i1 = absolute_pose_estimation_batched(tracks2D, points3D, first, intr4, model, need, True, max_error, us)
    retry = need & enough & (n1 == 0)
    if bool(retry.any()):
        p2, f2, n2, i2 = absolute_pose_estimation_batched(tracks2D, points3D, all_pts, intr4, model, retry, True, max_error, us)
        p1 = torch.where(retry[:, None, None], p2, p1)
        f1 = torch.where(retry, f2, f1)
        n1 = torch.where(retry, n2, n1)
        i1 = torch.where(retry[:, None], i2, i1)
    ok = need & (n1 > 0)
    rep.absolute_pose_ok = ok
    if not bool(ok.any()):
        return
    poses[ok] = p1[ok]
    if not shared_camera:
        intr4[ok, 0] = f1[ok]
    flags = ok.to(torch.uint8) * FLAG_ACTIVE
    if not shared_camera:
        flags = flags | (FLAG_FOCAL | FLAG_EXTRA)
    opt = default_pose_options()
    r2 = pose_refinement_batched(poses, intr4, points3D, tracks2D, i1, flags, model, opt)
    rep.kernel_launches += r2.kernel_launches + 2


def init_refine_pose(extrinsics, intrinsics, extra_params, inlier, points3D, tracks, valid_track_mask_init, image_size,
                     init_idx, max_reproj_error=12, shared_camera=False, camera_type="SIMPLE_PINHOLE"):
    """vggsfm/utils/triangulation.py:482-647, same arguments and return tuple.  As in the reference,
    ``max_reproj_error`` is accepted and unused, the query frame counts every track as inlier, and the
    initial pair (frames 0 and init_idx+1) is not refined again."""
    global last_report
    model = camera_model_id(camera_type)
    S, P = tracks.shape[0], tracks.shape[1]
    assert len(intrinsics) == S and inlier.shape[0] == S - 1 and inlier.shape[1] == P and len(valid_track_mask_init) == P
    inl = torch.cat([torch.ones_like(inlier[0:1]), inlier], dim=0)[:, valid_track_mask_init]
    tracks2D = tracks[:, valid_track_mask_init]
    poses = extrinsics.double().contiguous().clone()
    intr4 = _intr4(intrinsics, extra_params, model)
    opt = default_pose_options()
    opt.min_inliers = 50                                                           # :585
    active = torch.ones(S, dtype=torch.bool, device=poses.device)
    active[0] = False
    active[init_idx + 1] = False
    rep = _run_frames(poses, intr4, points3D, tracks2D, inl, active, model, shared_camera, opt)
    last_report = rep
    return _finish(poses, intr4, extrinsics, intrinsics, extra_params, model, image_size.max())
