"""The two-view stage on device tensors -- mirror of ``vggsfm.two_view_geo`` (estimate_preliminary.py,
fundamental.py, utils.py), same names, arguments and returns.

The reference scores every pair's 3 x max_ransac_iters 7-point candidates against every match as one
[B, K, N, 3] float32 tensor (or, with ``loopresidual``, a Python loop over pairs).  Here the whole of
``estimate_fundamental`` is five launches of csrc/twoview.cu (``vgg_estimate_fundamental``) with nothing of size
pairs x candidates x matches ever stored, and the relative pose is one more (``vgg_relative_pose_from_fundamental``).
The minimal samples are drawn on the host with the reference's own ``np.random.randint`` calls, so a seeded run sees
the reference's 7-point sets.  There is no fallback path: CPU tensors raise.

``vggsfm.runners.runner.estimate_preliminary_cameras`` (with ``use_poselib: False``) can be rebound to
``estimate_preliminary_cameras`` below, and ``estimate_preliminary_cameras_poselib`` (the default configurations,
``use_poselib: True``) to ``estimate_preliminary_cameras_poselib``: PoseLib's LO-MSAC restated as
csrc/twoview_msac.cu (``vgg_estimate_fundamental_msac``), so the default configuration runs without PoseLib.
"""
from __future__ import annotations

import ctypes
import types

import numpy as np
import torch

from . import _lib


def _need_cuda(t, what):
    if not t.is_cuda:
        raise RuntimeError(f"vggsfm_b200.two_view.{what} needs CUDA tensors (no CPU fallback)")


def generate_samples(N, target_num, sample_num, expand_ratio=2):
    """utils.py:39-60: duplicate-free index rows drawn with np.random.randint.  Where the reference would return fewer
    than ``target_num`` rows (and then fail at ``.view``), this raises ValueError."""
    sample_idx = np.random.randint(0, N, size=(target_num * expand_ratio, sample_num))
    sorted_array = np.sort(sample_idx, axis=1)
    has_duplicates = (np.diff(sorted_array, axis=1) == 0).any(axis=1)
    safe = sample_idx[np.where(~has_duplicates)[0]][:target_num]
    if len(safe) < target_num:
        raise ValueError(f"only {len(safe)} of {target_num} duplicate-free {sample_num}-point samples drawn from "
                         f"{N} points")
    return safe


def _points(p):
    if p.dtype == torch.float64:
        return p.contiguous(), 1
    return p.float().contiguous(), 0


def estimate_fundamental(points1, points2, max_ransac_iters=4096, max_error=1, lo_num=300, valid_mask=None,
                         squared=True, second_refine=True, loopresidual=False, return_residuals=False, samples=None):
    """fundamental.py:43-183.  points1/points2 [B,N,2] CUDA (float32 or float64).  Returns (best_fmat [B,3,3] f64,
    best_inlier_num [B] int64, best_inlier_mask [B,N] bool[, best_residuals [B,N] f64]).  ``loopresidual`` is
    accepted and ignored (nothing of size B x K x N is stored).  ``samples`` ([T,7] int) replaces the draw."""
    _need_cuda(points1, "estimate_fundamental")
    L = _lib.lib()
    B, N, _ = points1.shape
    dev = points1.device
    if samples is None:
        samples = generate_samples(N, max_ransac_iters, 7)
    smp = np.ascontiguousarray(np.asarray(samples, dtype=np.int32))
    T = smp.shape[0]
    thr = float(max_error) ** 2 if squared else float(max_error)
    p1, f64 = _points(points1)
    p2, _ = _points(points2.to(p1.dtype))
    vm = valid_mask.to(torch.uint8).contiguous() if valid_mask is not None else None
    fmat = torch.empty(B, 3, 3, dtype=torch.float64, device=dev)
    num = torch.empty(B, dtype=torch.int32, device=dev)
    mask = torch.empty(B, N, dtype=torch.uint8, device=dev)
    res = torch.empty(B, N, dtype=torch.float64, device=dev)
    nb = ctypes.c_size_t()
    _lib.check(L.vgg_twoview_workspace_bytes(B, N, T, int(lo_num), ctypes.byref(nb)), "vgg_twoview_workspace_bytes")
    ws = torch.empty(max(nb.value, 256), dtype=torch.uint8, device=dev)
    with torch.cuda.device(dev):
        stream = torch.cuda.current_stream(dev).cuda_stream
        _lib.check(L.vgg_estimate_fundamental(B, N, p1.data_ptr(), p2.data_ptr(), f64,
                                              vm.data_ptr() if vm is not None else None, smp.ctypes.data, T,
                                              int(lo_num), thr, 1 if squared else 0, 1 if second_refine else 0,
                                              fmat.data_ptr(), num.data_ptr(), mask.data_ptr(), res.data_ptr(),
                                              ws.data_ptr(), ws.numel(), stream), "vgg_estimate_fundamental")
    out = (fmat, num.long(), mask.bool())
    return out + (res,) if return_residuals else out


def inlier_by_fundamental(fmat, tracks, max_error=0.5):
    """utils.py:300-322: Sampson inliers of the (frame 0, frame s) matches of tracks [B,S,N,2] under
    fmat [B,S-1,3,3] -> [B,S-1,N] bool, one ``vgg_fundamental_inliers`` launch."""
    _need_cuda(tracks, "inlier_by_fundamental")
    L = _lib.lib()
    B, S, N, _ = tracks.shape
    left, f64 = _points(tracks[:, 0:1].expand(-1, S - 1, -1, -1).reshape(B * (S - 1), N, 2))
    right, _ = _points(tracks[:, 1:].reshape(B * (S - 1), N, 2).to(left.dtype))
    F = fmat.reshape(B * (S - 1), 3, 3).double().contiguous()
    mask = torch.empty(B * (S - 1), N, dtype=torch.uint8, device=tracks.device)
    with torch.cuda.device(tracks.device):
        stream = torch.cuda.current_stream(tracks.device).cuda_stream
        _lib.check(L.vgg_fundamental_inliers(B * (S - 1), N, left.data_ptr(), right.data_ptr(), f64, F.data_ptr(),
                                             float(max_error) ** 2, 1, mask.data_ptr(), stream),
                   "vgg_fundamental_inliers")
    return mask.bool().reshape(B, S - 1, N)


def build_default_kmat(width, height, B, S, N, device=None, dtype=None):
    """estimate_preliminary.py:244-272."""
    f = float(max(width, height))
    K = torch.tensor([[f, 0, width / 2], [0, f, height / 2], [0, 0, 1]], device=device, dtype=dtype)
    kmat = K[None].repeat(B * (S - 1), 1, 1)
    fl = torch.full((B * (S - 1), 4), f, device=device, dtype=dtype)
    pp = torch.tensor([width / 2, height / 2] * 2, device=device, dtype=dtype)[None].repeat(B * (S - 1), 1)
    return kmat, kmat.clone(), fl, pp


def essential_from_fundamental(fmat, kmat1, kmat2, points1=None, points2=None, focal_length=None, principal_point=None,
                               max_error=4, squared=True, compute_residual=False):
    """fundamental.py:186-246 without the residual branch (compute_residual=False is all the pipeline uses)."""
    if compute_residual:
        raise NotImplementedError("essential_from_fundamental(compute_residual=True) is not part of the CUDA path")
    return kmat2.transpose(-2, -1) @ fmat @ kmat1, None, None


def relative_pose_from_fundamental(fmat, points1, points2, width, height):
    """E = K^T F K, decompose_essential_matrix + remove_cheirality (estimate_preliminary.py:159-164) in one launch.
    Returns (R [B,3,3] f64, t [B,3] f64, E [B,3,3] f64), OpenCV convention."""
    _need_cuda(points1, "relative_pose_from_fundamental")
    L = _lib.lib()
    B, N, _ = points1.shape
    dev = points1.device
    p1, f64 = _points(points1)
    p2, _ = _points(points2.to(p1.dtype))
    F = fmat.double().contiguous()
    R = torch.empty(B, 3, 3, dtype=torch.float64, device=dev)
    t = torch.empty(B, 3, dtype=torch.float64, device=dev)
    E = torch.empty(B, 3, 3, dtype=torch.float64, device=dev)
    with torch.cuda.device(dev):
        stream = torch.cuda.current_stream(dev).cuda_stream
        _lib.check(L.vgg_relative_pose_from_fundamental(B, N, p1.data_ptr(), p2.data_ptr(), f64, F.data_ptr(),
                                                        float(width), float(height), R.data_ptr(), t.data_ptr(),
                                                        E.data_ptr(), stream), "vgg_relative_pose_from_fundamental")
    return R, t, E


def estimate_preliminary_cameras(tracks, tracks_vis, width, height, tracks_score=None, max_error=0.5, lo_num=300,
                                 max_ransac_iters=4096, predict_essential=False, predict_homo=False,
                                 loopresidual=False):
    """estimate_preliminary.py:98-241.  tracks [B,S,N,2] CUDA, tracks_vis [B,S,N].  Returns (pred_cameras with .R,
    .T in PyTorch3D convention [B*S,3,3] / [B*S,3], preliminary_dict with fmat, fmat_inlier_mask, R_opencv, t_opencv,
    default_intri, emat_fromf, fmat_residuals).  predict_essential, predict_homo and loopresidual are accepted and
    ignored, as in the reference."""
    _need_cuda(tracks, "estimate_preliminary_cameras")
    B, S, N, _ = tracks.shape
    dev, dt = tracks.device, tracks.dtype
    query = tracks[:, 0:1].expand(-1, S - 1, -1, -1).reshape(B * (S - 1), N, 2)
    ref = tracks[:, 1:].reshape(B * (S - 1), N, 2)
    valid = (tracks_vis >= 0.05)[:, 1:].reshape(B * (S - 1), N)
    if tracks_score is not None:
        valid = valid & (tracks_score >= 0.5)[:, 1:].reshape(B * (S - 1), N)
    fmat, _, fmask, fres = estimate_fundamental(query, ref, max_error=max_error, lo_num=lo_num,
                                                max_ransac_iters=max_ransac_iters, valid_mask=valid,
                                                return_residuals=True)
    kmat1, kmat2, _, _ = build_default_kmat(width, height, B, S, N, device=dev, dtype=torch.float64)
    R, t, E = relative_pose_from_fundamental(fmat, query, ref, width, height)
    R = R.to(dt).reshape(B, S - 1, 3, 3)
    t = t.to(dt).reshape(B, S - 1, 3)
    R_pad = torch.eye(3, device=dev, dtype=dt)[None].repeat(B, 1, 1).unsqueeze(1)
    t_pad = torch.zeros(3, device=dev, dtype=dt)[None].repeat(B, 1).unsqueeze(1)
    R_opencv = torch.cat([R_pad, R], dim=1).reshape(B * S, 3, 3)
    t_opencv = torch.cat([t_pad, t], dim=1).reshape(B * S, 3)
    # OpenCV -> PyTorch3D (estimate_preliminary.py:198-220), then relative to the first camera
    Rp = R_opencv.clone().permute(0, 2, 1)
    Tp = t_opencv.clone()
    Tp[:, :2] *= -1
    Rp[:, :, :2] *= -1
    se3 = torch.zeros(B * S, 4, 4, device=dev, dtype=dt)
    se3[:, :3, :3] = Rp
    se3[:, 3, :3] = Tp
    se3[:, 3, 3] = 1.0
    R0 = se3[0:1, :3, :3].transpose(1, 2)
    inv0 = torch.cat([torch.cat([R0, -se3[0:1, 3:, :3].bmm(R0)], dim=1), se3[0:1, :, 3:]], dim=-1)
    rel = torch.bmm(inv0.expand(B * S, -1, -1), se3)
    rel[..., :3, 3] = 0.0
    rel[..., 3, 3] = 1.0
    pred_cameras = types.SimpleNamespace(R=rel[:, :3, :3].clone(), T=rel[:, 3, :3].clone())
    preliminary_dict = {
        "fmat": fmat.to(dt).reshape(B, S - 1, 3, 3),
        "fmat_inlier_mask": fmask.reshape(B, S - 1, -1),
        "R_opencv": R_opencv.reshape(B, S, 3, 3),
        "t_opencv": t_opencv.reshape(B, S, 3),
        "default_intri": kmat1.to(dt).reshape(B, S - 1, 3, 3),
        "emat_fromf": E.to(dt),
        "fmat_residuals": fres.to(dt).reshape(B, S - 1, -1),
    }
    return pred_cameras, preliminary_dict


def estimate_fundamental_msac(points1, points2, valid_mask=None, max_error=0.5, max_iterations=20000,
                              min_iterations=1000, seed=0, workspace=None):
    """poselib.estimate_fundamental (LO-MSAC, real focal check, no progressive sampling) for every pair at once.
    points1/points2 [B,N,2] CUDA float32 or float64 pixels, valid_mask [B,N] bool or None.  Returns (fmat [B,3,3] f64,
    inlier_num [B] int64, inlier_mask [B,N] bool, iterations [B] int64).  ``workspace`` (a uint8 CUDA tensor) is
    used instead of a fresh one when it is large enough."""
    _need_cuda(points1, "estimate_fundamental_msac")
    L = _lib.lib()
    B, N, _ = points1.shape
    dev = points1.device
    p1, f64 = _points(points1)
    p2, _ = _points(points2.to(p1.dtype))
    vm = valid_mask.to(torch.uint8).contiguous() if valid_mask is not None else None
    fmat = torch.empty(B, 3, 3, dtype=torch.float64, device=dev)
    num = torch.empty(B, dtype=torch.int32, device=dev)
    mask = torch.empty(B, N, dtype=torch.uint8, device=dev)
    iters = torch.empty(B, dtype=torch.int32, device=dev)
    nb = ctypes.c_size_t()
    _lib.check(L.vgg_msac_fundamental_workspace_bytes(B, N, int(max_iterations), int(min_iterations), ctypes.byref(nb)),
               "vgg_msac_fundamental_workspace_bytes")
    ws = workspace if workspace is not None and workspace.numel() >= nb.value else \
        torch.empty(max(nb.value, 256), dtype=torch.uint8, device=dev)
    with torch.cuda.device(dev):
        stream = torch.cuda.current_stream(dev).cuda_stream
        _lib.check(L.vgg_estimate_fundamental_msac(B, N, p1.data_ptr(), p2.data_ptr(), f64,
                                                   vm.data_ptr() if vm is not None else None, float(max_error),
                                                   int(max_iterations), int(min_iterations), int(seed),
                                                   fmat.data_ptr(), num.data_ptr(), mask.data_ptr(), iters.data_ptr(),
                                                   ws.data_ptr(), ws.numel(), stream), "vgg_estimate_fundamental_msac")
    return fmat, num.long(), mask.bool(), iters.long()


def estimate_preliminary_cameras_poselib(tracks, tracks_vis, width, height, tracks_score=None, max_error=0.5,
                                         max_ransac_iters=20000, predict_essential=False, lo_num=None,
                                         predict_homo=False, loopresidual=False):
    """estimate_preliminary.py:37-95.  tracks [B,S,N,2] CUDA, tracks_vis [B,S,N].  Returns (None, {"fmat":
    [1, B(S-1), 3, 3] f64, "fmat_inlier_mask": [1, B(S-1), N] bool}).  As in the reference, the left points of every
    pair are tracks[0, 0] (batch 0's query frame, also for the pairs of later batches), only matches with
    tracks_vis >= 0.05 take part, and tracks_score, predict_essential, lo_num, predict_homo and loopresidual are
    accepted and ignored.  A pair with fewer than 7 valid matches gets F = 0 and an empty mask (the reference fails)."""
    _need_cuda(tracks, "estimate_preliminary_cameras_poselib")
    B, S, N, _ = tracks.shape
    left = tracks[0, 0][None].expand(B * (S - 1), N, 2)
    right = tracks[:, 1:].reshape(B * (S - 1), N, 2)
    valid = (tracks_vis >= 0.05)[:, 1:].reshape(B * (S - 1), N)
    fmat, _, mask, _ = estimate_fundamental_msac(left, right, valid, max_error=max_error,
                                                 max_iterations=max_ransac_iters, min_iterations=1000, seed=0)
    return None, {"fmat": fmat[None], "fmat_inlier_mask": mask[None]}
