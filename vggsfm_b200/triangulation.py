"""Triangulation side of the hot path -- same names, arguments and return values as the reference's
vggsfm/utils/triangulation.py and vggsfm/utils/triangulation_helpers.py, running in libvggsfm_b200.so.

Drop-in: these functions can be monkey-patched onto ``vggsfm.utils.triangulation`` /
``vggsfm.utils.triangulation_helpers`` (see INTEGRATION.md).  CUDA tensors only; no fallback.
"""
from __future__ import annotations

import ctypes
import itertools
from typing import Optional

import numpy as np
import torch

from . import _lib


def _stream(dev):
    return torch.cuda.current_stream(dev).cuda_stream


def _need_cuda(t, name):
    if not t.is_cuda:
        raise RuntimeError(f"vggsfm_b200: {name} must be a CUDA tensor (there is no CPU fallback)")


def _f64c(t):
    return t.to(torch.float64).contiguous()


def generate_combinations(N):
    """vggsfm/utils/triangulation_helpers.py:638-645."""
    return np.array(list(itertools.combinations(range(N), 2)), dtype=np.int64)


def draw_ransac_pairs(S: int, max_ransac_iters: int) -> np.ndarray:
    """Hypothesis frame pairs exactly as triangulation.py:804-813 draws them: all C(S,2) pairs when
    there are at most max_ransac_iters of them, else a prefix of a CPU ``torch.randperm`` (global RNG)."""
    comb = generate_combinations(S)
    if max_ransac_iters > len(comb):
        return comb
    return comb[torch.randperm(len(comb))[:max_ransac_iters].numpy()]


def cam_from_img(pred_tracks, intrinsics, extra_params=None):
    """vggsfm/utils/triangulation_helpers.py:398-428.  pred_tracks [S,N,2], intrinsics [S,3,3],
    extra_params [S,1] or None -> tracks_normalized [S,N,2] in torch's promoted dtype; with
    extra_params the reference's iterative_undistortion semantics (distortion.py:27-99), in float64."""
    _need_cuda(pred_tracks, "pred_tracks")
    L = _lib.lib()
    S, N, _ = pred_tracks.shape
    dt = torch.promote_types(pred_tracks.dtype, intrinsics.dtype)
    if dt not in (torch.float32, torch.float64):
        dt = torch.float32
    dev = pred_tracks.device
    uv = pred_tracks.to(dt).contiguous()
    f2 = torch.stack([intrinsics[:, 0, 0], intrinsics[:, 1, 1]], dim=-1).to(dt).contiguous()
    pp2 = torch.stack([intrinsics[:, 0, 2], intrinsics[:, 1, 2]], dim=-1).to(dt).contiguous()
    out = torch.empty_like(uv)
    with torch.cuda.device(dev):
        _lib.check(L.vgg_normalize_tracks(S, N, uv.data_ptr(), f2.data_ptr(), pp2.data_ptr(),
                                          1 if dt == torch.float64 else 0, out.data_ptr(), _stream(dev)),
                   "vgg_normalize_tracks")
        if extra_params is None:
            return out
        if extra_params.dim() != 2 or extra_params.shape[1] != 1:
            raise ValueError("Unsupported number of distortion parameters")   # distortion.py:153-154
        tn = _f64c(out)
        k = _f64c(extra_params[:, 0])
        res = torch.empty_like(tn)
        ws = torch.empty(64, dtype=torch.uint8, device=dev)
        iters = ctypes.c_int()
        _lib.check(L.vgg_undistort_simple_radial(S, N, tn.data_ptr(), k.data_ptr(), 100, 1e-10, 1e-6, res.data_ptr(),
                                                 ctypes.byref(iters), ws.data_ptr(), ws.numel(), _stream(dev)),
                   "vgg_undistort_simple_radial")
    return res.to(torch.promote_types(dt, extra_params.dtype))


_tri_ws: dict = {}


def triangulate_tracks(extrinsics, tracks_normalized, max_ransac_iters=256, lo_num=50, max_angular_error=2,
                       min_tri_angle=1.5, track_vis=None, track_score=None, max_tri_points_num=819200,
                       ransac_pairs: Optional[np.ndarray] = None):
    """vggsfm/utils/triangulation.py:677-773 (LORANSAC multi-view triangulation).

    extrinsics [S,3,4], tracks_normalized [S,N,2], track_vis/track_score [S,N].
    Returns (points [N,3] float64, inlier_num [N] int64, inlier_mask [N,S] bool).
    One fused kernel handles all N tracks, so `max_tri_points_num` (a memory-chunking knob of the
    reference) is accepted and ignored.  `ransac_pairs` overrides the host RNG draw (tests, sharding)."""
    _need_cuda(tracks_normalized, "tracks_normalized")
    L = _lib.lib()
    S, N, _ = tracks_normalized.shape
    dev = tracks_normalized.device
    pairs = ransac_pairs if ransac_pairs is not None else draw_ransac_pairs(S, max_ransac_iters)
    H0 = len(pairs)
    pairs_t = torch.from_numpy(np.ascontiguousarray(pairs, dtype=np.int32)).to(dev)
    E = _f64c(extrinsics.reshape(S, 12))
    tn = _f64c(tracks_normalized)
    if track_vis is None:
        raise ValueError("track_vis is required (triangulation.py:871 dereferences it)")
    vis = track_vis.to(torch.float32).contiguous()
    score = track_score.to(torch.float32).contiguous() if track_score is not None else None
    nbytes = ctypes.c_size_t()
    _lib.check(L.vgg_tri_workspace_bytes(S, N, H0, lo_num, ctypes.byref(nbytes)), "vgg_tri_workspace_bytes")
    key = (str(dev),)
    ws = _tri_ws.get(key)
    if ws is None or ws.numel() < nbytes.value:
        ws = torch.empty(nbytes.value, dtype=torch.uint8, device=dev)
        _tri_ws[key] = ws
    pts = torch.empty(N, 3, dtype=torch.float64, device=dev)
    num = torch.empty(N, dtype=torch.int64, device=dev)
    mask = torch.empty(N, S, dtype=torch.uint8, device=dev)
    with torch.cuda.device(dev):
        _lib.check(L.vgg_triangulate_tracks(S, N, E.data_ptr(), tn.data_ptr(), vis.data_ptr(),
                                            score.data_ptr() if score is not None else None, pairs_t.data_ptr(), H0,
                                            lo_num, float(max_angular_error), float(min_tri_angle), pts.data_ptr(),
                                            num.data_ptr(), mask.data_ptr(), ws.data_ptr(), ws.numel(), _stream(dev)),
                   "vgg_triangulate_tracks")
    return pts, num, mask.bool()


triangulate = triangulate_tracks   # the name BASELINE.json's north_star uses


def triangulate_by_pair(extrinsics, tracks_normalized):
    """vggsfm/utils/triangulation.py:45-135.  extrinsics [B,S,3,4], tracks_normalized [B,S,N,2] with B == 1
    (the reference asserts batch size 1, models/triangulator.py:78-80).
    Returns (points_3d_pair [S-1,N,3], cheirality_mask [S-1,N] bool, triangles [S-1,N] degrees)."""
    _need_cuda(tracks_normalized, "tracks_normalized")
    L = _lib.lib()
    B, S, N, _ = tracks_normalized.shape
    assert B == 1, "batch size must be 1"
    dev = tracks_normalized.device
    E = _f64c(extrinsics[0].reshape(S, 12))
    tn = _f64c(tracks_normalized[0])
    pts = torch.empty(S - 1, N, 3, dtype=torch.float64, device=dev)
    che = torch.empty(S - 1, N, dtype=torch.uint8, device=dev)
    ang = torch.empty(S - 1, N, dtype=torch.float64, device=dev)
    ws = torch.empty(S * 24 + 64, dtype=torch.uint8, device=dev)
    with torch.cuda.device(dev):
        _lib.check(L.vgg_triangulate_by_pair(S, N, E.data_ptr(), tn.data_ptr(), pts.data_ptr(), che.data_ptr(),
                                             ang.data_ptr(), ws.data_ptr(), ws.numel(), _stream(dev)),
                   "vgg_triangulate_by_pair")
    return pts, che.bool(), ang


def filter_all_points3D(points3D, points2D, extrinsics, intrinsics, extra_params=None, max_reproj_error=4,
                        min_tri_angle=1.5, check_triangle=True, return_detail=False, hard_max=300,
                        max_points_num=819200):
    """vggsfm/utils/triangulation_helpers.py:133-307.  points3D [P,3], points2D [S,P,2], extrinsics [S,3,4],
    intrinsics [S,3,3], extra_params [S,1]|None.  Returns (valid [P] bool, inlier_detail [S,P] bool | None).
    `max_points_num` (reference memory chunking) is accepted and ignored."""
    _need_cuda(points2D, "points2D")
    L = _lib.lib()
    S, P, _ = points2D.shape
    dev = points2D.device
    if P == 0:
        return (torch.zeros(0, dtype=torch.bool, device=dev),
                torch.zeros(S, 0, dtype=torch.bool, device=dev) if return_detail else None)
    X = _f64c(points3D)
    is64 = points2D.dtype == torch.float64
    uv = points2D.contiguous() if points2D.dtype in (torch.float32, torch.float64) else points2D.float().contiguous()
    E = _f64c(extrinsics.reshape(S, 12))
    K = _f64c(intrinsics.reshape(S, 9))
    ex = _f64c(extra_params[:, 0]) if extra_params is not None else None
    valid = torch.empty(P, dtype=torch.uint8, device=dev)
    detail = torch.empty(S, P, dtype=torch.uint8, device=dev) if return_detail else None
    ws = torch.empty(S * 24 + 64, dtype=torch.uint8, device=dev)
    with torch.cuda.device(dev):
        _lib.check(L.vgg_filter_points3d(S, P, X.data_ptr(), uv.data_ptr(), 1 if is64 else 0, E.data_ptr(), K.data_ptr(),
                                         ex.data_ptr() if ex is not None else None, float(max_reproj_error),
                                         float(min_tri_angle), 1 if check_triangle else 0, float(hard_max),
                                         valid.data_ptr(), detail.data_ptr() if detail is not None else None,
                                         ws.data_ptr(), ws.numel(), _stream(dev)), "vgg_filter_points3d")
    return valid.bool(), (detail.bool() if detail is not None else None)


def filter_observations(points3D, obs_uv, obs_frame, obs_point, extrinsics, intrinsics, extra_params=None,
                        max_reproj_error=4, min_tri_angle=1.5):
    """filter_all_points3D on observations given as a list (COO obs_uv [M,2], obs_frame [M], obs_point [M] into
    points3D [P,3], any order) instead of the [S,P] grid (vgg_filter_observations).  Returns (keep [M] bool in the
    caller's order: reprojection error <= max_reproj_error at positive depth, valid [P] bool: >= 2 kept observations
    and one kept pair with a triangulation angle >= min_tri_angle degrees).  The per-observation arithmetic is the grid
    filter's; unlike the grid filter, an unobserved frame never counts (COLMAP's FilterAllPoints3D)."""
    from . import bundle_adjustment as ba
    _need_cuda(obs_uv, "obs_uv")
    L = _lib.lib()
    S, P = extrinsics.shape[0], points3D.shape[0]
    dev = obs_uv.device
    lst = ba.obs_list(obs_uv, obs_frame, obs_point, S, P)
    M = lst.frame.shape[0]
    keep_l = torch.zeros(M, dtype=torch.uint8, device=dev)
    valid = torch.zeros(P, dtype=torch.uint8, device=dev)
    X = _f64c(points3D)
    E = _f64c(extrinsics.reshape(S, 12))
    K = _f64c(intrinsics.reshape(S, 9))
    ex = _f64c(extra_params[:, 0]) if extra_params is not None else None
    ws = torch.empty(S * 24 + 64, dtype=torch.uint8, device=dev)
    ol = lst.struct()
    with torch.cuda.device(dev):
        _lib.check(L.vgg_filter_observations(S, P, ctypes.byref(ol), X.data_ptr(), E.data_ptr(), K.data_ptr(),
                                             ex.data_ptr() if ex is not None else None, float(max_reproj_error),
                                             float(min_tri_angle), keep_l.data_ptr(), valid.data_ptr(), ws.data_ptr(),
                                             ws.numel(), _stream(dev)), "vgg_filter_observations")
    keep = torch.zeros(M, dtype=torch.bool, device=dev)
    keep[lst.order] = keep_l.bool()
    return keep, valid.bool()


def project_3D_points(points3D, extrinsics, intrinsics=None, extra_params=None, return_points_cam=False, default=0,
                      only_points_cam=False):
    """vggsfm/utils/triangulation_helpers.py:311-355: points2D [S,P,2] (and points_cam [S,3,P])."""
    _need_cuda(points3D, "points3D")
    L = _lib.lib()
    P = points3D.shape[0]
    S = extrinsics.shape[0]
    dev = points3D.device
    X = _f64c(points3D)
    E = _f64c(extrinsics.reshape(S, 12))
    K = _f64c(intrinsics.reshape(S, 9)) if intrinsics is not None else None
    ex = _f64c(extra_params[:, 0]) if extra_params is not None else None
    want_cam = return_points_cam or only_points_cam
    out2d = None if only_points_cam else torch.empty(S, P, 2, dtype=torch.float64, device=dev)
    outcam = torch.empty(S, 3, P, dtype=torch.float64, device=dev) if want_cam else None
    with torch.cuda.device(dev):
        _lib.check(L.vgg_project_points(S, P, X.data_ptr(), E.data_ptr(), K.data_ptr() if K is not None else None,
                                        ex.data_ptr() if ex is not None else None,
                                        out2d.data_ptr() if out2d is not None else None,
                                        outcam.data_ptr() if outcam is not None else None, _stream(dev)),
                   "vgg_project_points")
    if only_points_cam:
        return outcam
    if return_points_cam:
        return out2d, outcam
    return out2d
