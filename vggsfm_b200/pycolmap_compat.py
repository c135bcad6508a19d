"""``pycolmap``-shaped entry points on the CUDA kernels -- the reference's own third-party seam.

Every BA / pose call of the reference is a call into ``pycolmap`` (SURVEY section 0.2): ``pycolmap.bundle_adjustment``
(vggsfm/utils/triangulation.py:213,1050,1142; runners/video_runner.py:508), ``pycolmap.pose_refinement``
(triangulation.py:387,590; video_runner.py:1001), ``pycolmap.absolute_pose_estimation`` (triangulation.py:413-430;
video_runner.py:991), ``pycolmap.ObservationManager`` (video_runner.py:510-512), ``pycolmap.BundleAdjuster`` +
``pyceres.solve`` (video_runner.py:1321-1331), plus the container classes.  This module offers those names with the
same call signatures, so that

    import vggsfm_b200.pycolmap_compat as pycolmap          # instead of: import pycolmap

lets the reference's UNMODIFIED ``vggsfm/utils/triangulation.py`` / ``tensor_to_pycolmap.py`` drive the CUDA path
object by object (one launch per call -- the batched mirrors in ``bundle_adjustment.py`` / ``pose_refinement.py`` are the
fast way in; this one is the zero-patch way).  Options carry the fields the reference touches.  All arithmetic runs in
libvggsfm_b200.so on the current CUDA device; objects live on the host like pycolmap's.
"""
from __future__ import annotations

import enum

import numpy as np
import torch

from . import bundle_adjustment as _ba
from . import pose_refinement as _pr
from . import triangulation as _tri
from .reconstruction import (Camera, Image, ListPoint2D, Point2D, Point3D, Reconstruction, Rigid3d, Rotation3d,  # noqa: F401
                             Track, TrackElement)


def _dev():
    if not torch.cuda.is_available():
        raise RuntimeError("vggsfm_b200.pycolmap_compat needs a CUDA device (no CPU fallback)")
    return torch.device("cuda", torch.cuda.current_device())


class _SolverOptions:
    """The Ceres options COLMAP's BundleAdjustmentOptions exposes; defaults of COLMAP 3.10 [3P-memory]."""

    def __init__(self):
        self.function_tolerance = 0.0
        self.gradient_tolerance = 1e-4
        self.parameter_tolerance = 0.0
        self.max_num_iterations = 100
        self.max_linear_solver_iterations = 200
        self.min_linear_solver_iterations = 0
        self.linear_solver_type = "DENSE_SCHUR"      # or "ITERATIVE_SCHUR" (PCG, for problems the dense solve cannot hold)
        self.eta = 0.1
        self.minimizer_progress_to_stdout = False
        self.num_threads = -1


class LossFunctionType(enum.Enum):
    """COLMAP's BundleAdjustmentOptions::LossFunctionType: the robust loss on every reprojection residual."""
    TRIVIAL = 0
    SOFT_L1 = 1
    CAUCHY = 2


class BundleAdjustmentOptions:
    def __init__(self):
        self.solver_options = _SolverOptions()
        self.loss_function_type = LossFunctionType.TRIVIAL
        self.loss_function_scale = 1.0                 # pixels
        self.refine_focal_length = True
        self.refine_principal_point = False
        self.refine_extra_params = True
        self.refine_extrinsics = True
        self.print_summary = False

    def _native(self):
        """(vgg_ba_options, the linear-solver and loss keywords of bundle_adjustment.bundle_adjustment)."""
        o = _ba.default_options()
        so = self.solver_options
        o.function_tolerance, o.gradient_tolerance, o.parameter_tolerance = so.function_tolerance, so.gradient_tolerance, so.parameter_tolerance
        o.max_num_iterations = int(so.max_num_iterations)
        lin = dict(linear_solver_type=so.linear_solver_type, min_linear_solver_iterations=int(so.min_linear_solver_iterations),
                   max_linear_solver_iterations=int(so.max_linear_solver_iterations), eta=float(so.eta))
        lt = self.loss_function_type
        lin.update(loss_function_type=lt.name if isinstance(lt, LossFunctionType) else str(lt),
                   loss_function_scale=float(self.loss_function_scale))
        return o, lin


class BundleAdjustmentConfig:
    """Which images / points take part and which are constant (video_runner.py:817-829)."""

    def __init__(self):
        self.images, self.constant_poses, self.constant_positions = [], set(), {}
        self.variable_points, self.constant_points = set(), set()
        self.constant_intrinsics = set()

    def add_image(self, image_id):
        self.images.append(int(image_id))

    def set_constant_cam_pose(self, image_id):
        self.constant_poses.add(int(image_id))

    def set_constant_cam_positions(self, image_id, idxs):
        self.constant_positions[int(image_id)] = list(idxs)

    def set_constant_cam_intrinsics(self, camera_id):
        self.constant_intrinsics.add(int(camera_id))

    def add_variable_point(self, point3D_id):
        self.variable_points.add(int(point3D_id))

    def add_constant_point(self, point3D_id):
        self.constant_points.add(int(point3D_id))


def _dense(reconstruction, image_ids=None):
    """Scene object -> the dense arrays of the CUDA path.  Returns a dict of numpy arrays + id lists."""
    ims = reconstruction.images
    image_ids = sorted(i for i, im in ims.items() if im.registered) if image_ids is None else list(image_ids)
    pids = sorted(reconstruction.points3D.keys())
    col = {p: k for k, p in enumerate(pids)}
    S, P = len(image_ids), len(pids)
    tracks = np.zeros((S, P, 2))
    masks = np.zeros((S, P), dtype=bool)
    extr = np.zeros((S, 3, 4))
    K = np.zeros((S, 3, 3))
    cams = [reconstruction.cameras[ims[i].camera_id] for i in image_ids]
    radial = cams[0].model == "SIMPLE_RADIAL"
    extra = np.zeros((S, 1)) if radial else None
    for s, iid in enumerate(image_ids):
        im = ims[iid]
        extr[s] = im.cam_from_world.matrix()
        K[s] = cams[s].calibration_matrix()
        if radial:
            extra[s, 0] = cams[s].params[3]
        xys, ids = im._arrays()
        for k in range(len(ids)):
            c = col.get(int(ids[k]))
            if c is not None:
                tracks[s, c] = xys[k]
                masks[s, c] = True
    xyz = np.stack([reconstruction.points3D[p].xyz for p in pids]) if P else np.zeros((0, 3))
    shared = len({c.camera_id for c in cams}) == 1 and S > 1
    return dict(image_ids=image_ids, pids=pids, tracks=tracks, masks=masks, extr=extr, K=K, extra=extra, xyz=xyz,
                shared=shared, camera_type=cams[0].model, cams=cams)


def _write_back(reconstruction, d, pts, extr, K, extra, valid_idx, alive=None):
    pts, extr, K = pts.cpu().numpy(), extr.cpu().numpy(), K.cpu().numpy()
    extra = extra.cpu().numpy() if extra is not None else None
    vi = valid_idx.cpu().numpy()
    alive = alive.cpu().numpy() if alive is not None else np.ones(len(vi), dtype=bool)
    for k, c in enumerate(vi):
        pid = d["pids"][int(c)]
        if alive[k]:
            reconstruction.points3D[pid].xyz = pts[k].copy()
        else:
            reconstruction.delete_point3D(pid)
    for s, iid in enumerate(d["image_ids"]):
        im = reconstruction.images[iid]
        im.cam_from_world = Rigid3d(Rotation3d(extr[s][:, :3]), extr[s][:, 3])
        cam = reconstruction.cameras[im.camera_id]
        prm = cam.params.copy()
        prm[0] = K[s, 0, 0]
        if extra is not None:
            prm[3] = extra[s, 0]
        cam.params = prm


def bundle_adjustment(reconstruction, options=None):
    """``pycolmap.bundle_adjustment(reconstruction, options)``: COLMAP's BundleAdjustmentController on the CUDA LM
    (gauge, negative-depth filter, Normalize(10)) -- in place on the object, like pycolmap."""
    options = options or BundleAdjustmentOptions()
    native, lin = options._native()
    d = _dense(reconstruction)
    dev = _dev()
    t = lambda a: torch.from_numpy(np.ascontiguousarray(a)).to(dev)
    pts, extr, K, extra, valid_idx, summ = _ba.bundle_adjustment(
        t(d["xyz"]), t(d["extr"]), t(d["K"]), t(d["extra"]) if d["extra"] is not None else None, t(d["tracks"]), t(d["masks"]),
        shared_camera=d["shared"], camera_type=d["camera_type"], options=native, max_points3D_val=float("inf"),
        refine_focal_length=options.refine_focal_length, refine_extra_params=options.refine_extra_params,
        filter_reconstruction=False, **lin)
    _write_back(reconstruction, d, pts, extr, K, extra, valid_idx, summ.alive)
    reconstruction.summary = summ
    return summ


class ObservationManager:
    """``pycolmap.ObservationManager(reconstruction)`` for the two calls of VideoRunner.joint_BA (video_runner.py:510-512)."""

    def __init__(self, reconstruction):
        self.reconstruction = reconstruction

    def filter_all_points3D(self, max_reproj_error, min_tri_angle):
        rec = self.reconstruction
        d = _dense(rec)
        dev = _dev()
        t = lambda a: torch.from_numpy(np.ascontiguousarray(a)).to(dev)
        ex = t(d["extra"]) if d["extra"] is not None else None
        _, detail = _tri.filter_all_points3D(t(d["xyz"]), t(d["tracks"]), t(d["extr"]), t(d["K"]), extra_params=ex,
                                            max_reproj_error=max_reproj_error, min_tri_angle=min_tri_angle,
                                            check_triangle=False, return_detail=True, hard_max=-1)
        ok_tri, _ = _tri.filter_all_points3D(t(d["xyz"]), t(d["tracks"]), t(d["extr"]), t(d["K"]), extra_params=ex,
                                             max_reproj_error=max_reproj_error, min_tri_angle=min_tri_angle,
                                             check_triangle=True, hard_max=-1)
        keep_obs = (t(d["masks"]) & detail).cpu().numpy()
        ok = ((keep_obs.sum(0) >= 2) & ok_tri.cpu().numpy())
        self._apply(d, keep_obs & ok[None], ok)

    def filter_observations_with_negative_depth(self):
        rec = self.reconstruction
        d = _dense(rec)
        depth = np.einsum("sj,nj->sn", d["extr"][:, 2, :3], d["xyz"]) + d["extr"][:, 2, 3][:, None]
        keep_obs = d["masks"] & (depth >= np.finfo(np.float64).eps)
        ok = keep_obs.sum(0) >= 2
        self._apply(d, keep_obs & ok[None], ok)

    def _apply(self, d, keep_obs, ok):
        rec = self.reconstruction
        for c, pid in enumerate(d["pids"]):
            if not ok[c]:
                rec.delete_point3D(pid)
                continue
            pt = rec.points3D[pid]
            kept = []
            for e in pt.track.elements:
                s = d["image_ids"].index(e.image_id) if e.image_id in d["image_ids"] else -1
                if s >= 0 and not keep_obs[s, c]:
                    rec.images[e.image_id].points2D[e.point2D_idx].point3D_id = Point2D.INVALID
                else:
                    kept.append(e)
            pt.track.elements = kept


class _RansacOptions:
    def __init__(self):
        self.max_error = 12.0
        self.min_inlier_ratio = 0.1
        self.confidence = 0.99999
        self.min_num_trials = 100
        self.max_num_trials = 10000


class AbsolutePoseEstimationOptions:
    def __init__(self):
        self.estimate_focal_length = False
        self.ransac = _RansacOptions()


class AbsolutePoseRefinementOptions:
    def __init__(self):
        self.refine_focal_length = False
        self.refine_extra_params = False
        self.print_summary = False


def _cam4(camera):
    p = camera.params
    return np.array([p[0], p[1], p[2], p[3] if camera.model == "SIMPLE_RADIAL" else 0.0])


def pose_refinement(cam_from_world, points2D, points3D, inlier_mask, camera, refinement_options=None):
    """``pycolmap.pose_refinement``: one frame of the batched kernel; ``camera`` is updated in place like pycolmap's."""
    ro = refinement_options or AbsolutePoseRefinementOptions()
    dev = _dev()
    model = _ba.camera_model_id(camera.model)
    poses = torch.from_numpy(cam_from_world.matrix()[None].copy()).to(dev)
    intr4 = torch.from_numpy(_cam4(camera)[None].copy()).to(dev)
    flags = _pr.FLAG_ACTIVE | (_pr.FLAG_FOCAL if ro.refine_focal_length else 0) | (_pr.FLAG_EXTRA if ro.refine_extra_params else 0)
    rep = _pr.pose_refinement_batched(poses, intr4, torch.from_numpy(np.asarray(points3D, dtype=np.float64)).to(dev),
                                      torch.from_numpy(np.asarray(points2D, dtype=np.float32))[None].to(dev),
                                      torch.from_numpy(np.asarray(inlier_mask).astype(np.uint8))[None].to(dev),
                                      torch.tensor([flags], dtype=torch.uint8, device=dev), model, _pr.default_pose_options())
    E = poses[0].cpu().numpy()
    it = intr4[0].cpu().numpy()
    prm = camera.params.copy()
    prm[0] = it[0]
    if camera.model == "SIMPLE_RADIAL":
        prm[3] = it[3]
    camera.params = prm
    return {"cam_from_world": Rigid3d(Rotation3d(E[:, :3]), E[:, 3]), "num_iterations": int(rep.iterations[0])}


def absolute_pose_estimation(points2D, points3D, camera, estimation_options=None, refinement_options=None, return_covariance=False):
    """``pycolmap.absolute_pose_estimation``: P3P LO-RANSAC (+ focal ladder) then refinement on the inliers; ``None`` when
    no model was found.  ``camera`` is updated in place (focal from the ladder, then the refinement)."""
    eo = estimation_options or AbsolutePoseEstimationOptions()
    ro = refinement_options or AbsolutePoseRefinementOptions()
    dev = _dev()
    model = _ba.camera_model_id(camera.model)
    p2 = torch.from_numpy(np.asarray(points2D, dtype=np.float32))[None].to(dev)
    p3 = torch.from_numpy(np.asarray(points3D, dtype=np.float64)).to(dev)
    P = p3.shape[0]
    intr4 = torch.from_numpy(_cam4(camera)[None].copy()).to(dev)
    poses, focal, ninl, inl = _pr.absolute_pose_estimation_batched(p2, p3, torch.ones(1, P, dtype=torch.bool, device=dev), intr4, model,
                                                                   estimate_focal_length=eo.estimate_focal_length,
                                                                   max_error=eo.ransac.max_error)
    if int(ninl[0]) == 0:
        return None
    prm = camera.params.copy()
    prm[0] = float(focal[0])
    camera.params = prm
    E = poses[0].cpu().numpy()
    ans = pose_refinement(Rigid3d(Rotation3d(E[:, :3]), E[:, 3]), points2D, points3D, inl[0].cpu().numpy(), camera, ro)
    ans["num_inliers"] = int(ninl[0])
    ans["inliers"] = inl[0].cpu().numpy()
    return ans
