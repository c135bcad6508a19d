"""CPU oracle for absolute-pose refinement (motion-only BA) -- TEST INFRASTRUCTURE ONLY.

PARITY UNPINNED.  ``pycolmap.pose_refinement`` (pycolmap 3.10.0, pin: the reference's install.sh:41)
is COLMAP 3.10 ``RefineAbsolutePose`` (src/colmap/estimators/pose.cc) on Ceres 2.x; neither is
in the reference nor installable, and the reference holds no golden vectors for it.
Restated from the published algorithm [3P-memory]:
  * one ``ReprojErrorConstantPoint3DCostFunction<CameraModel>`` per inlier correspondence,
    wrapped in ``ceres::CauchyLoss(1.0)``;
  * quaternion manifold on the rotation, translation free, principal point constant, focal
    length / extra parameter refined per ``refine_focal_length`` / ``refine_extra_params``;
  * solver: DENSE_QR, gradient_tolerance 1.0, max_num_iterations 100, everything else Ceres
    defaults (function_tolerance 1e-6, parameter_tolerance 1e-8, radius 1e4, Jacobi scaling).
  * Ceres ``Corrector`` for a loss with rho'' <= 0: residual and Jacobian scaled by sqrt(rho').
Anchored on the reference's call sites vggsfm/utils/triangulation.py:260-479 (refine_pose) and
:482-647 (init_refine_pose): what goes in (pose, points2D, points3D, inlier_mask, camera,
options with refine_focal_length/refine_extra_params) and what is read back (cam_from_world,
camera.params).  Validated against scipy.optimize.least_squares(loss="cauchy") and finite
differences in tests/test_pose_oracle.py.

State layout as oracle/ba_oracle.py: pose [3,4] R|t, intr [4] = f,cx,cy,k, tangent columns
[delta(3) half-angle left perturbation, t(3), f, k].
"""
from __future__ import annotations

import dataclasses
import numpy as np

from .ba_oracle import SIMPLE_PINHOLE, SIMPLE_RADIAL, exp_so3

NO_CONVERGENCE, CONV_GRADIENT, CONV_FUNCTION, CONV_PARAMETER, MIN_RADIUS, FAILURE, SKIPPED = 0, 1, 2, 3, 4, 5, 6


@dataclasses.dataclass
class PoseOptions:
    """COLMAP AbsolutePoseRefinementOptions + Ceres defaults [3P-memory]."""
    max_num_iterations: int = 100
    function_tolerance: float = 1e-6
    gradient_tolerance: float = 1.0
    parameter_tolerance: float = 1e-8
    initial_trust_region_radius: float = 1e4
    max_trust_region_radius: float = 1e16
    min_trust_region_radius: float = 1e-32
    min_relative_decrease: float = 1e-3
    min_lm_diagonal: float = 1e-6
    max_lm_diagonal: float = 1e32
    max_num_consecutive_invalid_steps: int = 5
    loss_function_scale: float = 1.0


def residual_jacobian(pose, intr, X, uv, model):
    """Raw (uncorrected) residuals r[P,2] and Jacobian J[P,2,8] of one camera against constant points."""
    R, t = pose[:, :3], pose[:, 3]
    RX = X @ R.T
    p = RX + t
    iz = 1.0 / p[:, 2]
    u, v = p[:, 0] * iz, p[:, 1] * iz
    f, cx, cy = intr[0], intr[1], intr[2]
    k = intr[3] if model == SIMPLE_RADIAL else 0.0
    r2 = u * u + v * v
    d = 1.0 + k * r2
    r = np.stack([f * d * u + cx - uv[:, 0], f * d * v + cy - uv[:, 1]], axis=-1)
    a00 = f * (d + 2.0 * k * u * u)
    a01 = f * (2.0 * k * u * v)
    a11 = f * (d + 2.0 * k * v * v)
    Jp = np.zeros((len(X), 2, 3))
    Jp[:, 0, 0] = a00 * iz
    Jp[:, 0, 1] = a01 * iz
    Jp[:, 0, 2] = -(a00 * u + a01 * v) * iz
    Jp[:, 1, 0] = a01 * iz
    Jp[:, 1, 1] = a11 * iz
    Jp[:, 1, 2] = -(a01 * u + a11 * v) * iz
    J = np.zeros((len(X), 2, 8))
    a1, a2, a3 = RX[:, 0:1], RX[:, 1:2], RX[:, 2:3]
    J[:, :, 0] = 2.0 * (-a3 * Jp[:, :, 1] + a2 * Jp[:, :, 2])
    J[:, :, 1] = 2.0 * (a3 * Jp[:, :, 0] - a1 * Jp[:, :, 2])
    J[:, :, 2] = 2.0 * (-a2 * Jp[:, :, 0] + a1 * Jp[:, :, 1])
    J[:, :, 3:6] = Jp
    J[:, 0, 6] = d * u
    J[:, 1, 6] = d * v
    if model == SIMPLE_RADIAL:
        J[:, 0, 7] = f * u * r2
        J[:, 1, 7] = f * v * r2
    return r, J


def cauchy(s, a):
    """ceres::CauchyLoss(a): rho(s) = b log(1 + s/b), b = a^2.  Returns rho, rho'."""
    b = a * a
    return b * np.log1p(s / b), 1.0 / (1.0 + s / b)


def robust_cost(pose, intr, X, uv, model, a):
    r, _ = residual_jacobian(pose, intr, X, uv, model)
    rho, _ = cauchy(np.sum(r * r, axis=-1), a)
    return 0.5 * float(np.sum(rho))


def free_columns(model, refine_focal, refine_extra):
    free = np.ones(8, dtype=bool)
    free[6] = bool(refine_focal)
    free[7] = bool(refine_extra) and model == SIMPLE_RADIAL
    return free


def plus(pose, intr, delta):
    new_pose = pose.copy()
    new_pose[:, :3] = exp_so3(2.0 * delta[0:3]) @ pose[:, :3]
    new_pose[:, 3] = pose[:, 3] + delta[3:6]
    new_intr = intr.copy()
    new_intr[0] += delta[6]
    new_intr[3] += delta[7]
    return new_pose, new_intr


def pose_refinement(pose, intr, points3D, points2D, inlier_mask, model, refine_focal=True, refine_extra=True,
                    options: PoseOptions | None = None, trace: list | None = None):
    """pycolmap.pose_refinement(cam_from_world, points2D, points3D, inlier_mask, camera, options).

    Returns (pose[3,4], intr[4], summary dict).  Ceres TrustRegionMinimizer + LevenbergMarquardtStrategy
    semantics as in oracle/ba_oracle.lm_solve; the 8x8 damped normal equations are solved by Cholesky
    where Ceres uses QR on the stacked system (same minimiser of |J d + r|^2 + |D d|^2)."""
    opt = options or PoseOptions()
    pose = np.array(pose, dtype=np.float64)
    intr = np.array(intr, dtype=np.float64)
    m = np.asarray(inlier_mask, dtype=bool)
    X = np.asarray(points3D, dtype=np.float64)[m]
    uv = np.asarray(points2D, dtype=np.float64)[m]
    free = free_columns(model, refine_focal, refine_extra)
    a = opt.loss_function_scale

    def evaluate(pose, intr):
        r, J = residual_jacobian(pose, intr, X, uv, model)
        rho, rho1 = cauchy(np.sum(r * r, axis=-1), a)
        J = J * free[None, None, :]
        Jm = J.reshape(-1, 8)
        w = np.repeat(rho1, 2)
        H = Jm.T @ (Jm * w[:, None])
        g = Jm.T @ (r.reshape(-1) * w)
        return 0.5 * float(np.sum(rho)), H, g

    summary = {"iterations": 0, "successful": 0, "termination": NO_CONVERGENCE, "num_residuals": 2 * len(X)}
    if len(X) == 0:
        summary.update(initial_cost=0.0, final_cost=0.0, termination=CONV_GRADIENT)
        return pose, intr, summary
    cost, H, g = evaluate(pose, intr)
    summary["initial_cost"] = cost
    radius = opt.initial_trust_region_radius
    if not (np.isfinite(cost) and np.isfinite(g[free]).all()):
        # Ceres: the initial residual / Jacobian evaluation fails -> FAILURE before the first iteration [3P-memory]
        summary.update(final_cost=cost, final_radius=radius, termination=FAILURE)
        return pose, intr, summary
    sc = 1.0 / (1.0 + np.sqrt(np.diag(H)))
    decrease_factor = 2.0
    invalid = 0
    it = 0
    grad_max = float(np.max(np.abs(g[free])))
    if trace is not None:
        trace.append({"it": 0, "accepted": True, "cost": cost, "grad_max": grad_max})
    if grad_max <= opt.gradient_tolerance:
        summary.update(final_cost=cost, final_radius=radius, termination=CONV_GRADIENT)
        return pose, intr, summary
    while True:
        if it >= opt.max_num_iterations:
            break
        if radius < opt.min_trust_region_radius:
            summary["termination"] = MIN_RADIUS
            break
        it += 1
        Hs = H * sc[:, None] * sc[None, :]
        dd = np.clip(np.diag(Hs), opt.min_lm_diagonal, opt.max_lm_diagonal)
        A = Hs + np.diag(dd / radius)
        b = -g * sc
        A[~free, :] = 0.0
        A[:, ~free] = 0.0
        A[~free, ~free] = 1.0
        b[~free] = 0.0
        ok = True
        try:
            L = np.linalg.cholesky(A)
            y = np.linalg.solve(L.T, np.linalg.solve(L, b))
        except np.linalg.LinAlgError:
            ok = False
        if ok:
            delta = y * sc
            model_change = 0.5 * (np.sum(y * y * dd / radius * free) - np.sum(delta * g))
            ok = bool(np.all(np.isfinite(delta))) and model_change > 0
        if not ok:
            invalid += 1
            if invalid >= opt.max_num_consecutive_invalid_steps:
                summary["termination"] = FAILURE
                break
            radius *= 0.5
            if trace is not None:
                trace.append({"it": it, "invalid": True})
            continue
        invalid = 0
        c_pose, c_intr = plus(pose, intr, delta)
        c_cost = robust_cost(c_pose, c_intr, X, uv, model, a)
        # ambient norms: quaternion(4) + t(3) + camera params (f,cx,cy[,k])
        nd = np.linalg.norm(delta[0:3])
        step_norm = np.sqrt(2.0 - 2.0 * np.cos(nd) + np.sum(delta[3:8] ** 2))
        x_norm = np.sqrt(1.0 + np.sum(pose[:, 3] ** 2) + np.sum(intr[:3] ** 2) + (intr[3] ** 2 if model == SIMPLE_RADIAL else 0.0))
        cost_change = cost - c_cost
        rho = cost_change / model_change
        if trace is not None:
            trace.append({"it": it, "cost": cost, "candidate_cost": c_cost, "model_change": model_change, "rho": rho,
                          "radius": radius, "step_norm": step_norm, "x_norm": x_norm})
        if step_norm <= opt.parameter_tolerance * (x_norm + opt.parameter_tolerance):
            summary["termination"] = CONV_PARAMETER
            break
        if abs(cost_change) <= opt.function_tolerance * cost:
            # Ceres 2.x: FunctionToleranceReached() returns before HandleSuccessfulStep() -> candidate discarded
            summary["termination"] = CONV_FUNCTION
            break
        if rho > opt.min_relative_decrease:
            pose, intr = c_pose, c_intr
            cost, H, g = evaluate(pose, intr)
            summary["successful"] += 1
            radius = min(opt.max_trust_region_radius, radius / max(1.0 / 3.0, 1.0 - (2.0 * rho - 1.0) ** 3))
            decrease_factor = 2.0
            grad_max = float(np.max(np.abs(g[free])))
            if trace is not None:
                trace.append({"it": it, "accepted": True, "cost": cost, "grad_max": grad_max})
            if grad_max <= opt.gradient_tolerance:
                summary["termination"] = CONV_GRADIENT
                break
        else:
            radius /= decrease_factor
            decrease_factor *= 2.0
    summary["iterations"] = it
    summary["final_cost"] = cost
    summary["final_radius"] = radius
    return pose, intr, summary


def pose_refinement_batched(poses, intr, points3D, tracks2D, inlier, model, active, refine_focal, refine_extra,
                            options: PoseOptions | None = None):
    """Frame loop of refine_pose / init_refine_pose for per-frame cameras.  active/refine_* are [S] bools."""
    S = len(poses)
    out_p = np.array(poses, dtype=np.float64).copy()
    out_i = np.array(intr, dtype=np.float64).copy()
    summ = []
    for s in range(S):
        if not active[s]:
            summ.append({"termination": SKIPPED, "iterations": 0})
            continue
        out_p[s], out_i[s], sm = pose_refinement(out_p[s], out_i[s], points3D, tracks2D[s], inlier[s], model,
                                                  bool(refine_focal[s]), bool(refine_extra[s]), options)
        summ.append(sm)
    return out_p, out_i, summ


def frame_loop(poses, intr, points3D, tracks2D, inlier, active, model, shared_camera, max_reproj_error=0.0,
               min_inliers=0, options: PoseOptions | None = None, traces: list | None = None):
    """The python frame loop both reference callers share (triangulation.py:341-441, :542-608) in array form.

    * pre-filter (refine_pose only, :298-315): inlier AND depth > 0 AND squared reprojection error <= max^2,
      evaluated for ALL frames at the input cameras before the loop;
    * a frame is refined when active and its inlier count is > min_inliers;
    * shared camera: one camera object, created from frame 0's intrinsics, refined by frame 0 only
      (refine flags are switched off for ridx > 0, :373-375) and read back for every frame.
    Returns (poses, intr, used_mask, summaries).  ``traces``: a list that receives one ``pose_refinement`` trace per
    frame (empty for a frame that is not refined)."""
    poses = np.array(poses, dtype=np.float64).copy()
    intr = np.array(intr, dtype=np.float64).copy()
    S = len(poses)
    used = np.asarray(inlier, dtype=bool).copy()
    if max_reproj_error > 0:
        for s in range(S):
            r, _ = residual_jacobian(poses[s], intr[s], np.asarray(points3D, np.float64), np.asarray(tracks2D[s], np.float64), model)
            e = np.sum(r * r, axis=-1)
            pz = (np.asarray(points3D, np.float64) @ poses[s][:, :3].T + poses[s][:, 3])[:, 2]
            e[pz <= 0] = 1e9
            used[s] &= e <= max_reproj_error ** 2
    summ = []
    cam = intr[0].copy() if shared_camera else None
    for s in range(S):
        if shared_camera:
            intr[s] = cam
        rf = (not shared_camera) or s == 0
        trace = []
        if traces is not None:
            traces.append(trace)
        if active[s] and used[s].sum() > min_inliers:
            poses[s], intr[s], sm = pose_refinement(poses[s], intr[s], points3D, tracks2D[s], used[s], model, rf, rf, options,
                                                    trace)
            if shared_camera:
                cam = intr[s].copy()
        else:
            sm = {"termination": SKIPPED if not active[s] else 7, "iterations": 0}
        summ.append(sm)
    return poses, intr, used, summ
