"""CPU oracle for the bundle-adjustment half of the hot path -- TEST INFRASTRUCTURE ONLY.

PARITY UNPINNED.  The arithmetic restated here lives in third-party engines that are not
in the reference and could not be installed:
  * pycolmap 3.10.0 (pin: the reference's install.sh:41) -- COLMAP 3.10
    ``BundleAdjustmentController::Run`` / ``BundleAdjuster`` / ``ReprojErrorCostFunction`` /
    ``SimplePinholeCameraModel`` / ``SimpleRadialCameraModel`` / ``Reconstruction::Normalize``
  * pyceres 2.3 (install.sh:42) -- Ceres 2.x ``TrustRegionMinimizer`` +
    ``LevenbergMarquardtStrategy`` + (DENSE|SPARSE)_SCHUR.
The reference holds no golden vectors at this boundary (SURVEY.md section 8c), so this file
restates the published algorithm and is anchored on the reference's own call sites:
  vggsfm/utils/triangulation.py:1020-1073 (global_BA), :1076-1209 (iterative_global_BA),
  :1212-1218 (filter_reconstruction -> normalize(5.0, 0.1, 0.9, True)),
  vggsfm/utils/tensor_to_pycolmap.py:16-160 (what goes in), :163-214 (what comes out),
  vggsfm/utils/triangulation_helpers.py:626-635 (option preset),
  vggsfm/utils/triangulation_helpers.py:358-395 + vggsfm/utils/distortion.py:102-123
  (the in-repo statement of the same projection model).
It is validated against scipy.optimize.least_squares and finite differences in
tests/test_ba_oracle.py.

State layout (shared with the CUDA path, see DESIGN.md):
  poses   [S,3,4] float64   cam_from_world R|t
  intr    [S,4]   float64   f, cx, cy, k   (k ignored for SIMPLE_PINHOLE)
  points  [N,3]   float64
  uv      [S,N,2] float32-representable pixel observations, mask [S,N] bool
Camera tangent block (dc columns): [delta(3) half-angle left perturbation, t(3), f, k];
reduced-system index of frame s, column i is s*dc+i; shared intrinsics follow at S*dc.

LM control (lm_solve), as the CUDA loop (csrc/ba_solve.cu) must follow it:
  * terminations NO_CONVERGENCE, CONVERGENCE_GRADIENT / _FUNCTION / _PARAMETER, MIN_TRUST_REGION_RADIUS and
    FAILURE_INVALID_STEPS (max_num_consecutive_invalid_steps invalid steps in a row); the Python binding of the CUDA
    solver reports the same names.
  * a step is invalid when the linear solve fails or gives a non-finite step, or when the model change is not > 0;
    the radius then halves and decrease_factor is kept.
  * the gradient max-norm propagates NaN, so a NaN gradient never reads as converged.
  * trace: one dict per iteration with "outcome" 1 accepted / 0 rejected or terminating / 2 invalid and the radius
    the iteration ran with (an invalid step's halving shows in the next row); valid steps also carry cost_change and
    x_norm (|x| of ParameterToleranceReached), accepted steps the new gmax.  summary["initial_gmax"] is iteration 0's.
  * known differences from Ceres 2.x [3P-memory]: Ceres ends with FAILURE at iteration 0 when the initial residual
    evaluation fails (a NaN or inf observation); here such a problem runs into invalid steps instead (same
    termination, parameters unchanged).  Ceres gives a candidate that fails to evaluate the cost DBL_MAX, which
    rejects the step; here a non-finite candidate cost also makes rho non-finite and rejects it, but the CUDA loop
    counts it as an invalid step.  No input with a finite initial cost and float32 observations was found that makes
    the candidate cost non-finite, so that branch has no test (tests/test_ba_lm_edges_gpu.py).  A point block whose
    damped 3x3 Cholesky fails (a one-view point at radius >= 1e14) makes the CUDA step invalid, where Ceres inverts the
    block explicitly (DESIGN.md section 4.2); lm_solve here raises numpy's LinAlgError on it.
"""
from __future__ import annotations

import dataclasses
import numpy as np

SIMPLE_PINHOLE = 0
SIMPLE_RADIAL = 1

INTR_CONST = 0       # intrinsics not refined: dc = 6, ns = 0
INTR_PER_FRAME = 1   # one camera per frame: dc = 6 + ni, ns = 0
INTR_SHARED = 2      # one camera for all frames: dc = 6, ns = ni


def n_intr(model: int) -> int:
    return 1 if model == SIMPLE_PINHOLE else 2


def dims(model: int, mode: int):
    ni = n_intr(model)
    if mode == INTR_CONST:
        return 6, 0
    if mode == INTR_PER_FRAME:
        return 6 + ni, 0
    return 6, ni


@dataclasses.dataclass
class LMOptions:
    """Ceres solver options as COLMAP 3.10's BundleAdjustmentOptions sets them [3P-memory]."""
    max_num_iterations: int = 100
    function_tolerance: float = 0.0
    gradient_tolerance: float = 1e-4
    parameter_tolerance: float = 0.0
    initial_trust_region_radius: float = 1e4
    max_trust_region_radius: float = 1e16
    min_trust_region_radius: float = 1e-32
    min_relative_decrease: float = 1e-3
    min_lm_diagonal: float = 1e-6
    max_lm_diagonal: float = 1e32
    max_num_consecutive_invalid_steps: int = 10
    jacobi_scaling: bool = True

    @staticmethod
    def prepare_ba_options() -> "LMOptions":
        """vggsfm/utils/triangulation_helpers.py:626-635: tolerances x10, 50 iterations."""
        o = LMOptions()
        o.function_tolerance *= 10
        o.gradient_tolerance *= 10
        o.parameter_tolerance *= 10
        o.max_num_iterations = 50
        return o


# ----------------------------------------------------------------------------------------------
# projection model and analytic Jacobians
# ----------------------------------------------------------------------------------------------

def project(poses, intr, points, model):
    """COLMAP SimplePinhole/SimpleRadial ImgFromCam of R X + t.  Returns uvhat[S,N,2], depth[S,N]."""
    R = poses[:, :, :3]
    t = poses[:, :, 3]
    p = np.einsum("sij,nj->sni", R, points) + t[:, None, :]
    with np.errstate(divide="ignore", invalid="ignore"):
        u = p[..., 0] / p[..., 2]
        v = p[..., 1] / p[..., 2]
    f = intr[:, 0][:, None]
    cx = intr[:, 1][:, None]
    cy = intr[:, 2][:, None]
    if model == SIMPLE_RADIAL:
        k = intr[:, 3][:, None]
        d = 1.0 + k * (u * u + v * v)
    else:
        d = 1.0
    return np.stack([f * d * u + cx, f * d * v + cy], axis=-1), p[..., 2]


def residuals_and_jacobians(poses, intr, points, uv, mask, model):
    """Per-observation residual r[S,N,2] and Jacobians wrt the camera tangent block
    (all 8 columns: delta(3), t(3), f, k) and the point: Jc[S,N,2,8], Jp[S,N,2,3].
    Masked-out observations give exact zeros, selected with np.where rather than multiplied by the mask: their uv,
    their point and their camera may be NaN or inf (ba_blocks_ref.c skips them, csrc/ba_obs.h selects)."""
    S, N = mask.shape
    R = poses[:, :, :3]
    t = poses[:, :, 3]
    RX = np.einsum("sij,nj->sni", R, points)
    p = RX + t[:, None, :]
    pz = np.where(mask, p[..., 2], 1.0)
    iz = 1.0 / pz
    u = p[..., 0] * iz
    v = p[..., 1] * iz
    f = intr[:, 0][:, None]
    cx = intr[:, 1][:, None]
    cy = intr[:, 2][:, None]
    k = intr[:, 3][:, None] if model == SIMPLE_RADIAL else np.zeros((S, 1))
    r2 = u * u + v * v
    d = 1.0 + k * r2
    res = np.stack([f * d * u + cx - uv[..., 0], f * d * v + cy - uv[..., 1]], axis=-1)

    # d(uhat,vhat)/d(u,v) = f * A
    a00 = f * (d + 2.0 * k * u * u)
    a01 = f * (2.0 * k * u * v)
    a11 = f * (d + 2.0 * k * v * v)
    # d(u,v)/dp = iz * [[1,0,-u],[0,1,-v]]
    Jproj = np.zeros((S, N, 2, 3))
    Jproj[..., 0, 0] = a00 * iz
    Jproj[..., 0, 1] = a01 * iz
    Jproj[..., 0, 2] = -(a00 * u + a01 * v) * iz
    Jproj[..., 1, 0] = a01 * iz
    Jproj[..., 1, 1] = a11 * iz
    Jproj[..., 1, 2] = -(a01 * u + a11 * v) * iz

    Jp = np.einsum("snij,sjk->snik", Jproj, R)
    Jc = np.zeros((S, N, 2, 8))
    # dp/d(delta) = -2 [RX]_x   (Ceres QuaternionManifold::Plus: q_new = [cos|d|, sinc d] * q)
    a1, a2, a3 = RX[..., 0], RX[..., 1], RX[..., 2]
    Jc[..., 0] = 2.0 * (-a3[..., None] * Jproj[..., 1] + a2[..., None] * Jproj[..., 2])
    Jc[..., 1] = 2.0 * (a3[..., None] * Jproj[..., 0] - a1[..., None] * Jproj[..., 2])
    Jc[..., 2] = 2.0 * (-a2[..., None] * Jproj[..., 0] + a1[..., None] * Jproj[..., 1])
    Jc[..., 3:6] = Jproj
    Jc[..., 0, 6] = d * u
    Jc[..., 1, 6] = d * v
    if model == SIMPLE_RADIAL:
        Jc[..., 0, 7] = f * u * r2
        Jc[..., 1, 7] = f * v * r2
    keep = mask[..., None, None]
    return np.where(mask[..., None], res, 0.0), np.where(keep, Jc, 0.0), np.where(keep, Jp, 0.0)


def build_blocks(poses, intr, points, uv, mask, model, mode, point_const=None):
    """Normal-equation blocks of 0.5*sum|r|^2 (what the fused CUDA kernel emits).

    Returns dict: cost, g_c[S,dc], H_cc[S,dc,dc], g_p[N,3], H_pp[N,3,3], W[S,dc,N,3],
    and for INTR_SHARED also g_s[ns], H_ss[ns,ns], H_cs[S,6,ns], W_s[ns,N,3]."""
    dc, ns = dims(model, mode)
    ni = n_intr(model)
    res, Jc8, Jp = residuals_and_jacobians(poses, intr, points, uv, mask, model)
    if point_const is not None:
        Jp = np.where(np.asarray(point_const, dtype=bool)[None, :, None, None], 0.0, Jp)
    Jc = Jc8[..., :dc]
    out = {
        "cost": 0.5 * float(np.sum(res * res)),
        "g_c": np.einsum("snri,snr->si", Jc, res),
        "H_cc": np.einsum("snri,snrj->sij", Jc, Jc),
        "g_p": np.einsum("snri,snr->ni", Jp, res),
        "H_pp": np.einsum("snri,snrj->nij", Jp, Jp),
        "W": np.einsum("snri,snrj->sinj", Jc, Jp),
    }
    if mode == INTR_SHARED:
        Js = Jc8[..., 6:6 + ni]
        out["g_s"] = np.einsum("snri,snr->i", Js, res)
        out["H_ss"] = np.einsum("snri,snrj->ij", Js, Js)
        out["H_cs"] = np.einsum("snri,snrj->sij", Jc, Js)
        out["W_s"] = np.einsum("snri,snrj->inj", Js, Jp)
    return out


_C_LIB = None


def _load_c():
    """oracle/_build/libba_blocks_ref.so (oracle/ba_blocks_ref.c) if it has been built, else None."""
    global _C_LIB
    if _C_LIB is None:
        import ctypes
        import os
        path = os.path.join(os.path.dirname(os.path.abspath(__file__)), "_build", "libba_blocks_ref.so")
        _C_LIB = ctypes.CDLL(path) if os.path.exists(path) else False
    return _C_LIB or None


def build_blocks_c(poses, intr, points, uv, mask, model, mode, point_const=None):
    """Same outputs as build_blocks(), evaluated by the C/OpenMP restatement (oracle/ba_blocks_ref.c)."""
    import ctypes
    lib = _load_c()
    if lib is None:
        raise RuntimeError("oracle/_build/libba_blocks_ref.so not built (make -C oracle)")
    S, N = mask.shape
    dc, ns = dims(model, mode)
    c = lambda a, dt=np.float64: np.ascontiguousarray(a, dtype=dt)
    uvc, mk, po, it, pt = c(uv), c(mask, np.uint8), c(poses), c(intr), c(points)
    pcn = c(point_const, np.uint8) if point_const is not None else None
    Wfull = np.empty((S * dc + max(ns, 1), N, 3))        # camera rows then shared rows, one allocation
    out = {"g_c": np.empty((S, dc)), "H_cc": np.empty((S, dc, dc)), "g_p": np.empty((N, 3)), "H_pp": np.empty((N, 3, 3)),
           "W": Wfull[:S * dc].reshape(S, dc, N, 3), "W_full": Wfull[:S * dc + ns]}
    cost = np.zeros(1)
    g_s, H_ss = np.zeros(2), np.zeros(4)
    H_cs = np.zeros((S, 6, max(ns, 1)))
    W_s = Wfull[S * dc:]
    P = lambda a: a.ctypes.data_as(ctypes.c_void_p)
    rc = lib.ba_blocks_ref(S, N, P(uvc), P(mk), P(po), P(it), P(pt), P(pcn) if pcn is not None else None, model, mode,
                           P(cost), P(out["g_c"]), P(out["H_cc"]), P(out["g_p"]), P(out["H_pp"]), P(out["W"]), P(g_s),
                           P(H_ss), P(H_cs), P(W_s))
    if rc != 0:
        raise RuntimeError("ba_blocks_ref failed")
    out["cost"] = float(cost[0])
    if mode == INTR_SHARED:
        out["g_s"] = g_s[:ns].copy()
        out["H_ss"] = H_ss[:ns * ns].reshape(ns, ns).copy()
        out["H_cs"] = H_cs
        out["W_s"] = W_s
    return out


def cost_only(poses, intr, points, uv, mask, model):
    with np.errstate(invalid="ignore", over="ignore"):
        uvh, _ = project(poses, intr, points, model)
        r = np.where(mask[..., None], uvh - uv, 0.0)
    return 0.5 * float(np.sum(r * r))


# ----------------------------------------------------------------------------------------------
# manifold update
# ----------------------------------------------------------------------------------------------

def exp_so3(phi):
    """Rodrigues; phi [...,3] rotation vectors -> [...,3,3]."""
    th = np.linalg.norm(phi, axis=-1)
    small = th < 1e-12
    ths = np.where(small, 1.0, th)
    a = np.where(small, 1.0 - th * th / 6.0, np.sin(ths) / ths)
    b = np.where(small, 0.5 - th * th / 24.0, (1.0 - np.cos(ths)) / (ths * ths))
    K = np.zeros(phi.shape[:-1] + (3, 3))
    K[..., 0, 1] = -phi[..., 2]
    K[..., 0, 2] = phi[..., 1]
    K[..., 1, 0] = phi[..., 2]
    K[..., 1, 2] = -phi[..., 0]
    K[..., 2, 0] = -phi[..., 1]
    K[..., 2, 1] = phi[..., 0]
    return np.eye(3) + a[..., None, None] * K + b[..., None, None] * (K @ K)


def apply_step(poses, intr, points, d_cam, d_shared, d_pts, model, mode):
    """x (+) delta in the tangent parameterisation above.  d_cam [S,dc], d_shared [ns], d_pts [N,3].  A parameter whose
    step is exactly zero is copied (as cam_update_kernel / point_step_kernel do), so a constant or unobserved one comes
    back as given even when it is NaN or inf."""
    ni = n_intr(model)
    add = lambda x, d: np.where(d == 0.0, x, x + d)
    new_poses = poses.copy()
    rot = np.any(d_cam[:, 0:3] != 0.0, axis=1)[:, None, None]
    with np.errstate(invalid="ignore"):
        new_poses[:, :, :3] = np.where(rot, exp_so3(2.0 * d_cam[:, 0:3]) @ poses[:, :, :3], poses[:, :, :3])
    new_poses[:, :, 3] = add(poses[:, :, 3], d_cam[:, 3:6])
    new_intr = intr.copy()
    cols = [0, 3][:ni]
    if mode == INTR_PER_FRAME:
        for j, c in enumerate(cols):
            new_intr[:, c] = add(intr[:, c], d_cam[:, 6 + j])
    elif mode == INTR_SHARED:
        for j, c in enumerate(cols):
            new_intr[:, c] = add(intr[:, c], d_shared[j])
    return new_poses, new_intr, add(points, d_pts)


# ----------------------------------------------------------------------------------------------
# Levenberg-Marquardt with a direct Schur solve (Ceres semantics)
# ----------------------------------------------------------------------------------------------

def default_param_const(S, model, mode, refine_focal=True, refine_extra=True, gauge=True, const_pose=None):
    """uint8[D] mask of constant reduced parameters.  Gauge as COLMAP's
    BundleAdjustmentController::Run [3P-memory]: first image pose constant, x of the second
    image's translation constant."""
    dc, ns = dims(model, mode)
    D = S * dc + ns
    c = np.zeros(D, dtype=bool)
    if gauge:
        c[0:6] = True
        if S > 1:
            c[dc + 3] = True
    if const_pose is not None:
        for s in np.nonzero(const_pose)[0]:
            c[s * dc:s * dc + 6] = True
    ni = n_intr(model)
    flags = [refine_focal, refine_extra][:ni]
    for j, fl in enumerate(flags):
        if not fl:
            if mode == INTR_PER_FRAME:
                c[np.arange(S) * dc + 6 + j] = True
            elif mode == INTR_SHARED:
                c[S * dc + j] = True
    return c


def _assemble_camera_system(blk, S, dc, ns):
    """Dense [D,D] camera Hessian and [D] gradient from the compact blocks."""
    D = S * dc + ns
    H = np.zeros((D, D))
    g = np.zeros(D)
    for s in range(S):
        H[s * dc:(s + 1) * dc, s * dc:(s + 1) * dc] = blk["H_cc"][s]
    g[:S * dc] = blk["g_c"].reshape(-1)
    if ns:
        for s in range(S):
            H[s * dc:s * dc + 6, S * dc:] = blk["H_cs"][s]
            H[S * dc:, s * dc:s * dc + 6] = blk["H_cs"][s].T
        H[S * dc:, S * dc:] = blk["H_ss"]
        g[S * dc:] = blk["g_s"]
    return H, g


def _full_W(blk, S, dc, ns):
    """[D, N, 3] coupling blocks (camera rows then shared rows)."""
    if "W_full" in blk:
        return blk["W_full"]
    W = blk["W"].reshape(S * dc, *blk["W"].shape[2:])
    if ns:
        W = np.concatenate([W, blk["W_s"]], axis=0)
    return W


def _x_norm(poses, intr, points, S, dc, ns, param_const, point_const):
    """|x| of Ceres' reduced program in AMBIENT coordinates (TrustRegionMinimizer::ParameterToleranceReached uses
    x_norm_ = x_.norm()): every non-constant parameter block counts in full -- unit quaternion (1.0) and translation per
    image whose block is not constant (a block held partly constant through a SubsetManifold, e.g. the second image's
    translation or a camera with a fixed principal point, is still non-constant), camera parameter blocks (f,cx,cy[,k])
    unless no intrinsic is refined, free points. [3P-memory]"""
    cams, pts = _x_norm_parts(poses, intr, points, S, dc, ns, param_const, point_const)
    return np.sqrt(cams + pts)


def _x_norm_parts(poses, intr, points, S, dc, ns, param_const, point_const):
    """(camera part, point part) of |x|^2.  With track shards the camera part is the same on every rank and the point
    part covers this rank's points only: it has to be summed over the ranks before |x| is formed, or each rank tests
    the parameter tolerance against its own |x| and the ranks may stop at different iterations."""
    pc = np.asarray(param_const, dtype=bool)
    ni = dc - 6 if ns == 0 else ns
    nparam = 3 + (1 if ni == 2 else 0) if ni else 0
    tot = 0.0
    for s in range(S):
        c = pc[s * dc:(s + 1) * dc]
        if not c[0:3].all():
            tot += 1.0
        if not c[3:6].all():
            tot += float(np.sum(poses[s][:, 3] ** 2))
        if dc > 6 and not c[6:dc].all():
            tot += float(np.sum(intr[s][:3] ** 2)) + (float(intr[s][3] ** 2) if dc == 8 else 0.0)
    if ns and not pc[S * dc:].all():
        tot += float(np.sum(intr[0][:3] ** 2)) + (float(intr[0][3] ** 2) if ns == 2 else 0.0)
    free = ~np.asarray(point_const, dtype=bool)
    return tot, float(np.sum(points[free] ** 2))


def lm_solve(poses, intr, points, uv, mask, model, mode, param_const=None, point_const=None,
             options: LMOptions | None = None, trace: list | None = None, allreduce=None, use_c=False):
    """Ceres-style trust-region LM (TrustRegionMinimizer + LevenbergMarquardtStrategy) with the
    points eliminated by a Schur complement and the reduced camera system solved by Cholesky.

    ``allreduce`` (optional) is an object with ``.sum(ndarray) -> ndarray`` and ``.max(float) -> float``
    reducing across track shards; used by the world_size>1 gloo tests to check the sharding algebra.  Returns (poses, intr, points, summary)."""
    opt = options or LMOptions()
    S, N = mask.shape
    dc, ns = dims(model, mode)
    D = S * dc + ns
    ar = allreduce.sum if allreduce is not None else (lambda a: a)
    armax = allreduce.max if allreduce is not None else (lambda a: a)
    if param_const is None:
        param_const = default_param_const(S, model, mode)
    if point_const is None:
        point_const = np.zeros(N, dtype=bool)
    # A point that no valid observation sees, and every camera parameter of a frame that sees nothing, is not in Ceres'
    # problem: constant here whatever the flags say, so that its values (NaN or inf allowed) reach neither |x| nor the step.
    # Frames are summed over track shards (a frame is in the problem if any shard sees it).
    mask = np.asarray(mask, dtype=bool)
    point_const = np.asarray(point_const, dtype=bool) | ~mask.any(axis=0)
    frame_seen = np.asarray(ar(mask.any(axis=1).astype(np.float64))) != 0.0
    param_const = np.asarray(param_const, dtype=bool).copy()
    param_const[:S * dc] |= np.repeat(~frame_seen, dc)
    free_c = ~param_const

    def evaluate(poses, intr, points):
        blk = (build_blocks_c if use_c else build_blocks)(poses, intr, points, uv, mask, model, mode, point_const)
        Hc, gc = _assemble_camera_system(blk, S, dc, ns)
        return blk, Hc, gc

    import time as _time
    _t0 = _time.perf_counter()
    blk, Hc, gc = evaluate(poses, intr, points)
    _t_init = _time.perf_counter() - _t0        # initial evaluation (not an LM iteration): bench.py subtracts it
    cost = float(ar(np.array([blk["cost"]]))[0])
    Hc_diag = ar(np.diag(Hc).copy())
    gc_glob = ar(gc.copy())
    # Jacobi scaling, fixed at the initial point (Ceres: 1 / (1 + sqrt(sum J^2)))
    if opt.jacobi_scaling:
        sc_c = 1.0 / (1.0 + np.sqrt(Hc_diag))
        sc_p = 1.0 / (1.0 + np.sqrt(np.einsum("nii->ni", blk["H_pp"])))
    else:
        sc_c = np.ones(D)
        sc_p = np.ones((N, 3))

    def grad_max_norm(gc_glob, gp):
        a = np.max(np.abs(gc_glob[free_c])) if free_c.any() else 0.0
        b = np.max(np.abs(gp[~point_const])) if (~point_const).any() else 0.0
        return float(armax(np.max([a, b])))          # NaN propagates (Python's max() drops a NaN second argument)

    radius = opt.initial_trust_region_radius
    decrease_factor = 2.0
    summary = {"iterations": 0, "successful": 0, "initial_cost": cost, "termination": "NO_CONVERGENCE",
               "initial_eval_s": _t_init}
    gmax = grad_max_norm(gc_glob, blk["g_p"])
    summary["initial_gmax"] = gmax
    if gmax <= opt.gradient_tolerance:
        summary.update(termination="CONVERGENCE_GRADIENT", final_cost=cost)
        return poses, intr, points, summary
    invalid_steps = 0
    it = 0
    while True:
        if it >= opt.max_num_iterations:
            break
        if radius < opt.min_trust_region_radius:
            summary["termination"] = "MIN_TRUST_REGION_RADIUS"
            break
        it += 1
        # ---- point blocks: V = Dp H_pp Dp + diag(clamp(diag))/radius ; M = Dp L^-T
        Hpp_s = blk["H_pp"] * sc_p[:, :, None] * sc_p[:, None, :]
        dpp = np.clip(np.einsum("nii->ni", Hpp_s), opt.min_lm_diagonal, opt.max_lm_diagonal)
        V = Hpp_s + np.einsum("ni,ij->nij", dpp / radius, np.eye(3))
        V[point_const] = np.eye(3)
        L = np.linalg.cholesky(V)
        Linv = np.linalg.inv(L)
        M = sc_p[:, :, None] * np.transpose(Linv, (0, 2, 1))      # Dp L^-T
        M[point_const] = 0.0
        q = np.einsum("nji,nj->ni", M, blk["g_p"])                # L^-1 Dp g_p = M^T g_p
        # ---- Schur complement (local shard), then sum over shards
        W = _full_W(blk, S, dc, ns)                               # [D,N,3]
        Z = (W[:, :, 0:1] * M[None, :, 0, :] + W[:, :, 1:2] * M[None, :, 1, :] + W[:, :, 2:3] * M[None, :, 2, :]).reshape(D, N * 3)
        S_raw = Hc - Z @ Z.T
        rhs_raw = -(gc - Z @ q.reshape(-1))
        S_raw = ar(S_raw)
        rhs_raw = ar(rhs_raw)
        # ---- scale, damp, fix gauge, solve
        dcc = np.clip(Hc_diag * sc_c * sc_c, opt.min_lm_diagonal, opt.max_lm_diagonal)
        A = S_raw * sc_c[:, None] * sc_c[None, :] + np.diag(dcc / radius)
        b = rhs_raw * sc_c
        A[param_const, :] = 0.0
        A[:, param_const] = 0.0
        A[param_const, param_const] = 1.0
        b[param_const] = 0.0
        ok = True
        try:
            Lc = np.linalg.cholesky(A)
            y = np.linalg.solve(Lc, b)
            dcs = np.linalg.solve(Lc.T, y)                          # scaled camera step
        except np.linalg.LinAlgError:
            ok = False
        if ok and not np.all(np.isfinite(dcs)):
            ok = False
        if not ok:
            invalid_steps += 1
            if trace is not None:
                trace.append({"it": it, "invalid": True, "outcome": 2, "cost": cost, "radius": radius})
            if invalid_steps >= opt.max_num_consecutive_invalid_steps:
                summary["termination"] = "FAILURE_INVALID_STEPS"
                break
            radius *= 0.5
            continue
        d_c = dcs * sc_c                                           # unscaled camera step
        # ---- back-substitution: dp = M M^T (-(g_p + W^T d_c))
        w = np.tensordot(d_c, W, axes=(0, 0))
        ypt = -(blk["g_p"] + w)
        d_p = np.einsum("nij,nj->ni", M, np.einsum("nji,nj->ni", M, ypt))
        # ---- model cost change: 0.5*(delta^T D^2 delta - delta^T g)  (== -(J d)^T (f + J d/2))
        dps = d_p / np.where(sc_p == 0, 1.0, sc_p)
        # the point part of |x|^2 rides in the same reduction (a rank-local |x| would split the ranks' decisions)
        x_cams, x_pts = _x_norm_parts(poses, intr, points, S, dc, ns, param_const, point_const)
        pt_terms = np.array([np.sum(np.where(point_const[:, None], 0.0, dps * dps * dpp / radius)) - np.sum(d_p * blk["g_p"]),
                             np.sum(d_p * d_p), x_pts])
        pt_terms = ar(pt_terms)
        quad = np.sum(dcs * dcs * dcc / radius * free_c) - np.sum(d_c * gc_glob) + pt_terms[0]
        model_change = 0.5 * quad
        if not (model_change > 0):
            invalid_steps += 1
            if trace is not None:
                trace.append({"it": it, "invalid": True, "outcome": 2, "cost": cost, "radius": radius,
                              "model_change": model_change})
            if invalid_steps >= opt.max_num_consecutive_invalid_steps:
                summary["termination"] = "FAILURE_INVALID_STEPS"
                break
            radius *= 0.5
            continue
        invalid_steps = 0
        d_cam = d_c[:S * dc].reshape(S, dc)
        d_sh = d_c[S * dc:]
        c_poses, c_intr, c_points = apply_step(poses, intr, points, d_cam, d_sh, d_p, model, mode)
        c_blk, c_Hc, c_gc = evaluate(c_poses, c_intr, c_points)
        c_cost = float(ar(np.array([c_blk["cost"]]))[0])
        step_norm = float(np.sqrt(np.sum(d_c * d_c) + pt_terms[1]))
        cost_change = cost - c_cost
        rho = cost_change / model_change
        x_norm = np.sqrt(x_cams + pt_terms[2])
        rec = {"it": it, "cost": cost, "candidate_cost": c_cost, "model_change": model_change, "rho": rho,
               "radius": radius, "step_norm": step_norm, "cost_change": cost_change, "x_norm": x_norm, "outcome": 0}
        if trace is not None:
            trace.append(rec)
        if step_norm <= opt.parameter_tolerance * (x_norm + opt.parameter_tolerance):
            summary["termination"] = "CONVERGENCE_PARAMETER"
            break
        if abs(cost_change) <= opt.function_tolerance * cost:
            # Ceres 2.x: FunctionToleranceReached() returns before HandleSuccessfulStep() -> candidate discarded
            summary["termination"] = "CONVERGENCE_FUNCTION"
            break
        if rho > opt.min_relative_decrease:
            rec["outcome"] = 1
            poses, intr, points, cost = c_poses, c_intr, c_points, c_cost
            blk, Hc, gc = c_blk, c_Hc, c_gc
            Hc_diag = ar(np.diag(Hc).copy())
            gc_glob = ar(gc.copy())
            summary["successful"] += 1
            radius = min(opt.max_trust_region_radius, radius / max(1.0 / 3.0, 1.0 - (2.0 * rho - 1.0) ** 3))
            decrease_factor = 2.0
            gmax = grad_max_norm(gc_glob, blk["g_p"])
            rec["gmax"] = gmax
            if gmax <= opt.gradient_tolerance:
                summary["termination"] = "CONVERGENCE_GRADIENT"
                break
        else:
            radius = radius / decrease_factor
            decrease_factor *= 2.0
    summary["iterations"] = it
    summary["final_cost"] = cost
    summary["final_radius"] = radius
    return poses, intr, points, summary


# ----------------------------------------------------------------------------------------------
# COLMAP wrapper semantics around the solve
# ----------------------------------------------------------------------------------------------

def filter_negative_depth(poses, points, mask):
    """ObservationManager::FilterObservationsWithNegativeDepth [3P-memory]: drop observations whose
    depth r3.X + t3 < eps; deleting an observation from a track of length <= 2 deletes the point.
    Processed in image order then point2D order like COLMAP.  Returns (mask, point_alive)."""
    eps = np.finfo(np.float64).eps
    depth = np.einsum("sj,nj->sn", poses[:, 2, :3], points) + poses[:, 2, 3][:, None]
    mask = mask.copy()
    bad = mask & ~(depth >= eps)
    alive = np.ones(points.shape[0], dtype=bool)
    if bad.any():
        length = mask.sum(axis=0)
        for s, n in zip(*np.nonzero(bad)):
            if not alive[n]:
                continue
            if length[n] <= 2:
                alive[n] = False
                mask[:, n] = False
            else:
                mask[s, n] = False
                length[n] -= 1
    return mask, alive


def normalize(poses, points, extent=10.0, p0=0.1, p1=0.9, alive=None):
    """Reconstruction::Normalize(extent, p0, p1, use_images=True) [3P-memory]: similarity that puts
    the robust (p0..p1 percentile, float32-cast, per-axis sorted) bounding box of the projection
    centres at extent, centred on the mean of the kept sorted coordinates."""
    S = poses.shape[0]
    if S < 2:
        return poses, points
    R = poses[:, :, :3]
    t = poses[:, :, 3]
    centers = -np.einsum("sji,sj->si", R, t)
    c32 = np.sort(centers.astype(np.float32), axis=0)
    n = S
    P0 = int(p0 * (n - 1)) if n > 3 else 0
    P1 = int(p1 * (n - 1)) if n > 3 else n - 1
    bmin = c32[P0].astype(np.float64)
    bmax = c32[P1].astype(np.float64)
    mean = c32[P0:P1 + 1].astype(np.float64).sum(axis=0) / (P1 - P0 + 1)
    old_extent = np.linalg.norm(bmax - bmin)
    scale = 1.0 if old_extent < np.finfo(np.float64).eps else extent / old_extent
    tr = -scale * mean
    new_points = scale * points + tr
    if alive is not None:
        new_points = np.where(alive[:, None], new_points, points)
    new_poses = poses.copy()
    new_poses[:, :, 3] = scale * t - np.einsum("sij,j->si", R, tr)
    return new_poses, new_points


def bundle_adjustment(points3d, extrinsics, intrinsics, extra_params, tracks, masks,
                      shared_camera=False, camera_type="SIMPLE_PINHOLE", options: LMOptions | None = None,
                      max_points3D_val=3000.0, trace=None):
    """batch_matrix_to_pycolmap -> pycolmap.bundle_adjustment -> filter_reconstruction ->
    pycolmap_to_batch_matrix, on arrays (vggsfm/utils/triangulation.py:1033-1063).

    points3d [P,3], extrinsics [S,3,4], intrinsics [S,3,3], extra_params [S,1]|None,
    tracks [S,P,2], masks [S,P].  Returns (points3D [P',3], extrinsics, intrinsics, extra_params,
    valid_idx, summary) with P' = number of tracks having >= 2 inliers (ids compacted in order,
    tensor_to_pycolmap.py:62-70)."""
    model = SIMPLE_RADIAL if camera_type == "SIMPLE_RADIAL" else SIMPLE_PINHOLE
    if camera_type not in ("SIMPLE_PINHOLE", "SIMPLE_RADIAL"):
        raise ValueError(f"Camera type {camera_type} is not supported yet")
    masks = np.asarray(masks, dtype=bool)
    valid_idx = np.nonzero(masks.sum(axis=0) >= 2)[0]
    pts = np.asarray(points3d, dtype=np.float64)[valid_idx].copy()
    uv = np.asarray(tracks, dtype=np.float64)[:, valid_idx]
    m = masks[:, valid_idx].copy()
    # points with any coordinate >= max_points3D_val get no observations (tensor_to_pycolmap.py:131-133)
    m[:, ~(pts < max_points3D_val).all(axis=1)] = False
    poses = np.asarray(extrinsics, dtype=np.float64).copy()
    S = poses.shape[0]
    K = np.asarray(intrinsics, dtype=np.float64)
    intr = np.zeros((S, 4))
    intr[:, 0] = K[:, 0, 0]
    intr[:, 1] = K[:, 0, 2]
    intr[:, 2] = K[:, 1, 2]
    if model == SIMPLE_RADIAL:
        intr[:, 3] = np.asarray(extra_params, dtype=np.float64)[:, 0]
    mode = INTR_SHARED if shared_camera else INTR_PER_FRAME
    if shared_camera:
        intr[:] = intr[0]
    m, alive = filter_negative_depth(poses, pts, m)
    point_const = ~(m.any(axis=0))          # points without observations are not in the problem
    poses, intr, pts, summary = lm_solve(poses, intr, pts, uv, m, model, mode,
                                         point_const=point_const, options=options, trace=trace)
    poses, pts = normalize(poses, pts, 10.0, 0.1, 0.9, alive)    # BundleAdjustmentController::Run
    poses, pts = normalize(poses, pts, 5.0, 0.1, 0.9, alive)     # filter_reconstruction, triangulation.py:1217
    pts = np.where(alive[:, None], pts, 0.0)                     # deleted ids read back as zeros (:180-184)
    K_out = np.zeros((S, 3, 3))
    K_out[:, 0, 0] = intr[:, 0]
    K_out[:, 1, 1] = intr[:, 0]
    K_out[:, 0, 2] = intr[:, 1]
    K_out[:, 1, 2] = intr[:, 2]
    K_out[:, 2, 2] = 1.0
    extra_out = intr[:, 3:4].copy() if model == SIMPLE_RADIAL else None
    return pts, poses, K_out, extra_out, valid_idx, summary
