"""Bundle adjustment on device tensors -- the host-side mirror of the reference's BA call surface.

Replaces ``batch_matrix_to_pycolmap -> pycolmap.bundle_adjustment -> filter_reconstruction ->
pycolmap_to_batch_matrix`` (vggsfm/utils/triangulation.py:1033-1063, :1128-1165 and
vggsfm/utils/tensor_to_pycolmap.py:16-214): the O(S*P) Python object-graph marshalling and the CPU
Ceres solve become one C-ABI call, ``vgg_ba_solve``, on tensors that never leave the GPU.

PyTorch is used here for device memory, streams and a handful of index/compaction ops only; all
arithmetic of the solve runs in libvggsfm_b200.so.  There is no fallback path.
"""
from __future__ import annotations

import ctypes
import dataclasses
import threading
from typing import Optional

import torch

from . import _lib
from ._lib import BALinearSolver, BAOptions, BAProblem, BASummary

SIMPLE_PINHOLE = 0
SIMPLE_RADIAL = 1
INTR_CONST = 0
INTR_PER_FRAME = 1
INTR_SHARED = 2

LINEAR_SOLVER_TYPES = {"DENSE_SCHUR": 0, "ITERATIVE_SCHUR": 1}
# COLMAP's BundleAdjustmentOptions::LossFunctionType (VGG_LOSS_* of include/vggsfm_b200.h)
LOSS_FUNCTION_TYPES = {"TRIVIAL": 0, "SOFT_L1": 1, "CAUCHY": 2}
CG_TERMINATION = {0: "SUCCESS", 1: "NO_CONVERGENCE", 2: "FAILURE"}

TERMINATION = {0: "NO_CONVERGENCE", 1: "CONVERGENCE_GRADIENT", 2: "CONVERGENCE_FUNCTION",
               3: "CONVERGENCE_PARAMETER", 4: "MIN_TRUST_REGION_RADIUS", 5: "FAILURE_INVALID_STEPS"}


def camera_model_id(camera_type: str) -> int:
    if camera_type == "SIMPLE_PINHOLE":
        return SIMPLE_PINHOLE
    if camera_type == "SIMPLE_RADIAL":
        return SIMPLE_RADIAL
    # same error as tensor_to_pycolmap.py:97-100
    raise ValueError(f"Camera type {camera_type} is not supported yet")


def dims(model: int, mode: int):
    dc, ns = ctypes.c_int(), ctypes.c_int()
    _lib.check(_lib.lib().vgg_ba_dims(model, mode, ctypes.byref(dc), ctypes.byref(ns)), "vgg_ba_dims")
    return dc.value, ns.value


def default_options() -> BAOptions:
    """pycolmap.BundleAdjustmentOptions() defaults (triangulator.py:254, triangulation.py:1128-1129)."""
    o = BAOptions()
    _lib.lib().vgg_ba_default_options(ctypes.byref(o))
    return o


def prepare_ba_options() -> BAOptions:
    """vggsfm/utils/triangulation_helpers.py:626-635."""
    o = default_options()
    o.function_tolerance *= 10
    o.gradient_tolerance *= 10
    o.parameter_tolerance *= 10
    o.max_num_iterations = 50
    return o


def default_param_const(S: int, model: int, mode: int, device, refine_focal_length=True, refine_extra_params=True,
                        gauge=True, const_pose: Optional[torch.Tensor] = None) -> torch.Tensor:
    """uint8[D]: COLMAP's gauge (first pose constant, x of the second translation constant) plus
    refine_* flags and explicitly constant poses (video_runner.py:817-819)."""
    dc, ns = dims(model, mode)
    c = torch.zeros(S * dc + ns, dtype=torch.uint8)
    if gauge:
        c[0:6] = 1
        if S > 1:
            c[dc + 3] = 1
    if const_pose is not None:
        for s in torch.nonzero(const_pose.cpu()).flatten().tolist():
            c[s * dc:s * dc + 6] = 1
    ni = 1 if model == SIMPLE_PINHOLE else 2
    for j, fl in enumerate([refine_focal_length, refine_extra_params][:ni]):
        if not fl:
            if mode == INTR_PER_FRAME:
                c[torch.arange(S) * dc + 6 + j] = 1
            elif mode == INTR_SHARED:
                c[S * dc + j] = 1
    return c.to(device)


def linear_solver(linear_solver_type="DENSE_SCHUR", min_linear_solver_iterations=0, max_linear_solver_iterations=500,
                  eta=0.1) -> BALinearSolver:
    """Ceres' linear-solver options of the LM loop (defaults: Ceres' own).  ITERATIVE_SCHUR runs preconditioned CG on the
    reduced camera system without forming it (SCHUR_JACOBI), for problems whose dense reduced system does not fit."""
    if linear_solver_type not in LINEAR_SOLVER_TYPES:
        raise ValueError(f"linear_solver_type must be one of {sorted(LINEAR_SOLVER_TYPES)}, not {linear_solver_type!r}")
    lin = BALinearSolver()
    _lib.lib().vgg_ba_default_linear_solver(ctypes.byref(lin))
    lin.type = LINEAR_SOLVER_TYPES[linear_solver_type]
    lin.min_linear_solver_iterations = int(min_linear_solver_iterations)
    lin.max_linear_solver_iterations = int(max_linear_solver_iterations)
    lin.eta = float(eta)
    return lin


def workspace_bytes(S: int, N: int, model: int, mode: int, iterative: bool = False, obs: bool = False) -> int:
    """Bytes of the solve's workspace: vgg_ba_workspace_bytes (direct), vgg_ba_workspace_bytes_iterative, or with obs
    vgg_ba_workspace_bytes_obs (the iterative solve on an observation list)."""
    nbytes = ctypes.c_size_t()
    L = _lib.lib()
    fn = L.vgg_ba_workspace_bytes_obs if obs else L.vgg_ba_workspace_bytes_iterative if iterative else \
        L.vgg_ba_workspace_bytes
    _lib.check(fn(S, N, model, mode, ctypes.byref(nbytes)), fn.__name__)
    return nbytes.value


_ws_local = threading.local()


def workspace(S: int, N: int, model: int, mode: int, device, iterative: bool = False, obs: bool = False) -> torch.Tensor:
    """The solve's workspace, cached by shape per host thread, as the library's own caches are: two threads solving
    the same shape (track-shard ranks in one process) never share one."""
    cache = _ws_local.__dict__.setdefault("cache", {})
    key = (S, N, model, mode, str(device), iterative, obs)
    ws = cache.get(key)
    if ws is None:
        with torch.cuda.device(device):
            nbytes = ctypes.c_size_t(workspace_bytes(S, N, model, mode, iterative, obs))
        if len(cache) > 4:
            cache.clear()
        ws = torch.empty(nbytes.value, dtype=torch.uint8, device=device)
        cache[key] = ws
    return ws


def loss_function_id(loss_function_type: str) -> int:
    """VGG_LOSS_* of one of COLMAP's loss names: TRIVIAL, SOFT_L1 or CAUCHY."""
    if loss_function_type not in LOSS_FUNCTION_TYPES:
        raise ValueError(f"loss_function_type must be one of {sorted(LOSS_FUNCTION_TYPES)}, not {loss_function_type!r}")
    return LOSS_FUNCTION_TYPES[loss_function_type]


def _problem(uv, mask, poses, intr, points, model, mode, param_const, point_const, loss_function_type="TRIVIAL",
             loss_function_scale=1.0):
    S, N = mask.shape
    assert uv.dtype == torch.float32 and uv.is_contiguous() and uv.shape == (S, N, 2)
    assert mask.dtype == torch.uint8 and mask.is_contiguous()
    for t in (poses, intr, points):
        assert t.dtype == torch.float64 and t.is_contiguous() and t.is_cuda
    assert poses.shape == (S, 3, 4) and intr.shape == (S, 4) and points.shape == (N, 3)
    p = BAProblem()
    p.S, p.N, p.camera_model, p.intr_mode = S, N, model, mode
    p.uv, p.mask = uv.data_ptr(), mask.data_ptr()
    p.param_const = param_const.data_ptr() if param_const is not None else None
    p.point_const = point_const.data_ptr() if point_const is not None else None
    p.poses, p.intr, p.points = poses.data_ptr(), intr.data_ptr(), points.data_ptr()
    p.loss_function_type = loss_function_id(loss_function_type)
    p.loss_function_scale = float(loss_function_scale)
    return p


def build_blocks(uv, mask, poses, intr, points, model, mode, point_const=None, tracks_per_warp=0,
                 loss_function_type="TRIVIAL", loss_function_scale=1.0):
    """One launch of the fused residual+Jacobian+block kernel (vgg_ba_build_blocks).  Returns a dict of
    device tensors: cost[1], camrec[S,KR], g_p[N,3], H_pp[N,6], W[N,pitch,3] (track-major, pitch = D rounded
    up to even), shared[8].  ``tracks_per_warp``: 0 lets the library choose; otherwise a positive multiple of 4
    (the kernel loads the observations of 4 tracks at a time), anything else raises.  With a robust loss the blocks
    are those of the corrected residuals and Jacobians and the cost is 0.5 sum rho (as lm_solve)."""
    L = _lib.lib()
    S, N = mask.shape
    dc, ns = dims(model, mode)
    KR = L.vgg_ba_camrec_len(model, mode)
    dev = uv.device
    # the five accumulators carved back to back (cost | shared | camrec | g_p | H_pp, 32-double aligned) like the
    # solver's own workspace, so the library zeroes them with ONE memset
    al = lambda n: (n + 31) // 32 * 32
    offs, tot = {}, 0
    for name, n in (("cost", 8), ("shared", 8), ("camrec", S * KR), ("g_p", N * 3), ("H_pp", N * 6)):
        offs[name] = (tot, n)
        tot += al(n)
    flat = torch.empty(tot, dtype=torch.float64, device=dev)
    view = lambda name, shape: flat[offs[name][0]:offs[name][0] + offs[name][1]].view(*shape)
    out = {
        "cost": view("cost", (8,))[:1],
        "camrec": view("camrec", (S, KR)),
        "g_p": view("g_p", (N, 3)),
        "H_pp": view("H_pp", (N, 6)),
        "W": torch.empty(N, (S * dc + ns + 1) // 2 * 2, 3, dtype=torch.float64, device=dev),
        "shared": view("shared", (8,)),
    }
    p = _problem(uv, mask, poses, intr, points, model, mode, None, point_const, loss_function_type, loss_function_scale)
    with torch.cuda.device(dev):
        st = torch.cuda.current_stream().cuda_stream
        _lib.check(L.vgg_ba_build_blocks(ctypes.byref(p), out["cost"].data_ptr(), out["camrec"].data_ptr(),
                                         out["g_p"].data_ptr(), out["H_pp"].data_ptr(), out["W"].data_ptr(),
                                         out["shared"].data_ptr(), tracks_per_warp, st), "vgg_ba_build_blocks")
    return out


def schur(uv, mask, poses, intr, points, model, mode, blocks, scale_p, radius, min_diag=1e-6, max_diag=1e32,
          point_const=None, loss_function_type="TRIVIAL", loss_function_scale=1.0):
    """Schur complement of `blocks` (vgg_ba_schur; the coupling blocks are rebuilt from the observations and the
    state, so blocks["W"] is not read; pass the loss `blocks` were built with).  Returns (Sraw[D,Dpad] lower-valid,
    rhs[D])."""
    L = _lib.lib()
    S, N = mask.shape
    dc, ns = dims(model, mode)
    D = S * dc + ns
    Dpad = (D + 2 + 127) // 128 * 128          # same rule as csrc/ba_solve.cu make_layout
    dev = uv.device
    ws = workspace(S, N, model, mode, dev)
    Sraw = torch.empty(D, Dpad, dtype=torch.float64, device=dev)
    rhs = torch.empty(Dpad, dtype=torch.float64, device=dev)
    p = _problem(uv, mask, poses, intr, points, model, mode, None, point_const, loss_function_type, loss_function_scale)
    dpad = ctypes.c_int()
    with torch.cuda.device(dev):
        st = torch.cuda.current_stream().cuda_stream
        _lib.check(L.vgg_ba_schur(ctypes.byref(p), blocks["camrec"].data_ptr(), blocks["g_p"].data_ptr(),
                                  blocks["H_pp"].data_ptr(), blocks["shared"].data_ptr(),
                                  scale_p.data_ptr(), radius, min_diag, max_diag, ws.data_ptr(), ws.numel(),
                                  Sraw.data_ptr(), rhs.data_ptr(), ctypes.byref(dpad), st), "vgg_ba_schur")
    assert dpad.value == Dpad
    return Sraw, rhs[:D]


@dataclasses.dataclass
class Summary:
    iterations: int
    successful: int
    termination: str
    initial_cost: float
    final_cost: float
    final_radius: float
    device_ms: float
    kernel_launches: int
    trace: Optional[torch.Tensor] = None
    linear_solver: str = "DENSE_SCHUR"
    cg_iterations: int = 0                    # CG iterations over all LM iterations (ITERATIVE_SCHUR)
    cg_trace: Optional[torch.Tensor] = None   # [iterations, 4]: CG iterations, termination (CG_TERMINATION), zeta, |r|/|b|
    alive: Optional[torch.Tensor] = None      # [P'] points the negative-depth filter kept (bundle_adjustment only)
    mask: Optional[torch.Tensor] = None       # [S,P'] observations that were in the problem (bundle_adjustment only)
    keep: Optional[torch.Tensor] = None       # [M] observations that were in the problem (bundle_adjustment_obs only)


def check_allreduce(allreduce, linear_solver_type="DENSE_SCHUR"):
    """ValueError, before anything runs, for a hook lm_solve cannot use: an object without a callable ``bind``, or a hook
    with a fabric attached together with ITERATIVE_SCHUR (the fabric reduces the dense reduced system, which the
    iterative solve never forms)."""
    if allreduce is None:
        return
    if not callable(getattr(allreduce, "bind", None)):
        raise ValueError(f"allreduce must be an all-reduce hook with a bind(workspace) method "
                         f"(vggsfm_b200.dist.AllReduceHook), not {type(allreduce).__name__}")
    if linear_solver_type == "ITERATIVE_SCHUR" and getattr(allreduce, "fabric", None) is not None:
        raise ValueError("ITERATIVE_SCHUR reduces through the all-reduce hook, not a fabric: pass AllReduceHook() "
                         "without a fabric")


def lm_solve(uv, mask, poses, intr, points, model, mode, param_const=None, point_const=None,
             options: Optional[BAOptions] = None, allreduce=None, want_trace=False, linear_solver_type="DENSE_SCHUR",
             min_linear_solver_iterations=0, max_linear_solver_iterations=500, eta=0.1, loss_function_type="TRIVIAL",
             loss_function_scale=1.0) -> Summary:
    """In-place Levenberg-Marquardt on device tensors (vgg_ba_solve).  `allreduce` is a
    vggsfm_b200.dist.AllReduceHook for track-sharded multi-GPU runs.  A rank whose shard holds no track (N = 0:
    shard_range gives empty tail shards when the tracks are few) still takes part in every reduction: it solves 16
    masked-out padding tracks, as bundle_adjustment() pads, and leaves its empty `points` untouched.
    linear_solver_type="ITERATIVE_SCHUR" solves each step by PCG (vgg_ba_solve_iterative_sharded) with the three CG
    options, on one GPU or, with `allreduce`, over track shards: every rank sums its assembly once per LM iteration and
    the Schur part of every CG matvec through the hook, and all ranks take the same CG and LM decisions.  A hook with a
    fabric attached raises ValueError with ITERATIVE_SCHUR, and so does an object without a callable ``bind``, before
    anything runs.
    loss_function_type / loss_function_scale: COLMAP's BundleAdjustmentOptions loss (TRIVIAL, SOFT_L1 or CAUCHY at a
    scale in pixels) on every observation; the costs of the summary are then 0.5 sum rho(|r|^2).  An unknown name raises
    ValueError, a robust loss with a scale that is not finite and > 0 raises from the library before anything runs."""
    loss_function_id(loss_function_type)
    lin = linear_solver(linear_solver_type, min_linear_solver_iterations, max_linear_solver_iterations, eta)
    iterative = linear_solver_type == "ITERATIVE_SCHUR"
    check_allreduce(allreduce, linear_solver_type)
    L = _lib.lib()
    S, N = mask.shape
    dev = uv.device
    if param_const is None:
        param_const = default_param_const(S, model, mode, dev)
    if N == 0:
        n = pad_tracks(1)
        uv = torch.zeros(S, n, 2, dtype=torch.float32, device=dev)
        mask = torch.zeros(S, n, dtype=torch.uint8, device=dev)
        points = torch.zeros(n, 3, dtype=torch.float64, device=dev)
        points[:, 2] = 1.0
        point_const = torch.ones(n, dtype=torch.uint8, device=dev)
        N = n
    opt = options or default_options()
    ws = workspace(S, N, model, mode, dev, iterative=True) if iterative else workspace(S, N, model, mode, dev)
    p = _problem(uv, mask, poses, intr, points, model, mode, param_const, point_const, loss_function_type,
                 loss_function_scale)
    summ = BASummary()
    trace = torch.zeros(max(1, opt.max_num_iterations), 8, dtype=torch.float64) if want_trace else None
    cg_trace = torch.zeros(max(1, opt.max_num_iterations), 4, dtype=torch.float64) if iterative else None
    cb = allreduce.bind(ws) if allreduce is not None else _lib.ALLREDUCE_FN()
    fabric = getattr(allreduce, "fabric", None)
    with torch.cuda.device(dev):
        st = torch.cuda.current_stream().cuda_stream
        if iterative:
            rc = L.vgg_ba_solve_iterative_sharded(ctypes.byref(p), ctypes.byref(opt), ctypes.byref(lin), ws.data_ptr(),
                                                  ws.numel(), cb, None, ctypes.byref(summ),
                                                  trace.data_ptr() if trace is not None else None, cg_trace.data_ptr(),
                                                  st)
        elif fabric is not None:
            fs = fabric.struct()
            rc = L.vgg_ba_solve_fabric(ctypes.byref(p), ctypes.byref(opt), ws.data_ptr(), ws.numel(), cb, None,
                                       ctypes.byref(fs), ctypes.byref(summ),
                                       trace.data_ptr() if trace is not None else None, st)
        else:
            rc = L.vgg_ba_solve(ctypes.byref(p), ctypes.byref(opt), ws.data_ptr(), ws.numel(), cb, None,
                                ctypes.byref(summ), trace.data_ptr() if trace is not None else None, st)
    _lib.check(rc, "vgg_ba_solve_iterative" if iterative else "vgg_ba_solve")
    out = Summary(summ.iterations, summ.successful, TERMINATION.get(summ.termination, "?"), summ.initial_cost,
                  summ.final_cost, summ.final_radius, summ.device_ms, summ.kernel_launches,
                  trace[:summ.iterations] if trace is not None else None, linear_solver_type)
    if iterative:
        out.cg_trace = cg_trace[:summ.iterations]
        out.cg_iterations = int(out.cg_trace[:, 0].sum().item())
    return out


@dataclasses.dataclass
class ObsList:
    """An observation list as vgg_ba_solve_iterative_obs takes it (include/vggsfm_b200.h vgg_ba_obs_list), device
    tensors: uv [M,2] f32, frame / point [M] and frame_obs [M] i32 point-major, track_start [N+1], frame_start [S+1];
    order [M]: entry i of the list is the caller's observation order[i]."""
    uv: torch.Tensor
    frame: torch.Tensor
    point: torch.Tensor
    track_start: torch.Tensor
    frame_start: torch.Tensor
    frame_obs: torch.Tensor
    order: torch.Tensor

    def struct(self) -> "_lib.BAObsList":
        return _lib.BAObsList(self.uv.shape[0], self.uv.data_ptr(), self.frame.data_ptr(), self.point.data_ptr(),
                              self.track_start.data_ptr(), self.frame_start.data_ptr(), self.frame_obs.data_ptr())


def obs_list(obs_uv, obs_frame, obs_point, S: int, N: int) -> ObsList:
    """The list of COO observations (obs_uv [M,2], obs_frame [M], obs_point [M], any order) on S frames and N points:
    sorted point-major by (point, frame), with its track segments and its frame-major permutation (stable sorts).
    ValueError for shapes, indices outside [0, S) x [0, N), or a second observation of one point in one frame."""
    M = obs_frame.shape[0]
    if obs_uv.shape != (M, 2) or obs_frame.shape != (M,) or obs_point.shape != (M,):
        raise ValueError(f"observations must be obs_uv [M,2], obs_frame [M], obs_point [M]; got "
                         f"{tuple(obs_uv.shape)}, {tuple(obs_frame.shape)}, {tuple(obs_point.shape)}")
    if M >= 2 ** 30:
        raise ValueError(f"at most 2^30 - 1 observations, not {M}")
    dev = obs_uv.device
    fr, pt = obs_frame.to(dev, torch.int64), obs_point.to(dev, torch.int64)
    if M and (fr.min() < 0 or fr.max() >= S or pt.min() < 0 or pt.max() >= N):
        raise ValueError(f"observation frames must lie in [0, {S}) and points in [0, {N})")
    key, order = torch.sort(pt * S + fr, stable=True)
    if M > 1 and bool((key[1:] == key[:-1]).any()):
        raise ValueError("a point is observed twice in one frame (duplicate (point, frame) observations)")
    fr, pt = fr[order], pt[order]
    zero = torch.zeros(1, dtype=torch.int64, device=dev)
    track_start = torch.cat([zero, torch.cumsum(torch.bincount(pt, minlength=N), 0)])
    frame_start = torch.cat([zero, torch.cumsum(torch.bincount(fr, minlength=S), 0)])
    frame_obs = torch.sort(fr, stable=True).indices
    i32 = lambda t: t.to(torch.int32).contiguous()
    return ObsList(obs_uv[order].to(torch.float32).contiguous(), i32(fr), i32(pt), i32(track_start), i32(frame_start),
                   i32(frame_obs), order)


def lm_solve_obs(obs_uv, obs_frame, obs_point, poses, intr, points, model, mode, param_const=None, point_const=None,
                 options: Optional[BAOptions] = None, allreduce=None, want_trace=False, min_linear_solver_iterations=0,
                 max_linear_solver_iterations=500, eta=0.1, loss_function_type="TRIVIAL",
                 loss_function_scale=1.0) -> Summary:
    """lm_solve with ITERATIVE_SCHUR on observations given as a list instead of the [S, N] grid
    (vgg_ba_solve_iterative_obs): COO (obs_uv [M,2], obs_frame [M], obs_point [M]) in any order, each one valid; memory
    O(M) for the list and O(S + N) for the workspace.  The CG options, loss, allreduce (each rank passes the observations
    of its own tracks) and trace are lm_solve's.  A point or frame without observations is constant and comes back bit
    for bit.  ValueError (obs_list) for malformed observations."""
    loss_function_id(loss_function_type)
    lin = linear_solver("ITERATIVE_SCHUR", min_linear_solver_iterations, max_linear_solver_iterations, eta)
    check_allreduce(allreduce, "ITERATIVE_SCHUR")
    L = _lib.lib()
    S, N = poses.shape[0], points.shape[0]
    dev = poses.device
    if param_const is None:
        param_const = default_param_const(S, model, mode, dev)
    if N == 0:
        if obs_frame.shape[0] > 0:
            raise ValueError("observations given for a problem without points")
        # a rank without tracks: padding points without observations (constant), as lm_solve pads
        N = pad_tracks(1)
        points = torch.zeros(N, 3, dtype=torch.float64, device=dev)
        points[:, 2] = 1.0
        point_const = None
    lst = obs_list(obs_uv, obs_frame, obs_point, S, N)
    opt = options or default_options()
    ws = workspace(S, N, model, mode, dev, iterative=True, obs=True)
    p = BAProblem()                      # no grid: uv = mask = NULL
    p.S, p.N, p.camera_model, p.intr_mode = S, N, model, mode
    p.uv, p.mask = None, None
    p.param_const = param_const.data_ptr()
    p.point_const = point_const.data_ptr() if point_const is not None else None
    for t in (poses, intr, points):
        assert t.dtype == torch.float64 and t.is_contiguous() and t.is_cuda
    p.poses, p.intr, p.points = poses.data_ptr(), intr.data_ptr(), points.data_ptr()
    p.loss_function_type = loss_function_id(loss_function_type)
    p.loss_function_scale = float(loss_function_scale)
    ol = lst.struct()
    summ = BASummary()
    trace = torch.zeros(max(1, opt.max_num_iterations), 8, dtype=torch.float64) if want_trace else None
    cg_trace = torch.zeros(max(1, opt.max_num_iterations), 4, dtype=torch.float64)
    cb = allreduce.bind(ws) if allreduce is not None else _lib.ALLREDUCE_FN()
    with torch.cuda.device(dev):
        st = torch.cuda.current_stream().cuda_stream
        rc = L.vgg_ba_solve_iterative_obs(ctypes.byref(p), ctypes.byref(ol), ctypes.byref(opt), ctypes.byref(lin),
                                          ws.data_ptr(), ws.numel(), cb, None, ctypes.byref(summ),
                                          trace.data_ptr() if trace is not None else None, cg_trace.data_ptr(), st)
    _lib.check(rc, "vgg_ba_solve_iterative_obs")
    out = Summary(summ.iterations, summ.successful, TERMINATION.get(summ.termination, "?"), summ.initial_cost,
                  summ.final_cost, summ.final_radius, summ.device_ms, summ.kernel_launches,
                  trace[:summ.iterations] if trace is not None else None, "ITERATIVE_SCHUR")
    out.cg_trace = cg_trace[:summ.iterations]
    out.cg_iterations = int(out.cg_trace[:, 0].sum().item())
    return out


# --------------------------------------------------------------------------------------------------
# COLMAP wrapper semantics around the solve, on device
# --------------------------------------------------------------------------------------------------

def filter_negative_depth(poses, points, mask):
    """ObservationManager::FilterObservationsWithNegativeDepth: drop observations with depth < eps;
    a track left with < 2 observations is deleted.  (mask bool [S,N]) -> (mask, alive[N])."""
    eps = torch.finfo(torch.float64).eps
    depth = torch.einsum("sj,nj->sn", poses[:, 2, :3], points) + poses[:, 2, 3][:, None]
    bad = mask & ~(depth >= eps)
    length = mask.sum(dim=0)
    nbad = bad.sum(dim=0)
    alive = (nbad == 0) | ((length - nbad) >= 2)
    mask = mask & ~bad & alive[None]
    return mask, alive


def normalize(poses, points, extent=10.0, p0=0.1, p1=0.9, alive=None):
    """Reconstruction::Normalize(extent, p0, p1, use_images=True) as restated in oracle/ba_oracle.py."""
    S = poses.shape[0]
    if S < 2:
        return poses, points
    R = poses[:, :, :3]
    t = poses[:, :, 3]
    centers = -torch.einsum("sji,sj->si", R, t)
    c32 = torch.sort(centers.to(torch.float32), dim=0).values
    P0 = int(p0 * (S - 1)) if S > 3 else 0
    P1 = int(p1 * (S - 1)) if S > 3 else S - 1
    bmin = c32[P0].double()
    bmax = c32[P1].double()
    mean = c32[P0:P1 + 1].double().sum(dim=0) / (P1 - P0 + 1)
    old_extent = torch.linalg.norm(bmax - bmin)
    scale = torch.where(old_extent < torch.finfo(torch.float64).eps, torch.ones_like(old_extent), extent / old_extent)
    tr = -scale * mean
    new_points = scale * points + tr
    if alive is not None:
        new_points = torch.where(alive[:, None], new_points, points)
    new_poses = poses.clone()
    new_poses[:, :, 3] = scale * t - torch.einsum("sij,j->si", R, tr)
    return new_poses, new_points


def pad_tracks(n: int, multiple: int = 16) -> int:
    return (n + multiple - 1) // multiple * multiple


def bundle_adjustment(points3d, extrinsics, intrinsics, extra_params, tracks, masks, shared_camera=False,
                      camera_type="SIMPLE_PINHOLE", options: Optional[BAOptions] = None, max_points3D_val=3000.0,
                      allreduce=None, want_trace=False, refine_focal_length=True, refine_extra_params=True,
                      const_pose=None, const_points=None, gauge=True, do_normalize=True, filter_reconstruction=True,
                      drop_negative_depth=True, linear_solver_type="DENSE_SCHUR", min_linear_solver_iterations=0,
                      max_linear_solver_iterations=500, eta=0.1, loss_function_type="TRIVIAL", loss_function_scale=1.0):
    """Tensor-in / tensor-out equivalent of batch_matrix_to_pycolmap + pycolmap.bundle_adjustment +
    filter_reconstruction + pycolmap_to_batch_matrix (triangulation.py:1033-1063).

    points3d [P,3], extrinsics [S,3,4], intrinsics [S,3,3], extra_params [S,1]|None, tracks [S,P,2],
    masks [S,P] bool -- CUDA tensors.  Returns (points3D [P',3] f64, extrinsics [S,3,4] f64,
    intrinsics [S,3,3] f64, extra_params [S,1]|None, valid_idx [P'], Summary).  linear_solver_type and the CG options
    as lm_solve (ITERATIVE_SCHUR runs over track shards through `allreduce` too; a hook with a fabric raises ValueError
    with it before anything runs), and so are
    loss_function_type and loss_function_scale (COLMAP's BundleAdjustmentOptions defaults: TRIVIAL, 1.0)."""
    model = camera_model_id(camera_type)
    loss_function_id(loss_function_type)
    lin_kw = dict(linear_solver_type=linear_solver_type, min_linear_solver_iterations=min_linear_solver_iterations,
                  max_linear_solver_iterations=max_linear_solver_iterations, eta=eta)
    linear_solver(**lin_kw)
    check_allreduce(allreduce, linear_solver_type)
    dev = tracks.device
    if not tracks.is_cuda:
        raise RuntimeError("vggsfm_b200.bundle_adjustment needs CUDA tensors (no CPU fallback)")
    masks = masks.bool()
    valid_idx = torch.nonzero(masks.sum(dim=0) >= 2).flatten()   # tensor_to_pycolmap.py:62-64
    pts = points3d.double()[valid_idx].contiguous()
    P = pts.shape[0]
    m = masks[:, valid_idx]
    m = m & (pts < max_points3D_val).all(dim=1)[None]          # tensor_to_pycolmap.py:131-133
    poses = extrinsics.double().contiguous().clone()
    S = poses.shape[0]
    intr = torch.zeros(S, 4, dtype=torch.float64, device=dev)
    intr[:, 0] = intrinsics[:, 0, 0]
    intr[:, 1] = intrinsics[:, 0, 2]
    intr[:, 2] = intrinsics[:, 1, 2]
    if model == SIMPLE_RADIAL:
        intr[:, 3] = extra_params[:, 0]
    if shared_camera:
        mode = INTR_SHARED
        intr[:] = intr[0].clone()
    else:
        mode = INTR_PER_FRAME
    if not (refine_focal_length or refine_extra_params):
        mode = INTR_CONST
    if drop_negative_depth:                                    # BundleAdjustmentController::Run only
        m, alive = filter_negative_depth(poses, pts, m)
    else:
        alive = torch.ones(P, dtype=torch.bool, device=dev)
    point_const = ~m.any(dim=0)
    if const_points is not None:
        point_const = point_const | const_points[valid_idx]
    # pad the track axis to a multiple of 16 so the kernels take the TMA path (padding is masked out)
    Pp = pad_tracks(max(P, 1))
    uv = torch.zeros(S, Pp, 2, dtype=torch.float32, device=dev)
    uv[:, :P] = tracks[:, valid_idx].float()
    mk = torch.zeros(S, Pp, dtype=torch.uint8, device=dev)
    mk[:, :P] = m.to(torch.uint8)
    X = torch.zeros(Pp, 3, dtype=torch.float64, device=dev)
    X[:P] = pts
    X[P:, 2] = 1.0
    pc = torch.ones(Pp, dtype=torch.uint8, device=dev)
    pc[:P] = point_const.to(torch.uint8)
    param_const = default_param_const(S, model, mode, dev, refine_focal_length, refine_extra_params, gauge, const_pose)
    summary = lm_solve(uv, mk, poses, intr, X, model, mode, param_const, pc, options, allreduce, want_trace, **lin_kw,
                       loss_function_type=loss_function_type, loss_function_scale=loss_function_scale)
    pts = X[:P]
    if do_normalize:
        poses, pts = normalize(poses, pts, 10.0, 0.1, 0.9, alive)   # BundleAdjustmentController::Run
        if filter_reconstruction:
            poses, pts = normalize(poses, pts, 5.0, 0.1, 0.9, alive)    # filter_reconstruction (triangulation.py:1217)
    pts = torch.where(alive[:, None], pts, torch.zeros_like(pts))
    summary.alive, summary.mask = alive, m
    K = torch.zeros(S, 3, 3, dtype=torch.float64, device=dev)
    K[:, 0, 0] = intr[:, 0]
    K[:, 1, 1] = intr[:, 0]
    K[:, 0, 2] = intr[:, 1]
    K[:, 1, 2] = intr[:, 2]
    K[:, 2, 2] = 1.0
    extra_out = intr[:, 3:4].clone() if model == SIMPLE_RADIAL else None
    return pts, poses, K, extra_out, valid_idx, summary


run_ba = bundle_adjustment   # the name BASELINE.json's north_star uses for this call


def bundle_adjustment_obs(points3d, extrinsics, intrinsics, extra_params, obs_uv, obs_frame, obs_point,
                          shared_camera=False, camera_type="SIMPLE_PINHOLE", options: Optional[BAOptions] = None,
                          max_points3D_val=3000.0, allreduce=None, want_trace=False, refine_focal_length=True,
                          refine_extra_params=True, const_pose=None, const_points=None, gauge=True, do_normalize=True,
                          filter_reconstruction=True, drop_negative_depth=True, min_linear_solver_iterations=0,
                          max_linear_solver_iterations=500, eta=0.1, loss_function_type="TRIVIAL",
                          loss_function_scale=1.0):
    """bundle_adjustment with ITERATIVE_SCHUR on observations given as a list (COO obs_uv [M,2], obs_frame [M],
    obs_point [M] into points3d [P,3], any order) instead of the [S,P] grid, with the same COLMAP wrapper semantics:
    points with >= 2 observations kept and renumbered in id order, the max_points3D_val clamp, the negative-depth filter
    per observation, the gauge, the constant sets and both normalisations.  Returns bundle_adjustment's tuple
    (points3D [P',3], extrinsics, intrinsics, extra_params, valid_idx [P'], Summary); Summary.alive is as there and
    Summary.keep [M] bool (in the caller's order) replaces Summary.mask: the observations that were in the problem."""
    model = camera_model_id(camera_type)
    loss_function_id(loss_function_type)
    linear_solver("ITERATIVE_SCHUR", min_linear_solver_iterations, max_linear_solver_iterations, eta)
    check_allreduce(allreduce, "ITERATIVE_SCHUR")
    dev = obs_uv.device
    if not obs_uv.is_cuda:
        raise RuntimeError("vggsfm_b200.bundle_adjustment_obs needs CUDA tensors (no CPU fallback)")
    S, P0 = extrinsics.shape[0], points3d.shape[0]
    fr, pt = obs_frame.to(dev, torch.int64), obs_point.to(dev, torch.int64)
    M = fr.shape[0]
    if M and (pt.min() < 0 or pt.max() >= P0 or fr.min() < 0 or fr.max() >= S):
        raise ValueError(f"observation frames must lie in [0, {S}) and points in [0, {P0})")
    count = torch.bincount(pt, minlength=P0)
    valid_idx = torch.nonzero(count >= 2).flatten()                  # tensor_to_pycolmap.py:62-64
    new_id = torch.full((P0,), -1, dtype=torch.int64, device=dev)
    new_id[valid_idx] = torch.arange(valid_idx.numel(), device=dev)
    pts = points3d.double()[valid_idx].contiguous()
    P = pts.shape[0]
    cp = new_id[pt]
    m = (cp >= 0) & (pts < max_points3D_val).all(dim=1)[cp.clamp(min=0)]   # tensor_to_pycolmap.py:131-133
    poses = extrinsics.double().contiguous().clone()
    intr = torch.zeros(S, 4, dtype=torch.float64, device=dev)
    intr[:, 0] = intrinsics[:, 0, 0]
    intr[:, 1] = intrinsics[:, 0, 2]
    intr[:, 2] = intrinsics[:, 1, 2]
    if model == SIMPLE_RADIAL:
        intr[:, 3] = extra_params[:, 0]
    if shared_camera:
        mode = INTR_SHARED
        intr[:] = intr[0].clone()
    else:
        mode = INTR_PER_FRAME
    if not (refine_focal_length or refine_extra_params):
        mode = INTR_CONST
    cpc = cp.clamp(min=0)
    if drop_negative_depth:                                          # filter_negative_depth, per observation
        depth = (poses[fr, 2, :3] * pts[cpc]).sum(dim=1) + poses[fr, 2, 3]
        bad = m & ~(depth >= torch.finfo(torch.float64).eps)
        length = torch.bincount(cpc[m], minlength=P)
        nbad = torch.bincount(cpc[bad], minlength=P)
        alive = (nbad == 0) | ((length - nbad) >= 2)
        m = m & ~bad & alive[cpc]
    else:
        alive = torch.ones(P, dtype=torch.bool, device=dev)
    point_const = torch.bincount(cpc[m], minlength=P) == 0
    if const_points is not None:
        point_const = point_const | const_points[valid_idx]
    param_const = default_param_const(S, model, mode, dev, refine_focal_length, refine_extra_params, gauge, const_pose)
    X = pts.clone()
    summary = lm_solve_obs(obs_uv[m], fr[m], cpc[m], poses, intr, X, model, mode, param_const,
                           point_const.to(torch.uint8), options, allreduce, want_trace, min_linear_solver_iterations,
                           max_linear_solver_iterations, eta, loss_function_type, loss_function_scale)
    pts = X
    if do_normalize:
        poses, pts = normalize(poses, pts, 10.0, 0.1, 0.9, alive)   # BundleAdjustmentController::Run
        if filter_reconstruction:
            poses, pts = normalize(poses, pts, 5.0, 0.1, 0.9, alive)    # filter_reconstruction (triangulation.py:1217)
    pts = torch.where(alive[:, None], pts, torch.zeros_like(pts))
    summary.alive, summary.keep = alive, m
    K = torch.zeros(S, 3, 3, dtype=torch.float64, device=dev)
    K[:, 0, 0] = intr[:, 0]
    K[:, 1, 1] = intr[:, 0]
    K[:, 0, 2] = intr[:, 1]
    K[:, 1, 2] = intr[:, 2]
    K[:, 2, 2] = 1.0
    extra_out = intr[:, 3:4].clone() if model == SIMPLE_RADIAL else None
    return pts, poses, K, extra_out, valid_idx, summary


# --------------------------------------------------------------------------------------------------
# mirrors of the reference's BA drivers (vggsfm/utils/triangulation.py:1020-1242)
# --------------------------------------------------------------------------------------------------

from .reconstruction import Reconstruction   # noqa: E402  (pycolmap-shaped scene object, vggsfm_b200/reconstruction.py)


def _reconstruction(pts, extr, K, extra, tracks, masks, image_size, camera_type, shared_camera, summary, alive=None):
    """The ``pycolmap.Reconstruction`` the reference returns, as its duck-typed stand-in (lazy: a few array
    references until a caller touches ``.images / .cameras / .points3D``)."""
    return Reconstruction.from_batch_matrix(pts, extr, K, tracks, masks, image_size, shared_camera=shared_camera,
                                            camera_type=camera_type, extra_params=extra, summary=summary, alive=alive)


def _revert_negative_focal(extr_new, K_new, extra_new, extr_old, K_old, extra_old):
    """triangulation.py:1066-1071 / 1158-1165: cameras whose optimised focal is negative keep their old values."""
    bad = K_new[:, 0, 0] < 0
    if bad.any():
        extr_new[bad] = extr_old[bad].to(extr_new.dtype)
        K_new[bad] = K_old[bad].to(K_new.dtype)
        if extra_new is not None:
            extra_new[bad] = extra_old[bad].to(extra_new.dtype)
    return extr_new, K_new, extra_new


def global_BA(triangulated_points, valid_tracks, pred_tracks, inlier_mask, extrinsics, intrinsics, extra_params,
              image_size, shared_camera=False, camera_type="SIMPLE_PINHOLE", allreduce=None,
              linear_solver_type="DENSE_SCHUR", min_linear_solver_iterations=0, max_linear_solver_iterations=200,
              eta=0.1):
    """vggsfm/utils/triangulation.py:1020-1073 with the same arguments and return tuple
    (points3D_opt, extrinsics, intrinsics, extra_params, reconstruction).  The linear-solver options are
    bundle_adjustment()'s; max_linear_solver_iterations defaults to the 200 of prepare_ba_options."""
    BA_points = triangulated_points[valid_tracks]
    BA_tracks = pred_tracks[:, valid_tracks]
    BA_inlier_masks = inlier_mask[valid_tracks].transpose(0, 1)
    pts, extr, K, extra, valid_idx, summary = bundle_adjustment(
        BA_points, extrinsics, intrinsics, extra_params, BA_tracks, BA_inlier_masks, shared_camera=shared_camera,
        camera_type=camera_type, options=prepare_ba_options(), allreduce=allreduce,
        linear_solver_type=linear_solver_type, min_linear_solver_iterations=min_linear_solver_iterations,
        max_linear_solver_iterations=max_linear_solver_iterations, eta=eta)
    extr, K, extra = _revert_negative_focal(extr, K, extra, extrinsics, intrinsics, extra_params)
    rec = _reconstruction(pts, extr, K, extra, BA_tracks[:, valid_idx], summary.mask, image_size, camera_type,
                          shared_camera, summary, summary.alive)
    return pts, extr, K, extra, rec


def init_BA(extrinsics, intrinsics, extra_params, tracks, points_3d_pair, inlier, image_size, shared_camera=False,
            init_max_reproj_error=0.5, camera_type="SIMPLE_PINHOLE"):
    """vggsfm/utils/triangulation.py:138-257 with the same arguments and return tuple
    (points3D_opt, extrinsics, intrinsics, extra_params, filtered_valid_track_mask, reconstruction, init_idx):
    two-frame BA of the query frame and the frame with the most triangulation inliers, then the reprojection
    filter at ``init_max_reproj_error``.  Like the reference it writes the optimised pair back INTO the
    extrinsics / intrinsics / extra_params it was given (:243-246) and does not call filter_reconstruction."""
    from . import triangulation as tri
    init_idx = int(torch.argmax(inlier.sum(dim=-1)).item())
    init_indices = [0, init_idx + 1]
    toBA_extrinsics = extrinsics[init_indices]
    toBA_intrinsics = intrinsics[init_indices]
    toBA_extra = extra_params[init_indices] if extra_params is not None else None
    toBA_masks = inlier[init_idx].unsqueeze(0)
    toBA_masks = torch.cat([torch.ones_like(toBA_masks), toBA_masks], dim=0)
    valid_track = toBA_masks.sum(dim=0) >= 2
    toBA_masks = toBA_masks[:, valid_track]
    toBA_points = points_3d_pair[init_idx][valid_track]
    toBA_tracks = tracks[init_indices][:, valid_track]
    pts, extr, K, extra, valid_idx, summary = bundle_adjustment(
        toBA_points, toBA_extrinsics, toBA_intrinsics, toBA_extra, toBA_tracks, toBA_masks, shared_camera=shared_camera,
        camera_type=camera_type, options=prepare_ba_options(), filter_reconstruction=False)
    rec = _reconstruction(pts, extr, K, extra, toBA_tracks[:, valid_idx], summary.mask, image_size, camera_type,
                          shared_camera, summary, summary.alive)
    ok, _ = tri.filter_all_points3D(pts, toBA_tracks, extr, K, extra, check_triangle=False,
                                    max_reproj_error=init_max_reproj_error)
    points3D_opt = pts[ok]
    filtered = valid_track.clone()
    filtered[valid_track] = ok
    extrinsics[init_indices] = extr.to(extrinsics.dtype)
    intrinsics[init_indices] = K.to(intrinsics.dtype)
    if extra_params is not None:
        extra_params[init_indices] = extra.to(extra_params.dtype)
    return points3D_opt, extrinsics, intrinsics, extra_params, filtered, rec, init_idx


def get_valid_frame_mask(intrinsics, extrinsics, extra_params, scale):
    """vggsfm/utils/triangulation.py:1222-1242."""
    valid = (intrinsics[:, 0, 0] >= 0.1 * scale) & (intrinsics[:, 0, 0] <= 30 * scale)
    if extra_params is not None:
        if extra_params.dim() == 1:
            extra_params = extra_params[:, None]
        valid = valid & (extra_params.abs() <= 1.0).all(dim=-1)
    return valid & (extrinsics[:, :, 3].abs() <= 30).all(-1)


def iterative_global_BA(pred_tracks, intrinsics, extrinsics, pred_vis, pred_score, valid_tracks, points3D_opt,
                        image_size, shared_camera=False, min_valid_track_length=2, max_reproj_error=1,
                        ba_options=None, lastBA=False, camera_type="SIMPLE_PINHOLE", extra_params=None,
                        allreduce=None, linear_solver_type="DENSE_SCHUR", min_linear_solver_iterations=0,
                        max_linear_solver_iterations=200, eta=0.1):
    """vggsfm/utils/triangulation.py:1076-1209: re-triangulate (128 hypotheses) -> keep the last BA's points for
    already-valid tracks -> reprojection/triangle filter -> BA (default options) -> filter again -> compaction.
    Same arguments; returns (points3D_opt, extrinsics, intrinsics, extra_params, valid_tracks, BA_inlier_masks,
    reconstruction).  The linear-solver options are bundle_adjustment()'s (max 200 as in prepare_ba_options)."""
    from . import triangulation as tri
    tn = tri.cam_from_img(pred_tracks, intrinsics, extra_params)
    best_points, best_num, best_mask = tri.triangulate_tracks(extrinsics, tn, track_vis=pred_vis, track_score=pred_score,
                                                             max_ransac_iters=128)
    best_points[valid_tracks] = points3D_opt.to(best_points.dtype)                      # :1110
    _, filtered = tri.filter_all_points3D(best_points, pred_tracks, extrinsics, intrinsics, extra_params=extra_params,
                                          max_reproj_error=max_reproj_error, return_detail=True)
    valid_tracks = filtered.sum(dim=0) >= min_valid_track_length
    BA_points = best_points[valid_tracks]
    BA_tracks = pred_tracks[:, valid_tracks]
    BA_inlier_masks = filtered[:, valid_tracks]
    pts, extr, K, extra, valid_idx, summary = bundle_adjustment(
        BA_points, extrinsics, intrinsics, extra_params, BA_tracks, BA_inlier_masks, shared_camera=shared_camera,
        camera_type=camera_type, options=ba_options or default_options(), allreduce=allreduce,
        linear_solver_type=linear_solver_type, min_linear_solver_iterations=min_linear_solver_iterations,
        max_linear_solver_iterations=max_linear_solver_iterations, eta=eta)
    rec = _reconstruction(pts, extr, K, extra, BA_tracks[:, valid_idx], summary.mask, image_size, camera_type,
                          shared_camera, summary, summary.alive)        # the BA'd, filter_reconstruction'd object (:1146)
    if valid_idx.numel() != BA_points.shape[0]:
        # tracks with < 2 inliers never reach this point (min_valid_track_length >= 2), kept for safety
        full = torch.zeros(BA_points.shape[0], 3, dtype=pts.dtype, device=pts.device)
        full[valid_idx] = pts
        pts = full
    extr, K, extra = _revert_negative_focal(extr, K, extra, extrinsics, intrinsics, extra_params)
    _, filtered = tri.filter_all_points3D(pts, pred_tracks[:, valid_tracks], extr, K, extra_params=extra,
                                          max_reproj_error=max_reproj_error, return_detail=True)
    valid_after = filtered.sum(dim=0) >= min_valid_track_length
    valid_tmp = valid_tracks.clone()
    valid_tmp[valid_tracks] = valid_after
    valid_tracks = valid_tmp
    pts = pts[valid_after]
    BA_inlier_masks = filtered[:, valid_after]
    if lastBA:
        # :1186-1199: rebuilt from the filtered tensors, then filter_reconstruction's normalize(5.0, 0.1, 0.9, True);
        # normalize() takes and returns (poses, points)
        e2, p2 = normalize(extr, pts, 5.0, 0.1, 0.9)
        rec = _reconstruction(p2, e2, K, extra, pred_tracks[:, valid_tracks], BA_inlier_masks, image_size, camera_type,
                              shared_camera, summary)
    return pts, extr, K, extra, valid_tracks, BA_inlier_masks, rec
