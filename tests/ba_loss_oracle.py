"""Float64 restatement of bundle adjustment under a robust loss -- TEST INFRASTRUCTURE ONLY.

COLMAP 3.10's BundleAdjustmentOptions puts ``loss_function_type`` (TRIVIAL, SOFT_L1, CAUCHY) at
``loss_function_scale`` a on every reprojection residual block; the losses are Ceres 2.x's [3P-memory].  With the
observation's s = |r|^2, b = a^2 and c = 1 / b:

  * CauchyLoss(a):  rho = b log(1 + s c),            rho' = max(DBL_MIN, 1 / (1 + s c)),    rho'' = -c rho'^2
  * SoftLOneLoss(a): rho = 2 b (sqrt(1 + s c) - 1),  rho' = max(DBL_MIN, 1 / sqrt(1 + s c)), rho'' = -c rho' / (2 (1 + s c))
  * the cost of an observation is rho(s) / 2;
  * Ceres' Corrector: when rho'' <= 0 (always, for both) or s = 0, residual and Jacobian are scaled by sqrt(rho'), and
    every normal-equation block, gradient, Jacobi scale and model change follows from the scaled pair.

Cauchy's rho and rho' are oracle/pose_oracle.py's ``cauchy`` (pose refinement wraps every residual in CauchyLoss), used
here with Ceres' DBL_MIN clamp; SoftL1 and rho'' are restated below, nowhere else.  rho is evaluated in forms without
cancellation (log1p; 2 s / (1 + sqrt(1 + s c)) for SoftL1 where sqrt(1 + s c) < 2), which are the same functions and let
a large scale reduce to the trivial loss to rounding, as the kernels do (csrc/ba_obs.h).

The LM loops of oracle/ba_oracle.py and oracle/ba_pcg_oracle.py run as they are: ``robust()`` swaps the linearisation
both of them call -- ``ba_oracle.residuals_and_jacobians`` (blocks, the CG model change) and ``ba_oracle.build_blocks``
(whose cost becomes 0.5 sum rho) -- for the corrected one while it is active, the same single point at which the CUDA
path applies the loss.  TRIVIAL never swaps anything, so its results are those of the oracles bit for bit.
"""
from __future__ import annotations

import contextlib
import sys

import numpy as np

from oracle import ba_oracle as bo
from oracle import ba_pcg_oracle as bpo
from oracle.pose_oracle import cauchy

LOSS_TYPES = ("TRIVIAL", "SOFT_L1", "CAUCHY")
DBL_MIN = sys.float_info.min


def loss_rho(s, loss_type, scale):
    """(rho, rho', rho'') of Ceres' loss at s = |r|^2 (arrays of s's shape)."""
    if loss_type not in LOSS_TYPES:
        raise ValueError(f"unknown loss {loss_type!r}")
    s = np.asarray(s, dtype=np.float64)
    if loss_type == "TRIVIAL":
        return s.copy(), np.ones_like(s), np.zeros_like(s)
    b = scale * scale
    c = 1.0 / b
    with np.errstate(invalid="ignore", divide="ignore", over="ignore"):
        if loss_type == "CAUCHY":
            rho, rho1 = cauchy(s, scale)
            rho1 = np.maximum(DBL_MIN, rho1)
            rho2 = -c * rho1 * rho1
        else:
            t = np.sqrt(1.0 + s * c)
            rho = np.where(t < 2.0, 2.0 * s / (1.0 + t), 2.0 * b * (t - 1.0))
            rho1 = np.maximum(DBL_MIN, 1.0 / t)
            rho2 = -(c * rho1) / (2.0 * (1.0 + s * c))
    return rho, rho1, rho2


def cost_only(poses, intr, points, uv, mask, model, loss_function_type="TRIVIAL", loss_function_scale=1.0):
    """0.5 sum rho(|r|^2) over the valid observations (residuals as ba_oracle.residuals_and_jacobians forms them)."""
    res, _, _ = _raw_rj(poses, intr, points, uv, mask, model)
    rho, _, _ = loss_rho(np.sum(res * res, axis=-1), loss_function_type, loss_function_scale)
    return 0.5 * float(np.sum(np.where(mask, rho, 0.0)))


_raw_rj = bo.residuals_and_jacobians
_raw_build_blocks = bo.build_blocks


@contextlib.contextmanager
def robust(loss_function_type="TRIVIAL", loss_function_scale=1.0):
    """Within the block, the oracles' linearisation is that of the loss (see the module docstring)."""
    loss_rho(0.0, loss_function_type, loss_function_scale)           # name check
    if loss_function_type == "TRIVIAL":
        yield
        return
    assert bo.residuals_and_jacobians is _raw_rj and bo.build_blocks is _raw_build_blocks, "robust() does not nest"

    def residuals_and_jacobians(poses, intr, points, uv, mask, model):
        res, Jc, Jp = _raw_rj(poses, intr, points, uv, mask, model)
        _, rho1, rho2 = loss_rho(np.sum(res * res, axis=-1), loss_function_type, loss_function_scale)
        assert np.all(~(rho2 > 0.0))                                    # the Corrector's alpha = 0 branch
        k = np.sqrt(rho1)
        return res * k[..., None], Jc * k[..., None, None], Jp * k[..., None, None]

    def build_blocks(poses, intr, points, uv, mask, model, mode, point_const=None):
        out = _raw_build_blocks(poses, intr, points, uv, mask, model, mode, point_const)
        out["cost"] = cost_only(poses, intr, points, uv, mask, model, loss_function_type, loss_function_scale)
        return out

    # callers that prefer oracle/ba_blocks_ref.c when it is built (it evaluates the trivial loss) take numpy instead
    load_c = bo._load_c
    bo.residuals_and_jacobians, bo.build_blocks, bo._load_c = residuals_and_jacobians, build_blocks, lambda: None
    try:
        yield
    finally:
        bo.residuals_and_jacobians, bo.build_blocks, bo._load_c = _raw_rj, _raw_build_blocks, load_c


def build_blocks(poses, intr, points, uv, mask, model, mode, point_const=None, loss_function_type="TRIVIAL",
                 loss_function_scale=1.0):
    """ba_oracle.build_blocks of the loss: blocks of the corrected residuals and Jacobians, cost 0.5 sum rho."""
    with robust(loss_function_type, loss_function_scale):
        return bo.build_blocks(poses, intr, points, uv, mask, model, mode, point_const)


def jd_model_change(poses, intr, points, uv, mask, model, mode, d_c, d_p, point_const, loss_function_type="TRIVIAL",
                    loss_function_scale=1.0):
    """ba_pcg_oracle.jd_model_change of the loss: -(J d)^T (f + J d / 2) with the corrected f and J."""
    with robust(loss_function_type, loss_function_scale):
        return bpo.jd_model_change(poses, intr, points, uv, mask, model, mode, d_c, d_p, point_const)


def lm_solve(poses, intr, points, uv, mask, model, mode, linear_solver="dense_schur", loss_function_type="TRIVIAL",
             loss_function_scale=1.0, **kw):
    """ba_oracle.lm_solve ("dense_schur"; its allreduce keyword included) or ba_pcg_oracle.lm_solve
    ("iterative_schur", with the CG keywords) under the loss.  Returns (poses, intr, points, summary)."""
    if kw.get("use_c") and loss_function_type != "TRIVIAL":
        raise ValueError("oracle/ba_blocks_ref.c evaluates the trivial loss only")
    with robust(loss_function_type, loss_function_scale):
        if linear_solver == "dense_schur":
            return bo.lm_solve(poses, intr, points, uv, mask, model, mode, **kw)
        return bpo.lm_solve(poses, intr, points, uv, mask, model, mode, linear_solver=linear_solver, **kw)


def with_outliers(c, frac=0.1, lo=20.0, hi=80.0, seed=0):
    """ba_case dict c with a fraction `frac` of its valid observations displaced by lo..hi pixels in a random direction
    (a learned tracker's gross outliers); the displaced (frame, track) pairs are returned under "outlier"."""
    rng = np.random.default_rng(seed)
    mask = np.asarray(c["mask"], dtype=bool)
    pick = mask & (rng.uniform(size=mask.shape) < frac)
    ang = rng.uniform(0.0, 2.0 * np.pi, size=mask.shape)
    mag = rng.uniform(lo, hi, size=mask.shape)
    off = np.stack([np.cos(ang), np.sin(ang)], axis=-1) * mag[..., None]
    uv = np.where(pick[..., None], c["uv"] + off, c["uv"])
    uv = uv.astype(np.float32).astype(np.float64)                      # what the float32 observations hold
    return dict(c, uv=uv, outlier=pick)
