"""CPU checks of oracle/pose_oracle.py (the restatement of pycolmap.pose_refinement -- parity unpinned, so it is
validated against finite differences, an independent minimiser, and the reference's documented loop semantics)."""
import numpy as np
import pytest

from oracle import pose_oracle as po
from oracle.ba_oracle import exp_so3, project


def _case(model, P=240, seed=0, outliers=16):
    rng = np.random.default_rng(seed)
    X = rng.normal(size=(P, 3)) + np.array([0, 0, 6.0])
    R = exp_so3(rng.normal(size=3) * 0.2)
    t = rng.normal(size=3) * 0.3
    pose = np.concatenate([R, t[:, None]], 1)
    intr = np.array([500.0, 320, 240, 0.05])
    uv, _ = project(pose[None], intr[None], X, model)
    uv = uv[0] + rng.normal(size=(P, 2)) * 0.5
    uv[:outliers] += rng.normal(size=(outliers, 2)) * 40
    p0 = pose.copy()
    p0[:, :3] = exp_so3(np.array([0.02, -0.01, 0.015])) @ p0[:, :3]
    p0[:, 3] += 0.05
    i0 = intr.copy()
    i0[0] *= 1.05
    return pose, intr, X, uv.astype(np.float32).astype(np.float64), p0, i0


@pytest.mark.parametrize("model", [0, 1])
def test_jacobian_finite_differences(model):
    _, _, X, uv, p0, i0 = _case(model)
    r, J = po.residual_jacobian(p0, i0, X, uv, model)
    eps = 1e-6
    for c in range(8 if model == 1 else 7):
        d = np.zeros(8)
        d[c] = eps
        rp, _ = po.residual_jacobian(*po.plus(p0, i0, d), X, uv, model)
        rm, _ = po.residual_jacobian(*po.plus(p0, i0, -d), X, uv, model)
        num = (rp - rm) / (2 * eps)
        assert np.allclose(num, J[:, :, c], rtol=1e-5, atol=1e-5 * np.abs(J[:, :, c]).max()), c


@pytest.mark.parametrize("model", [0, 1])
def test_reaches_local_minimum_of_cauchy_cost(model):
    from scipy.optimize import minimize
    _, _, X, uv, p0, i0 = _case(model)
    o = po.PoseOptions(function_tolerance=1e-15, gradient_tolerance=1e-9, parameter_tolerance=1e-14)
    p1, i1, sm = po.pose_refinement(p0, i0, X, uv, np.ones(len(X), bool), model, options=o)
    assert sm["final_cost"] < 0.5 * sm["initial_cost"]

    def fun(x):
        pp, ii = po.plus(p1, i1, np.concatenate([x[:6] * 1e-3, [x[6], x[7] * 1e-3 if model == 1 else 0.0]]))
        return po.robust_cost(pp, ii, X, uv, model, 1.0)
    res = minimize(fun, np.zeros(8), method="BFGS", options=dict(gtol=1e-10))
    assert res.fun >= sm["final_cost"] * (1 - 1e-9)


def test_default_options_stop_and_flags():
    pose, intr, X, uv, p0, i0 = _case(1)
    p1, i1, sm = po.pose_refinement(p0, i0, X, uv, np.ones(len(X), bool), 1)
    assert sm["termination"] in (po.CONV_GRADIENT, po.CONV_FUNCTION, po.CONV_PARAMETER) and sm["iterations"] < 30
    assert abs(i1[0] - intr[0]) < 2.0 and np.abs(p1[:, 3] - pose[:, 3]).max() < 0.02
    # principal point never moves; focal / extra stay put when their flags are off
    assert i1[1] == i0[1] and i1[2] == i0[2]
    _, i2, _ = po.pose_refinement(p0, i0, X, uv, np.ones(len(X), bool), 1, refine_focal=False, refine_extra=True)
    assert i2[0] == i0[0] and i2[3] != i0[3]
    _, i3, _ = po.pose_refinement(p0, i0, X, uv, np.ones(len(X), bool), 1, refine_focal=True, refine_extra=False)
    assert i3[3] == i0[3] and i3[0] != i0[0]
    # SIMPLE_PINHOLE ignores k altogether
    _, i4, _ = po.pose_refinement(p0, i0, X, uv, np.ones(len(X), bool), 0)
    assert i4[3] == i0[3]


def test_frame_loop_shared_camera_semantics():
    """triangulation.py:341-375: one camera object; frame 0 refines it, later frames see the update and keep it fixed."""
    rng = np.random.default_rng(3)
    S, P = 4, 200
    X = rng.normal(size=(P, 3)) + np.array([0, 0, 6.0])
    poses = np.stack([np.concatenate([exp_so3(rng.normal(size=3) * 0.1), rng.normal(size=(3, 1)) * 0.2], 1) for _ in range(S)])
    intr = np.tile(np.array([500.0, 320, 240, 0.0]), (S, 1))
    uv, _ = project(poses, intr, X, 0)
    uv = uv + rng.normal(size=uv.shape) * 0.3
    intr0 = intr.copy()
    intr0[:, 0] = 520.0
    inl = np.ones((S, P), bool)
    inl[2, 60:] = False                                  # 60 inliers only: frame 2 is not refined at min_inliers=100
    p1, i1, used, summ = po.frame_loop(poses, intr0, X, uv, inl, np.ones(S, bool), 0, True, 12.0, 100)
    assert np.all(i1 == i1[0]) and abs(i1[0, 0] - 500.0) < 3.0
    assert summ[2]["termination"] == 7 and np.array_equal(p1[2], poses[2])
    assert summ[1]["termination"] in (1, 2, 3)
    # per-frame cameras: every refined frame moves its own focal
    p2, i2, _, _ = po.frame_loop(poses, intr0, X, uv, inl, np.ones(S, bool), 0, False, 12.0, 100)
    assert i2[2, 0] == 520.0 and len(set(np.round(i2[[0, 1, 3], 0], 9))) == 3
    # the pre-filter drops observations behind the camera or beyond max_reproj_error at the input pose
    uv_bad = uv.copy()
    uv_bad[1, :10] += 50.0
    _, _, used2, _ = po.frame_loop(poses, intr, X, uv_bad, inl, np.zeros(S, bool), 0, False, 12.0, 0)
    assert not used2[1, :10].any() and used2[1, 10:].all()


@pytest.mark.parametrize("bad", ["nan", "camera_plane"])
def test_non_finite_start_fails_at_iteration_zero(bad):
    """A non-finite residual at the starting point (a NaN observation, or a point exactly on the camera plane; nothing
    filters them when max_reproj_error is 0, as in init_refine_pose) ends the solve with FAILURE before the first
    iteration and leaves pose and intrinsics untouched -- Ceres' failed initial evaluation [3P-memory]."""
    _, _, X, uv, p0, i0 = _case(1)
    X, uv = X.copy(), uv.copy()
    if bad == "nan":
        uv[7, 0] = np.nan
    else:
        p0 = p0.copy()
        p0[2, 3] = 0.0                                    # the world origin is then exactly at depth 0
        X[7] = 0.0
    trace = []
    p1, i1, sm = po.pose_refinement(p0, i0, X, uv, np.ones(len(X), bool), 1, trace=trace)
    assert sm["termination"] == po.FAILURE and sm["iterations"] == 0 and sm["successful"] == 0
    assert not np.isfinite(sm["initial_cost"]) and not np.isfinite(sm["final_cost"])
    assert sm["final_radius"] == po.PoseOptions().initial_trust_region_radius
    assert np.array_equal(p1, p0) and np.array_equal(i1, i0) and trace == []
    # the same observation outside the inlier set does not matter
    m = np.ones(len(X), bool)
    m[7] = False
    _, _, sm2 = po.pose_refinement(p0, i0, X, uv, m, 1)
    assert sm2["termination"] in (po.CONV_GRADIENT, po.CONV_FUNCTION, po.CONV_PARAMETER) and sm2["iterations"] > 0


def test_trace_records_gradient_at_every_accepted_point():
    _, _, X, uv, p0, i0 = _case(0)
    trace = []
    _, _, sm = po.pose_refinement(p0, i0, X, uv, np.ones(len(X), bool), 0, trace=trace)
    acc = [t for t in trace if t.get("accepted")]
    assert acc[0]["it"] == 0 and abs(acc[0]["cost"] - sm["initial_cost"]) == 0
    assert len(acc) == sm["successful"] + 1 and acc[-1]["cost"] == sm["final_cost"]
    assert all(a["grad_max"] > 0 for a in acc)
    steps = [t for t in trace if "step_norm" in t]
    assert len(steps) == sm["iterations"] and all(t["x_norm"] > 1 for t in steps)
