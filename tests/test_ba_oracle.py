"""CPU tests of the BA oracle itself (no GPU): analytic Jacobians vs finite differences, the LM solve vs
scipy.optimize.least_squares, and the COLMAP wrapper semantics.  The BA oracle is 'parity unpinned'
(pycolmap absent), so these are the checks that anchor it."""
import numpy as np
import pytest

from oracle import ba_oracle as bo
from tests.helpers import ba_case


@pytest.mark.parametrize("cam,mode", [("SIMPLE_PINHOLE", bo.INTR_PER_FRAME), ("SIMPLE_RADIAL", bo.INTR_SHARED),
                                      ("SIMPLE_RADIAL", bo.INTR_PER_FRAME)])
def test_jacobians_vs_finite_differences(cam, mode):
    c = ba_case(5, 30, cam, mode, seed=4)
    S, N = c["mask"].shape
    model = c["model"]
    res, Jc, Jp = bo.residuals_and_jacobians(c["poses"], c["intr"], c["points"], c["uv"], c["mask"], model)

    def resid(p, i, x):
        uvh, _ = bo.project(p, i, x, model)
        return (uvh - c["uv"]) * c["mask"][..., None]

    eps = 1e-6
    ni = bo.n_intr(model)
    for col in range(6 + ni):
        d = np.zeros((S, 6 + ni))
        d[:, col] = eps
        pp, ii, xx = bo.apply_step(c["poses"], c["intr"], c["points"], d, np.zeros(2), 0 * c["points"], model, bo.INTR_PER_FRAME)
        pm, im, xm = bo.apply_step(c["poses"], c["intr"], c["points"], -d, np.zeros(2), 0 * c["points"], model, bo.INTR_PER_FRAME)
        fd = (resid(pp, ii, xx) - resid(pm, im, xm)) / (2 * eps)
        assert np.abs(fd - Jc[..., col]).max() <= 1e-5 * max(1.0, np.abs(Jc[..., col]).max())
    for col in range(3):
        d = np.zeros_like(c["points"])
        d[:, col] = eps
        fd = (resid(c["poses"], c["intr"], c["points"] + d) - resid(c["poses"], c["intr"], c["points"] - d)) / (2 * eps)
        assert np.abs(fd - Jp[..., col]).max() <= 1e-5 * np.abs(Jp[..., col]).max()


@pytest.mark.parametrize("cam,mode", [("SIMPLE_PINHOLE", bo.INTR_PER_FRAME), ("SIMPLE_RADIAL", bo.INTR_SHARED)])
def test_lm_optimum_matches_scipy(cam, mode):
    from scipy.optimize import least_squares
    c = ba_case(6, 40, cam, mode, seed=3)
    S, N = c["mask"].shape
    model = c["model"]
    p2, i2, x2, summ = bo.lm_solve(c["poses"], c["intr"], c["points"], c["uv"], c["mask"], model, mode)
    assert summ["termination"] == "CONVERGENCE_GRADIENT"
    dc, ns = bo.dims(model, mode)
    pc = bo.default_param_const(S, model, mode)
    free = np.nonzero(~pc)[0]

    def fun(x):
        d = np.zeros(S * dc + ns)
        d[free] = x[:len(free)]
        pp, ii, xx = bo.apply_step(c["poses"], c["intr"], c["points"], d[:S * dc].reshape(S, dc), d[S * dc:],
                                   x[len(free):].reshape(N, 3), model, mode)
        uvh, _ = bo.project(pp, ii, xx, model)
        return ((uvh - c["uv"]) * c["mask"][..., None]).reshape(-1)

    r = least_squares(fun, np.zeros(len(free) + 3 * N), method="trf", xtol=1e-15, ftol=1e-15, gtol=1e-12,
                      x_scale="jac", max_nfev=200)
    assert abs(r.cost - summ["final_cost"]) <= 1e-9 * r.cost


def test_negative_depth_and_normalize():
    c = ba_case(6, 20, "SIMPLE_PINHOLE", bo.INTR_PER_FRAME, seed=9, invisible_frac=0.0)
    pts = c["points"].copy()
    pts[3] = [0, 0, -2.0]
    mask, alive = bo.filter_negative_depth(c["poses"], pts, c["mask"])
    assert not alive[3] and not mask[:, 3].any() and alive.sum() == 19
    poses, X = bo.normalize(c["poses"], pts, 5.0, 0.1, 0.9)
    centers = -np.einsum("sji,sj->si", poses[:, :, :3], poses[:, :, 3])
    cs = np.sort(centers.astype(np.float32), axis=0)
    ext = np.linalg.norm(cs[int(0.9 * 5)] - cs[int(0.1 * 5)])
    assert abs(ext - 5.0) < 1e-5
    # projections are invariant under the similarity
    uv0, _ = bo.project(c["poses"], c["intr"], pts, c["model"])
    uv1, _ = bo.project(poses, c["intr"], X, c["model"])
    assert np.abs(uv0 - uv1).max() < 1e-8


@pytest.mark.parametrize("cam,mode", [("SIMPLE_PINHOLE", bo.INTR_PER_FRAME), ("SIMPLE_RADIAL", bo.INTR_SHARED),
                                      ("SIMPLE_RADIAL", bo.INTR_CONST)])
def test_c_restatement_matches_numpy(cam, mode):
    if bo._load_c() is None:
        pytest.skip("oracle/_build/libba_blocks_ref.so not built")
    c = ba_case(7, 50, cam, mode, seed=8)
    pc = np.zeros(50, dtype=bool)
    pc[::5] = True
    a = bo.build_blocks(c["poses"], c["intr"], c["points"], c["uv"], c["mask"], c["model"], mode, pc)
    b = bo.build_blocks_c(c["poses"], c["intr"], c["points"], c["uv"], c["mask"], c["model"], mode, pc)
    assert abs(a["cost"] - b["cost"]) <= 1e-12 * a["cost"]
    for k in a:
        if k != "cost":
            assert np.abs(a[k] - b[k]).max() <= 1e-11 * max(1.0, np.abs(a[k]).max()), k


def test_lm_trace_fields():
    """lm_solve's trace: the outcome of every iteration, cost_change, x_norm and (after a success) gmax as the solver
    decided with them; an invalid step records the radius it ran with; a NaN gradient is not convergence."""
    c = ba_case(8, 60, "SIMPLE_PINHOLE", bo.INTR_PER_FRAME, seed=4)
    S, N = c["mask"].shape
    pc = bo.default_param_const(S, c["model"], c["mode"])
    ptc = np.zeros(N, dtype=bool)
    trace = []
    o = bo.LMOptions()
    o.max_num_iterations = 6
    p, i, x, summ = bo.lm_solve(c["poses"], c["intr"], c["points"], c["uv"], c["mask"], c["model"], c["mode"],
                                options=o, trace=trace)
    assert len(trace) == summ["iterations"] and sum(r["outcome"] == 1 for r in trace) == summ["successful"]
    dc, ns = bo.dims(c["model"], c["mode"])
    for r in trace:
        assert r["cost_change"] == r["cost"] - r["candidate_cost"] and r["outcome"] == int(r["rho"] > 1e-3)
        assert ("gmax" in r) == (r["outcome"] == 1)
    assert trace[0]["x_norm"] == bo._x_norm(c["poses"], c["intr"], c["points"], S, dc, ns, pc, ptc)
    assert trace[-1]["outcome"] == 1                 # the returned state is the last row's candidate
    blk = bo.build_blocks(p, i, x, c["uv"], c["mask"], c["model"], c["mode"])
    _, gc = bo._assemble_camera_system(blk, S, dc, ns)
    g = max(np.abs(gc[~pc]).max(), np.abs(blk["g_p"]).max())
    assert abs(trace[-1]["gmax"] - g) <= 1e-12 * g
    # NaN observation: invalid steps, each recording the radius it ran with; no convergence on a NaN gradient
    uv = c["uv"].copy()
    uv[2, 7] = np.nan
    mask = c["mask"].copy()
    mask[2, 7] = True
    trace = []
    o = bo.LMOptions()
    o.gradient_tolerance = 1e30
    o.max_num_consecutive_invalid_steps = 4
    p2, _, _, summ = bo.lm_solve(c["poses"], c["intr"], c["points"], uv, mask, c["model"], c["mode"], options=o,
                                 trace=trace)
    assert np.isnan(summ["initial_gmax"]) and summ["termination"] == "FAILURE_INVALID_STEPS"
    assert [r["outcome"] for r in trace] == [2, 2, 2, 2]
    assert [r["radius"] for r in trace] == [1e4, 5e3, 2.5e3, 1.25e3]
    assert np.array_equal(p2, c["poses"])
