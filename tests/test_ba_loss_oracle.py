"""The robust-loss restatement of bundle adjustment (tests/ba_loss_oracle.py) against closed forms, finite differences
and scipy.optimize.least_squares, and its trivial path against the plain oracles."""
import numpy as np
import pytest

from oracle import ba_oracle as bo
from oracle import ba_pcg_oracle as bpo
from tests import ba_loss_oracle as lo
from tests.helpers import ba_case, so3_log

ROBUST = ("SOFT_L1", "CAUCHY")


def _closed_form(s, loss, a):
    """Ceres' expressions as written (log(1 + s c), 2 b (sqrt(1 + s c) - 1)), in extended precision where numpy has it"""
    s = np.asarray(s, dtype=np.longdouble)
    b = np.longdouble(a) * np.longdouble(a)
    c = 1 / b
    if loss == "CAUCHY":
        rho = b * np.log1p(s * c)
        rho1 = np.maximum(np.longdouble(lo.DBL_MIN), 1 / (1 + s * c))
        return rho, rho1, -c * rho1 * rho1
    t = np.sqrt(1 + s * c)
    rho = 2 * b * (s * c) / (t + 1)
    rho1 = np.maximum(np.longdouble(lo.DBL_MIN), 1 / t)
    return rho, rho1, -(c * rho1) / (2 * (1 + s * c))


@pytest.mark.parametrize("loss", ROBUST)
@pytest.mark.parametrize("a", [1e-3, 0.5, 1.0, 4.0, 1e6])
def test_rho_matches_closed_form(loss, a):
    s = np.concatenate([[0.0], np.logspace(-12, 12, 97), [3.0, 1e300]])
    rho, rho1, rho2 = lo.loss_rho(s, loss, a)
    r, r1, r2 = _closed_form(s, loss, a)
    for got, ref in ((rho, r), (rho1, r1), (rho2, r2)):
        ref = ref.astype(np.float64)
        np.testing.assert_allclose(got, ref, rtol=4e-15, atol=0.0)
    assert rho[0] == 0.0 and rho1[0] == 1.0                       # s = 0: the weight of a masked observation
    assert np.all(rho2 <= 0.0)                                     # the Corrector's alpha = 0 branch, everywhere


@pytest.mark.parametrize("loss", ROBUST)
def test_rho_at_infinity_and_nan(loss):
    rho, rho1, rho2 = lo.loss_rho(np.array([np.inf, np.nan]), loss, 1.0)
    assert rho[0] == np.inf and rho1[0] == lo.DBL_MIN and rho2[0] <= 0.0   # Ceres' DBL_MIN clamp
    assert np.isnan(rho[1])


@pytest.mark.parametrize("loss", ROBUST)
def test_scale_limits(loss):
    s = np.logspace(-6, 6, 25)
    # very large scale: the trivial loss to rounding (no cancellation in rho)
    rho, rho1, _ = lo.loss_rho(s, loss, 1e8)
    np.testing.assert_allclose(rho, s, rtol=1e-9)
    np.testing.assert_allclose(rho1, 1.0, rtol=1e-9)
    # very small scale: rho grows like 2 a |r| (SoftL1) or b log(s / b) (Cauchy)
    a = 1e-4
    s = s[s >= 1.0]
    rho, _, _ = lo.loss_rho(s, loss, a)
    ref = 2.0 * a * np.sqrt(s) if loss == "SOFT_L1" else a * a * np.log(s / (a * a))
    np.testing.assert_allclose(rho, ref, rtol=1e-3)


def test_unknown_loss_raises():
    with pytest.raises(ValueError):
        lo.loss_rho(1.0, "HUBER", 1.0)


def _outlier_case(S, N, cam, mode, seed, invisible_frac=0.2):
    c = ba_case(S, N, cam, mode, seed=seed, invisible_frac=invisible_frac)
    return lo.with_outliers(c, seed=seed)


@pytest.mark.parametrize("loss,a", [("SOFT_L1", 0.5), ("CAUCHY", 1.0), ("CAUCHY", 4.0)])
@pytest.mark.parametrize("cam,mode", [("SIMPLE_RADIAL", bo.INTR_PER_FRAME), ("SIMPLE_PINHOLE", bo.INTR_SHARED)])
def test_robust_gradient_matches_finite_differences(loss, a, cam, mode):
    """g = J'^T r' of the corrected pair is the gradient of 0.5 sum rho: central differences through apply_step"""
    S, N = 4, 40
    c = _outlier_case(S, N, cam, mode, seed=5)
    model = c["model"]
    dc, ns = bo.dims(model, mode)
    blk = lo.build_blocks(c["poses"], c["intr"], c["points"], c["uv"], c["mask"], model, mode,
                          loss_function_type=loss, loss_function_scale=a)
    Hc, gc = bo._assemble_camera_system(blk, S, dc, ns)
    D = S * dc + ns

    def cost(d_c, d_p):
        p, i, x = bo.apply_step(c["poses"], c["intr"], c["points"], d_c[:S * dc].reshape(S, dc), d_c[S * dc:], d_p,
                                model, mode)
        return lo.cost_only(p, i, x, c["uv"], c["mask"], model, loss, a)

    assert blk["cost"] == pytest.approx(cost(np.zeros(D), np.zeros((N, 3))), rel=1e-15)
    h = 1e-6
    fd_c = np.zeros(D)
    for j in range(D):
        e = np.zeros(D)
        e[j] = h
        fd_c[j] = (cost(e, np.zeros((N, 3))) - cost(-e, np.zeros((N, 3)))) / (2.0 * e[j])
    np.testing.assert_allclose(gc, fd_c, rtol=2e-5, atol=2e-5 * np.abs(gc).max())
    fd_p = np.zeros((N, 3))
    for n in range(0, N, 3):
        for k in range(3):
            e = np.zeros((N, 3))
            e[n, k] = h
            fd_p[n, k] = (cost(np.zeros(D), e) - cost(np.zeros(D), -e)) / (2.0 * h)
    np.testing.assert_allclose(blk["g_p"][::3], fd_p[::3], rtol=2e-5, atol=2e-5 * np.abs(blk["g_p"]).max())


@pytest.mark.parametrize("loss,scipy_loss", [("CAUCHY", "cauchy"), ("SOFT_L1", "soft_l1")])
@pytest.mark.parametrize("a", [1.0, 4.0])
def test_robust_minimum_matches_scipy(loss, scipy_loss, a):
    """the oracle's robust LM minimum on a C1-size problem (8 x 256, SIMPLE_PINHOLE, constant intrinsics) against
    scipy.optimize.least_squares with one residual |r| per observation, whose cost 0.5 a^2 sum rho_scipy(s / a^2) is
    0.5 sum rho(s) exactly; the gauge as the oracle's (first pose and the x of the second translation constant)"""
    from scipy.optimize import least_squares
    from scipy.sparse import lil_matrix
    S, N = 8, 256
    mode = bo.INTR_CONST
    c = _outlier_case(S, N, "SIMPLE_PINHOLE", mode, seed=3, invisible_frac=0.0)
    model = c["model"]
    opt = bo.LMOptions(max_num_iterations=300, gradient_tolerance=1e-10, function_tolerance=0.0,
                       parameter_tolerance=0.0)                     # runs until a step no longer changes the cost
    p_o, i_o, x_o, summ = lo.lm_solve(c["poses"], c["intr"], c["points"], c["uv"], c["mask"], model, mode,
                                      loss_function_type=loss, loss_function_scale=a, options=opt)
    assert summ["final_cost"] < 0.5 * summ["initial_cost"]

    mask = c["mask"]
    si, ni = np.nonzero(mask)
    free = np.ones(S * 6, dtype=bool)
    free[0:6] = False
    free[6 + 3] = False
    nf = int(free.sum())

    def unpack(x):
        d = np.zeros(S * 6)
        d[free] = x[:nf]
        return d.reshape(S, 6), x[nf:].reshape(N, 3)

    def state(x):
        d, X = unpack(x)
        p, _, _ = bo.apply_step(c["poses"], c["intr"], c["points"], d, np.zeros(0), np.zeros((N, 3)), model, mode)
        return p, X

    def fun(x):
        p, X = state(x)
        uvh, _ = bo.project(p, c["intr"], X, model)
        r = (uvh - c["uv"])[si, ni]
        return np.sqrt(np.sum(r * r, axis=-1))

    sp = lil_matrix((len(si), nf + 3 * N), dtype=int)
    col = np.full(S * 6, -1)
    col[free] = np.arange(nf)
    for k, (s, n) in enumerate(zip(si, ni)):
        for j in col[s * 6:(s + 1) * 6]:
            if j >= 0:
                sp[k, j] = 1
        sp[k, nf + 3 * n:nf + 3 * n + 3] = 1
    # scipy's cost at the oracle's minimum is the oracle's cost ...
    d_o = np.zeros((S, 6))
    d_o[:, 0:3] = 0.5 * so3_log(p_o[:, :, :3] @ c["poses"][:, :, :3].transpose(0, 2, 1))
    d_o[:, 3:6] = p_o[:, :, 3] - c["poses"][:, :, 3]
    x_or = np.concatenate([d_o.reshape(-1)[free], x_o.reshape(-1)])
    f = fun(x_or)
    assert 0.5 * np.sum(lo.loss_rho(f * f, loss, a)[0]) == pytest.approx(summ["final_cost"], rel=1e-12)
    # ... and scipy, started there, finds no lower cost and stays
    res = least_squares(fun, x_or, jac_sparsity=sp, loss=scipy_loss, f_scale=a, method="trf", x_scale="jac",
                        ftol=1e-15, xtol=1e-15, gtol=1e-15, max_nfev=100)
    assert res.cost >= summ["final_cost"] * (1.0 - 1e-12)
    p_s, X_s = state(res.x)
    assert np.abs(X_s - x_o).max() < 1e-6 * max(1.0, np.abs(x_o).max())


@pytest.mark.parametrize("cam,mode", [("SIMPLE_RADIAL", bo.INTR_SHARED), ("SIMPLE_PINHOLE", bo.INTR_PER_FRAME)])
def test_trivial_path_is_the_oracle_bit_for_bit(cam, mode):
    c = _outlier_case(6, 64, cam, mode, seed=9)
    args = (c["poses"], c["intr"], c["points"], c["uv"], c["mask"], c["model"], mode)
    opt = bo.LMOptions(max_num_iterations=8)
    ref_blk = bo.build_blocks(*args)
    blk = lo.build_blocks(*args, loss_function_type="TRIVIAL", loss_function_scale=3.0)
    assert blk["cost"] == ref_blk["cost"]
    for k in ref_blk:
        if k != "cost":
            assert np.array_equal(blk[k], ref_blk[k])
    for solver, ref_fn in (("dense_schur", bo.lm_solve), ("iterative_schur", bpo.lm_solve)):
        ref = ref_fn(*args, options=opt) if solver == "dense_schur" else ref_fn(*args, options=opt,
                                                                                  linear_solver=solver)
        out = lo.lm_solve(*args, linear_solver=solver, options=opt)
        for r, o in zip(ref[:3], out[:3]):
            assert np.array_equal(r, o)
        assert ref[3]["final_cost"] == out[3]["final_cost"] and ref[3]["iterations"] == out[3]["iterations"]


def test_robust_leaves_the_oracles_as_they_were():
    c = _outlier_case(4, 32, "SIMPLE_PINHOLE", bo.INTR_CONST, seed=1)
    args = (c["poses"], c["intr"], c["points"], c["uv"], c["mask"], c["model"], bo.INTR_CONST)
    before = bo.build_blocks(*args)["cost"]
    robust = lo.build_blocks(*args, loss_function_type="CAUCHY")["cost"]
    assert robust < before
    assert bo.build_blocks(*args)["cost"] == before
    with pytest.raises(RuntimeError):
        with lo.robust("CAUCHY"):
            raise RuntimeError("inside")
    assert bo.build_blocks(*args)["cost"] == before
