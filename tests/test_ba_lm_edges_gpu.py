"""The trust-region control of vgg_ba_solve against oracle/ba_oracle.py lm_solve: every termination, rejected and invalid
steps, the radius cap, jacobi_scaling = 0, constant cameras or points, non-finite observations, and reduced systems of
order D > 7000 (where the backward substitution is cuBLAS Dtrsv on the mirrored row-major factor).

What must match exactly: termination, iterations, successful steps and each iteration's outcome (trace column 7:
accepted 1 / rejected 0 / invalid 2).  Where no step was accepted the returned parameters must be bit-identical to the
input.  For CONVERGENCE_FUNCTION the returned state is the last accepted iterate: final_cost == trace[-1, 1] (the cost
the terminating iteration started from) != trace[-1, 2].

Bars: the rounding bands of tests/ba_harness.py (costs EPS_COST, model change EPS_MODEL, rho e_rho, the radius its
running bar), and its whole-solve bars for the final parameters.  They hold only while cost_change is well above the
rounding of the cost, so every case here stops before the minimum: by a gradient / function / parameter tolerance
placed between two iterations of an oracle run without tolerances, or by max_num_iterations.

Margins (asserted on the oracle's trace, printed per case as the smallest ratio margin / band): no decision may lie
within its band -- rho vs min_relative_decrease (e_rho), |cost_change| vs function_tolerance cost (e_cc), gmax vs
gradient_tolerance and step_norm vs parameter_tolerance (|x| + parameter_tolerance) (1e-9 relative), radius vs
min_trust_region_radius (its radius bar).

Non-finite values.  A NaN or inf observation under a valid mask makes the initial cost and the gradient non-finite:
every step is invalid and the solve ends in FAILURE_INVALID_STEPS (or MIN_TRUST_REGION_RADIUS when the halved radius
gets there first), with the parameters unchanged; with a gradient_tolerance above every finite gradient entry it must
not stop as converged at iteration 0 (the gradient max-norm propagates NaN).  A finite-cost start whose candidate cost
is non-finite (Ceres: cost DBL_MAX, a rejected step; the CUDA loop: an invalid step) has no deterministic input here:
the observations are float32, so a residual near 1e154 has to come from a float64 principal point, which moves the whole
frame's residuals together and keeps the candidate within a small factor of the initial cost -- that branch is untested.
"""
import ctypes
import functools

import numpy as np
import pytest

from oracle import ba_oracle as bo
from tests.ba_harness import (SHAPES, between, check_decisions, check_one_step, device_solve, first_drop, options,
                              oracle_solve)
from tests.helpers import ba_case, banded_ba_case, shuffled_twin

pytestmark = pytest.mark.gpu

C3 = (400, 4096, "SIMPLE_RADIAL", bo.INTR_SHARED)


def _case(shape, seed=11):
    S, N, cam, mode = shape
    if shape == C3:
        return ba_case(S, N, cam, mode, seed=0, invisible_frac=0.0)
    return ba_case(S, N, cam, mode, seed=seed)


@functools.lru_cache(maxsize=None)
def _probe(shape, iters):
    """the oracle's trace with every tolerance off: where the gradient / function / parameter tests would fire"""
    _, opt = options(max_num_iterations=iters, gradient_tolerance=0.0)
    ref = oracle_solve(_case(shape), opt=opt, use_c=bo._load_c() is not None)
    return ref["s"], ref["trace"]


def _solve(c, uv=None, mask=None, param_const=None, point_const=None, check_margins=True, label="", **kw):
    """run both solvers on the same input and compare them (tests/ba_harness.py check_decisions); returns (oracle
    summary, oracle trace, GPU summary, GPU trace)"""
    import torch
    S, N = (c["mask"] if mask is None else mask).shape
    pc = bo.default_param_const(S, c["model"], c["mode"]) if param_const is None else param_const
    ptc = np.zeros(N, dtype=bool) if point_const is None else point_const
    o, opt = options(**kw)
    ref = oracle_solve(c, uv, mask, pc, ptc, opt, use_c=bo._load_c() is not None)
    got = device_solve(c, torch.device("cuda:0"), uv=uv, mask=mask, param_const=pc, point_const=ptc, options=o)
    check_decisions(got, ref, opt, c, margins=check_margins, label=label)
    return ref["s"], ref["trace"], got["s"], got["trace"]


def _label(shape, what):
    S, N, cam, mode = shape
    return f"{what} {S}x{N} {cam} mode={mode}"


# ------------------------------------------------------------------------------------------------------------------
# terminations
# ------------------------------------------------------------------------------------------------------------------

@pytest.mark.parametrize("shape", SHAPES[:3] + [C3])
def test_gradient_at_iteration_zero(cuda_dev, shape):
    summ, _ = _probe(shape, 1)
    _, _, s, _ = _solve(_case(shape), gradient_tolerance=10.0 * summ["initial_gmax"], label=_label(shape, "gradient@0"))
    assert s.termination == "CONVERGENCE_GRADIENT" and s.iterations == 0


@pytest.mark.parametrize("shape", SHAPES)
def test_gradient_after_successes(cuda_dev, shape):
    """gradient_tolerance placed below the gmax of the start and the first accepted iterate and above a later one"""
    summ, trace = _probe(shape, 5)
    g = [summ["initial_gmax"]] + [r["gmax"] for r in trace if r["outcome"] == 1]
    k, gtol = first_drop(g, 2)
    _, _, s, _ = _solve(_case(shape), gradient_tolerance=gtol, label=_label(shape, "gradient"))
    assert s.termination == "CONVERGENCE_GRADIENT" and s.successful == k >= 2


def test_gradient_c3(cuda_dev):
    """gradient_tolerance between the gmax of the 2nd and the 3rd accepted iterate"""
    summ, trace = _probe(C3, 3)
    g = [r["gmax"] for r in trace]
    assert all(r["outcome"] == 1 for r in trace) and g[2] < g[1] < summ["initial_gmax"]
    _, _, s, _ = _solve(_case(C3), gradient_tolerance=between(g[2], g[1]), label=_label(C3, "gradient"))
    assert s.termination == "CONVERGENCE_GRADIENT" and s.iterations == 3


@pytest.mark.parametrize("shape", SHAPES + [C3])
def test_function_tolerance(cuda_dev, shape):
    """a function_tolerance that fires at the 3rd valid iteration or later: the candidate is discarded"""
    _, trace = _probe(shape, 3 if shape == C3 else 12)
    assert all(r["outcome"] != 2 for r in trace)
    at, ftol = first_drop([abs(r["cost_change"]) / r["cost"] for r in trace], 2)
    _, trace, s, _ = _solve(_case(shape), function_tolerance=ftol, label=_label(shape, "function"))
    assert s.termination == "CONVERGENCE_FUNCTION" and s.iterations == at + 1
    assert s.successful == sum(r["outcome"] == 1 for r in trace) >= 2


@pytest.mark.parametrize("shape", SHAPES + [C3])
def test_parameter_tolerance(cuda_dev, shape):
    """parameter_tolerance > 0 runs xnorm_kernel (at C3 one 1024-thread CTA sums 4096 points and 400 cameras)"""
    _, trace = _probe(shape, 3 if shape == C3 else 12)
    assert all(r["outcome"] != 2 for r in trace)
    at, ptol = first_drop([r["step_norm"] / r["x_norm"] for r in trace], 1)
    _, trace, s, _ = _solve(_case(shape), parameter_tolerance=ptol, label=_label(shape, "parameter"))
    assert s.termination == "CONVERGENCE_PARAMETER" and s.iterations == at + 1 and s.successful == at


@pytest.mark.parametrize("iters", [1, 2, 3])
@pytest.mark.parametrize("shape", SHAPES[:2])
def test_no_convergence(cuda_dev, shape, iters):
    _, _, s, _ = _solve(_case(shape), max_num_iterations=iters, label=_label(shape, f"max {iters} iterations"))
    assert s.termination == "NO_CONVERGENCE" and s.iterations == iters


@pytest.mark.parametrize("shape", SHAPES[2:4])
def test_min_radius_at_start(cuda_dev, shape):
    _, _, s, _ = _solve(_case(shape), initial_trust_region_radius=1e-3, min_trust_region_radius=1e-2,
                        label=_label(shape, "radius below the minimum at the start"))
    assert s.termination == "MIN_TRUST_REGION_RADIUS" and s.iterations == 0


@pytest.mark.parametrize("shape", SHAPES[:2] + SHAPES[4:])
def test_min_radius_by_rejections(cuda_dev, shape):
    """min_relative_decrease = 10: every step is rejected, radius = 1e4 / 2^(k (k + 1) / 2) exactly, and the 8th
    iteration would run below 1e-3"""
    _, _, s, tr = _solve(_case(shape), min_relative_decrease=10.0, min_trust_region_radius=1e-3,
                         label=_label(shape, "rejections"))
    assert s.termination == "MIN_TRUST_REGION_RADIUS" and s.iterations == 7 and s.successful == 0
    assert tr[:, 5].tolist() == [1e4 / 2.0 ** (k * (k + 1) // 2) for k in range(7)]
    assert s.final_radius == 1e4 / 2.0 ** 28


@pytest.mark.parametrize("shape", SHAPES[1:3])
def test_radius_cap(cuda_dev, shape):
    _, _, s, tr = _solve(_case(shape), max_trust_region_radius=2e4, max_num_iterations=8,
                         label=_label(shape, "radius cap"))
    assert s.termination == "NO_CONVERGENCE"
    acc = np.nonzero(tr[:, 7] == 1)[0]
    assert len(acc) >= 2 and tr[acc[0] + 1, 5] == 2e4 and (tr[:, 5] <= 2e4).all()


@pytest.mark.parametrize("shape", [SHAPES[0], SHAPES[1], SHAPES[4]])
def test_no_jacobi_scaling(cuda_dev, shape):
    _, _, s, _ = _solve(_case(shape), jacobi_scaling=False, max_num_iterations=4,
                        label=_label(shape, "jacobi_scaling = 0"))
    assert s.termination == "NO_CONVERGENCE" and s.successful >= 2


# ------------------------------------------------------------------------------------------------------------------
# non-finite observations: invalid steps
# ------------------------------------------------------------------------------------------------------------------

def _bad_observation(c, value):
    uv, mask = c["uv"].copy(), c["mask"].copy()
    uv[2, 7] = value
    mask[2, 7] = True
    return uv, mask


@pytest.mark.parametrize("max_invalid", [10, 3])
@pytest.mark.parametrize("value", [np.nan, np.inf])
@pytest.mark.parametrize("shape", [SHAPES[0], SHAPES[1], SHAPES[4]])
def test_failure_on_non_finite_observation(cuda_dev, shape, value, max_invalid):
    c = _case(shape)
    uv, mask = _bad_observation(c, value)
    _, _, s, tr = _solve(c, uv, mask, max_num_consecutive_invalid_steps=max_invalid,
                         label=_label(shape, f"uv = {value}, {max_invalid} invalid steps"))
    assert s.termination == "FAILURE_INVALID_STEPS" and s.iterations == max_invalid and s.successful == 0
    assert tr[:, 5].tolist() == [1e4 / 2.0 ** k for k in range(max_invalid)]       # the radius each step ran with


@pytest.mark.parametrize("max_invalid,termination", [(4, "FAILURE_INVALID_STEPS"), (5, "MIN_TRUST_REGION_RADIUS")])
def test_invalid_steps_meet_min_radius(cuda_dev, max_invalid, termination):
    """after 4 invalid steps the radius is 625 < 700: the 4th step ends the solve first when 4 are allowed"""
    c = _case(SHAPES[2])
    uv, mask = _bad_observation(c, np.nan)
    _, _, s, _ = _solve(c, uv, mask, max_num_consecutive_invalid_steps=max_invalid, min_trust_region_radius=700.0,
                        label=f"NaN observation, {max_invalid} invalid steps, min radius 700")
    assert s.termination == termination and s.iterations == 4


@pytest.mark.parametrize("shape", [SHAPES[0], SHAPES[3]])
def test_nan_gradient_is_not_convergence(cuda_dev, shape):
    """a gradient_tolerance above every finite gradient entry: a NaN entry still keeps the solve going"""
    c = _case(shape)
    uv, mask = _bad_observation(c, np.nan)
    summ, _, s, _ = _solve(c, uv, mask, gradient_tolerance=1e30, label=_label(shape, "NaN gradient, tolerance 1e30"))
    assert np.isnan(summ["initial_gmax"])
    assert s.termination == "FAILURE_INVALID_STEPS" and s.iterations == 10


# ------------------------------------------------------------------------------------------------------------------
# structure-only / motion-only
# ------------------------------------------------------------------------------------------------------------------

@pytest.mark.parametrize("shape", SHAPES[:3])
def test_structure_only(cuda_dev, shape):
    c = _case(shape)
    S, N = c["mask"].shape
    dc, ns = bo.dims(c["model"], c["mode"])
    pc = np.ones(S * dc + ns, dtype=bool)
    _, _, s, _ = _solve(c, param_const=pc, max_num_iterations=3, label=_label(shape, "every camera parameter constant"))
    assert s.successful >= 1


@pytest.mark.parametrize("shape", SHAPES[3:])
def test_motion_only(cuda_dev, shape):
    c = _case(shape)
    _, _, s, _ = _solve(c, point_const=np.ones(c["mask"].shape[1], dtype=bool), max_num_iterations=3,
                        label=_label(shape, "every point constant"))
    assert s.successful >= 1


@pytest.mark.parametrize("shape", [SHAPES[0], SHAPES[1]])
def test_frame_without_observation(cuda_dev, shape):
    c = _case(shape)
    mask = c["mask"].copy()
    mask[4] = False
    _, _, s, _ = _solve(c, mask=mask, max_num_iterations=4, label=_label(shape, "frame 4 sees nothing"))
    assert s.termination == "NO_CONVERGENCE" and s.successful >= 2


# ------------------------------------------------------------------------------------------------------------------
# reduced systems of order D > 7000
# ------------------------------------------------------------------------------------------------------------------

def _big_case(name):
    if name == "1000x2048":       # D = 7000: the own backward substitution's last order
        return ba_case(1000, 2048, "SIMPLE_PINHOLE", bo.INTR_PER_FRAME, seed=41)
    if name == "1001x2048":       # D = 7007: cuBLAS Dtrsv
        return ba_case(1001, 2048, "SIMPLE_PINHOLE", bo.INTR_PER_FRAME, seed=42)
    if name == "1001x6000":       # D = 7007, banded (video-like)
        return banded_ba_case(1001, 6000, "SIMPLE_PINHOLE", bo.INTR_PER_FRAME, life=24, seed=43)
    raise KeyError(name)


@pytest.mark.parametrize("name,band", [("1000x2048", None), ("1001x2048", None), ("1001x6000", None),
                                       ("1001x6000", "0")])
def test_big_step_backward_error(cuda_dev, name, band):
    """one LM step at D = 7000 / 7007 in the full damped system (test_lm_step_gpu.py's backward error <= 1e-12); band
    "0": the banded case's shuffled twin, which takes the dense path"""
    c = _big_case(name)
    if band == "0":
        c = shuffled_twin(c)
    S, N = c["mask"].shape
    dc, ns = bo.dims(c["model"], c["mode"])
    pc = bo.default_param_const(S, c["model"], c["mode"])
    ptc = np.zeros(N, dtype=bool)
    o, _ = options(max_num_iterations=1, function_tolerance=0.0, gradient_tolerance=0.0, parameter_tolerance=0.0)
    got = device_solve(c, cuda_dev, param_const=pc, options=o)
    check_one_step(c, got, pc, ptc, label=f"big step {name}{' shuffled' if band == '0' else ''}: D = {S * dc + ns}")


def test_big_trajectory(cuda_dev):
    """3 LM iterations at D = 7007 (cuBLAS back-substitution in every one) against the oracle"""
    _, _, s, _ = _solve(_big_case("1001x2048"), max_num_iterations=3, check_margins=False,
                        label="1001x2048 D = 7007, 3 iterations")
    assert s.iterations == 3 and s.successful >= 1


@pytest.mark.parametrize("n", [7001, 8009])
def test_cholesky_above_7000(cuda_dev, n):
    """csrc/chol.cu at more than 55 panels in one captured graph against numpy.linalg.cholesky"""
    import torch
    from vggsfm_b200 import _lib
    rng = np.random.default_rng(n)
    G = rng.normal(size=(n, n)) * 0.05
    A = G + G.T
    A += np.diag(np.abs(A).sum(1) + 1.0)          # diagonally dominant, so SPD
    lda = (n + 127) // 128 * 128
    buf = torch.zeros(n, lda, dtype=torch.float64, device=cuda_dev)
    buf[:, :n] = torch.from_numpy(np.tril(A)).to(cuda_dev)
    ws = torch.empty(((n + 127) // 128) * 131072 + 1024, dtype=torch.uint8, device=cuda_dev)
    info = ctypes.c_int(-1)
    L = _lib.lib()
    _lib.check(L.vgg_cholesky_lower(n, lda, buf.data_ptr(), ws.data_ptr(), ws.numel(), ctypes.byref(info),
                                    torch.cuda.current_stream().cuda_stream), "vgg_cholesky_lower")
    assert info.value == 0
    ref = np.linalg.cholesky(A)
    full = buf.cpu().numpy()[:, :n]
    err = np.abs(np.tril(full) - ref).max() / np.abs(ref).max()
    print(f"cholesky n = {n}: max |L - L_lapack| / max |L| = {err:.2e}")
    assert err <= 1e-10
    assert np.array_equal(np.triu(full, 1), np.tril(full, -1).T)
