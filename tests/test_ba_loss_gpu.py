"""Bundle adjustment under a robust loss (vgg_ba_problem.loss_function_type / loss_function_scale: SOFT_L1, CAUCHY) on
the GPU against the float64 restatement (tests/ba_loss_oracle.py), on problems with about 10 % of the observations
displaced by 20-80 px, so that the weights sqrt(rho') are far from 1.

The bars are those of the trivial loss's tests, which the robust path shares kernel for kernel: blocks at 1e-10 relative
and the Schur complement per entry at 1e-12 sqrt(S_ii S_jj) (test_ba_gpu.py); one LM step at backward error <= 1e-12 in
the full damped system, initial and candidate cost within 1e-12, model change and step norm within 1e-10
(tests/ba_harness.py check_one_step); whole solves with termination, iterations and every iteration's outcome exact,
and no decision of the oracle's run inside its rounding band; DENSE_SCHUR solves also with every iteration and the
final state at the bars of tests/ba_harness.py check_decisions (final cost within EPS_COST)."""
import ctypes

import numpy as np
import pytest

from oracle import ba_oracle as bo
from tests import ba_loss_oracle as lo
from tests.ba_harness import (EPS_COST, SHAPES, assert_clear, check_decisions, check_one_step, check_outcomes,
                              device_args, device_solve, options, oracle_solve, relerr)
from tests.emulated_ranks import run_shards
from tests.helpers import (ba_case, banded_ba_case, hidden_case, rotation_angle_deg, shuffled_twin, to_dev,
                           unpack_camrec)

pytestmark = pytest.mark.gpu

LOSSES = [("SOFT_L1", 0.5), ("SOFT_L1", 1.0), ("SOFT_L1", 4.0), ("CAUCHY", 0.5), ("CAUCHY", 1.0), ("CAUCHY", 4.0)]


def _case(S, N, cam, mode, seed=11, invisible_frac=0.2):
    return lo.with_outliers(ba_case(S, N, cam, mode, seed=seed, invisible_frac=invisible_frac), seed=seed + 100)


# ---- blocks and Schur complement ---------------------------------------------------------------------------------

C2 = (50, 2048, "SIMPLE_RADIAL", bo.INTR_SHARED)


@pytest.mark.parametrize("shape,loss,a", [(sh, l, a) for sh in SHAPES for l, a in LOSSES] +
                         [(C2, "SOFT_L1", 1.0), (C2, "CAUCHY", 1.0)])
def test_blocks_and_schur_match_oracle(cuda_dev, shape, loss, a):
    S, N, cam, mode = shape
    c = _case(S, N, cam, mode, seed=S + N)
    pconst = np.zeros(N, dtype=bool)
    pconst[::7] = True
    _check_blocks_and_schur(cuda_dev, c, pconst, loss, a)


def test_blocks_and_schur_match_oracle_c3(cuda_dev):
    """C3: 400 x 4096, SIMPLE_RADIAL, shared camera, CAUCHY at 1 px"""
    c = _case(400, 4096, "SIMPLE_RADIAL", bo.INTR_SHARED, seed=0, invisible_frac=0.0)
    _check_blocks_and_schur(cuda_dev, c, np.zeros(4096, dtype=bool), "CAUCHY", 1.0)


def _check_blocks_and_schur(dev, c, pconst, loss, a):
    import torch
    from vggsfm_b200 import bundle_adjustment as ba
    S, N = c["mask"].shape
    model, mode = c["model"], c["mode"]
    dc, ns = bo.dims(model, mode)
    D = S * dc + ns
    kw = dict(loss_function_type=loss, loss_function_scale=a)
    ref = lo.build_blocks(c["poses"], c["intr"], c["points"], c["uv"], c["mask"], model, mode, pconst, **kw)
    args = device_args(c, dev)
    ptc = to_dev(pconst.astype(np.uint8), dev)
    out = ba.build_blocks(*args, point_const=ptc, **kw)
    torch.cuda.synchronize()
    g_c, H_cc, H_cs, g_s, H_ss = unpack_camrec(out["camrec"].cpu().numpy(), out["shared"].cpu().numpy(), S, dc, ns)
    tol = 1e-10
    assert abs(out["cost"].item() - ref["cost"]) <= tol * ref["cost"]
    assert relerr(g_c, ref["g_c"]) < tol and relerr(H_cc, ref["H_cc"]) < tol
    assert relerr(out["g_p"].cpu().numpy(), ref["g_p"]) < tol
    Hpp = out["H_pp"].cpu().numpy()
    assert relerr(np.stack([Hpp[:, [0, 1, 2]], Hpp[:, [1, 3, 4]], Hpp[:, [2, 4, 5]]], axis=1), ref["H_pp"]) < tol
    W = out["W"].cpu().numpy()
    assert relerr(W[:, :S * dc].reshape(N, S, dc, 3).transpose(1, 2, 0, 3), ref["W"]) < tol
    if ns:
        assert relerr(W[:, S * dc:S * dc + ns].transpose(1, 0, 2), ref["W_s"]) < tol
        assert relerr(H_cs, ref["H_cs"]) < tol and relerr(g_s, ref["g_s"]) < tol and relerr(H_ss, ref["H_ss"]) < tol
    # Schur complement of the robust blocks
    Hc, gc = bo._assemble_camera_system(ref, S, dc, ns)
    radius = 37.0
    sc_p = 1.0 / (1.0 + np.sqrt(np.einsum("nii->ni", ref["H_pp"])))
    Hs = ref["H_pp"] * sc_p[:, :, None] * sc_p[:, None, :]
    dpp = np.clip(np.einsum("nii->ni", Hs), 1e-6, 1e32)
    V = Hs + np.einsum("ni,ij->nij", dpp / radius, np.eye(3))
    V[pconst] = np.eye(3)
    M = sc_p[:, :, None] * np.transpose(np.linalg.inv(np.linalg.cholesky(V)), (0, 2, 1))
    M[pconst] = 0.0
    q = np.einsum("nji,nj->ni", M, ref["g_p"])
    Z = np.einsum("dnj,njk->dnk", bo._full_W(ref, S, dc, ns), M).reshape(D, N * 3)
    S_ref = Hc - Z @ Z.T
    rhs_ref = -(gc - Z @ q.reshape(-1))
    Sraw, rhs = ba.schur(*args, out, to_dev(sc_p, dev), radius, point_const=ptc, **kw)
    torch.cuda.synchronize()
    Sraw = Sraw.cpu().numpy()[:, :D]
    # per entry within 1e-12 sqrt(S_ii S_jj), times the cancellation max_i H_ii / S_ii where the elimination of the
    # points removes most of a camera's diagonal (the rounding of H - Z Z^T scales with H, not with S)
    d = np.sqrt(np.diag(S_ref))
    ratio = (np.abs(Sraw - S_ref) / np.outer(d, d))[np.tril_indices(D)].max()
    cancel = max(1.0, float(np.max(np.diag(Hc) / np.diag(S_ref))))
    print(f"{S}x{N} {loss} {a}: max |dS_ij| / sqrt(S_ii S_jj) = {ratio:.3g}, cancellation {cancel:.3g}")
    assert ratio < 1e-12 * cancel
    assert np.abs(rhs.cpu().numpy() - rhs_ref).max() < 1e-9 * np.abs(rhs_ref).max()


# ---- one LM step -------------------------------------------------------------------------------------------------

def _one_step(c, dev, loss, a, label=""):
    S, N = c["mask"].shape
    param_const = bo.default_param_const(S, c["model"], c["mode"])
    point_const = ~c["mask"].any(axis=0)
    o, _ = options(max_num_iterations=1, function_tolerance=0.0, gradient_tolerance=0.0, parameter_tolerance=0.0)
    got = device_solve(c, dev, param_const=param_const, point_const=point_const, options=o, loss=(loss, a))
    check_one_step(c, got, param_const, point_const, loss=(loss, a), label=label)


@pytest.mark.parametrize("loss,a", [("SOFT_L1", 1.0), ("CAUCHY", 0.5), ("CAUCHY", 4.0)])
@pytest.mark.parametrize("shape", SHAPES)
def test_one_lm_step(cuda_dev, shape, loss, a):
    _one_step(_case(*shape), cuda_dev, loss, a, f"{shape} {loss} {a}")


@pytest.mark.parametrize("loss", ["SOFT_L1", "CAUCHY"])
def test_one_lm_step_banded(cuda_dev, loss):
    """160 x 4003 sequential problem in creation order (band plan on) and its shuffled twin (band plan off)"""
    c = lo.with_outliers(banded_ba_case(160, 4003, "SIMPLE_RADIAL", bo.INTR_SHARED, life=24, seed=4), seed=5)
    _one_step(c, cuda_dev, loss, 1.0, "banded")
    _one_step(shuffled_twin(c), cuda_dev, loss, 1.0, "shuffled")


# ---- whole solves against the oracle's LM decisions --------------------------------------------------------------

def _solve_both(c, dev, loss, a, iters, solver="DENSE_SCHUR"):
    o, opt = options(max_num_iterations=iters, function_tolerance=0.0, gradient_tolerance=0.0, parameter_tolerance=0.0)
    ref = oracle_solve(c, opt=opt, linear_solver=solver, loss=(loss, a))
    got = device_solve(c, dev, options=o, linear_solver=solver, loss=(loss, a))
    label = f"{c['mask'].shape} {solver} {loss} {a}"
    if solver == "DENSE_SCHUR":
        check_decisions(got, ref, opt, c, label=label, cost_bar=EPS_COST)
    else:
        # a truncated CG step ends at the first iteration with zeta < eta; the two CG runs may place that test on
        # either side at a close iteration, so the steps agree to the CG's truncation, not to rounding
        # (test_ba_iterative_gpu.py)
        assert_clear(ref["trace"], opt)
        check_outcomes(got, ref, label)
        assert abs(got["s"].final_cost - ref["s"]["final_cost"]) <= 1e-5 * ref["s"]["final_cost"]
    return got["s"], ref["s"]


@pytest.mark.parametrize("loss,a", [("SOFT_L1", 0.5), ("CAUCHY", 1.0), ("CAUCHY", 4.0)])
@pytest.mark.parametrize("shape", SHAPES)
def test_solve_decisions_match_oracle(cuda_dev, shape, loss, a):
    _solve_both(_case(*shape), cuda_dev, loss, a, iters=6)


@pytest.mark.parametrize("loss", ["SOFT_L1", "CAUCHY"])
@pytest.mark.parametrize("shape", SHAPES[:3])
def test_iterative_solve_decisions_match_oracle(cuda_dev, shape, loss):
    """ITERATIVE_SCHUR: CG on the robust reduced system and Ceres' model change -(J d)^T (f + J d / 2) of the corrected
    f and J"""
    _solve_both(_case(*shape), cuda_dev, loss, 1.0, iters=4, solver="ITERATIVE_SCHUR")


# ---- edges ------------------------------------------------------------------------------------------------------

def _run(c, dev, iters=5, loss=None):
    """loss (type, scale) None: lm_solve's default loss"""
    got = device_solve(c, dev, options=options(max_num_iterations=iters)[0], loss=loss)
    return got["s"], (got["poses"], got["intr"], got["points"])


@pytest.mark.parametrize("loss", ["SOFT_L1", "CAUCHY"])
def test_hidden_values_change_nothing(cuda_dev, loss):
    """NaN / inf behind the mask: the clean twin's results bit for bit (s = 0 and rho' = 1 for a masked observation)"""
    for pv, uvv in ((np.nan, np.nan), (np.inf, -np.inf)):
        dirty, clean, hidden = hidden_case(10, 200, "SIMPLE_RADIAL", bo.INTR_PER_FRAME, 7, pv, uvv,
                                      case=_case(10, 200, "SIMPLE_RADIAL", bo.INTR_PER_FRAME, seed=7))
        clean = dict(clean, poses=dirty["poses"])
        sd, xd = _run(dirty, cuda_dev, loss=(loss, 1.0))
        sc, xc = _run(clean, cuda_dev, loss=(loss, 1.0))
        s2, x2 = _run(clean, cuda_dev, loss=(loss, 1.0))
        # a hidden point is not in the problem: it comes back as given (NaN / inf in the dirty twin)
        assert np.array_equal(xd[2][hidden], dirty["points"][hidden], equal_nan=True)
        keep = np.setdiff1d(np.arange(xd[2].shape[0]), hidden)
        xd, xc, x2 = ((x[0], x[1], x[2][keep]) for x in (xd, xc, x2))
        assert np.array_equal(sd.trace.numpy()[:, 7], sc.trace.numpy()[:, 7])
        if sc.final_cost == s2.final_cost and all(np.array_equal(u, v, equal_nan=True) for u, v in zip(xc, x2)):
            assert sd.final_cost == sc.final_cost and np.array_equal(sd.trace.numpy(), sc.trace.numpy())
            for u, v in zip(xd, xc):
                assert np.array_equal(u, v, equal_nan=True)
        else:                # two clean runs differ (the block kernels add with float atomics): hold to their spread
            spread = max(abs(s2.final_cost - sc.final_cost), 1e-13 * sc.final_cost)
            assert abs(sd.final_cost - sc.final_cost) <= 10 * spread
            for u, v in zip(xd, xc):
                both = np.isfinite(v)
                assert np.array_equal(np.isfinite(u), both) and np.allclose(u[both], v[both], rtol=1e-9, atol=1e-9)


@pytest.mark.parametrize("loss", ["TRIVIAL", "SOFT_L1", "CAUCHY"])
def test_non_finite_residual_gives_invalid_steps(cuda_dev, loss):
    c = _case(8, 256, "SIMPLE_PINHOLE", bo.INTR_PER_FRAME)
    s_, n_ = np.argwhere(c["mask"])[5]
    c["uv"] = c["uv"].copy()
    c["uv"][s_, n_, 0] = np.inf
    s, x = _run(c, cuda_dev, iters=20, loss=(loss, 1.0))
    assert s.termination in ("FAILURE_INVALID_STEPS", "MIN_TRUST_REGION_RADIUS") and s.successful == 0
    assert np.all(s.trace.numpy()[:, 7] == 2)
    assert not np.isfinite(s.initial_cost)
    for u, v in zip(x, (c["poses"], c["intr"], c["points"])):
        assert np.array_equal(u, v)


def test_explicit_trivial_is_the_default(cuda_dev):
    c = _case(8, 256, "SIMPLE_RADIAL", bo.INTR_SHARED)
    sa, xa = _run(c, cuda_dev)
    sb, xb = _run(c, cuda_dev, loss=("TRIVIAL", 7.0))
    sc, xc = _run(c, cuda_dev)
    if sa.final_cost == sc.final_cost and all(np.array_equal(u, v) for u, v in zip(xa, xc)):
        assert sb.final_cost == sa.final_cost and np.array_equal(sb.trace.numpy(), sa.trace.numpy())
        for u, v in zip(xa, xb):
            assert np.array_equal(u, v)
    else:                                    # two default runs differ (float atomics): hold TRIVIAL to their spread
        assert abs(sb.final_cost - sa.final_cost) <= 1e-12 * sa.final_cost


@pytest.mark.parametrize("loss", ["SOFT_L1", "CAUCHY"])
def test_large_scale_is_trivial(cuda_dev, loss):
    c = _case(8, 256, "SIMPLE_PINHOLE", bo.INTR_PER_FRAME)
    st, xt = _run(c, cuda_dev, iters=3)
    sr, xr = _run(c, cuda_dev, iters=3, loss=(loss, 1e8))
    assert abs(sr.initial_cost - st.initial_cost) <= 1e-9 * st.initial_cost
    assert abs(sr.final_cost - st.final_cost) <= 1e-9 * st.final_cost
    assert np.array_equal(sr.trace.numpy()[:, 7], st.trace.numpy()[:, 7])
    assert np.abs(xr[2] - xt[2]).max() <= 1e-9 * np.abs(xt[2]).max()


def test_cauchy_rejects_outliers(cuda_dev):
    """from the same perturbed start, CAUCHY's median rotation error to the ground truth is well below TRIVIAL's"""
    c = lo.with_outliers(ba_case(20, 600, "SIMPLE_PINHOLE", bo.INTR_PER_FRAME, seed=2, noise_px=0.3), frac=0.1, seed=3)
    gt = c["scene"].extrinsics[:, :, :3]
    st, xt = _run(c, cuda_dev, iters=50)
    sr, xr = _run(c, cuda_dev, iters=50, loss=("CAUCHY", 1.0))
    rel = lambda R: R[1:] @ R[0].T                      # rotations relative to the first frame: free of the gauge
    et = np.median(rotation_angle_deg(rel(xt[0][:, :, :3]), rel(gt)))
    er = np.median(rotation_angle_deg(rel(xr[0][:, :, :3]), rel(gt)))
    print(f"median rotation error: TRIVIAL {et:.3e} deg, CAUCHY {er:.3e} deg")
    assert er < 0.5 * et


def test_sharded_cauchy_matches_unsharded(cuda_dev):
    """two and three emulated ranks (tests/emulated_ranks.py) with CAUCHY against the unsharded robust solve"""
    c = _case(12, 512, "SIMPLE_RADIAL", bo.INTR_SHARED, seed=3)
    o, _ = options(max_num_iterations=8)
    cauchy = ("CAUCHY", 1.0)
    ref = device_solve(c, cuda_dev, options=o, loss=cauchy)
    for K in (2, 3):
        res, _ = run_shards(c["mask"].shape[1], K, lambda r, lo_, hi_, hook: device_solve(
            c, cuda_dev, lo_, hi_, options=o, allreduce=hook, loss=cauchy), device=cuda_dev)
        for x in res:
            s = x["s"]
            assert s.termination == ref["s"].termination and s.iterations == ref["s"].iterations
            assert np.array_equal(x["trace"][:, 7], ref["trace"][:, 7])
            assert np.isclose(s.final_cost, ref["s"].final_cost, rtol=1e-9, atol=0)
            assert np.abs(x["poses"] - ref["poses"]).max() < 1e-8
            assert np.abs(x["points"] - ref["points"][x["lo"]:x["hi"]]).max() < 1e-8


# ---- argument errors and the pycolmap-shaped options ---------------------------------------------------------------

@pytest.mark.parametrize("ltype,scale", [(3, 1.0), (-1, 1.0), (1, 0.0), (2, -1.0), (2, np.nan), (1, np.inf)])
def test_bad_loss_is_einval_before_any_launch(cuda_dev, ltype, scale):
    import torch
    from vggsfm_b200 import _lib
    from vggsfm_b200 import bundle_adjustment as ba
    L = _lib.lib()
    c = _case(8, 256, "SIMPLE_PINHOLE", bo.INTR_PER_FRAME)
    uv, mask, poses, intr, pts, model, mode = device_args(c, cuda_dev)
    S, N = mask.shape
    pc = ba.default_param_const(S, model, mode, cuda_dev)
    p = ba._problem(uv, mask, poses, intr, pts, model, mode, pc, None)
    p.loss_function_type, p.loss_function_scale = ltype, scale
    before = [t.clone() for t in (poses, intr, pts)]
    st = torch.cuda.current_stream().cuda_stream
    ws = ba.workspace(S, N, model, mode, cuda_dev)
    summ = _lib.BASummary()
    assert L.vgg_ba_solve(ctypes.byref(p), None, ws.data_ptr(), ws.numel(), _lib.ALLREDUCE_FN(), None,
                          ctypes.byref(summ), None, st) == -1
    lin = ba.linear_solver("ITERATIVE_SCHUR")
    wsi = ba.workspace(S, N, model, mode, cuda_dev, iterative=True)
    assert L.vgg_ba_solve_iterative(ctypes.byref(p), None, ctypes.byref(lin), wsi.data_ptr(), wsi.numel(),
                                    ctypes.byref(summ), None, None, st) == -1
    sentinel = torch.full((1 << 16,), 7.0, dtype=torch.float64, device=cuda_dev)
    o = sentinel.data_ptr()
    assert L.vgg_ba_build_blocks(ctypes.byref(p), o, o, o, o, None, o, 0, st) == -1
    assert L.vgg_ba_schur(ctypes.byref(p), o, o, o, o, o, 1.0, 1e-6, 1e32, ws.data_ptr(), ws.numel(), o, o, None,
                          st) == -1
    torch.cuda.synchronize()
    assert torch.all(sentinel == 7.0)
    for t, b in zip((poses, intr, pts), before):
        assert torch.equal(t, b)


def test_unknown_loss_name_raises(cuda_dev):
    from vggsfm_b200 import bundle_adjustment as ba
    c = _case(8, 256, "SIMPLE_PINHOLE", bo.INTR_PER_FRAME)
    with pytest.raises(ValueError):
        ba.lm_solve(*device_args(c, cuda_dev), loss_function_type="HUBER")
    with pytest.raises(ValueError):
        ba.lm_solve(*device_args(c, cuda_dev), loss_function_type="cauchy")


def test_pycolmap_options_carry_the_loss(cuda_dev):
    """BundleAdjustmentOptions with CAUCHY through the reference's call sequence (test_pycolmap_compat_gpu.py) gives the
    scene of bundle_adjustment(..., loss_function_type="CAUCHY"), and another one than the default loss"""
    import torch
    from vggsfm_b200 import bundle_adjustment as ba
    from vggsfm_b200 import pycolmap_compat as pycolmap
    from vggsfm_b200.reconstruction import batch_matrix_to_pycolmap, pycolmap_to_batch_matrix
    from vggsfm_b200.synthetic import make_scene, perturb
    S, N = 7, 150
    sc = make_scene(S, N, "SIMPLE_PINHOLE", seed=21, invisible_frac=0.3)
    extr, K, extra, pts = perturb(sc, seed=22)
    tracks = lo.with_outliers(dict(uv=sc.tracks.astype(np.float64), mask=sc.mask), seed=23)["uv"].astype(np.float32)
    t = torch.from_numpy
    size = torch.tensor([1024, 1024])

    def via_options(loss):
        rec = batch_matrix_to_pycolmap(t(pts), t(extr), t(K), t(tracks), t(sc.mask), size, camera_type="SIMPLE_PINHOLE")
        opt = pycolmap.BundleAdjustmentOptions()
        assert opt.loss_function_type == pycolmap.LossFunctionType.TRIVIAL and opt.loss_function_scale == 1.0
        opt.solver_options.gradient_tolerance *= 10
        opt.solver_options.max_num_iterations = 50
        if loss is not None:
            opt.loss_function_type = loss
        summ = pycolmap.bundle_adjustment(rec, opt)
        rec.normalize(5.0, 0.1, 0.9, True)
        return summ, pycolmap_to_batch_matrix(rec, device="cpu", camera_type="SIMPLE_PINHOLE")

    s_c, (p_c, e_c, _, _) = via_options(pycolmap.LossFunctionType.CAUCHY)
    s_t, (p_t, e_t, _, _) = via_options(None)
    dev = cuda_dev
    out = ba.bundle_adjustment(to_dev(pts, dev), to_dev(extr, dev), to_dev(K, dev), None, to_dev(tracks, dev),
                               to_dev(sc.mask, dev), camera_type="SIMPLE_PINHOLE", options=ba.prepare_ba_options(),
                               loss_function_type="CAUCHY")
    assert s_c.iterations == out[5].iterations
    assert np.abs(p_c.numpy() - out[0].cpu().numpy()).max() < 1e-9
    assert np.abs(e_c.numpy() - out[1].cpu().numpy()).max() < 1e-9
    assert np.abs(e_c.numpy() - e_t.numpy()).max() > 1e-6          # a different scene from the default loss
    assert s_c.final_cost != s_t.final_cost
