"""ITERATIVE_SCHUR (csrc/ba_pcg.cu, vgg_ba_solve_iterative) against the float64 oracle (oracle/ba_pcg_oracle.py) and the
direct solve.

Reduced operator, right-hand side and preconditioner (vgg_dev_pcg_probe): the oracle forms the scaled, damped, pinned
reduced matrix A and b explicitly from its own blocks; the kernels rebuild every coupling block per observation and never
form A.  Entry i of y = A x is a sum of m_i products (the D terms of the camera-Hessian row and 3 per observation of
frame i, each itself a short sum), so per entry

    |y_i - y_ref_i|  <=  (m_i + 64) 2^-53 T_i,   T_i = sum_j (|Dc H_cc Dc|_ij + (|Dc Z| |Dc Z|^T)_ij) |x_j| + damp_i |x_i|,

the usual bound of a recursively summed dot product of m terms, on the absolute terms, with 64 for the blocks' own
rounding.  b gets the same bar with T_i = |sc_i| (|g_i| + sum |Z q|_i).  A dropped observation or a wrong block moves
an entry by about one term, far above the bar.

Whole solves reach the direct solver's final cost within 1e-9 relative; one LM step matches the oracle's CG iteration
count and termination exactly, with every zeta of the oracle's CG at least 1e-6 from eta and its rho outside its band
(tests/ba_harness.py assert_clear), so that no decision sits within rounding of its threshold."""
import ctypes

import numpy as np
import pytest

from oracle import ba_oracle as bo
from oracle import ba_pcg_oracle as po
from tests.ba_harness import assert_clear, device_solve, options, oracle_solve
from tests.helpers import ba_case, banded_ba_case, to_dev

pytestmark = pytest.mark.gpu

EPS = 2.0 ** -53
RADIUS = 1e4


def _effective(c, pc=None, ptc=None):
    S, N = c["mask"].shape
    dc, ns = bo.dims(c["model"], c["mode"])
    mask = c["mask"].astype(bool)
    pc = bo.default_param_const(S, c["model"], c["mode"]) if pc is None else np.asarray(pc, bool).copy()
    pc[:S * dc] |= np.repeat(~mask.any(axis=1), dc)
    ptc = (np.zeros(N, bool) if ptc is None else np.asarray(ptc, bool)) | ~mask.any(axis=0)
    return pc, ptc


def _oracle_system(c, pc, ptc, radius=RADIUS):
    S, N = c["mask"].shape
    dc, ns = bo.dims(c["model"], c["mode"])
    mask = c["mask"].astype(bool)
    unseen = ~mask.any(axis=0)
    pts = np.where(unseen[:, None], 0.0, c["points"])       # hidden values never reach the oracle
    pts[unseen, 2] = 1.0
    poses = c["poses"].copy()
    poses[~mask.any(axis=1)] = np.eye(3, 4)
    blk = bo.build_blocks(poses, c["intr"], pts, np.where(mask[..., None], c["uv"], 0.0), mask, c["model"], c["mode"],
                          ptc)
    Hc, gc = bo._assemble_camera_system(blk, S, dc, ns)
    hd = np.diag(Hc).copy()
    sc_c = 1.0 / (1.0 + np.sqrt(hd))
    sc_p = 1.0 / (1.0 + np.sqrt(np.einsum("nii->ni", blk["H_pp"])))
    A, b, M, dpp, dcc, W = po.reduced_system(blk, Hc, gc, sc_c, sc_p, hd, pc, ptc, radius, S, dc, ns)
    Z = np.einsum("dnk,nkj->dnj", W, M).reshape(W.shape[0], -1)
    q = np.einsum("nji,nj->ni", M, blk["g_p"]).reshape(-1)
    absZ = np.abs(Z * sc_c[:, None])
    absZ[pc] = 0.0
    Hs = np.abs(Hc * sc_c[:, None] * sc_c[None, :])
    Hs[pc, :] = 0.0
    Hs[:, pc] = 0.0
    return dict(A=A, b=b, sc_c=sc_c, sc_p=sc_p, absZ=absZ, Hs=Hs, dcc=dcc, gc=gc, Zq=np.abs(Z) @ np.abs(q),
                S=S, dc=dc, ns=ns)


def _probe(c, pc, ptc, sc_p, sc_c, x, dev, radius=RADIUS):
    import torch
    from vggsfm_b200 import _lib
    from vggsfm_b200 import bundle_adjustment as ba
    S, N = c["mask"].shape
    dc, ns = bo.dims(c["model"], c["mode"])
    D = S * dc + ns
    L = _lib.lib()
    t = lambda a, dt=None: to_dev(a, dev, dt)
    uv, mask = t(c["uv"], torch.float32), t(c["mask"], torch.uint8)
    poses, intr, pts = t(c["poses"].reshape(S, 3, 4)), t(c["intr"]), t(c["points"])
    ptc_t, pc_t = t(ptc, torch.uint8), t(pc, torch.uint8)      # held: the problem struct keeps raw pointers
    blk = ba.build_blocks(uv, mask, poses, intr, pts, c["model"], c["mode"], point_const=ptc_t)
    p = ba._problem(uv, mask, poses, intr, pts, c["model"], c["mode"], pc_t, ptc_t)
    ws = ba.workspace(S, N, c["model"], c["mode"], dev, iterative=True)
    nblk = 3 * S + (1 if ns else 0)
    y = torch.empty(D, dtype=torch.float64, device=dev)
    b = torch.empty(D, dtype=torch.float64, device=dev)
    pinv = torch.empty(nblk, 3, 3, dtype=torch.float64, device=dev)
    state = torch.empty(32, dtype=torch.float64, device=dev)
    scp, scc, xt = t(sc_p), t(sc_c), t(x)
    with torch.cuda.device(dev):
        st = torch.cuda.current_stream().cuda_stream
        _lib.check(L.vgg_dev_pcg_probe(ctypes.byref(p), blk["camrec"].data_ptr(), blk["g_p"].data_ptr(),
                                       blk["H_pp"].data_ptr(), blk["shared"].data_ptr(), scp.data_ptr(), scc.data_ptr(),
                                       radius, 1e-6, 1e32, xt.data_ptr(), ws.data_ptr(), ws.numel(), y.data_ptr(),
                                       b.data_ptr(), pinv.data_ptr(), state.data_ptr(), st), "vgg_dev_pcg_probe")
    return y.cpu().numpy(), b.cpu().numpy(), pinv.cpu().numpy(), state.cpu().numpy()


def _check_probe(c, dev, pc=None, ptc=None, seed=0, twin=None):
    pc, ptc = _effective(c, pc, ptc)
    ref = _oracle_system(c, pc, ptc)
    D = ref["A"].shape[0]
    x = np.random.default_rng(seed).standard_normal(D)
    x[pc] = 0.0
    y, b, pinv, _ = _probe(c, pc, ptc, ref["sc_p"], ref["sc_c"], x, dev)
    T = (ref["Hs"] + ref["absZ"] @ ref["absZ"].T) @ np.abs(x) + ref["dcc"] / RADIUS * np.abs(x) + np.where(pc, np.abs(x), 0)
    m = D + 3 * int(c["mask"].sum())
    bar = (m + 64) * EPS * T
    err = np.abs(y - ref["A"] @ x)
    bad = np.nonzero(err > bar)[0]
    assert bad.size == 0, (f"matvec: {bad.size} entries over the bar, first {bad[:8]}: y {y[bad[:4]]} ref "
                           f"{(ref['A'] @ x)[bad[:4]]} x {x[bad[:4]]} bar {bar[bad[:4]]}")
    Tb = ref["sc_c"] * (np.abs(ref["gc"]) + ref["Zq"])
    errb = np.abs(b - ref["b"])
    assert (errb <= (m + 64) * EPS * Tb + 0.0).all(), f"rhs: worst {np.max(errb / np.maximum(Tb, 1e-300)):.3g}"
    assert not b[pc].any()
    _, ok, store = po.schur_jacobi(ref["A"], ref["S"], ref["dc"], ref["ns"])
    assert ok
    for k, (r0, nb) in enumerate(po.parameter_blocks(ref["S"], ref["dc"], ref["ns"])):
        if nb:
            # the inverse of a block of condition kappa is good to ~kappa times the rounding of the block
            kappa = np.linalg.cond(ref["A"][r0:r0 + nb, r0:r0 + nb])
            d = np.abs(pinv[k][:nb, :nb] - store[k][:nb, :nb]).max()
            assert d <= 1e-11 * max(kappa, 1.0) * np.abs(store[k]).max(), (k, d, kappa)
    if twin is not None:
        # the hidden values reach nothing: the twin meets the clean problem's bars (the kernels' f64 atomics add in
        # an arbitrary order, so two runs agree to rounding, not bit for bit)
        y2, b2, p2, _ = _probe(twin, pc, ptc, ref["sc_p"], ref["sc_c"], x, dev)
        assert np.isfinite(y2).all() and np.isfinite(b2).all() and np.isfinite(p2).all()
        assert (np.abs(y2 - ref["A"] @ x) <= bar).all()
        assert (np.abs(b2 - ref["b"]) <= (m + 64) * EPS * Tb).all()


PAIRS = [("SIMPLE_PINHOLE", bo.INTR_CONST), ("SIMPLE_PINHOLE", bo.INTR_PER_FRAME), ("SIMPLE_PINHOLE", bo.INTR_SHARED),
         ("SIMPLE_RADIAL", bo.INTR_CONST), ("SIMPLE_RADIAL", bo.INTR_PER_FRAME), ("SIMPLE_RADIAL", bo.INTR_SHARED)]


@pytest.mark.parametrize("cam,mode", PAIRS)
def test_operator_c1_edges(cuda_dev, cam, mode):
    """C1 (8 x 256) with a constant pose, constant points, a frame and a point that nothing sees; the twin hides NaN and
    inf in the unseen frame's pose, the unseen point and masked uv, and must give the same bits."""
    c = ba_case(8, 256, cam, mode, seed=11)
    c["mask"][5] = False
    c["mask"][:, 17] = False
    const_pose = np.zeros(8, bool)
    const_pose[3] = True
    pc = bo.default_param_const(8, c["model"], mode, const_pose=const_pose)
    ptc = np.zeros(256, bool)
    ptc[::9] = True
    clean = dict(c, uv=np.where(c["mask"][..., None], c["uv"], 0.0), points=c["points"].copy(), poses=c["poses"].copy())
    clean["points"][17] = [0.0, 0.0, 1.0]
    clean["poses"][5] = np.eye(3, 4)
    dirty = dict(clean, uv=clean["uv"].copy(), points=clean["points"].copy(), poses=clean["poses"].copy())
    dirty["points"][17] = np.nan
    dirty["poses"][5] = np.inf
    dirty["uv"][~c["mask"]] = np.nan
    _check_probe(clean, cuda_dev, pc, ptc, twin=dirty)


@pytest.mark.parametrize("name", ["C2", "C3", "banded160x4003"])
def test_operator_large(cuda_dev, name):
    if name == "C2":
        c = ba_case(50, 2048, "SIMPLE_PINHOLE", bo.INTR_PER_FRAME, seed=1)
    elif name == "C3":
        c = ba_case(400, 4096, "SIMPLE_RADIAL", bo.INTR_SHARED, seed=0, invisible_frac=0.0)
    else:
        c = banded_ba_case(160, 4003, "SIMPLE_RADIAL", bo.INTR_SHARED, life=24, seed=31)
        c["mask"][77] = False
        c["mask"][:, 1234] = False
    _check_probe(c, cuda_dev)


def _solve(c, dev, iterative, opt=None, **lin):
    return device_solve(c, dev, options=opt, linear_solver="ITERATIVE_SCHUR" if iterative else "DENSE_SCHUR", **lin)["s"]


def _tight(max_it=100):
    return options(function_tolerance=1e-13, gradient_tolerance=1e-10, max_num_iterations=max_it)[0]


@pytest.mark.parametrize("name", ["C1", "C2"])
def test_one_lm_step_matches_oracle(cuda_dev, name):
    c = ba_case(8, 256, "SIMPLE_PINHOLE", bo.INTR_PER_FRAME, seed=0) if name == "C1" else \
        ba_case(50, 2048, "SIMPLE_PINHOLE", bo.INTR_PER_FRAME, seed=1)
    o, opt = options(max_num_iterations=1)
    summ = _solve(c, cuda_dev, True, o)
    ref = oracle_solve(c, opt=opt, linear_solver="ITERATIVE_SCHUR")
    trace, cs = ref["trace"], ref["cg"][0]
    assert_clear(trace, opt, cg=ref["cg"])
    got = summ.cg_trace[0].numpy()
    assert int(got[0]) == cs["summary"]["iterations"] and int(got[1]) == cs["summary"]["termination"]
    assert abs(got[2] - cs["summary"]["zeta"]) <= 1e-6 * max(1.0, abs(cs["summary"]["zeta"]))
    tr = summ.trace[0].numpy()
    ref = trace[0]
    assert abs(tr[3] - ref["model_change"]) <= 1e-8 * abs(ref["model_change"])
    assert abs(tr[2] - ref["candidate_cost"]) <= 1e-9 * abs(ref["candidate_cost"])
    assert abs(tr[6] - ref["step_norm"]) <= 1e-8 * abs(ref["step_norm"])


@pytest.mark.parametrize("name,rel", [("C2", 1e-9), ("C3", 1e-8), ("banded1000", 1e-4)])
def test_whole_solve_reaches_the_direct_minimum(cuda_dev, name, rel):
    """C2 converges (function tolerance) in both solvers, at the same iteration and cost.  C3 stops at the 100-iteration
    cap in both, a few 1e-9 apart.  On the banded 1000-frame problem the CG reaches its 500-iteration cap at every LM
    step (the Schur-Jacobi preconditioner is weak on the long, drifting sequence), so the steps stay inexact and the two
    solves end 2e-5 apart after 100 iterations."""
    if name == "C2":
        c = ba_case(50, 2048, "SIMPLE_PINHOLE", bo.INTR_PER_FRAME, seed=1)
    elif name == "C3":
        c = ba_case(400, 4096, "SIMPLE_RADIAL", bo.INTR_SHARED, seed=0, invisible_frac=0.0)
    else:
        c = banded_ba_case(1000, 12000, "SIMPLE_PINHOLE", bo.INTR_SHARED, life=24, seed=7)
    sd = _solve(c, cuda_dev, False, _tight())
    # a CG solved to rounding (eta 1e-12): the same minimum as the direct solve.  With Ceres' eta = 0.1 the truncated
    # steps converge far more slowly on these problems (at C2 the oracle's own iterative LM is 2.5 % above the minimum
    # after 100 iterations, DESIGN 4.8), which says nothing about the kernels.
    si = _solve(c, cuda_dev, True, _tight(), eta=1e-12, max_linear_solver_iterations=500)
    print(f"{name}: direct {sd.final_cost:.12g} ({sd.iterations} it, {sd.termination}), iterative {si.final_cost:.12g} "
          f"({si.iterations} it, {si.termination}, {si.cg_iterations} CG it, {si.kernel_launches} launches)")
    assert si.termination != "FAILURE_INVALID_STEPS"
    assert abs(si.final_cost - sd.final_cost) <= rel * sd.final_cost


@pytest.mark.parametrize("mn,mx", [(0, 0), (0, 1), (0, 2), (1, 2), (2, 2), (0, 200), (2, 200), (200, 200)])
def test_cg_iteration_limits(cuda_dev, mn, mx):
    c = ba_case(50, 2048, "SIMPLE_PINHOLE", bo.INTR_PER_FRAME, seed=1)
    summ = _solve(c, cuda_dev, True, _tight(4), min_linear_solver_iterations=mn, max_linear_solver_iterations=mx)
    for it, term, *_ in summ.cg_trace.numpy():
        it, term = int(it), int(term)
        assert 1 <= it <= max(1, mx)
        if term == po.SUCCESS:
            assert it >= mn
        if term == po.NO_CONVERGENCE:
            assert it == max(1, mx)


def test_multi_gpu_and_bad_options_are_refused(cuda_dev):
    import torch
    from vggsfm_b200 import _lib
    from vggsfm_b200 import bundle_adjustment as ba
    c = ba_case(8, 256, "SIMPLE_PINHOLE", bo.INTR_PER_FRAME, seed=0)
    with pytest.raises(ValueError):
        ba.lm_solve(
            to_dev(c["uv"], cuda_dev, torch.float32), to_dev(c["mask"], cuda_dev, torch.uint8),
            to_dev(c["poses"], cuda_dev), to_dev(c["intr"], cuda_dev), to_dev(c["points"], cuda_dev), c["model"],
            c["mode"], allreduce=object(), linear_solver_type="ITERATIVE_SCHUR")
    with pytest.raises(ValueError):
        ba.linear_solver("SPARSE_SCHUR")
    L = _lib.lib()
    summ = _lib.BASummary()
    for lin in (ba.linear_solver("DENSE_SCHUR"), ba.linear_solver("ITERATIVE_SCHUR", 3, 2),
                ba.linear_solver("ITERATIVE_SCHUR", eta=0.0)):
        rc = L.vgg_ba_solve_iterative(None, None, ctypes.byref(lin), None, 0, ctypes.byref(summ), None, None, None)
        assert rc == -1


def test_joint_ba_beyond_the_direct_workspace(cuda_dev):
    """The final joint BA of a 2500-frame synthetic sequence with 2048 new points per window (the tools/video_c5.py
    generator): the direct solve's workspace exceeds an 80 GB card; the iterative one solves it."""
    import time
    import torch
    from tools.video_c5 import final_problem_arrays
    from vggsfm_b200 import bundle_adjustment as ba
    tracks, masks, xyz, extr, K = final_problem_arrays(2500, 2048, dev=cuda_dev)
    S, P = masks.shape
    direct = ba.workspace_bytes(S, ba.pad_tracks(P), ba.SIMPLE_PINHOLE, ba.INTR_SHARED)
    assert direct > 80e9
    torch.cuda.reset_peak_memory_stats(cuda_dev)
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    *_, summ = ba.bundle_adjustment(xyz, extr, K.expand(S, -1, -1), None, tracks, masks, shared_camera=True,
                                    options=ba.default_options(), filter_reconstruction=False,
                                    linear_solver_type="ITERATIVE_SCHUR")
    torch.cuda.synchronize()
    dt = time.perf_counter() - t0
    peak = torch.cuda.max_memory_allocated(cuda_dev)
    print(f"joint BA {S} x {P}: direct workspace {direct / 1e9:.1f} GB, iterative peak {peak / 1e9:.2f} GB, "
          f"{summ.iterations} LM it in {dt:.1f} s, {summ.cg_iterations} CG it, {summ.termination}, "
          f"cost {summ.initial_cost:.6g} -> {summ.final_cost:.6g}")
    assert summ.termination != "FAILURE_INVALID_STEPS"
    assert summ.final_cost < 1e-3 * summ.initial_cost
    assert peak < 80e9
