"""Values the masks hide from the bundle adjustment, on the GPU: NaN, inf and huge values under masks.

A hidden value is the uv of an observation whose mask is 0, the coordinates of a point that no valid observation sees,
or the pose of a frame that no valid observation sees (tests/helpers.py hidden_case).  The solve must not let any of
them reach what it computes or returns, so every case here runs the problem with hidden values and its clean twin (the
same problem with uv = 0, points at (0, 0, 1) and the original pose in those places) and holds the two to the bars the
existing files use: blocks at 1e-10 (test_ba_gpu.py), the Schur complement at 1e-12 sqrt(S_ii S_jj), one LM step at a
backward error of 1e-12 in the clean twin's damped system, whole solves with identical decisions and costs within
EPS_COST (tests/ba_harness.py).  Hidden parameters come back bit for bit as given.

bundle_adjustment() makes such input itself: a triangulated point with a NaN or a coordinate >= max_points3D_val is
given no observations but keeps its coordinates (as pycolmap's input conversion drops them)."""
import numpy as np
import pytest

from oracle import ba_oracle as bo
from tests.ba_harness import (EPS_COST, SHAPES, check_one_step, check_same_solve, device_args, device_solve,
                              first_drop, options, oracle_solve, relerr)
from tests.helpers import banded_ba_case, hidden_case, rotation_angle_deg, to_dev, unpack_camrec

pytestmark = pytest.mark.gpu

FLT_MAX = float(np.finfo(np.float32).max)
MODES = [(cam, mode) for cam in ("SIMPLE_PINHOLE", "SIMPLE_RADIAL")
         for mode in (bo.INTR_CONST, bo.INTR_PER_FRAME, bo.INTR_SHARED)]


def _blocks(c, dev, tracks_per_warp=0, point_const=None):
    import torch
    from vggsfm_b200 import bundle_adjustment as ba
    args = device_args(c, dev)
    pc = None if point_const is None else to_dev(point_const.astype(np.uint8), dev)
    out = ba.build_blocks(*args, point_const=pc, tracks_per_warp=tracks_per_warp)
    torch.cuda.synchronize()
    return args, {k: v.cpu().numpy() if hasattr(v, "cpu") else v for k, v in out.items()}, out


# ------------------------------------------------------------------------------------------------------------------
# normal-equation blocks
# ------------------------------------------------------------------------------------------------------------------

BLOCK_CASES = [(8, 256, cam, mode, tpw, None) for cam, mode in MODES for tpw in (0, 4, 36)] + [
    (5, 100, "SIMPLE_RADIAL", bo.INTR_PER_FRAME, 0, 2),       # N % 16 != 0: non-TMA W path
    (70, 1001, "SIMPLE_PINHOLE", bo.INTR_SHARED, 0, 40),      # N % 4 != 0: scalar observation loads, 3 frame groups
    (33, 130, "SIMPLE_RADIAL", bo.INTR_CONST, 36, 32),        # the hidden frame is alone in frame group 1
]


@pytest.mark.parametrize("S,N,cam,mode,tpw,hframe", BLOCK_CASES)
def test_blocks_equal_clean_twin(cuda_dev, S, N, cam, mode, tpw, hframe):
    dirty, clean, hidden = hidden_case(S, N, cam, mode, S + N + tpw, np.nan, np.nan, n_hidden=5, hidden_frame=hframe)
    dirty["points"][hidden[1]] = np.inf
    dirty["points"][hidden[2]] = 1e308
    off = ~dirty["mask"]
    dirty["uv"][off] = np.array([np.nan, np.inf, -FLT_MAX])[np.arange(off.sum()) % 3][:, None]
    pconst = np.zeros(N, dtype=bool)
    pconst[::7] = True
    pconst[hidden[3]] = True                       # a hidden point that is also flagged constant
    _, ref, _ = _blocks(clean, cuda_dev, tpw, pconst)
    _, got, _ = _blocks(dirty, cuda_dev, tpw, pconst)
    dc, ns = bo.dims(clean["model"], mode)
    assert np.isfinite(got["cost"]).all() and abs(got["cost"].item() - ref["cost"].item()) <= 1e-10 * ref["cost"].item()
    for k in ("camrec", "g_p", "H_pp", "W", "shared"):
        assert np.isfinite(got[k]).all(), k
    assert relerr(got["camrec"], ref["camrec"]) < 1e-10
    assert relerr(got["g_p"], ref["g_p"]) < 1e-10 and relerr(got["H_pp"], ref["H_pp"]) < 1e-10
    assert relerr(got["W"][:, :S * dc + ns], ref["W"][:, :S * dc + ns]) < 1e-10
    if ns:
        assert relerr(got["shared"][:5], ref["shared"][:5]) < 1e-10
    assert not got["g_p"][hidden].any() and not got["H_pp"][hidden].any() and not got["W"][hidden].any()
    if hframe is not None:
        g_c, H_cc, _, _, _ = unpack_camrec(got["camrec"], got["shared"], S, dc, ns)
        assert not g_c[hframe].any() and not H_cc[hframe].any()


# ------------------------------------------------------------------------------------------------------------------
# Schur complement
# ------------------------------------------------------------------------------------------------------------------

def _schur(c, dev, sc_p, radius):
    import torch
    from vggsfm_b200 import bundle_adjustment as ba
    args, _, out = _blocks(c, dev)
    Sraw, rhs = ba.schur(*args, out, to_dev(sc_p, dev), radius)
    torch.cuda.synchronize()
    return Sraw.cpu().numpy(), rhs.cpu().numpy()


@pytest.mark.parametrize("name", ["dense 8x256", "banded 160x2050", "C3"])
def test_schur_equals_clean_twin(cuda_dev, name):
    if name == "dense 8x256":
        dirty, clean, _ = hidden_case(8, 256, "SIMPLE_PINHOLE", bo.INTR_PER_FRAME, 5, np.nan, np.nan, hidden_frame=3)
    elif name == "banded 160x2050":
        case = banded_ba_case(160, 2050, "SIMPLE_RADIAL", bo.INTR_SHARED, life=24, seed=41)
        dirty, clean, _ = hidden_case(0, 2050, None, None, 6, np.inf, np.nan, n_hidden=20, hidden_frame=77, case=case)
    else:
        dirty, clean, _ = hidden_case(400, 4096, "SIMPLE_RADIAL", bo.INTR_SHARED, 0, np.nan, np.nan, n_hidden=16,
                                      hidden_frame=200)
    S = clean["mask"].shape[0]
    dc, ns = bo.dims(clean["model"], clean["mode"])
    D = S * dc + ns
    _, blk, _ = _blocks(clean, cuda_dev)
    Hpp = blk["H_pp"]
    sc_p = 1.0 / (1.0 + np.sqrt(Hpp[:, [0, 3, 5]]))
    S_ref, rhs_ref = _schur(clean, cuda_dev, sc_p, 37.0)
    S_got, rhs_got = _schur(dirty, cuda_dev, sc_p, 37.0)
    S_ref, S_got = S_ref[:, :D], S_got[:, :D]
    low = np.tril_indices(D)
    d = np.sqrt(np.abs(np.diag(S_ref)))
    d = np.where(d > 0, d, 1.0)                    # the hidden frame's rows are exact zeros in both
    assert np.isfinite(S_got[low]).all() and np.isfinite(rhs_got[:D]).all()
    ratio = (np.abs(S_got - S_ref) / np.outer(d, d))[low].max()
    print(f"schur {name}: max |dS_ij| / sqrt(S_ii S_jj) = {ratio:.3g}")
    assert ratio < 1e-12
    assert np.abs(rhs_got[:D] - rhs_ref[:D]).max() < 1e-9 * np.abs(rhs_ref[:D]).max()


# ------------------------------------------------------------------------------------------------------------------
# LM solve
# ------------------------------------------------------------------------------------------------------------------

def _gpu_solve(c, dev, **kw):
    S, N = c["mask"].shape
    return device_solve(c, dev, param_const=bo.default_param_const(S, c["model"], c["mode"]),
                        point_const=np.zeros(N, dtype=bool), options=options(**kw)[0])


def _hidden_frames(c):
    return np.nonzero(~c["mask"].any(axis=1))[0]


def _assert_hidden_as_given(dirty, got, hidden):
    assert np.array_equal(got["points"][hidden].view(np.uint64), dirty["points"][hidden].view(np.uint64))
    hf = _hidden_frames(dirty)
    assert np.array_equal(got["poses"][hf].view(np.uint64), dirty["poses"][hf].view(np.uint64))
    if dirty["mode"] != bo.INTR_SHARED:
        assert np.array_equal(got["intr"][hf].view(np.uint64), dirty["intr"][hf].view(np.uint64))


@pytest.mark.parametrize("name", ["dense 8x256", "dense 45x700", "banded 160x4003"])
def test_one_step_in_clean_twins_system(cuda_dev, name):
    """one LM iteration on the problem with hidden values: its step has a backward error <= 1e-12 in the clean twin's
    damped system (hidden points and frames are constant there), and the trace's model change and step norm are the
    clean twin's at that step"""
    if name == "dense 8x256":
        dirty, clean, hidden = hidden_case(8, 256, "SIMPLE_PINHOLE", bo.INTR_PER_FRAME, 21, np.nan, np.nan, hidden_frame=4)
    elif name == "dense 45x700":
        dirty, clean, hidden = hidden_case(45, 700, "SIMPLE_RADIAL", bo.INTR_SHARED, 23, np.inf, np.nan, n_hidden=9)
    else:       # the band hint is on for this problem (tests/test_lm_step_gpu.py)
        case = banded_ba_case(160, 4003, "SIMPLE_RADIAL", bo.INTR_SHARED, life=24, seed=31)
        dirty, clean, hidden = hidden_case(0, 4003, None, None, 31, np.nan, FLT_MAX, n_hidden=12, hidden_frame=77,
                                           case=case)
    S, N = clean["mask"].shape
    model, mode = clean["model"], clean["mode"]
    dc, ns = bo.dims(model, mode)
    got = _gpu_solve(dirty, cuda_dev, max_num_iterations=1, function_tolerance=0.0, gradient_tolerance=0.0,
                     parameter_tolerance=0.0)
    _assert_hidden_as_given(dirty, got, hidden)
    hf = _hidden_frames(clean)
    got = dict(got, poses=got["poses"].copy(), intr=got["intr"].copy(), points=got["points"].copy())
    got["poses"][hf] = clean["poses"][hf]
    got["points"][hidden] = clean["points"][hidden]
    if mode != bo.INTR_SHARED:
        got["intr"][hf] = clean["intr"][hf]
    point_const = ~clean["mask"].any(axis=0)
    param_const = bo.default_param_const(S, model, mode)
    param_const[:S * dc] |= np.repeat(~clean["mask"].any(axis=1), dc)
    check_one_step(clean, got, param_const, point_const, label=f"hidden-value step {name}")


def _compare_solves(dirty, clean, hidden, dev, label, **kw):
    """the problem with hidden values and its clean twin through the whole solve: identical decisions, costs within
    EPS_COST, the visible parameters at the whole-solve bars, hidden parameters bit for bit as given"""
    d, c = _gpu_solve(dirty, dev, **kw), _gpu_solve(clean, dev, **kw)
    s_d, tr_d, s_c, tr_c = d["s"], d["trace"], c["s"], c["trace"]
    assert (s_d.termination, s_d.iterations, s_d.successful) == (s_c.termination, s_c.iterations, s_c.successful), \
        (label, s_d.termination, s_c.termination, s_d.iterations, s_c.iterations)
    assert [int(v) for v in tr_d[:, 7]] == [int(v) for v in tr_c[:, 7]], (label, tr_d[:, 7], tr_c[:, 7])
    assert abs(s_d.initial_cost - s_c.initial_cost) <= EPS_COST * s_c.initial_cost
    for k in range(s_c.iterations):
        for col in (1, 2):
            assert abs(tr_d[k, col] - tr_c[k, col]) <= EPS_COST * max(tr_c[k, 1], tr_c[k, 2]), (label, k, tr_d[k], tr_c[k])
        assert tr_d[k, 5] == tr_c[k, 5] or abs(tr_d[k, 5] - tr_c[k, 5]) <= 1e-6 * tr_c[k, 5], (label, k)
    _assert_hidden_as_given(dirty, d, hidden)
    keep = np.setdiff1d(np.arange(clean["mask"].shape[1]), hidden)
    fr = np.setdiff1d(np.arange(clean["mask"].shape[0]), _hidden_frames(clean))
    check_same_solve(d, c, label, cost_bar=EPS_COST, frames=fr, points=keep)
    print(f"{label}: {s_d.termination} after {s_d.iterations} iterations ({s_d.successful} accepted)")
    return s_d


def _probe(clean, iters):
    """the oracle's trace of the clean twin with every tolerance off"""
    _, opt = options(max_num_iterations=iters, gradient_tolerance=0.0)
    trace = oracle_solve(clean, opt=opt, use_c=bo._load_c() is not None)["trace"]
    assert all(r["outcome"] != 2 for r in trace)
    return trace


@pytest.mark.parametrize("shape", SHAPES)
def test_solve_function_tolerance(cuda_dev, shape):
    """a function_tolerance that fires at the 3rd valid iteration or later (placed as test_ba_lm_edges_gpu.py places
    it, on the clean twin); hidden NaN / +inf points, inf uv in masked slots"""
    S, N, cam, mode = shape
    dirty, clean, hidden = hidden_case(S, N, cam, mode, 11, np.nan, np.inf, n_hidden=4)
    dirty["points"][hidden[0]] = np.inf
    trace = _probe(clean, 12)
    at, ftol = first_drop([abs(r["cost_change"]) / r["cost"] for r in trace], 2)
    s = _compare_solves(dirty, clean, hidden, cuda_dev, f"function {shape}", function_tolerance=ftol,
                        gradient_tolerance=0.0)
    assert s.termination == "CONVERGENCE_FUNCTION" and s.iterations == at + 1


@pytest.mark.parametrize("shape", SHAPES[:3])
def test_solve_parameter_tolerance(cuda_dev, shape):
    """parameter_tolerance > 0: |x| must leave out the hidden points, which are NOT flagged constant by the caller (a
    NaN among them would make |x| NaN and the test never fire)"""
    S, N, cam, mode = shape
    dirty, clean, hidden = hidden_case(S, N, cam, mode, 12, np.nan, np.nan, n_hidden=4)
    trace = _probe(clean, 12)
    at, ptol = first_drop([r["step_norm"] / r["x_norm"] for r in trace], 1)
    s = _compare_solves(dirty, clean, hidden, cuda_dev, f"parameter {shape}", parameter_tolerance=ptol,
                        gradient_tolerance=0.0)
    assert s.termination == "CONVERGENCE_PARAMETER" and s.iterations == at + 1


@pytest.mark.parametrize("shape", SHAPES)
def test_solve_unobserved_frame(cuda_dev, shape):
    """frame 2 (not the gauge frame) sees nothing and has a NaN pose; parameter_tolerance > 0 so that the frame's pose
    would enter |x| if it were not constant"""
    S, N, cam, mode = shape
    dirty, clean, hidden = hidden_case(S, N, cam, mode, 13, np.nan, np.nan, n_hidden=2, hidden_frame=2)
    s = _compare_solves(dirty, clean, hidden, cuda_dev, f"unobserved frame {shape}", max_num_iterations=6,
                        gradient_tolerance=0.0, parameter_tolerance=1e-30)
    assert s.termination == "NO_CONVERGENCE" and s.iterations == 6 and s.successful >= 3


# ------------------------------------------------------------------------------------------------------------------
# bundle_adjustment() wrapper
# ------------------------------------------------------------------------------------------------------------------

def test_bundle_adjustment_drops_non_finite_points(cuda_dev):
    """points3d rows of NaN and +inf on tracks with >= 2 inliers, NaN tracks in masked slots: the result equals the
    wrapper and the oracle run with those tracks deleted.  (-inf passes the < max_points3D_val filter and fails in
    pycolmap too: not a hidden value.)"""
    from vggsfm_b200 import bundle_adjustment as ba
    from tests.helpers import ba_case
    c = ba_case(10, 300, "SIMPLE_RADIAL", bo.INTR_SHARED, seed=5, invisible_frac=0.4)
    sc = c["scene"]
    mask = sc.mask.copy()
    pts = c["points"].copy()
    tracks = sc.tracks.copy()
    bad = np.array([11, 57, 58, 200])
    assert (mask[:, bad].sum(axis=0) >= 2).all()
    pts[bad[0]] = np.nan
    pts[bad[1], 1] = np.nan
    pts[bad[2]] = [np.inf, 0.0, 1.0]
    pts[bad[3], 2] = np.inf
    tracks[~mask] = np.nan
    keep = np.setdiff1d(np.arange(pts.shape[0]), bad)
    kw = dict(shared_camera=True, camera_type="SIMPLE_RADIAL")
    dev = cuda_dev
    run = lambda p, t, m: ba.bundle_adjustment(to_dev(p, dev), to_dev(c["poses"], dev), to_dev(c["K"], dev),
                                               to_dev(c["extra"], dev), to_dev(t, dev), to_dev(m, dev),
                                               options=ba.prepare_ba_options(), **kw)
    got = run(pts, tracks, mask)
    ref = run(pts[keep], np.where(mask[..., None], tracks, 0.0)[:, keep], mask[:, keep])
    ora = bo.bundle_adjustment(pts[keep], c["poses"], c["K"], c["extra"], sc.tracks[:, keep], mask[:, keep],
                               options=bo.LMOptions.prepare_ba_options(), **kw)
    vi = got[4].cpu().numpy()
    rows = np.isin(vi, keep)
    assert np.array_equal(vi[rows], keep[ref[4].cpu().numpy()])
    assert got[5].termination == ref[5].termination == ora[5]["termination"]
    assert got[5].iterations == ref[5].iterations == ora[5]["iterations"]
    P = got[0].cpu().numpy()
    for other, tol in ((ref[0].cpu().numpy(), 1e-7), (ora[0], 1e-6)):
        assert np.abs(P[rows] - other).max() < tol
    for other in ((ref[1].cpu().numpy(), ref[2].cpu().numpy(), ref[3].cpu().numpy()), (ora[1], ora[2], ora[3])):
        assert rotation_angle_deg(got[1].cpu().numpy()[:, :, :3], other[0][:, :, :3]).max() < 1e-6
        assert np.abs(got[1].cpu().numpy()[:, :, 3] - other[0][:, :, 3]).max() < 1e-6
        assert np.abs(got[2].cpu().numpy() - other[1]).max() < 1e-5
        assert np.abs(got[3].cpu().numpy() - other[2]).max() < 1e-7
    assert not np.isfinite(P[~rows]).all(axis=1).any()     # the dropped points come back non-finite, as given
