"""ITERATIVE_SCHUR on an observation list (vgg_ba_solve_iterative_obs, bundle_adjustment.lm_solve_obs) against the grid
solve of the same problem (vgg_ba_solve_iterative_sharded without a hook), the float64 oracle and itself on track shards.

The list holds exactly the grid's valid cells, so both solves add the same terms, in another order (the list kernels sum
a frame's observations in CTA chunks and a point's in one warp, the grid kernels in their own tiles).  As between the
sharded and the unsharded solve (tests/test_ba_iterative_sharded_gpu.py, whose docstring gives the measurements), CG
amplifies that rounding, so the bars are the same: termination, LM outcomes and per LM iteration the CG iteration count
and termination match exactly where assert_clear finds the grid run clear of its rounding bands; costs within 1e-5
relative and parameters within 1e-4 over the first few LM iterations."""
import ctypes

import numpy as np
import pytest

from oracle import ba_oracle as bo
from tests.ba_harness import SHAPES, assert_clear, device_solve, options, oracle_solve, radius_bar, trace_rows
from tests.emulated_ranks import run_shards
from tests.helpers import ba_case, banded_ba_case, hidden_case, to_dev
from tests.test_ba_iterative_sharded_gpu import _check

pytestmark = [pytest.mark.gpu, pytest.mark.usefixtures("cuda_dev")]

DEV = "cuda:0"
COST_BAR = 1e-5
PARAM_BAR = 1e-4


def coo(c, lo=0, hi=None, seed=None):
    """the valid cells of tracks [lo, hi) of case c as COO observations (uv, frame, point), frame-major as np.nonzero
    gives them, or in a random order with a seed"""
    hi = c["mask"].shape[1] if hi is None else hi
    f, n = np.nonzero(c["mask"][:, lo:hi])
    uv = c["uv"][:, lo:hi][f, n]
    if seed is not None:
        perm = np.random.default_rng(seed).permutation(len(f))
        f, n, uv = f[perm], n[perm], uv[perm]
    return uv, f, n


def list_solve(c, lo=0, hi=None, seed=None, options=None, allreduce=None, loss=None, param_const=None,
               point_const=None, max_cg=500):
    """lm_solve_obs of tracks [lo, hi) of case c, with device_solve's result dict"""
    import torch
    from vggsfm_b200 import bundle_adjustment as ba
    hi = c["mask"].shape[1] if hi is None else hi
    uv, f, n = coo(c, lo, hi, seed)
    poses, intr, pts = to_dev(c["poses"], DEV), to_dev(c["intr"], DEV), to_dev(c["points"][lo:hi], DEV)
    kw = {} if loss is None else dict(loss_function_type=loss[0], loss_function_scale=loss[1])
    s = ba.lm_solve_obs(to_dev(uv, DEV, torch.float32), to_dev(f.astype(np.int32), DEV), to_dev(n.astype(np.int32), DEV),
                        poses, intr, pts, c["model"], c["mode"],
                        param_const=None if param_const is None else to_dev(param_const.astype(np.uint8), DEV),
                        point_const=None if point_const is None else to_dev(point_const[lo:hi].astype(np.uint8), DEV),
                        options=options, allreduce=allreduce, want_trace=True, max_linear_solver_iterations=max_cg, **kw)
    torch.cuda.current_stream().synchronize()
    ran = s.iterations > 0
    return dict(poses=poses.cpu().numpy(), intr=intr.cpu().numpy(), points=pts.cpu().numpy(), s=s,
                trace=s.trace.numpy().copy() if ran else np.zeros((0, 8)),
                cg=s.cg_trace.numpy().copy() if ran else np.zeros((0, 4)),
                calls=allreduce.calls if allreduce is not None else 0, lo=lo, hi=hi)


def grid_solve(c, o, max_cg=500, **kw):
    return device_solve(c, DEV, options=o, linear_solver="ITERATIVE_SCHUR", max_linear_solver_iterations=max_cg, **kw)


def check_same(got, ref, label, bar=PARAM_BAR, clear=True, o=None):
    """got against ref at the module's bars; clear: the exact decisions are asserted where ref is clear of its bands"""
    s, s0 = got["s"], ref["s"]
    if clear:
        assert_clear(trace_rows(ref["trace"]), o, cg=ref["cg"])
    assert s.termination == s0.termination, (label, s.termination, s0.termination)
    assert (s.iterations, s.successful) == (s0.iterations, s0.successful), (label, s.iterations, s0.iterations)
    assert np.array_equal(got["trace"][:, 7], ref["trace"][:, 7]), (label, got["trace"][:, 7], ref["trace"][:, 7])
    assert np.array_equal(got["cg"][:, :2], ref["cg"][:, :2]), (label, got["cg"][:, :2], ref["cg"][:, :2])
    assert np.isclose(s.initial_cost, s0.initial_cost, rtol=1e-12, atol=0), (label, s.initial_cost, s0.initial_cost)
    assert np.isclose(s.final_cost, s0.final_cost, rtol=COST_BAR, atol=0), (label, s.final_cost, s0.final_cost)
    assert np.allclose(got["trace"][:, 2], ref["trace"][:, 2], rtol=COST_BAR, atol=0, equal_nan=True), label
    for k in ("poses", "intr", "points"):
        a, b = got[k], ref[k]
        fin = np.isfinite(b)
        assert np.array_equal(np.isfinite(a), fin), (label, k)
        scale = np.maximum(1.0, np.abs(b[fin])) if k == "intr" else 1.0
        assert np.all(np.abs(a[fin] - b[fin]) <= bar * scale), (label, k, np.abs(a[fin] - b[fin]).max())
    print(f"{label}: {s0.termination} after {s0.iterations} LM it, {int(ref['cg'][:, 0].sum())} CG it; final cost "
          f"{abs(s.final_cost / s0.final_cost - 1):.2e} relative, poses {np.nanmax(np.abs(got['poses'] - ref['poses'])):.2e}")


def _with_outliers(c, seed):
    rng = np.random.default_rng(seed)
    uv = c["uv"].copy()
    bad = c["mask"] & (rng.random(c["mask"].shape) < 0.1)
    uv[bad] += rng.uniform(20, 60, (int(bad.sum()), 2)) * rng.choice([-1.0, 1.0], (int(bad.sum()), 2))
    return dict(c, uv=uv)


# ------------------------------------------------------------------------------------------------------------------
# the list against the grid

@pytest.mark.parametrize("shape", SHAPES, ids=lambda s: f"{s[0]}x{s[1]}-{s[2]}-{s[3]}")
@pytest.mark.parametrize("loss", ["TRIVIAL", "CAUCHY"])
def test_shapes_match_grid(shape, loss):
    S, N, cam, mode = shape
    c = ba_case(S, N, cam, mode, seed=3)
    lf = None
    if loss == "CAUCHY":
        c, lf = _with_outliers(c, 5), ("CAUCHY", 1.0)
    o = options(max_num_iterations=3)[0]
    check_same(list_solve(c, options=o, loss=lf), grid_solve(c, o, loss=lf), f"{shape} {loss}", o=o)


def test_c2_matches_grid():
    c = ba_case(50, 2048, "SIMPLE_PINHOLE", bo.INTR_PER_FRAME, seed=1)
    o = options(max_num_iterations=10)[0]
    check_same(list_solve(c, options=o), grid_solve(c, o), "C2", o=o)


def test_c3_matches_grid():
    """400 x 4096 SIMPLE_RADIAL shared intrinsics, every cell an observation, prepare_ba_options, at most 200 CG"""
    from vggsfm_b200 import bundle_adjustment as ba
    c = ba_case(400, 4096, "SIMPLE_RADIAL", bo.INTR_SHARED, seed=0, invisible_frac=0.0)
    o = ba.prepare_ba_options()
    o.max_num_iterations = 3
    ref = grid_solve(c, o, max_cg=200)
    check_same(list_solve(c, options=o, max_cg=200), ref, "C3", bar=max(PARAM_BAR, radius_bar(trace_rows(ref["trace"]))),
               o=o)


def test_banded_matches_grid():
    c = banded_ba_case(160, 4003, "SIMPLE_RADIAL", bo.INTR_SHARED, life=24, seed=31)
    o = options(max_num_iterations=5)[0]
    check_same(list_solve(c, options=o), grid_solve(c, o), "banded", o=o)


def test_cauchy_with_outliers_matches_grid():
    c = _with_outliers(ba_case(12, 512, "SIMPLE_RADIAL", bo.INTR_PER_FRAME, seed=23), 23)
    o = options(max_num_iterations=3)[0]
    check_same(list_solve(c, options=o, loss=("CAUCHY", 1.0)), grid_solve(c, o, loss=("CAUCHY", 1.0)), "CAUCHY", o=o)


def test_one_lm_step_matches_oracle():
    """one LM iteration of the list solve in the float64 oracle's ITERATIVE_SCHUR (the list densified is the case's
    grid), at the bars of test_ba_iterative_gpu.py::test_one_lm_step_matches_oracle"""
    c = ba_case(50, 2048, "SIMPLE_PINHOLE", bo.INTR_PER_FRAME, seed=1)
    o, opt = options(max_num_iterations=1)
    got = list_solve(c, options=o)
    ref = oracle_solve(c, opt=opt, linear_solver="ITERATIVE_SCHUR")
    trace, cs = ref["trace"], ref["cg"][0]
    assert_clear(trace, opt, cg=ref["cg"])
    g = got["cg"][0]
    assert int(g[0]) == cs["summary"]["iterations"] and int(g[1]) == cs["summary"]["termination"]
    assert abs(g[2] - cs["summary"]["zeta"]) <= 1e-6 * max(1.0, abs(cs["summary"]["zeta"]))
    tr, r = got["trace"][0], trace[0]
    assert abs(tr[3] - r["model_change"]) <= 1e-8 * abs(r["model_change"])
    assert abs(tr[2] - r["candidate_cost"]) <= 1e-9 * abs(r["candidate_cost"])
    assert abs(tr[6] - r["step_norm"]) <= 1e-8 * abs(r["step_norm"])


# ------------------------------------------------------------------------------------------------------------------
# edges

def test_single_observation_point():
    c = ba_case(10, 240, "SIMPLE_RADIAL", bo.INTR_PER_FRAME, seed=41)
    mask = c["mask"].copy()
    for n in (0, 17, 239):
        mask[:, n] = False
        mask[n % 10, n] = True
    c = dict(c, mask=mask)
    o = options(max_num_iterations=3)[0]
    check_same(list_solve(c, options=o), grid_solve(c, o), "one observation", o=o)


def test_empty_segments_hold_hidden_values():
    """points and a frame without observations hold NaN / inf: returned bit for bit, and the rest of the solve is the
    clean twin's (which holds finite values there)"""
    o = options(max_num_iterations=3)[0]
    dirty, clean, hidden = hidden_case(12, 300, "SIMPLE_RADIAL", bo.INTR_PER_FRAME, seed=43, point_value=np.nan,
                                       uv_value=np.inf, hidden_frame=5)
    dirty["points"][hidden[0]] = np.inf
    got, twin = list_solve(dirty, options=o), list_solve(clean, options=o)
    assert np.array_equal(got["points"][hidden], dirty["points"][hidden], equal_nan=True)
    assert np.array_equal(got["poses"][5], dirty["poses"][5], equal_nan=True)
    assert np.array_equal(got["intr"][5], dirty["intr"][5])
    keep = np.ones(300, dtype=bool)
    keep[hidden] = False
    frames = np.arange(12) != 5
    got_c = dict(got, poses=got["poses"][frames], intr=got["intr"][frames], points=got["points"][keep])
    twin_c = dict(twin, poses=twin["poses"][frames], intr=twin["intr"][frames], points=twin["points"][keep])
    check_same(got_c, twin_c, "hidden values", o=o)


def test_long_segments():
    """every point seen by every frame, and every frame's segment (3000) longer than the frame kernels' chunk (1024)"""
    c = ba_case(12, 3000, "SIMPLE_PINHOLE", bo.INTR_SHARED, seed=47, invisible_frac=0.0)
    assert c["mask"].all()
    o = options(max_num_iterations=3)[0]
    check_same(list_solve(c, options=o), grid_solve(c, o), "long segments", o=o)


@pytest.mark.parametrize("M", [1023, 1024, 1025, 2047, 2049])
def test_tile_widths(M):
    """M at and around the frame kernels' chunk of 1024 positions; N = 8 k + 1 points, one past the point kernels'
    eight per CTA"""
    c = ba_case(8, 257, "SIMPLE_RADIAL", bo.INTR_PER_FRAME, seed=53, invisible_frac=0.0)
    rng = np.random.default_rng(M)
    cells = np.argwhere(c["mask"])
    keep = cells[rng.choice(len(cells), size=M, replace=False)]
    mask = np.zeros_like(c["mask"])
    mask[keep[:, 0], keep[:, 1]] = True
    c = dict(c, mask=mask)
    o = options(max_num_iterations=3)[0]
    check_same(list_solve(c, options=o), grid_solve(c, o), f"M={M}", o=o)


def test_shuffled_coo_matches_sorted():
    c = ba_case(16, 300, "SIMPLE_PINHOLE", bo.INTR_SHARED, seed=59)
    o = options(max_num_iterations=3)[0]
    check_same(list_solve(c, options=o, seed=7), list_solve(c, options=o), "shuffled", o=o)


# ------------------------------------------------------------------------------------------------------------------
# refusals

def _valid_list(c):
    import torch
    from vggsfm_b200 import bundle_adjustment as ba
    uv, f, n = coo(c)
    S, N = c["mask"].shape
    lst = ba.obs_list(to_dev(uv, DEV, torch.float32), to_dev(f.astype(np.int32), DEV), to_dev(n.astype(np.int32), DEV),
                      S, N)
    return {k: getattr(lst, k).cpu().numpy() for k in ("uv", "frame", "point", "track_start", "frame_start", "frame_obs")}


def _corrupt(a, which):
    """one malformed copy of a valid list per check of vgg_ba_solve_iterative_obs"""
    a = {k: v.copy() for k, v in a.items()}
    ts, fs, M = a["track_start"], a["frame_start"], len(a["frame"])
    n = int(np.argmax(np.diff(ts) >= 3))            # a point with at least three observations
    m = int(ts[n])
    if which == "track_start_order":
        ts[n + 1] = ts[n + 2] + 1
    elif which == "track_start_end":
        ts[-1] = M - 1
    elif which == "point":
        a["point"][m] = n + 1
    elif which == "frame_range":
        a["frame"][m] = len(fs) - 1
    elif which == "duplicate":
        a["frame"][m + 1] = a["frame"][m]
    elif which == "track_order":
        a["frame"][m], a["frame"][m + 1] = a["frame"][m + 1], a["frame"][m]
    elif which == "histogram":
        fs[1] += 1
    elif which == "frame_start_end":
        fs[-1] = M + 1
    elif which == "frame_obs_frame":
        j = int(np.nonzero(a["frame_obs"] == m)[0][0])
        a["frame_obs"][j] = m + 1                       # the point's next observation, in a later frame
    elif which == "frame_obs_order":
        j = int(fs[0])
        a["frame_obs"][j], a["frame_obs"][j + 1] = a["frame_obs"][j + 1], a["frame_obs"][j]
    return a


CORRUPTIONS = ["track_start_order", "track_start_end", "point", "frame_range", "duplicate", "track_order", "histogram",
               "frame_start_end", "frame_obs_frame", "frame_obs_order"]


@pytest.mark.parametrize("which", CORRUPTIONS)
def test_malformed_list_refused(which):
    """VGG_EINVAL before the LM loop: the summary and the trace are not written, the state is unchanged"""
    import torch
    from vggsfm_b200 import _lib
    from vggsfm_b200 import bundle_adjustment as ba
    c = ba_case(8, 64, "SIMPLE_PINHOLE", bo.INTR_PER_FRAME, seed=61)
    S, N = c["mask"].shape
    arrays = _corrupt(_valid_list(c), which)
    d = {k: to_dev(v, DEV) for k, v in arrays.items()}
    poses, intr, pts = to_dev(c["poses"], DEV), to_dev(c["intr"], DEV), to_dev(c["points"], DEV)
    p = _lib.BAProblem()
    p.S, p.N, p.camera_model, p.intr_mode = S, N, c["model"], c["mode"]
    pc = ba.default_param_const(S, c["model"], c["mode"], DEV)
    p.param_const, p.poses, p.intr, p.points = pc.data_ptr(), poses.data_ptr(), intr.data_ptr(), pts.data_ptr()
    ol = _lib.BAObsList(len(arrays["frame"]), *(d[k].data_ptr() for k in ("uv", "frame", "point", "track_start",
                                                                          "frame_start", "frame_obs")))
    ws = ba.workspace(S, N, c["model"], c["mode"], DEV, iterative=True, obs=True)
    lin = ba.linear_solver("ITERATIVE_SCHUR")
    summ = _lib.BASummary()
    summ.iterations, summ.termination = -7, -7
    trace = np.full((100, 8), 7.0)
    L = _lib.lib()
    rc = L.vgg_ba_solve_iterative_obs(ctypes.byref(p), ctypes.byref(ol), ctypes.byref(ba.default_options()),
                                      ctypes.byref(lin), ws.data_ptr(), ws.numel(), _lib.ALLREDUCE_FN(), None,
                                      ctypes.byref(summ), trace.ctypes.data, None,
                                      torch.cuda.current_stream().cuda_stream)
    torch.cuda.synchronize()
    assert rc == -1, (which, rc)
    assert "malformed observation list" in L.vgg_last_error().decode(), L.vgg_last_error()
    assert summ.iterations == -7 and summ.termination == -7 and (trace == 7.0).all()
    assert np.array_equal(poses.cpu().numpy(), c["poses"]) and np.array_equal(pts.cpu().numpy(), c["points"])


def test_lm_solve_obs_rejects_duplicates_and_shapes():
    import torch
    from vggsfm_b200 import bundle_adjustment as ba
    c = ba_case(8, 64, "SIMPLE_PINHOLE", bo.INTR_PER_FRAME, seed=61)
    uv, f, n = coo(c)
    args = (to_dev(c["poses"], DEV), to_dev(c["intr"], DEV), to_dev(c["points"], DEV), c["model"], c["mode"])
    dup = lambda a: np.concatenate([a, a[3:4]])
    with pytest.raises(ValueError, match="twice"):
        ba.lm_solve_obs(to_dev(dup(uv), DEV, torch.float32), to_dev(dup(f), DEV), to_dev(dup(n), DEV), *args)
    with pytest.raises(ValueError, match="obs_uv"):
        ba.lm_solve_obs(to_dev(uv[:-1], DEV, torch.float32), to_dev(f, DEV), to_dev(n, DEV), *args)
    with pytest.raises(ValueError, match="lie in"):
        ba.lm_solve_obs(to_dev(uv, DEV, torch.float32), to_dev(f + 8, DEV), to_dev(n, DEV), *args)


# ------------------------------------------------------------------------------------------------------------------
# track shards

@pytest.mark.parametrize("K", [2, 3, 8])
@pytest.mark.parametrize("name", ["C2", "banded"])
def test_track_shards(K, name):
    """each rank's list of its own tracks, against the unsharded list solve, at _check's bars: exact decisions and CG
    counts, the hook's call schedule, bit-identical CG traces and cameras across the ranks"""
    if name == "C2":
        c, o = ba_case(50, 2048, "SIMPLE_PINHOLE", bo.INTR_PER_FRAME, seed=1), options(max_num_iterations=10)[0]
    else:
        c = banded_ba_case(160, 4003, "SIMPLE_RADIAL", bo.INTR_SHARED, life=24, seed=31)
        o = options(max_num_iterations=5)[0]
    ref = list_solve(c, options=o)
    assert_clear(trace_rows(ref["trace"]), o, cg=ref["cg"])
    res, _ = run_shards(c["mask"].shape[1], K,
                        lambda r, lo, hi, hook: list_solve(c, lo=lo, hi=hi, options=o, allreduce=hook), device=DEV)
    _check(res, ref, f"list {name} K={K}")
