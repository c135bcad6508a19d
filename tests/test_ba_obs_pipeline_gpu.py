"""The observation list through the layers above the solve: the list point filter (triangulation.filter_observations)
against the grid's filter_all_points3D, bundle_adjustment_obs against bundle_adjustment(..., "ITERATIVE_SCHUR"), a
1000-frame C5 joint BA through joint_BA_obs / replace_from_obs against the grid SceneStore path, and the 8000-frame
joint BA whose grid would not fit on the card, built as a list and run through SceneStore.joint_bundle_adjustment.
Solve bars as tests/test_ba_obs_list_gpu.py (CG amplifies the rounding of the two summation orders)."""
import numpy as np
import pytest

from oracle import ba_oracle as bo
from tests.helpers import ba_case, to_dev

pytestmark = [pytest.mark.gpu, pytest.mark.usefixtures("cuda_dev")]

DEV = "cuda:0"
PARAM_BAR = 1e-4
COST_BAR = 1e-5
# peak device memory of the 8000-frame joint BA on the list path (measured 'frames8000' peak of tools/ba_obs_bench.py
# on an H100 80GB HBM3, DESIGN 4.10, plus margin)
PEAK_8000_GB = 12.0                    # measured: 8.75 GB


def _reproj_err(c, pts):
    """float64 reprojection error and depth of every cell [S,P]"""
    R, t = c["poses"][:, :, :3], c["poses"][:, :, 3]
    pc = np.einsum("sij,pj->spi", R, pts) + t[:, None]
    u, v = pc[..., 0] / pc[..., 2], pc[..., 1] / pc[..., 2]
    k = c["intr"][:, 3:4] if c["model"] == bo.SIMPLE_RADIAL else 0.0
    d = 1 + k * (u * u + v * v)
    x = c["intr"][:, 0:1] * d * u + c["intr"][:, 1:2]
    y = c["intr"][:, 0:1] * d * v + c["intr"][:, 2:3]
    return np.hypot(x - c["uv"][..., 0], y - c["uv"][..., 1]), pc[..., 2]


def test_filter_observations_matches_grid_filter():
    import torch
    from vggsfm_b200 import triangulation as tri
    c = ba_case(20, 600, "SIMPLE_RADIAL", bo.INTR_PER_FRAME, seed=71)
    err, depth = _reproj_err(c, c["points"])
    obs = c["mask"]
    e = np.sort(err[obs])
    thr = float(0.5 * (e[len(e) // 2 - 1] + e[len(e) // 2]))     # half the observations on each side
    # the two rules differ only for an unobserved cell that reprojects within the bound: the data has none, and every
    # observed error is clear of the threshold by 1e-9 relative
    uv_grid = np.where(obs[..., None], c["uv"], 0.0)
    err0, _ = _reproj_err(dict(c, uv=uv_grid), c["points"])
    assert not ((err0 <= thr) & (depth > 0) & ~obs).any()
    assert (np.abs(err[obs] - thr) > 1e-9 * thr).all()
    assert 0.3 < ((err[obs] <= thr) & (depth[obs] > 0)).mean() < 0.7
    S = obs.shape[0]
    K = np.zeros((S, 3, 3))
    K[:, 0, 0] = K[:, 1, 1] = c["intr"][:, 0]
    K[:, 0, 2], K[:, 1, 2], K[:, 2, 2] = c["intr"][:, 1], c["intr"][:, 2], 1.0
    X, E, Kd, ex = (to_dev(c["points"], DEV), to_dev(c["poses"], DEV), to_dev(K, DEV), to_dev(c["intr"][:, 3:4], DEV))
    valid_g, _ = tri.filter_all_points3D(X, to_dev(uv_grid, DEV, torch.float32), E, Kd, ex, max_reproj_error=thr,
                                         min_tri_angle=1.5, check_triangle=True, hard_max=-1)
    _, detail = tri.filter_all_points3D(X, to_dev(uv_grid, DEV, torch.float32), E, Kd, ex, max_reproj_error=thr,
                                        min_tri_angle=1.5, check_triangle=False, return_detail=True, hard_max=-1)
    f, n = np.nonzero(obs)
    perm = np.random.default_rng(3).permutation(len(f))
    f, n = f[perm], n[perm]
    keep, valid = tri.filter_observations(X, to_dev(c["uv"][f, n], DEV, torch.float32), to_dev(f, DEV), to_dev(n, DEV),
                                          E, Kd, ex, max_reproj_error=thr, min_tri_angle=1.5)
    assert np.array_equal(keep.cpu().numpy(), detail.cpu().numpy()[f, n])
    assert np.array_equal(valid.cpu().numpy(), valid_g.cpu().numpy())
    print(f"list filter: {int(keep.sum())} of {len(f)} observations kept, {int(valid.sum())} of {obs.shape[1]} points")


def test_bundle_adjustment_obs_matches_grid():
    """compaction (points with < 2 observations), the 3000 clamp, the negative-depth filter, gauge and both
    normalisations: the same kept points, alive flags and kept observations as bundle_adjustment, the solve at the
    list-vs-grid bars"""
    import torch
    from vggsfm_b200 import bundle_adjustment as ba
    c = ba_case(12, 400, "SIMPLE_RADIAL", bo.INTR_PER_FRAME, seed=73)
    mask, pts = c["mask"].copy(), c["points"].copy()
    mask[:, 5] = False
    mask[3, 5] = True                                  # one observation: not in the problem
    pts[9] = [4000.0, 0.0, 10.0]                       # past the clamp
    # a point behind one camera that sees it: that observation is dropped by the negative-depth filter
    R, t = c["poses"][0, :, :3], c["poses"][0, :, 3]
    pts[11] = R.T @ (np.array([0.0, 0.0, -3.0]) - t)
    mask[0, 11] = True
    S = mask.shape[0]
    K = np.zeros((S, 3, 3))
    K[:, 0, 0] = K[:, 1, 1] = c["intr"][:, 0]
    K[:, 0, 2], K[:, 1, 2], K[:, 2, 2] = c["intr"][:, 1], c["intr"][:, 2], 1.0
    o = ba.default_options()
    o.max_num_iterations = 3
    args = (to_dev(pts, DEV), to_dev(c["poses"], DEV), to_dev(K, DEV), to_dev(c["intr"][:, 3:4], DEV))
    g = ba.bundle_adjustment(*args, to_dev(c["uv"], DEV, torch.float32), to_dev(mask, DEV), camera_type="SIMPLE_RADIAL",
                             options=o, linear_solver_type="ITERATIVE_SCHUR")
    f, n = np.nonzero(mask)
    lst = ba.bundle_adjustment_obs(*args, to_dev(c["uv"][f, n], DEV, torch.float32), to_dev(f, DEV), to_dev(n, DEV),
                                   camera_type="SIMPLE_RADIAL", options=o)
    vi = g[4].cpu().numpy()
    assert np.array_equal(lst[4].cpu().numpy(), vi) and 5 not in vi and 9 in vi
    assert np.array_equal(lst[5].alive.cpu().numpy(), g[5].alive.cpu().numpy())
    pos = np.full(mask.shape[1], -1)
    pos[vi] = np.arange(len(vi))
    want = np.where(pos[n] >= 0, g[5].mask.cpu().numpy()[f, np.maximum(pos[n], 0)], False)
    assert np.array_equal(lst[5].keep.cpu().numpy(), want)
    assert not want[(f == 0) & (n == 11)].any() and not want[n == 9].any()
    sg, sl = g[5], lst[5]
    assert (sl.termination, sl.iterations, sl.successful) == (sg.termination, sg.iterations, sg.successful)
    assert np.array_equal(sl.cg_trace[:, :2].numpy(), sg.cg_trace[:, :2].numpy())
    assert abs(sl.final_cost / sg.final_cost - 1) <= COST_BAR
    for k in (0, 1, 2, 3):
        assert np.abs(lst[k].cpu().numpy() - g[k].cpu().numpy()).max() <= PARAM_BAR * max(1.0, np.abs(g[k].cpu().numpy()).max()), k


def _store(uv, fr, pt, pts, extr, dev):
    from tools.ba_obs_bench import store_of
    return store_of(uv, fr, pt, pts, extr, dev)


def test_scene_store_c5_list_matches_grid():
    """a 1000-frame C5 store: joint_BA_obs + replace_from_obs against the grid joint_bundle_adjustment
    (ITERATIVE_SCHUR, which the size rule leaves on the grid): identical kept points and observations, cameras and
    points within the bars"""
    import torch
    from tools.video_c5 import final_problem_arrays
    from vggsfm_b200 import bundle_adjustment as ba
    from vggsfm_b200 import video
    tracks, masks, pts, extr, K = final_problem_arrays(1000, 512, dev=torch.device(DEV))
    S, P = masks.shape
    assert video.grid_fits(S, P, DEV)
    f, n = torch.nonzero(masks, as_tuple=True)
    uv = tracks[f, n]
    o = ba.default_options()
    # the first two LM iterations: from the third on this problem's CG stops lie within rounding of eta (two grid runs
    # of the 2500-frame problem already end 156 and 157 CG iterations apart, tools/ba_obs_bench.py)
    o.max_num_iterations = 2
    sg = _store(uv, f, n, pts, extr, DEV)
    sg.joint_bundle_adjustment(0, S, K, None, linear_solver_type="ITERATIVE_SCHUR", options=o)
    summ_g = video.last_joint_summary
    assert summ_g.keep is None                           # the grid path
    sl = _store(uv, f, n, pts, extr, DEV)
    xyz, ouv, ofr, opt_, ex = sl.observations(0, S)
    out, e2, K2, _, keep, valid = video.joint_BA_obs(xyz, ex, K, None, ouv, ofr, opt_, options=o)
    sl.replace_from_obs(0, out, e2, ouv, ofr, opt_, keep, valid)
    summ_l = video.last_joint_summary
    assert (summ_l.termination, summ_l.iterations, summ_l.successful) == \
        (summ_g.termination, summ_g.iterations, summ_g.successful)
    assert np.array_equal(summ_l.cg_trace[:, :2].numpy(), summ_g.cg_trace[:, :2].numpy())
    assert abs(summ_l.final_cost / summ_g.final_cost - 1) <= COST_BAR
    assert sl.num_points == sg.num_points
    for k in ("obs_point", "obs_frame"):
        assert torch.equal(getattr(sl, k), getattr(sg, k)), k
    assert torch.equal(sl.obs_uv, sg.obs_uv)
    assert (sl.extri - sg.extri).abs().max().item() <= PARAM_BAR
    assert (sl.xyz.double() - sg.xyz.double()).abs().max().item() <= PARAM_BAR * max(1.0, sg.xyz.abs().max().item())
    print(f"C5 1000: {sg.num_points} of {P} points and {sg.obs_point.numel()} observations kept by both paths")


def test_8000_frames_take_the_list():
    """8000 frames at 2048 new points per window, built as a list window by window (never as a grid): its grid would
    need 9 S P > 70 GB, so SceneStore.joint_bundle_adjustment takes the list path; about 10 LM iterations without
    FAILURE, a final cost well below the initial one, peak device memory under PEAK_8000_GB"""
    import torch
    from tools.ba_obs_bench import final_problem_obs, store_of
    from vggsfm_b200 import bundle_adjustment as ba
    from vggsfm_b200 import video
    dev = torch.device(DEV)
    uv, fr, pt, pts, extr, K = final_problem_obs(8000, 2048, dev=dev)
    S, P = extr.shape[0], pts.shape[0]
    assert 9.0 * S * P > 70e9 and not video.grid_fits(S, P, dev)
    store = store_of(uv, fr, pt, pts, extr, dev)
    del uv, fr, pt
    o = ba.default_options()
    o.max_num_iterations = 10
    torch.cuda.synchronize()
    torch.cuda.reset_peak_memory_stats()
    store.joint_bundle_adjustment(0, S, K, None, linear_solver_type="ITERATIVE_SCHUR", max_linear_solver_iterations=100,
                                  options=o)
    torch.cuda.synchronize()
    peak = torch.cuda.max_memory_allocated() / 1e9
    s = video.last_joint_summary
    print(f"8000 frames: S={S} P={P} 9SP={9.0 * S * P / 1e9:.1f} GB, {s.iterations} LM it, {s.cg_iterations} CG it, "
          f"cost {s.initial_cost:.4g} -> {s.final_cost:.4g}, {s.termination}, peak {peak:.2f} GB")
    assert s.keep is not None                            # the list path
    assert s.termination != "FAILURE_INVALID_STEPS" and 5 <= s.iterations <= 10
    assert s.final_cost < 0.1 * s.initial_cost
    assert peak < PEAK_8000_GB
    assert store.num_points > 0.9 * P


def test_lm_solve_obs_without_points_rejects_observations():
    import torch
    from vggsfm_b200 import bundle_adjustment as ba
    c = ba_case(8, 64, "SIMPLE_PINHOLE", bo.INTR_PER_FRAME, seed=61)
    none = torch.zeros(0, 3, dtype=torch.float64, device=DEV)
    with pytest.raises(ValueError, match="without points"):
        ba.lm_solve_obs(torch.zeros(2, 2, device=DEV), torch.tensor([0, 1], device=DEV), torch.tensor([0, 0], device=DEV),
                        to_dev(c["poses"], DEV), to_dev(c["intr"], DEV), none, c["model"], c["mode"])
