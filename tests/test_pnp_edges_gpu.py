"""P3P LO-RANSAC absolute pose (csrc/pnp.cu: pnp_ransac_kernel + pnp_select_kernel) against oracle/pnp_oracle.py at the
production shape and at its edges: 400 x 4096 with and without the focal ladder, all 31 LO-RANSACs of a frame one by
one, the compaction of usable points across 256-point chunks, the shared-memory limit, sample edge values, degenerate
geometry, and the force_estimate branches of refine_pose.

Bars as in test_pnp_gpu.py: inlier count, focal and mask exact, pose 1e-8; and for every frame
num_inliers == inliers.sum() (pnp_select_kernel recomputes the mask independently of the count).

Near ties: counts and masks are compared exactly, so every oracle run asserts (through ``return_debug``) that no residual
of a scored pose lies within 1e-9 relative of the threshold and that no two supports with equal counts had residual sums
within 1e-9 relative.  A best support of exactly three inliers is the exception: every candidate then fits its own
sample and the sums are rounding noise, so only the count and that the pose fits its three inliers are checked.  A pose
that is a raw P3P candidate (no local optimisation improved on it) is held to 1e-7 instead of 1e-8 (RAW_P3P_POSE_TOL)."""
import numpy as np
import pytest

from oracle import pnp_oracle as pno
from oracle import pose_oracle as poo
from tests.helpers import to_dev
from vggsfm_b200.synthetic import make_scene

pytestmark = pytest.mark.gpu

NEAR_TIE = 1e-9
POSE_TOL = 1e-8
# a winner that is a raw closed-form P3P candidate (no local optimisation beat it): the kernel evaluates the quartic and
# its Ferrari / Cardano steps with CUDA's libm and contracted FMAs, numpy with glibc and separate roundings, and three
# Newton steps do not always polish the difference away.  Largest seen on an H100: 4.4e-8 (SIMPLE_RADIAL production
# scene; 1.5e-10 on the SIMPLE_PINHOLE one); every local-optimisation result agrees to POSE_TOL.
RAW_P3P_POSE_TOL = 1e-7
PNP_MAX_POINTS = 9751                 # 21 P + 16 bytes of dynamic shared memory <= 200 KB


def run_and_check(dev, tracks, X, masks, intr4, model, us, est_f=False, frames=None, check=None, max_error=12.0):
    """One vgg_absolute_pose_estimation launch; frames in `check` (default: every flagged frame) against the oracle.
    Returns (kernel outputs, the oracle debug records merged over the checked frames)."""
    import torch
    from vggsfm_b200 import pose_refinement as pr
    S, P = masks.shape
    flags = np.ones(S, bool) if frames is None else np.asarray(frames, bool)
    poses, focal, ninl, inl = pr.absolute_pose_estimation_batched(
        to_dev(tracks, dev), to_dev(X, dev), to_dev(masks, dev), to_dev(intr4, dev), model, frames=to_dev(flags, dev),
        estimate_focal_length=est_f, max_error=max_error, u_samples=torch.from_numpy(np.asarray(us, np.float64)))
    poses, focal, ninl, inl = poses.cpu().numpy(), focal.cpu().numpy(), ninl.cpu().numpy(), inl.cpu().numpy()
    assert np.array_equal(ninl, inl.sum(axis=1)), np.nonzero(ninl != inl.sum(axis=1))[0]
    assert not (inl & ~np.asarray(masks, bool)).any()              # inliers only among the usable points
    off = ~flags
    assert not ninl[off].any() and not inl[off].any() and not poses[off].any()
    assert np.array_equal(focal[off], intr4[off, 0])
    agg = pno.new_debug()
    for s in (np.nonzero(flags)[0] if check is None else check):
        r, d = pno.absolute_pose_estimation(tracks[s], X, intr4[s], model, us, estimate_focal_length=est_f,
                                            max_error=max_error, mask=masks[s], return_debug=True)
        agg["nsol_hist"] += d["nsol_hist"]
        agg["skipped"] += d["skipped"]
        agg["lo_not_last"] += d["lo_not_last"]
        if r is None:
            assert ninl[s] == 0 and not inl[s].any() and not poses[s].any() and focal[s] == intr4[s, 0], s
            continue
        assert ninl[s] == r["num_inliers"], (s, ninl[s], r["num_inliers"])
        assert focal[s] == r["focal"], (s, focal[s], r["focal"])
        if r["num_inliers"] == 3:                             # every candidate fits its own sample: the pose is a tie
            xn = (tracks[s][inl[s]].astype(np.float64) - intr4[s, 1:3]) / focal[s]
            if model == pno.SIMPLE_RADIAL:
                xn = pno.undistort_radial(xn, intr4[s, 3])
            assert (pno.residuals(poses[s], X[inl[s]], xn) <= (max_error / focal[s]) ** 2).all()
            continue
        assert np.array_equal(inl[s], r["inliers"]), (s, np.nonzero(inl[s] != r["inliers"])[0][:10])
        agg["thr_margin"] = min(agg["thr_margin"], d["thr_margin"])
        agg["tie_gap"] = min(agg["tie_gap"], d["tie_gap"])
        _check_pose(agg, s, poses[s], r["pose"], d["best_from_lo"])
    assert agg["thr_margin"] > NEAR_TIE and agg["tie_gap"] > NEAR_TIE, (agg["thr_margin"], agg["tie_gap"])
    return (poses, focal, ninl, inl), agg


def _check_pose(agg, s, got, want, from_lo):
    err = np.abs(got - want).max()
    if from_lo:
        assert err <= POSE_TOL, (s, err)
    else:
        assert err <= RAW_P3P_POSE_TOL, (s, err)
        agg["p3p_pose_err"] = max(agg.get("p3p_pose_err", 0.0), err)


def _intr(S, f, k, model):
    return np.tile(np.array([f, 512.0, 512.0, k if model == pno.SIMPLE_RADIAL else 0.0]), (S, 1))


def _model(cam):
    return pno.SIMPLE_RADIAL if cam == "SIMPLE_RADIAL" else pno.SIMPLE_PINHOLE


# seed 31 / 32: 400 x 4096, 25 % outliers, 20 % invisible; smallest margins printed by the test
@pytest.mark.parametrize("cam", ["SIMPLE_PINHOLE", "SIMPLE_RADIAL"])
def test_production_shape(cuda_dev, cam):
    """400 x 4096, default 128 trials.  Without the ladder every frame is flagged and 64 spread frames (0 and 399
    included) are checked; with the ladder 12 frames are flagged and all of them are checked, and every unflagged frame
    must come back with count 0, zero pose, an empty mask and focal = prior."""
    import torch
    from vggsfm_b200 import pose_refinement as pr
    S, P = 400, 4096
    model = _model(cam)
    sc = make_scene(S, P, cam, seed=31 if model == 0 else 32, noise_px=0.3, outlier_frac=0.25, invisible_frac=0.2)
    torch.manual_seed(5)
    us = pr.draw_pnp_samples().numpy()
    intr4 = _intr(S, 1000.0, 0.05, model)
    chk = np.unique(np.linspace(0, S - 1, 64).round().astype(int))
    _, a = run_and_check(cuda_dev, sc.tracks, sc.points3d, sc.mask, intr4, model, us, check=chk)
    intr4[:, 0] = 1000.0 * np.random.default_rng(7).uniform(0.7, 1.6, size=S)
    flagged = np.zeros(S, bool)
    flagged[np.unique(np.linspace(0, S - 1, 12).round().astype(int))] = True
    _, b = run_and_check(cuda_dev, sc.tracks, sc.points3d, sc.mask, intr4, model, us, est_f=True, frames=flagged)
    print(f"pnp 400x4096 {cam}: P3P solutions per trial {a['nsol_hist'].tolist()} / {b['nsol_hist'].tolist()}, "
          f"LO on an earlier candidate {a['lo_not_last']} / {b['lo_not_last']}, threshold margin "
          f"{min(a['thr_margin'], b['thr_margin']):.2e}, equal-count sum gap {min(a['tie_gap'], b['tie_gap']):.2e}, "
          f"largest raw-P3P pose difference {max(a.get('p3p_pose_err', 0), b.get('p3p_pose_err', 0)):.2e}")


@pytest.mark.parametrize("frame", [3, 11])
def test_every_focal_factor(cuda_dev, frame):
    """All 31 LO-RANSACs of one frame: 31 calls without the ladder, one per factor, with the prior set to the oracle's
    f0 * fac_k, each against the oracle's result at that focal; then the ladder call returns the first factor with the
    highest count, at the same focal to the bit."""
    S, P = 16, 800
    sc = make_scene(S, P, "SIMPLE_RADIAL", seed=41, noise_px=0.3, outlier_frac=0.25, invisible_frac=0.2)
    us = np.random.default_rng(42).uniform(size=(96, 3))
    f0 = 1000.0 * (1.45 if frame == 3 else 0.62)
    intr = np.array([f0, 512.0, 512.0, 0.05])
    r, d = pno.absolute_pose_estimation(sc.tracks[frame], sc.points3d, intr, 1, us, estimate_focal_length=True,
                                        mask=sc.mask[frame], return_debug=True)
    facs = d["factors"]
    rows = np.tile(intr, (31, 1))
    rows[:, 0] = [fc["focal"] for fc in facs]
    tr = np.repeat(sc.tracks[frame][None], 31, 0)
    mk = np.repeat(sc.mask[frame][None], 31, 0)
    (poses, focal, ninl, inl), agg = run_and_check(cuda_dev, tr, sc.points3d, mk, rows, 1, us, check=[])
    for k, fc in enumerate(facs):
        assert ninl[k] == fc["num_inliers"] and np.array_equal(inl[k], fc["inliers"]), k
        assert focal[k] == fc["focal"]
        if fc["num_inliers"]:
            _check_pose(agg, k, poses[k], fc["pose"], fc["from_lo"])
    assert d["thr_margin"] > NEAR_TIE and d["tie_gap"] > NEAR_TIE
    assert len(set(fc["num_inliers"] for fc in facs)) > 5             # the factors really differ
    (lp, lf, ln, li), _ = run_and_check(cuda_dev, sc.tracks[frame:frame + 1], sc.points3d, sc.mask[frame:frame + 1],
                                        intr[None], 1, us, est_f=True)
    best = int(np.argmax([fc["num_inliers"] for fc in facs]))
    assert lf[0] == facs[best]["focal"] == r["focal"] and ln[0] == facs[best]["num_inliers"]


@pytest.mark.parametrize("P", [3, 4, 255, 256, 257, 511, 512, 513])
def test_compaction(cuda_dev, P):
    """Usable points compacted in order across 256-point chunks: holes straddling every chunk boundary, a frame with
    exactly 3 usable points spread over the chunks, one with 2 (no minimal sample: count 0), one with all points."""
    cam = "SIMPLE_RADIAL" if P % 2 else "SIMPLE_PINHOLE"
    model = _model(cam)
    sc = make_scene(4, P, cam, seed=50 + P, noise_px=0.3, outlier_frac=0.2)
    m = sc.mask.copy()
    for c in range(256, P + 1, 256):
        m[0, max(0, c - 3):c + 2] = False
    m[0, :2] = False
    m[1] = False
    m[1, [0, P // 2, P - 1]] = True
    m[2] = False
    m[2, [1, P - 1]] = True
    m[3] = True
    us = np.random.default_rng(51).uniform(size=(64, 3))
    (_, _, ninl, inl), _ = run_and_check(cuda_dev, sc.tracks, sc.points3d, m, _intr(4, 1000.0, 0.05, model), model, us)
    assert ninl[2] == 0 and (ninl[1] == 3 or P == 3)
    assert not (inl[1] & ~m[1]).any()                             # the 3-inlier frame's mask lies on its usable points


def test_shared_memory_limit(cuda_dev):
    """P = 9751 needs 204 787 B of dynamic shared memory, just under the 200 KB cap: it runs and matches the oracle.
    P = 9752 is refused with VGG_EINVAL before any launch, and refine_pose(force_estimate=True) with more than 9751
    valid tracks raises instead of returning its lost frames unchanged."""
    import torch
    from vggsfm_b200 import pose_refinement as pr
    assert PNP_MAX_POINTS * 21 + 16 <= 200 * 1024 < (PNP_MAX_POINTS + 1) * 21 + 16
    sc = make_scene(2, PNP_MAX_POINTS + 1, "SIMPLE_PINHOLE", seed=61, noise_px=0.3, outlier_frac=0.25,
                    invisible_frac=0.2)
    us = np.random.default_rng(62).uniform(size=(48, 3))
    n = PNP_MAX_POINTS
    run_and_check(cuda_dev, sc.tracks[:, :n], sc.points3d[:n], sc.mask[:, :n], _intr(2, 1000.0, 0, 0), 0, us)
    with pytest.raises(RuntimeError, match=r"rc=-1\).*9751"):
        pr.absolute_pose_estimation_batched(to_dev(sc.tracks, cuda_dev), to_dev(sc.points3d, cuda_dev),
                                            to_dev(sc.mask, cuda_dev), to_dev(_intr(2, 1000.0, 0, 0), cuda_dev), 0,
                                            u_samples=torch.from_numpy(us))
    E = sc.extrinsics.copy()
    E[1, :, 3] += np.array([0.8, -0.3, 0.5])                     # frame 1 lost: needs the fall-back
    args = (to_dev(E, cuda_dev), to_dev(sc.intrinsics, cuda_dev), None, to_dev(sc.mask, cuda_dev),
            to_dev(sc.points3d, cuda_dev), to_dev(sc.tracks, cuda_dev),
            torch.ones(n + 1, dtype=torch.bool, device=cuda_dev), torch.tensor([1024, 1024], device=cuda_dev))
    with pytest.raises(RuntimeError, match="9751"):
        pr.refine_pose(*args, force_estimate=True)


@pytest.mark.parametrize("case", ["T1", "T3_edges", "T1024"])
def test_samples(cuda_dev, case):
    """One trial, 1024 trials, and the sample edges: u = 0.0, 1 - 2^-53 and 1.0 (clamped to n - 1), and a repeated index
    (the trial is skipped)."""
    sc = make_scene(4, 300, "SIMPLE_PINHOLE", seed=71, noise_px=0.3, outlier_frac=0.25, invisible_frac=0.2)
    rng = np.random.default_rng(72)
    if case == "T1":
        us = np.array([[0.11, 0.52, 0.93]])
    elif case == "T3_edges":
        us = np.array([[0.0, 0.5, 1.0 - 2.0 ** -53], [1.0, 0.0, 0.3], [0.25, 0.25, 0.7]])
    else:
        us = rng.uniform(size=(1024, 3))
    (_, _, ninl, _), d = run_and_check(cuda_dev, sc.tracks, sc.points3d, sc.mask, _intr(4, 1000.0, 0, 0), 0, us)
    if case == "T3_edges":
        assert d["skipped"] == 4 and d["nsol_hist"].sum() == 8
    else:
        assert d["nsol_hist"].sum() + d["skipped"] == 4 * len(us)


def test_degenerate_geometry(cuda_dev):
    """Exactly collinear sample triples and duplicated 3D points (no P3P solution: frame3 divides by zero), points behind
    every camera, candidates from a sample containing such a point, and a NaN observation -- each drawn by a planted
    sample, the rest random."""
    S, P = 3, 300
    sc = make_scene(S, P, "SIMPLE_PINHOLE", seed=81, noise_px=0.3, outlier_frac=0.2)
    X = sc.points3d.copy()
    X[0] = np.round(X[0] * 1024) / 1024
    X[1] = X[0] + [0.25, 0.0, 0.0]                               # exactly collinear along x
    X[2] = X[0] + [0.5, 0.0, 0.0]
    X[4] = X[3]                                                  # duplicated point
    X[6:10] = np.array([0.0, 0.0, -4.0]) + np.random.default_rng(82).normal(size=(4, 3)) * 0.3   # behind every camera
    uv = sc.tracks.copy()
    uv[:, 12, 0] = np.nan
    m = np.ones((S, P), bool)
    n = P
    pick = lambda *ids: [(i + 0.5) / n for i in ids]
    us = np.concatenate([np.array([pick(0, 1, 2), pick(2, 0, 1), pick(3, 4, 5), pick(6, 20, 21), pick(12, 13, 14)]),
                         np.random.default_rng(83).uniform(size=(60, 3))])
    (_, _, ninl, inl), d = run_and_check(cuda_dev, uv, X, m, _intr(S, 1000.0, 0, 0), 0, us)
    assert not inl[:, 6:10].any() and not inl[:, 12].any() and (ninl > 100).all()
    for s in range(S):                                           # the planted trials contribute no candidate
        xn = (uv[s].astype(np.float64) - 512.0) / 1000.0
        for ids in ((0, 1, 2), (2, 0, 1), (3, 4, 5), (12, 13, 14)):
            b = np.concatenate([xn[list(ids)], np.ones((3, 1))], 1)
            with np.errstate(all="ignore"):
                assert pno.p3p(b / np.linalg.norm(b, axis=1, keepdims=True), X[list(ids)]) == []


def test_radial_undistortion_diverges(cuda_dev):
    """SIMPLE_RADIAL with k = -0.3: x (1 + k r^2) peaks at r = 0.703, so observations beyond that distorted radius
    (the image corners at f = 1000) have no undistorted solution and the 20 Newton steps wander; they must come out
    identically (never inliers) and the rest must match."""
    S, P = 3, 300
    sc = make_scene(S, P, "SIMPLE_RADIAL", seed=91, noise_px=0.3, outlier_frac=0.2, k=-0.3)
    uv = sc.tracks.copy()
    uv[:, :4] = np.array([[0.0, 0.0], [1023.0, 0.0], [0.0, 1023.0], [1023.0, 1023.0]], np.float32)
    m = np.ones((S, P), bool)
    us = np.random.default_rng(92).uniform(size=(64, 3))
    (_, _, ninl, inl), _ = run_and_check(cuda_dev, uv, sc.points3d, m, _intr(S, 1000.0, -0.3, 1), 1, us)
    assert (ninl > 100).all() and not inl[:, :4].any()


def test_p3p_solution_counts_and_lo_restore(cuda_dev):
    """Trials with 1, 2, 3 and 4 P3P solutions all occur (3 is rare on random scenes), and local optimisation runs on a
    candidate that is not the last of its trial, where the kernel must restore the supports of the later candidates."""
    sc = make_scene(3, 400, "SIMPLE_PINHOLE", seed=21, noise_px=0.3, outlier_frac=0.25, invisible_frac=0.2)
    us = np.random.default_rng(22).uniform(size=(1024, 3))
    _, d = run_and_check(cuda_dev, sc.tracks, sc.points3d, sc.mask, _intr(3, 1000.0, 0, 0), 0, us)
    print(f"P3P solutions per trial {d['nsol_hist'].tolist()}, LO on an earlier candidate {d['lo_not_last']}")
    assert (d["nsol_hist"][1:] > 0).all() and d["lo_not_last"] > 0


def _oracle_force_estimate(p0, i0, X, uv, vis, model, shared, us, scale=1024.0):
    """refine_pose(force_estimate=True) composed from the oracles: the frame loop (12 px pre-filter, > 100 inliers),
    then triangulation.py:404-433 for the frames that need it -- P3P LO-RANSAC with the focal ladder on the visible
    matches when there are more than 50 of them, retried on all matches when that finds nothing, on all matches
    otherwise -- and the refinement on the RANSAC inliers."""
    S, P = vis.shape
    pe, ie, _, summ = poo.frame_loop(p0, i0, X, uv, vis, np.ones(S, bool), model, shared, 12.0, 100)
    need = np.array([sm["termination"] >= 6 for sm in summ]) | (ie[:, 0] < 0.1 * scale) | (ie[:, 0] > 30 * scale)
    ok = np.zeros(S, bool)
    branch = {}
    for s in np.nonzero(need)[0]:
        enough = vis[s].sum() > 50
        r = pno.absolute_pose_estimation(uv[s], X, ie[s], model, us, True, 12.0, mask=vis[s] if enough else None)
        branch[s] = "visible" if enough else "all"
        if enough and r is None:
            r = pno.absolute_pose_estimation(uv[s], X, ie[s], model, us, True, 12.0)
            branch[s] = "retry"
        if r is None:
            continue
        ok[s] = True
        intr = ie[s].copy()
        if not shared:
            intr[0] = r["focal"]
        pe[s], ie[s], _ = poo.pose_refinement(r["pose"], intr, X, uv[s], r["inliers"], model, not shared, not shared)
    return pe, ie, need, ok, branch


@pytest.mark.parametrize("cam,shared", [("SIMPLE_PINHOLE", False), ("SIMPLE_RADIAL", True)])
def test_force_estimate_branches(cuda_dev, cam, shared):
    """refine_pose(force_estimate=True) against the oracle composition on the same samples (torch.manual_seed, then
    draw_pnp_samples).  Lost frames in every branch: more than 50 visible matches and RANSAC succeeds (frame 2); more
    than 50 visible matches that are all NaN, so RANSAC finds nothing and the retry on all matches succeeds (frame 5);
    40 visible matches, so RANSAC runs on all matches at once (frame 7)."""
    import torch
    from vggsfm_b200 import pose_refinement as pr
    from vggsfm_b200.synthetic import perturb
    S, N = 10, 600
    model = _model(cam)
    sc = make_scene(S, N, cam, seed=101, noise_px=0.3, outlier_frac=0.05)
    extr0, _, _, _ = perturb(sc, rot_deg=0.2, trans_frac=0.005, focal_frac=0.0, seed=102)
    for s in (2, 5, 7):
        a = np.deg2rad(25.0)
        Ry = np.array([[np.cos(a), 0, np.sin(a)], [0, 1, 0], [-np.sin(a), 0, np.cos(a)]])
        extr0[s, :, :3] = Ry @ extr0[s, :, :3]
        extr0[s, :, 3] += np.array([0.8, -0.3, 0.5])
    vis = sc.vis > 0.05
    uv = sc.tracks.copy()
    vis[5] = False
    vis[5, :60] = True
    uv[5, :60] = np.nan
    vis[7] = False
    vis[7, 100:140] = True
    i0 = np.tile(np.array([1000.0, 512.0, 512.0, 0.05 if model else 0.0]), (S, 1))
    K = sc.intrinsics
    ex = to_dev(sc.extra_params, cuda_dev) if sc.extra_params is not None else None
    seed = 11
    torch.manual_seed(seed)
    E, K1, ex1, vmask = pr.refine_pose(to_dev(extr0, cuda_dev), to_dev(K, cuda_dev), ex, to_dev(vis, cuda_dev),
                                       to_dev(sc.points3d, cuda_dev), to_dev(uv, cuda_dev),
                                       torch.ones(N, dtype=torch.bool, device=cuda_dev),
                                       torch.tensor([1024, 1024], device=cuda_dev), shared_camera=shared,
                                       camera_type=cam, force_estimate=True)
    rep = pr.last_report
    torch.manual_seed(seed)
    us = pr.draw_pnp_samples().numpy()
    pe, ie, need, ok, branch = _oracle_force_estimate(extr0, i0, sc.points3d, uv.astype(np.float64), vis, model,
                                                      shared, us)
    assert branch == {2: "visible", 5: "retry", 7: "all"}, branch
    assert np.array_equal(rep.needs_absolute_pose.cpu().numpy(), need)
    assert np.array_equal(rep.absolute_pose_ok.cpu().numpy(), ok) and ok[[2, 5, 7]].all()
    assert bool(vmask.all())
    assert np.abs(E.cpu().numpy() - pe).max() <= 1e-8, np.abs(E.cpu().numpy() - pe).max()
    assert np.allclose(K1.cpu().numpy()[:, 0, 0], ie[:, 0], rtol=1e-9)
    if model == 1:
        assert np.allclose(ex1.cpu().numpy()[:, 0], ie[:, 3], atol=1e-9)
