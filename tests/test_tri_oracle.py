"""CPU: the triangulation oracle (oracle/tri_oracle.py) against the committed golden fixtures produced by
the reference itself (tools/make_golden.py, tools/make_golden_live.py)."""
import glob
import os

import numpy as np
import pytest

from oracle import tri_oracle as to

GOLDEN = sorted(glob.glob(os.path.join(os.path.dirname(__file__), "golden", "tri_*.npz")))


def load(path):
    g = dict(np.load(path))
    g["extra"] = g["extra_params"] if g["extra_params"].shape[0] else None
    return g


@pytest.mark.parametrize("path", GOLDEN, ids=[os.path.basename(p)[:-4] for p in GOLDEN])
def test_oracle_matches_reference_golden(path):
    g = load(path)
    tn = to.cam_from_img(g["tracks"].astype(np.float64), g["intrinsics"], g["extra"])
    assert np.abs(tn - g["tn"]).max() < 1e-12          # same iteration, same global stop
    pts, num, mask = to.triangulate_tracks(g["extrinsics"], g["tn"], g["pairs"], g["vis"], g["score"])
    if bool(g["pinned"]):
        assert np.array_equal(num, g["inlier_num"])
        assert np.array_equal(mask, g["inlier_mask"])
        assert np.abs(pts - g["points"]).max() <= 1e-9 * np.abs(g["points"]).max()
    else:
        # reference run with its unstable sort: tie order may differ, the outcome must still agree
        same = (num == g["inlier_num"])
        assert same.mean() >= 0.95
        close = np.linalg.norm(pts - g["points"], axis=1) <= 1e-3
        assert close.mean() >= 0.95
    v, d = to.filter_all_points3D(g["points"], g["tracks"].astype(np.float64), g["extrinsics"], g["intrinsics"],
                                  g["extra"], max_reproj_error=1.0, return_detail=True)
    assert np.array_equal(v, g["filt_valid"]) and np.array_equal(d, g["filt_detail"])
    v2, _ = to.filter_all_points3D(g["points"], g["tracks"].astype(np.float64), g["extrinsics"], g["intrinsics"],
                                   g["extra"], max_reproj_error=4.0, check_triangle=False)
    assert np.array_equal(v2, g["filt_valid_notri"])
    p2d, pcam = to.project_3D_points(g["points"], g["extrinsics"], g["intrinsics"], g["extra"])
    assert np.abs(p2d - g["proj2d"]).max() < 1e-8 and np.abs(pcam - g["projcam"]).max() < 1e-10
    bp, bche, bang = to.triangulate_by_pair(g["extrinsics"], g["tn"])
    assert np.array_equal(bche, g["pair_cheirality"])
    assert np.nanmax(np.abs(bp - g["pair_points"]) / (1 + np.abs(g["pair_points"]))) < 1e-7
    assert np.nanmax(np.abs(bang - g["pair_angle"])) < 1e-7


def test_oracle_matches_live_reference():
    """The reference's triangulate_tracks (stable sort, torch seed 3) on a 10 x 40 scene, stored by
    tools/make_golden_live.py; the oracle draws the same pairs from the same seed."""
    import torch
    from vggsfm_b200.synthetic import make_scene
    g = np.load(os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "reference_triangulate_10x40.npz"))
    sc = make_scene(10, 40, "SIMPLE_RADIAL", seed=21, invisible_frac=0.2, outlier_frac=0.1)
    torch.manual_seed(3)
    pairs = to.draw_pairs(10, 256)
    po, no, mo = to.triangulate_tracks(sc.extrinsics, g["tn"], pairs, sc.vis, sc.score)
    assert np.array_equal(no, g["num"]) and np.array_equal(mo, g["mask"])
    assert np.abs(po - g["points"]).max() < 1e-9


def test_oracle_matches_reference_edges():
    """tools/make_golden.py's edge fixture: slow undistortion (11, 47, 80 and 100 iterations, one call per k and one
    call mixing k) and a pinned triangulation with max_angular_error = 8 degrees."""
    g = np.load(os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "edges_undistort_gate8.npz"))
    assert list(g["und_iters"]) == [11, 47, 80, 100] and int(g["und_iters_mixed"]) == 80
    for c in range(len(g["und_k"])):
        tn_d = (g["und_uv"][c:c + 1].astype(np.float64) - 512.0) / 1000.0
        und, iters = to.iterative_undistortion(g["und_k"][c], tn_d)
        assert iters == g["und_iters"][c]
        assert np.abs(und - g["und_tn"][c]).max() < 1e-12
        tn = to.cam_from_img(g["und_uv"][c:c + 1].astype(np.float64), g["und_intrinsics"][c:c + 1], g["und_k"][c:c + 1])
        assert np.abs(tn - g["und_tn"][c]).max() < 1e-12
    C = len(g["und_tn_mixed"])
    tn_d = (g["und_uv"][:C].astype(np.float64) - 512.0) / 1000.0
    und, iters = to.iterative_undistortion(g["und_k"][:C, 0], tn_d)
    assert iters == int(g["und_iters_mixed"]) and np.abs(und - g["und_tn_mixed"]).max() < 1e-12
    tn = to.cam_from_img(g["tracks"].astype(np.float64), g["intrinsics"], g["extra_params"])
    assert np.abs(tn - g["tn"]).max() < 1e-12
    pts, num, mask = to.triangulate_tracks(g["extrinsics"], g["tn"], g["pairs"], g["vis"], g["score"],
                                           max_angular_error=float(g["max_angular_error"]))
    assert np.array_equal(num, g["inlier_num"]) and np.array_equal(mask, g["inlier_mask"])
    assert np.abs(pts - g["points"]).max() <= 1e-9 * np.abs(g["points"]).max()
    # the wide gate matters: at the default 2 degrees the same tracks keep fewer inliers
    _, num2, _ = to.triangulate_tracks(g["extrinsics"], g["tn"], g["pairs"], g["vis"], g["score"])
    assert num2.sum() < num.sum()


def _arc_centers(S, seed):
    rng = np.random.default_rng(seed)
    i = np.arange(S) / S
    return np.stack([-2.0 * i, 0.05 * rng.normal(size=S), 0.1 * np.sin(3 * i)], -1)


@pytest.mark.parametrize("S", [2, 3, 31, 64, 401])
def test_any_pair_search_equals_exhaustive(S):
    """The wide-first, early-exit search gives the exhaustive S x S answer, with and without an inlier mask, on random
    points and on the inputs where the answer is False and the whole search runs."""
    rng = np.random.default_rng(S)
    C = _arc_centers(S, S)
    X = np.concatenate([
        rng.normal(size=(40, 3)) * 0.5 + [0, 0, 4],          # ordinary points: mostly True
        rng.normal(size=(6, 3)) * 0.5 + [0, 0, 4e5],         # very distant: every pair far below the minimum
        C[rng.integers(0, S, 4)],                            # at a camera centre
        [[np.nan, 0, 4], [0, np.inf, 4], [np.nan] * 3],      # NaN / inf coordinates
    ])
    inl = rng.uniform(size=(S, len(X))) < 0.3
    for min_deg in (1.5, 10.0, 0.0):
        for mask in (None, inl):
            fast, best = to.any_pair_tri_angle(C, X, min_deg, mask, return_best=True)
            ref = to.any_pair_tri_angle_exhaustive(C, X, min_deg, mask)
            assert np.array_equal(fast, ref), (min_deg, mask is None)
            assert np.array_equal(fast, best >= min_deg)
        if min_deg > 0:
            assert not ref[40:46].any() and not ref[-3:].any()   # distant and NaN points: False after a full search
    # pure rotation: every centre equal; and a point at the end of a line of collinear centres
    same = np.zeros((S, 3))
    line = np.stack([np.arange(S, dtype=np.float64), np.zeros(S), np.zeros(S)], -1)
    for C2, X2 in ((same, X), (line, np.concatenate([line[:1], line[-1:], [[-5.0, 0, 0]]]))):
        fast = to.any_pair_tri_angle(C2, X2, 1.5)
        assert np.array_equal(fast, to.any_pair_tri_angle_exhaustive(C2, X2, 1.5)) and not fast.any()


def test_any_pair_search_best_angle_is_exact_near_the_minimum():
    """Within `margin` above min_deg the search keeps going, so the best pair angle it reports there is the maximum
    over every pair (the triangulation oracle's near-tie information relies on this)."""
    S = 50
    C = _arc_centers(S, 1)
    rng = np.random.default_rng(2)
    X = rng.normal(size=(64, 3)) * 0.5 + [0, 0, 4]
    full = np.array([max(to.tri_angle_deg(C[a], C[b], x) for a in range(S) for b in range(S)) for x in X])
    min_deg = float(np.median(full))
    _, best = to.any_pair_tri_angle(C, X, min_deg, margin=1.0, return_best=True)
    near = full < min_deg + 1.0
    assert near.any() and (~near).any()
    assert np.array_equal(best[near], full[near])
    assert (best[~near] >= min_deg + 1.0).all()


def test_triangulation_debug_reports_near_ties():
    """return_debug's near-tie fields are consistent with the returned scores, errors and angles."""
    import torch
    from vggsfm_b200.synthetic import make_scene
    sc = make_scene(12, 48, "SIMPLE_PINHOLE", seed=4, invisible_frac=0.2, outlier_frac=0.1)
    tn = to.cam_from_img(sc.tracks.astype(np.float64), sc.intrinsics)
    torch.manual_seed(1)
    pairs = to.draw_pairs(12, 40)
    thr = np.deg2rad(2.0)
    pts, num, mask, d = to.triangulate_tracks(sc.extrinsics, tn, pairs, sc.vis, sc.score, return_debug=True)
    ar = np.arange(48)
    assert np.array_equal(d["gate_dist"], np.abs(d["allE"][ar, d["best"]] - thr))
    assert (d["gate_dist_min"] <= d["gate_dist"].min(axis=1)).all()
    assert (d["score_margin"] >= 0).all()
    s = d["score"].copy()
    s[ar, d["best"]] = -np.inf
    assert (d["score_margin"] >= d["score"][ar, d["best"]] - s.max(axis=1)).all()
    lo = min(50, len(pairs))
    assert d["tri_dist"].shape == (48, lo + 10) and d["tri_dist0"].shape == (48, len(pairs))
    C = to.proj_centers(sc.extrinsics)
    for n in range(0, 48, 7):                 # the sign of tri_dist is the exhaustive angle test
        for j in range(lo + 10):
            x = d["allX"][n, len(pairs) + j]
            ok = to.any_pair_tri_angle_exhaustive(C, x[None], 1.5)[0]
            assert ok == (d["tri_dist"][n, j] >= 0)


def test_undistortion_quirk_is_reproduced():
    """SURVEY Appendix A.3: the reference's damped Newton stops ~4e-6 short of the true undistortion."""
    from vggsfm_b200.synthetic import make_scene
    sc = make_scene(4, 50, "SIMPLE_RADIAL", seed=5)
    k = sc.extra_params[:, 0]
    tn_d = (sc.tracks.astype(np.float64) - 512.0) / 1000.0
    und, iters = to.iterative_undistortion(k, tn_d)
    u, v = to.apply_distortion(k, und[..., 0], und[..., 1])
    err = np.abs(np.stack([u, v], -1) - tn_d).max()
    assert 2 <= iters < 100 and err < 1e-4
