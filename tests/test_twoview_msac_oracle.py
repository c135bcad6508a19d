"""CPU checks of oracle/poselib_oracle.py, the float64 restatement of poselib.estimate_fundamental that
csrc/twoview_msac.cu is held to: recovery on synthetic pairs with gross outliers, the stopping rule, the real focal
check, the LM, the sampler and the small-count edges."""
import numpy as np
import pytest

from oracle import poselib_oracle as po
from vggsfm_b200.synthetic import make_scene


def _skew(t):
    return np.array([[0.0, -t[2], t[1]], [t[2], 0.0, -t[0]], [-t[1], t[0], 0.0]])


def _gt_fmat(sc, s):
    R = sc.extrinsics[s, :, :3] @ sc.extrinsics[0, :, :3].T
    t = sc.extrinsics[s, :, 3] - R @ sc.extrinsics[0, :, 3]
    Ki = np.linalg.inv(sc.intrinsics[0])
    return Ki.T @ _skew(t) @ R @ Ki


def _clean_pair(N, seed, noise_px=0.0):
    sc = make_scene(2, N, seed=seed, noise_px=noise_px)
    return sc, sc.tracks[0].astype(np.float64), sc.tracks[1].astype(np.float64)


def test_recovers_inliers_and_rejects_planted_outliers():
    sc = make_scene(2, 2000, seed=5, noise_px=0.3, outlier_frac=0.2)
    from vggsfm_b200.synthetic import project_np
    uv, _ = project_np(sc.extrinsics, 1000.0, np.array([512.0, 512.0]), 0.0, sc.points3d)
    clean = (np.linalg.norm(sc.tracks - uv, axis=-1) < 3.0).all(0)
    # the ground-truth correspondences satisfy the ground-truth F
    G = _gt_fmat(sc, 1)
    r2 = po.sampson_sq(G, uv[0], uv[1])
    assert r2.max() < 1e-16
    F, mask, it = po.estimate_fundamental_pair(sc.tracks[0], sc.tracks[1], 1.0, 20000)
    assert (mask & clean).sum() >= 0.95 * clean.sum(), ((mask & clean).sum(), clean.sum())
    assert (mask & ~clean).sum() <= 0.01 * (~clean).sum() + 1
    assert abs(np.linalg.norm(F) - 1.0) < 1e-12
    Gn = G / np.linalg.norm(G)
    assert min(np.abs(F - Gn).max(), np.abs(F + Gn).max()) < 2e-3


def test_stop_counts():
    sc, x1, x2 = _clean_pair(300, 1, noise_px=0.1)
    d = po._new_debug()
    _, m, it = po.estimate_fundamental_pair(x1, x2, 1.0, 5000, 200, 0, d)
    assert m.all() and it == 201                                   # all inliers: min_iterations + 1
    _, m, it = po.estimate_fundamental_pair(x1, x2, 1.0, 150, 200, 0)
    assert it == 150                                               # max_iterations < min_iterations
    rng = np.random.default_rng(2)
    noise = rng.uniform(0, 1024, size=(300, 2))
    d = po._new_debug()
    _, m, it = po.estimate_fundamental_pair(x1, noise, 0.5, 400, 100, 0, d)
    assert it == 400, d["dyn"]                                     # pure noise: max_iterations
    x2b = x2.copy()
    bad = rng.uniform(size=300) < 0.4
    x2b[bad] = rng.uniform(0, 1024, size=(int(bad.sum()), 2))
    d = po._new_debug()
    _, m, it = po.estimate_fundamental_pair(x1, x2b, 1.0, 5000, 100, 0, d)
    last_it, cnt, dyn = d["dyn"][-1]
    assert dyn == po.dynamic_max_iter(cnt, 300, 100, 5000)[0]
    assert dyn == int(np.ceil(np.log(1 - 0.9999) / np.log(1 - (cnt / 300) ** 7)))
    assert it == max(100, dyn) + 1 and 101 < it < 5000, (it, dyn)


def test_real_focal_check():
    R = po.rodrigues(np.array([0.1, 0.3, -0.05]))
    t = np.array([1.0, 0.2, 0.1])
    K1, K2 = np.diag([2.0, 2.0, 1.0]), np.diag([3.0, 3.0, 1.0])
    F = np.linalg.inv(K2).T @ _skew(t) @ R @ np.linalg.inv(K1)
    keep, _, (f1, f2) = po.real_focal_check(F)
    assert keep and abs(f1 - 4.0) < 1e-9 and abs(f2 - 9.0) < 1e-9
    # the check reads the same Bougnoux values: a rank-2 matrix whose f1^2 or f2^2 comes out negative is dropped
    rng = np.random.default_rng(0)
    seen = 0
    for _ in range(200):
        U, S, Vt = np.linalg.svd(rng.normal(size=(3, 3)))
        M = U @ np.diag([S[0], S[1], 0.0]) @ Vt
        keep, _, (g1, g2) = po.real_focal_check(M)
        assert keep == (g1 >= 0 and g2 >= 0), (g1, g2)
        seen += not keep
    assert 0 < seen < 200
    assert not po.real_focal_check(np.full((3, 3), np.nan))[0]


def test_lm_never_increases_cost_and_converges_on_exact_inliers():
    sc, x1, x2 = _clean_pair(400, 7)
    s = po.shared_scale(x1, x2)
    y1, y2 = x1 / s, x2 / s
    G = _gt_fmat(sc, 1)
    G = G * np.array([s, s, 1.0])[:, None] * np.array([s, s, 1.0])[None]      # into the scaled frame
    rng = np.random.default_rng(3)
    F0 = G / np.linalg.norm(G) + rng.normal(size=(3, 3)) * 2e-4
    U, S, Vt = np.linalg.svd(F0)
    F0 = U @ np.diag([S[0], S[1], 0.0]) @ Vt
    for loss, c2, iters in (("truncated", (4.0 / s) ** 2, 25), ("cauchy", (1.0 / s) ** 2, 100)):
        d = po._lm_dbg()
        F = po.lm_refine(F0, y1, y2, loss, c2, iters, d)
        costs = d["costs"][0]
        assert all(b <= a for a, b in zip(costs, costs[1:]))
        Fn, Gn = F / np.linalg.norm(F), G / np.linalg.norm(G)
        assert min(np.abs(Fn - Gn).max(), np.abs(Fn + Gn).max()) < 1e-7, loss
        assert po.sampson_sq(F, y1, y2).max() < 1e-12


def test_sampler():
    a = po.RandomSampler(9, seed=0)
    b = po.RandomSampler(9, seed=0)
    for _ in range(500):
        s = a.sample()
        assert len(set(s)) == 7 and min(s) >= 0 and max(s) < 9
        assert s == b.sample()
    c = po.RandomSampler(9, seed=1)
    assert [c.sample() for _ in range(3)] != [po.RandomSampler(9, 0).sample() for _ in range(3)]
    st = 0
    first = []
    for _ in range(3):
        st = (st * 1103515245 + 12345) % (1 << 31)
        first.append(st % 1000)
    assert po.RandomSampler(1000, 0).sample()[:3] == first


@pytest.mark.parametrize("n", [0, 6])
def test_fewer_than_seven(n):
    sc, x1, x2 = _clean_pair(10, 3)
    F, m, it = po.estimate_fundamental_pair(x1[:n], x2[:n], 1.0, 100, 10)
    assert not F.any() and m.shape == (n,) and not m.any() and it == 0


@pytest.mark.parametrize("n,scene,polished", [(7, 17, False), (8, 25, True)])
def test_seven_and_eight_inliers_around_the_polish(n, scene, polished):
    # noise-free scenes whose true minimal models pass the real focal check (with the principal point at the image
    # corner, most seven-match scenes of this camera have no candidate that does, and then there is no model)
    sc, x1, x2 = _clean_pair(n, scene)
    d = po._new_debug()
    F, m, it = po.estimate_fundamental_pair(x1, x2, 1.0, 300, 100, 0, d)
    assert m.sum() == n and d["num"] == n and d["polished"] is polished and it == 101
    assert abs(np.linalg.norm(F) - 1.0) < 1e-12


def test_batch_quirk_uses_batch_zero_query():
    a = make_scene(3, 200, seed=1)
    b = make_scene(3, 200, seed=2)
    tracks = np.stack([a.tracks, b.tracks])
    vis = np.stack([a.vis, b.vis])
    out = po.estimate_preliminary_cameras_poselib(tracks, vis, 1024, 1024, max_error=1.0, max_ransac_iters=300,
                                                  min_iterations=50, pairs=[2])
    ref = po.estimate_fundamental_msac(tracks[0, :1], tracks[1, 1:2], vis[1, 1:2] >= 0.05, 1.0, 300, 50)
    assert np.array_equal(out["inlier_mask"], ref["inlier_mask"]) and np.allclose(out["fmat"], ref["fmat"])
