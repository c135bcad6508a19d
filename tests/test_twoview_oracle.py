"""CPU checks of oracle/twoview_oracle.py (the float64 restatement of vggsfm/two_view_geo) and of the argument checks
of vgg_estimate_fundamental, which run before anything touches a GPU."""
import ctypes
import os

import numpy as np
import pytest

from oracle import twoview_oracle as tvo
from vggsfm_b200.synthetic import make_scene

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")


def _h(p):
    return np.concatenate([p, np.ones(p.shape[:-1] + (1,))], -1)


def test_seven_point_roots_match_numpy_roots():
    """Every real root of det(l f1 + f2) gives a candidate with det 0 through the 7 points; trials with one and with
    three real roots both occur."""
    rng = np.random.default_rng(0)
    a = rng.uniform(0, 1000, (400, 7, 2))
    b = rng.uniform(0, 1000, (400, 7, 2))
    p1n, _ = tvo.normalize_points(a)
    p2n, _ = tvo.normalize_points(b)
    f1, f2 = tvo.null_basis(tvo._design_rows(p1n, p2n))
    F = tvo.run_7point(a, b)
    seen = set()
    for m in range(400):
        A, Bm = f1[m].reshape(3, 3), f2[m].reshape(3, 3)
        # det(l A + B) as a cubic in l, sampled at 4 points
        ls = np.array([-1.0, 0.0, 1.0, 2.0])
        c = np.polyfit(ls, [np.linalg.det(l * A + Bm) for l in ls], 3)
        real = np.sort([r.real for r in np.roots(c) if abs(r.imag) < 1e-9 * max(1, abs(r))])
        seen.add(len(real))
        cand = F[m]
        resid = np.abs(np.einsum("ni,kij,nj->kn", _h(b[m]), cand, _h(a[m])))
        for k in range(len(real)):
            assert resid[k].max() < 1e-6 * np.abs(cand[k]).max() * 1e6
            assert abs(np.linalg.det(cand[k])) < 1e-9 * np.abs(cand[k]).max() ** 3 * 1e6
        if len(real) == 1:                        # the two zero slots are both f2 / f2_22, denormalised
            assert np.allclose(cand[1], cand[2])
    assert {1, 3} <= seen


def test_solve_cubic_lower_order_branches():
    r = tvo.solve_cubic(np.array([[0.0, 0.0, 2.0, -4.0],       # linear: x = 2
                                  [0.0, 1.0, -3.0, 2.0],       # quadratic, two roots
                                  [0.0, 1.0, -2.0, 1.0],       # quadratic, double root
                                  [0.0, 1.0, 0.0, 1.0],        # quadratic, no real root
                                  [0.0, 0.0, 0.0, 5.0],        # zero order: unsolved
                                  [1.0, -6.0, 11.0, -6.0],     # three real roots 1 2 3
                                  [1.0, 0.0, 0.0, -8.0],       # one real root (Q = 0, R != 0): 2
                                  [1.0, -3.0, 3.0, -1.0]]))    # triple root 1
    assert np.allclose(r[0], [2, 0, 0]) and np.allclose(sorted(r[1][:2]), [1, 2]) and r[1][2] == 0
    assert np.allclose(r[2], [1, 1, 0]) and np.all(r[3] == 0) and np.all(r[4] == 0)
    assert np.allclose(sorted(r[5]), [1, 2, 3]) and np.allclose(r[6], [2, 0, 0]) and np.allclose(r[7], [1, 1, 1])


def test_eight_point_exact_on_noise_free_data():
    rng = np.random.default_rng(1)
    X = rng.normal(size=(50, 3)) + np.array([0, 0, 5.0])
    R = np.array([[np.cos(0.3), 0, np.sin(0.3)], [0, 1, 0], [-np.sin(0.3), 0, np.cos(0.3)]])
    t = np.array([-1.0, 0.2, 0.1])
    x1 = X[:, :2] / X[:, 2:] * 800 + 400
    Y = X @ R.T + t
    x2 = Y[:, :2] / Y[:, 2:] * 800 + 400
    F = tvo.run_8point(x1[None], x2[None], np.ones((1, 50), bool))[0]
    K = np.array([[800, 0, 400], [0, 800, 400], [0, 0, 1.0]])
    tx = np.array([[0, -t[2], t[1]], [t[2], 0, -t[0]], [-t[1], t[0], 0]])
    Fg = np.linalg.inv(K).T @ tx @ R @ np.linalg.inv(K)
    Fg = Fg / Fg[2, 2]
    assert np.abs(F / F[2, 2] - Fg).max() < 1e-9 * np.abs(Fg).max()
    assert tvo.sampson(x1, x2, F[None])[0].max() < 1e-10                               # px^2


def test_oracle_recovers_synthetic_epipolar_geometry():
    sc = make_scene(4, 300, seed=2, noise_px=0.0)
    np.random.seed(0)
    smp = tvo.generate_samples(300, 64)
    p1 = np.broadcast_to(sc.tracks[:1], (3, 300, 2))
    r = tvo.estimate_fundamental(p1, sc.tracks[1:], smp, max_error=1.0, lo_num=10)
    assert (r["inlier_num"] == 300).all()
    R, t, _, _ = tvo.relative_pose(r["fmat"], p1, sc.tracks[1:], 1024, 1024)
    for b in range(3):
        Rg, tg = sc.extrinsics[b + 1, :, :3], sc.extrinsics[b + 1, :, 3]
        # the default intrinsics (f = max(W, H) = 1024 against the scene's 1000 px) cost a fraction of a degree
        assert np.degrees(np.arccos(np.clip((np.trace(R[b].T @ Rg) - 1) / 2, -1, 1))) < 1.0
        assert np.abs(t[b] - tg / np.linalg.norm(tg)).max() < 1e-3


def test_generate_samples_raises_when_too_few_distinct_draws():
    np.random.seed(0)
    with pytest.raises(ValueError, match="duplicate-free"):
        tvo.generate_samples(7, 64)
    from vggsfm_b200 import two_view as tv
    np.random.seed(0)
    with pytest.raises(ValueError, match="duplicate-free"):
        tv.generate_samples(8, 100, 7)
    np.random.seed(3)
    a = tvo.generate_samples(500, 32)
    np.random.seed(3)
    assert np.array_equal(a, tv.generate_samples(500, 32, 7))


@pytest.mark.parametrize("name", sorted(f for f in os.listdir(GOLDEN) if f.startswith("twoview_")))
def test_oracle_matches_reference_golden(name):
    """tools/make_golden_twoview.py: the unmodified reference on float32 tracks, with its sample draws recorded.
    Counts and masks exact on every pair; F at the float32 level of the reference on the live pairs.  The relative
    pose and the residuals are checked on the reference's own F, which pins the decomposition, its orientation and the
    cheirality vote.  Candidate indices are not compared: the order of the three real roots of a trial follows the
    parameterisation of the null space, i.e. the basis (DESIGN.md section 3), and so does the dead pair's matrix."""
    g = np.load(os.path.join(GOLDEN, name))
    r = tvo.estimate_fundamental(g["points1"], g["points2"], g["samples"], max_error=float(g["max_error"]),
                                 lo_num=int(g["lo_num"]), valid_mask=g["valid"])
    assert np.array_equal(r["inlier_num"], g["inlier_num"])
    assert np.array_equal(r["inlier_mask"], g["inlier_mask"])
    live = g["inlier_num"] > 0
    assert live.sum() == len(live) - 1
    F, Fg = r["fmat"][live], g["fmat"][live]
    rel = np.abs(F - Fg).reshape(len(F), -1).max(-1) / np.abs(Fg).reshape(len(F), -1).max(-1)
    assert rel.max() < 2e-4, rel
    R, t, _, _ = tvo.relative_pose(g["fmat"].astype(np.float64), g["points1"], g["points2"], int(g["width"]),
                                   int(g["height"]))
    assert np.abs(R[live] - g["R"][live]).max() < 1e-5 and np.abs(t[live] - g["t"][live]).max() < 1e-5
    thr = float(g["max_error"]) ** 2
    for b in np.nonzero(live)[0]:
        res = tvo.sampson(g["points1"][b].astype(np.float64), g["points2"][b].astype(np.float64),
                          g["fmat"][b][None].astype(np.float64))[0]
        res = np.where(g["valid"][b], res, 1e6)
        assert np.all(np.abs(res - g["residuals"][b]) <= 1e-3 * np.maximum(res, thr))


def test_einval_before_launch():
    """Bad sizes and out-of-range samples return VGG_EINVAL before any CUDA call (host buffers suffice)."""
    from vggsfm_b200 import _lib
    L = _lib.lib()
    B, N, T = 2, 16, 8
    p = np.zeros((B, N, 2), np.float32)
    outs = [np.zeros((B, 9)), np.zeros(B, np.int32), np.zeros((B, N), np.uint8), np.zeros((B, N))]
    ws = np.zeros(1 << 20, np.uint8)

    def call(n=N, t=T, lo=4, smp=None):
        s = np.zeros((t, 7), np.int32) if smp is None else smp
        return L.vgg_estimate_fundamental(B, n, p.ctypes.data, p.ctypes.data, 0, None, s.ctypes.data, t, lo, 4.0, 1, 1,
                                          *[o.ctypes.data for o in outs], ws.ctypes.data, ws.nbytes, None)
    assert call(lo=3 * T + 1) == -1 and b"lo_num" in L.vgg_last_error()
    assert call(lo=0) == -1
    assert call(t=6) == -1 and call(n=6) == -1
    bad = np.tile(np.arange(7, dtype=np.int32), (T, 1))
    bad[3, 2] = N
    assert call(smp=bad) == -1 and b"sample" in L.vgg_last_error()
    bad[3, 2] = -1
    assert call(smp=bad) == -1
    nb = ctypes.c_size_t()
    assert L.vgg_twoview_workspace_bytes(400, 4096, 4096, 300, ctypes.byref(nb)) == 0 and nb.value < 200 * 2 ** 20


_W = np.array([[0.0, -1.0, 0.0], [1.0, 0.0, 0.0], [0.0, 0.0, 1.0]])


def _pinned_candidates(U, V):
    """The four (R, t) of decompose_essential_matrix from rotations U, V, with its orientation pin."""
    t = U[:, 2]
    if t[np.argmax(np.abs(t))] < 0:
        P = np.array([-1.0, 1.0, -1.0])
        U, V = U * P, V * P
    R1, R2, T = U @ _W @ V.T, U @ _W.T @ V.T, U[:, 2]
    return np.stack([R1, R1, R2, R2]), np.stack([T, -T, T, -T])


def _normal_matrix_route(E):
    """Float64 restatement of the decomposition through E^T E that tv_pose_kernel used before it moved to one-sided
    Jacobi: V = eigenvectors of E^T E (descending), u_i = E v_i / |E v_i|, u1 re-orthogonalised, u2 = u0 x u1."""
    w, Wv = np.linalg.eigh(E.T @ E)
    V = Wv[:, np.argsort(-w, kind="stable")]
    u0, u1 = (E @ V[:, i] for i in range(2))
    u0, u1 = u0 / np.linalg.norm(u0), u1 / np.linalg.norm(u1)
    u1 = u1 - (u0 @ u1) * u0
    u1 = u1 / np.linalg.norm(u1)
    if np.linalg.det(V) < 0:
        V[:, 2] = -V[:, 2]
    return _pinned_candidates(np.stack([u0, u1, np.cross(u0, u1)], 1), V)


@pytest.mark.parametrize("r", [1.0, 1 - 1e-12, 1e-2, 1e-4, 1e-6, 1e-8])
def test_singular_value_generator_plants_what_it_claims(r):
    rng = np.random.default_rng(int(-np.log10(r)) if r < 1 else 99)
    for width, height in ((1024, 1024), (1920, 1080), (480, 640)):
        F, E, U, V = tvo.fundamental_with_singular_values((1.0, r, 0.0), width, height, rng)
        assert np.linalg.det(U) > 0 and np.linalg.det(V) > 0
        assert np.abs(U.T @ U - np.eye(3)).max() < 1e-15 and np.abs(V.T @ V - np.eye(3)).max() < 1e-15
        K = tvo.default_kmat(width, height)
        Ek = K.T @ F @ K
        assert np.abs(Ek - E).max() < 1e-13
        s = np.linalg.svd(Ek, compute_uv=False)
        assert abs(s[0] - 1) < 1e-14 and abs(s[1] - r) < 1e-14 and s[2] < 1e-14
        Rs, ts = _pinned_candidates(U, V)
        for R in Rs:
            assert np.abs(R.T @ R - np.eye(3)).max() < 1e-14 and abs(np.linalg.det(R) - 1) < 1e-14
        assert np.abs(Ek.T @ ts[0]).max() < 1e-14            # t spans the left null space


@pytest.mark.parametrize("r", [1.0, 1 - 1e-12, 1e-2, 1e-4, 1e-6, 1e-8])
def test_pose_bar_passes_lapack_and_rejects_the_normal_matrix_route(r):
    """LAPACK's decomposition of K^T F K stays inside pose_bar around the planted candidates (all four, in order: the
    determinant fixes and the orientation pin make the order canonical); the E^T E route of the old kernel leaves it
    at sigma_2 / sigma_1 <= 1e-4 on every draw."""
    rng = np.random.default_rng(7)
    worst_lapack, best_normal = 0.0, np.inf
    for _ in range(12):
        F, E, U, V = tvo.fundamental_with_singular_values((1.0, r, 0.0), 1024, 768, rng)
        K = tvo.default_kmat(1024, 768)
        Ek = K.T @ F @ K
        bar = tvo.pose_bar(np.linalg.svd(Ek, compute_uv=False))
        Rp, tp = _pinned_candidates(U, V)
        Rs, ts = tvo.decompose_essential_matrix(Ek[None])
        worst_lapack = max(worst_lapack, max(np.abs(Rs[0] - Rp).max(), np.abs(ts[0] - tp).max()) / bar)
        Rn, tn = _normal_matrix_route(Ek)
        best_normal = min(best_normal, max(np.abs(Rn - Rp).max(), np.abs(tn - tp).max()) / bar)
    assert worst_lapack <= 0.25, worst_lapack
    if r <= 1e-4:
        assert best_normal > 1.0, best_normal


def test_pose_bar_is_inf_at_rank_one():
    assert tvo.pose_bar([1.0, 0.0, 0.0]) == np.inf
    assert tvo.pose_bar([2.0, 1e-3, 0.0]) == pytest.approx(96 * 2.0 ** -52 * 2e3)


def test_lapack_basis_of_rank_deficient_e():
    """What the oracle decomposes F = 0 and a rank-1 F into: F = 0 gives U = V = I, so R = W, W^T and t = e2; a rank-1
    E = a b^T gives rotations with t orthogonal to a (LAPACK's completion of the basis, not unique)."""
    Rs, ts = tvo.decompose_essential_matrix(np.zeros((1, 3, 3)))
    assert np.array_equal(Rs[0, 0], _W) and np.array_equal(Rs[0, 2], _W.T) and np.array_equal(ts[0, 0], [0, 0, 1])
    a, b = np.array([0.3, -0.5, 0.8]), np.array([1.0, 0.2, -0.4])
    Rs, ts = tvo.decompose_essential_matrix(np.outer(a, b)[None])
    for R in Rs[0]:
        assert np.isfinite(R).all() and np.abs(R.T @ R - np.eye(3)).max() < 1e-14 and abs(np.linalg.det(R) - 1) < 1e-14
    assert abs(ts[0, 0] @ a) < 1e-14 and abs(np.linalg.norm(ts[0, 0]) - 1) < 1e-14


def test_cheirality_margin_fields_on_a_hand_built_pair():
    """R = I, t = (1, 0, 0): window 1000.  Points at depth 2, 500 and 999.5 -> margins 0.998, 0.5, 5e-4; a point
    behind both cameras at -3 is not counted and its margin is (3 + eps32) / 1000 + 1 against the window, far larger."""
    R, t = np.eye(3), np.array([1.0, 0.0, 0.0])
    X = np.array([[0.1, 0.2, 2.0], [0.5, -0.3, 500.0], [1.0, 1.0, 999.5], [0.2, 0.1, -3.0]])
    Y = X @ R.T + t
    x1, x2 = X[:, :2] / X[:, 2:], Y[:, :2] / Y[:, 2:]
    for n, want_cnt, want_margin in ((1, 1, 0.998), (2, 2, 0.5), (3, 3, 5e-4), (4, 3, 5e-4)):
        cnt, margin = tvo.cheirality_counts(R, t, x1[:n], x2[:n], return_margin=True)
        assert cnt == want_cnt and margin == pytest.approx(want_margin, rel=1e-9), (n, cnt, margin)
    assert tvo.cheirality_counts(R, t, x1, x2) == 3
    # the relative pose of the same pair in pixels: the winner has every point in front, count_gap against the others
    f, w, h = 1000.0, 1000, 800
    K = tvo.default_kmat(w, h)
    Ki = np.linalg.inv(K)
    tx = np.array([[0, -t[2], t[1]], [t[2], 0, -t[0]], [-t[1], t[0], 0]])
    F = (Ki.T @ tx @ R @ Ki)[None]
    p1 = (x1 * f + [w / 2, h / 2])[None]
    p2 = (x2 * f + [w / 2, h / 2])[None]
    Rr, tr, _, counts, dbg = tvo.relative_pose(F, p1, p2, w, h, return_debug=True)
    d = dbg[0]
    assert d["k"] == int(np.argmax(counts[0])) and counts[0, d["k"]] == 3
    assert np.abs(Rr[0] - np.eye(3)).max() < 1e-12 and np.abs(tr[0] - t).max() < 1e-12
    others = [counts[0, j] for j in range(4) if j != d["k"]]
    assert d["count_gap"] == 3 - max(others)
    assert d["depth_margin"] <= 5e-4 * (1 + 1e-9) and np.allclose(d["sigma"], [1, 1, 0], atol=1e-12)


def test_mirror_refuses_cpu_tensors():
    import torch
    from vggsfm_b200 import two_view as tv
    with pytest.raises(RuntimeError, match="no CPU fallback"):
        tv.estimate_fundamental(torch.zeros(1, 16, 2), torch.zeros(1, 16, 2))
    with pytest.raises(RuntimeError, match="no CPU fallback"):
        tv.estimate_preliminary_cameras(torch.zeros(1, 3, 16, 2), torch.ones(1, 3, 16), 64, 64)
