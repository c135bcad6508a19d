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


def test_mirror_refuses_cpu_tensors():
    import torch
    from vggsfm_b200 import two_view as tv
    with pytest.raises(RuntimeError, match="no CPU fallback"):
        tv.estimate_fundamental(torch.zeros(1, 16, 2), torch.zeros(1, 16, 2))
    with pytest.raises(RuntimeError, match="no CPU fallback"):
        tv.estimate_preliminary_cameras(torch.zeros(1, 3, 16, 2), torch.ones(1, 3, 16), 64, 64)
