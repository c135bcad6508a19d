"""oracle/pnp_oracle.py (P3P + LO-RANSAC absolute pose, the restatement behind the refine_pose fall-back,
vggsfm/utils/triangulation.py:404-433): the P3P solver returns the true pose among its solutions, the quartic solver
agrees with numpy.roots, and the estimator recovers pose and focal length on scenes with gross outliers.  CPU only."""
import numpy as np
import pytest

from oracle import pnp_oracle as po
from tests.helpers import rotation_angle_deg
from vggsfm_b200.synthetic import make_scene


def test_quartic_matches_numpy_roots():
    rng = np.random.default_rng(0)
    for _ in range(200):
        c = rng.normal(size=5)
        if rng.uniform() < 0.2:
            c[3] = 0.0                                     # near-biquadratic after depression happens for symmetric inputs
        ref = np.roots(c)
        ref = np.sort(ref[np.abs(ref.imag) < 1e-9 * (1 + np.abs(ref.real))].real)
        got = np.sort(np.array(po.solve_quartic_real(*c)))
        # every well-separated real root is found
        for r in ref:
            others = ref[np.abs(ref - r) > 0]
            if len(others) and np.min(np.abs(others - r)) < 1e-4:
                continue
            assert len(got) and np.min(np.abs(got - r)) <= 1e-8 * (1 + abs(r)), (c, ref, got)


def test_p3p_contains_true_pose():
    rng = np.random.default_rng(1)
    sc = make_scene(6, 64, "SIMPLE_PINHOLE", seed=1, noise_px=0.0)
    for trial in range(100):
        s = rng.integers(0, 6)
        idx = rng.choice(64, 3, replace=False)
        E = sc.extrinsics[s]
        p = sc.points3d[idx] @ E[:, :3].T + E[:, 3]
        f = p / np.linalg.norm(p, axis=1, keepdims=True)
        sols = po.p3p(f, sc.points3d[idx])
        assert sols, trial
        err = min(np.abs(P - E).max() for P in sols)
        assert err < 1e-5, (trial, err)           # closed-form quartic: conditioning-limited; RANSAC refines locally


@pytest.mark.parametrize("cam,est_f", [("SIMPLE_PINHOLE", False), ("SIMPLE_RADIAL", False), ("SIMPLE_PINHOLE", True)])
def test_recovers_pose_with_outliers(cam, est_f):
    sc = make_scene(4, 300, cam, seed=5, noise_px=0.3, outlier_frac=0.3)
    rng = np.random.default_rng(2)
    us = rng.uniform(size=(64, 3))
    s = 2
    f_true, k = 1000.0, (0.05 if cam == "SIMPLE_RADIAL" else 0.0)
    f0 = f_true * (1.6 if est_f else 1.0)                      # a wrong prior focal when it is to be estimated
    model = po.SIMPLE_RADIAL if cam == "SIMPLE_RADIAL" else po.SIMPLE_PINHOLE
    r = po.absolute_pose_estimation(sc.tracks[s], sc.points3d, (f0, 512.0, 512.0, k), model, us, estimate_focal_length=est_f,
                                    max_error=12.0, mask=sc.mask[s])
    assert r is not None
    E = sc.extrinsics[s]
    uv_gt = sc.points3d @ E[:, :3].T + E[:, 3]
    clean = np.linalg.norm(sc.tracks[s] - (f_true * (uv_gt[:, :2] / uv_gt[:, 2:]) * (1 + k * ((uv_gt[:, :2] / uv_gt[:, 2:]) ** 2).sum(1, keepdims=True)) + 512.0), axis=1) < 3
    assert r["num_inliers"] >= 0.9 * int((clean & sc.mask[s]).sum())
    if est_f:
        # the sampled focal closest to the truth in the quadratic ladder: within the ladder's local spacing
        facs = po.focal_length_factors(True) * f0
        assert abs(r["focal"] - f_true) <= np.abs(np.diff(facs)).max()
        assert abs(r["focal"] - f_true) / f_true < 0.12
    else:
        assert r["focal"] == f0
        assert rotation_angle_deg(r["pose"][None, :, :3], E[None, :, :3]).max() < 0.05
        assert np.abs(r["pose"][:, 3] - E[:, 3]).max() < 0.01


def test_returns_none_without_enough_points():
    us = np.random.default_rng(0).uniform(size=(8, 3))
    assert po.absolute_pose_estimation(np.zeros((2, 2)), np.zeros((2, 3)), (1000.0, 512.0, 512.0, 0.0), 0, us) is None


def test_debug_record():
    """absolute_pose_estimation(return_debug=True): per-factor results agree with a direct lo_ransac at that focal,
    the winner is the first factor with the highest count, and the decision record is filled."""
    sc = make_scene(2, 300, "SIMPLE_PINHOLE", seed=5, noise_px=0.3, outlier_frac=0.3)
    us = np.random.default_rng(4).uniform(size=(48, 3))
    us[5] = [0.1, 0.1, 0.7]                                       # a repeated index: the trial is skipped
    intr = (1300.0, 512.0, 512.0, 0.0)
    r, dbg = po.absolute_pose_estimation(sc.tracks[1], sc.points3d, intr, 0, us, estimate_focal_length=True,
                                         mask=sc.mask[1], return_debug=True)
    facs = dbg["factors"]
    assert len(facs) == 31 and dbg["skipped"] == 31
    assert dbg["nsol_hist"].sum() == 31 * 47 and dbg["nsol_hist"][1:].sum() > 0
    counts = [f["num_inliers"] for f in facs]
    k = int(np.argmax(counts))
    assert r["focal"] == facs[k]["focal"] and r["num_inliers"] == counts[k]
    assert np.array_equal(r["inliers"], facs[k]["inliers"]) and np.array_equal(r["pose"], facs[k]["pose"])
    assert 0 < dbg["thr_margin"] < 1 and dbg["tie_gap"] > 0
    for j in (0, 17, 30):
        f = facs[j]["focal"]
        idx = np.nonzero(sc.mask[1])[0]
        xn = (sc.tracks[1][idx].astype(np.float64) - 512.0) / f
        d = po.new_debug()
        got = po.lo_ransac(sc.points3d[idx], xn, (12.0 / f) ** 2, us, d)
        if got is None:
            assert facs[j]["num_inliers"] == 0 and not facs[j]["inliers"].any()
            continue
        assert got[1] == facs[j]["num_inliers"] and got[2] == facs[j]["residual_sum"]
        assert np.array_equal(got[0], facs[j]["pose"]) and facs[j]["inliers"].sum() == got[1]
        assert d["nsol_hist"].sum() == 47 and d["thr_margin"] >= dbg["thr_margin"]
    # without the debug flag the result is the same
    r2 = po.absolute_pose_estimation(sc.tracks[1], sc.points3d, intr, 0, us, estimate_focal_length=True, mask=sc.mask[1])
    assert r2["focal"] == r["focal"] and np.array_equal(r2["pose"], r["pose"])


def test_debug_sees_lo_on_an_earlier_candidate():
    """Over a few hundred random trials some P3P samples have 3 or 4 solutions and local optimisation runs on a candidate
    that is not the last of its trial (the case in which the kernel restores the later candidates' supports)."""
    sc = make_scene(1, 400, "SIMPLE_PINHOLE", seed=11, noise_px=0.3, outlier_frac=0.2)
    us = np.random.default_rng(12).uniform(size=(400, 3))
    _, dbg = po.absolute_pose_estimation(sc.tracks[0], sc.points3d, (1000.0, 512.0, 512.0, 0.0), 0, us,
                                         mask=sc.mask[0], return_debug=True)
    assert dbg["nsol_hist"][2] > 0 and dbg["nsol_hist"][3:].sum() > 0
    assert dbg["lo_not_last"] > 0 and len(dbg["factors"]) == 1
