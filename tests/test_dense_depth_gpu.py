"""CUDA dense depth stage (csrc/dense_depth.cu via vggsfm_b200.dense_depth) against the float64/float32 numpy oracle.

Per frame the RANSAC decisions are exact: n_trials, n_inliers and the inlier mask, because the trial kernel computes
sklearn's float32 two-sample fit bitwise (oracle.fit_two == sgelsd) and the residuals in the same float64 operations.
The final fit on the inliers takes numpy's float32 means bitwise (oracle.mean_f32) and then solves the centred
least squares in float64 where sklearn runs sgelsd in float32, so the scale agrees to a few float32 ulps (rtol 2e-6).
With equal means, shift = ym - xm * c differs only through c: two roundings of the product and two of the difference
give |d shift| <= |xm| |d c| + 4u (|ym| + |xm c|), u = 2^-24, which is the shift's bar (SHIFT_ULPS = 4).  Given the
same scale and shift, the rescaled disparity and depth are bitwise equal, so the maps are compared after the oracle's
rescale with the kernel's scale / shift.  The decisions are only exact away from ties, so the oracle side asserts its
margins."""
import glob
import os
import re

import numpy as np
import pytest

from oracle import dense_depth_oracle as O
from vggsfm_b200 import dense_depth
from vggsfm_b200.reconstruction import Camera, Image, Reconstruction, Rigid3d, Rotation3d

pytestmark = pytest.mark.gpu
GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")
SCALE_RTOL = 2e-6
SHIFT_ULPS = 4
U32 = 2.0 ** -24


def check_fit(scale, shift, X, y, r, label=""):
    """The kernel's final scale / shift against the oracle's fit on the same inlier mask -> shift error / bar."""
    m = r["inlier_mask"]
    xm, ym = float(O.mean_f32(X[m])), float(O.mean_f32(y[m]))
    c = float(r["coef"])
    assert abs(float(scale) - c) <= SCALE_RTOL * abs(c), (label, float(scale), c)
    bar = abs(xm) * abs(float(scale) - c) + SHIFT_ULPS * U32 * (abs(ym) + abs(xm * c))
    err = abs(float(shift) - float(r["intercept"]))
    assert err <= bar, (label, float(shift), float(r["intercept"]), bar)
    return err / bar if bar > 0 else 0.0


def _scene(rng, shapes, n_samples, ratio, model="SIMPLE_PINHOLE", sky=0.05):
    rec = Reconstruction()
    sparse, disp, rgb = {}, {}, {}
    for f, (H, W) in enumerate(shapes):
        nm = f"frame_{f}.png"
        prm = [1.1 * max(H, W), W / 2, H / 2] + ([-0.05] if model == "SIMPLE_RADIAL" else [])
        rec.add_camera(Camera(model, W, H, np.array(prm), f))
        R = Rotation3d(np.concatenate([rng.normal(0, 0.1, 3), [1.0]])).matrix()
        rec.add_image(Image(id=f, name=nm, camera_id=f, cam_from_world=Rigid3d(Rotation3d(R), rng.normal(0, 1, 3))))
        yy, xx = np.mgrid[0:H, 0:W]
        depth = 2.0 + 1.5 * np.sin(xx / W * 3) + yy / H
        dm = (rng.uniform(0.5, 2) / depth + rng.uniform(-0.05, 0.05)).astype(np.float32)
        dm[rng.uniform(size=(H, W)) < sky] = 0
        n = n_samples if np.isscalar(n_samples) else n_samples[f]
        u, v = rng.uniform(-0.5, W - 0.5, n), rng.uniform(-0.5, H - 0.5, n)
        iu, iv = np.clip(np.round(u).astype(int), 0, W - 1), np.clip(np.round(v).astype(int), 0, H - 1)
        d = depth[iv, iu] * (1 + rng.normal(0, 1e-3, n))
        out = rng.uniform(size=n) > ratio
        d[out] = rng.uniform(0.5, 6, out.sum())
        sparse[nm], disp[nm] = np.column_stack([u, v, d]), dm
        rgb[nm] = rng.integers(0, 256, (H, W, 3), dtype=np.uint8)
    return rec, sparse, disp, rgb


def _check(rec, sparse, disp, rgb, seeds, visual=False, model="SIMPLE_PINHOLE", **kw):
    orig = {k: v.copy() for k, v in disp.items()}
    depth, pts, dbg = dense_depth.align_dense_depth_maps(rec, sparse, disp, rgb, visual, seeds=seeds,
                                                         return_debug=True, **kw)
    worst = 0.0
    for f, nm in enumerate(sparse):
        X, y, th = O.frame_samples(orig[nm], sparse[nm])
        np.testing.assert_array_equal(dbg["x"][f], X)
        np.testing.assert_array_equal(dbg["y"][f], y)
        assert dbg["threshold"][f] == th
        r = O.ransac_fit(X, y, th, int(seeds[f]), return_debug=True)
        assert r["debug"]["residual_margin"] > 1e-9, "oracle winner has a residual at the threshold"
        assert r["debug"]["score_gap"] > 1e-12, "oracle has an equal-count R^2 tie"
        assert dbg["n_trials"][f] == r["n_trials"], nm
        assert dbg["n_inliers"][f] == r["n_inliers"], nm
        np.testing.assert_array_equal(dbg["inlier_mask"][f], r["inlier_mask"])
        worst = max(worst, check_fit(dbg["scale"][f], dbg["shift"][f], X, y, r, nm))
        dref, depref, valid = O.apply_scale(orig[nm], dbg["scale"][f], dbg["shift"][f])
        np.testing.assert_array_equal(depth[nm].view(np.uint32), depref.view(np.uint32))
        np.testing.assert_array_equal(disp[nm].view(np.uint32), dref.view(np.uint32))
        if visual:
            im = rec.images[f]
            cam = rec.cameras[im.camera_id]
            M = im.cam_from_world.matrix()
            ref = O.unproject(depref, valid, model, cam.params, M[:, :3], M[:, 3], rgb[nm])
            assert pts[nm].shape == ref.shape
            np.testing.assert_array_equal(pts[nm][1], ref[1])
            if model == "SIMPLE_PINHOLE":
                np.testing.assert_allclose(pts[nm][0], ref[0], rtol=1e-12, atol=1e-12)
            else:
                # normalised coordinates: back through the pose, divide by depth
                cam_p = (pts[nm][0] - (im.cam_from_world.inverse().translation)) @ M[:, :3].T
                nrm = cam_p[:, :2] / cam_p[:, 2:3]
                H, W = depref.shape
                yy, xx = np.mgrid[0:H, 0:W]
                xy = np.column_stack([xx.ravel(), yy.ravel()])[valid.ravel()]
                np.testing.assert_allclose(nrm, O.cam_from_img(model, cam.params, xy), atol=1e-9)
                np.testing.assert_allclose(cam.img_from_cam(nrm), xy, atol=1e-6)
    print(f"largest shift error / bar: {worst:.3g}")
    return dbg


@pytest.mark.parametrize("path", sorted(p for p in glob.glob(os.path.join(GOLDEN, "dense_depth_*.npz"))
                                        if "write_array" not in p))
def test_reference_goldens(cuda_dev, path):
    z = np.load(path)
    F = len(z["seeds"])
    rec = Reconstruction()
    sparse, disp, rgb = {}, {}, {}
    for f in range(F):
        nm = f"image_{f}"
        H, W = z[f"disp_in_{f}"].shape
        rec.add_camera(Camera("SIMPLE_PINHOLE", W, H, z[f"cam_{f}"], f))
        P = z[f"pose_{f}"]
        rec.add_image(Image(id=f, name=nm, camera_id=f, cam_from_world=Rigid3d(Rotation3d(P[:, :3]), P[:, 3])))
        sparse[nm], disp[nm], rgb[nm] = z[f"uvd_{f}"], z[f"disp_in_{f}"].copy(), z[f"rgb_{f}"]
    visual = bool(z["visual"])
    depth, pts = dense_depth.align_dense_depth_maps(rec, sparse, disp, rgb, visual, seeds=z["seeds"])
    for f in range(F):
        nm = f"image_{f}"
        np.testing.assert_allclose(depth[nm], z[f"depth_{f}"], rtol=2e-5)
        assert ((depth[nm] == 0) == (z[f"depth_{f}"] == 0)).all()
        if visual:
            assert pts[nm].shape == z[f"points_{f}"].shape
            ref = z[f"points_{f}"]
            np.testing.assert_allclose(pts[nm], ref, rtol=2e-5, atol=2e-5 * np.abs(ref).max())


def test_400_frames_mixed_sizes(cuda_dev):
    rng = np.random.default_rng(0)
    shapes = [(1080, 1920), (480, 640), (720, 1280), (333, 517)] * 100
    rec, sparse, disp, rgb = _scene(rng, shapes, 4000, 0.6, sky=0.02)
    seeds = rng.integers(0, 2**31, len(shapes))
    _check(rec, sparse, disp, rgb, seeds)


@pytest.mark.parametrize("model", ["SIMPLE_PINHOLE", "SIMPLE_RADIAL"])
def test_small_frames_noise_and_visual(cuda_dev, model):
    rng = np.random.default_rng(1)
    shapes = [(40, 60), (41, 37), (64, 64), (50, 70)]
    rec, sparse, disp, rgb = _scene(rng, shapes, [2, 3, 256, 3000], 0.7, model=model, sky=0.0)
    nm = list(sparse)[3]                                      # pure noise: the 20000-trial cap
    sparse[nm][:, 2] = 1 / rng.uniform(1, 1e4, len(sparse[nm]))   # targets spread far beyond the threshold
    disp[nm][:] = rng.uniform(0.2, 1.0, disp[nm].shape).astype(np.float32)
    seeds = rng.integers(0, 2**31, len(shapes))
    dbg = _check(rec, sparse, disp, rgb, seeds, visual=True, model=model)
    assert dbg["n_trials"][3] == 20000


def test_rounding_clip_and_limits(cuda_dev):
    rng = np.random.default_rng(2)
    rec, sparse, disp, rgb = _scene(rng, [(30, 40), (31, 41)], 200, 0.9, sky=0.0)
    for nm, (H, W) in zip(sparse, [(30, 40), (31, 41)]):
        s = sparse[nm]
        s[:6, :2] = [[-0.5, 3], [W - 0.5, 3], [3, H - 0.5], [-0.5000001, 2], [2.5, 1.5], [W - 1.5, H - 1.5]]
        s[6:9, 2] = [-1.0, 0.0, 2e4]                         # depth <= 0 and > 1e4 reach the clip
        disp[nm][0, :5] = [-3.0, 1e9, 0.0, 1e-30, -1e-30]    # rescaled disparity <= 0 and > 10000
    _check(rec, sparse, disp, rgb, rng.integers(0, 2**31, 2))


def test_reference_errors_before_launch(cuda_dev):
    """The reference's errors and messages, raised before any RANSAC launch.  Samples that all fall out of bounds leave
    no kept sample: np.median of it is NaN, and sklearn rejects the NaN residual_threshold."""
    rng = np.random.default_rng(3)
    rec, sparse, disp, rgb = _scene(rng, [(30, 40)], 50, 0.9)
    nm = list(sparse)[0]
    with pytest.raises(ValueError, match="Too few points"):
        dense_depth.align_dense_depth_maps(rec, {nm: np.zeros((0, 3))}, disp, rgb)
    out_of_bounds = sparse[nm].copy()
    out_of_bounds[:, 0] = -5
    with pytest.raises(ValueError, match=re.escape(O.NAN_THRESHOLD_ERROR.format(np.float64(np.nan)))):
        dense_depth.align_dense_depth_maps(rec, {nm: out_of_bounds}, disp, rgb)
    with pytest.raises(TypeError):
        dense_depth.align_dense_depth_maps(rec, sparse, {nm: disp[nm].astype(np.float64)}, rgb)
    with pytest.raises(ValueError):
        dense_depth.align_dense_depth_maps(rec, sparse, disp, rgb, device="cpu")


def test_batches_by_memory_budget(cuda_dev):
    rng = np.random.default_rng(4)
    rec, sparse, disp, rgb = _scene(rng, [(60, 80), (61, 81), (59, 79)], 300, 0.8)
    seeds = rng.integers(0, 2**31, 3)
    _check(rec, sparse, disp, rgb, seeds, visual=True, memory_budget=60 * 80 * 60)


def test_end_to_end_synthetic_scene(cuda_dev):
    """Extraction from a Reconstruction, then alignment of a disparity rendered as a / depth_gt + b."""
    from vggsfm_b200.synthetic import make_scene
    sc = make_scene(6, 600, "SIMPLE_PINHOLE", seed=5)
    W, H = 640, 480
    rec = Reconstruction.from_batch_matrix(sc.points3d, sc.extrinsics, sc.intrinsics, sc.tracks, sc.mask,
                                           np.array([W, H]))
    pred = dense_depth.extract_sparse_depth_and_point_from_reconstruction(None, {"reconstruction": rec})
    rng = np.random.default_rng(6)
    disp, gt = {}, {}
    for nm, uvd in pred["sparse_depth"].items():
        # ground-truth depth: a plane fitted through the frame's sparse depths, rendered per pixel
        A = np.column_stack([uvd[:, 0], uvd[:, 1], np.ones(len(uvd))])
        coef = np.linalg.lstsq(A, uvd[:, 2], rcond=None)[0]
        yy, xx = np.mgrid[0:H, 0:W]
        d = np.clip(coef[0] * xx + coef[1] * yy + coef[2], 0.5, None)
        gt[nm] = d
        disp[nm] = (0.8 / d + 0.05).astype(np.float32)
        uvd[:, 2] = (A @ coef) * (1 + rng.normal(0, 1e-4, len(uvd)))
        out = rng.uniform(size=len(uvd)) < 0.2             # outliers beyond the loose squared-residual threshold
        uvd[out, 2] *= rng.uniform(4, 10, out.sum())
    depth, _ = dense_depth.align_dense_depth_maps(rec, pred["sparse_depth"], disp, {}, seeds=np.arange(len(disp)))
    for nm in disp:
        ok = depth[nm] > 0
        assert ok.mean() > 0.99
        np.testing.assert_allclose(depth[nm][ok], gt[nm][ok], rtol=1e-3)
