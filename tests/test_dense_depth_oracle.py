"""Dense depth stage on the host: the oracle against live sklearn and the reference goldens, write_array's bytes, the
stand-in camera / pose methods and the vectorised sparse-depth extraction (no GPU)."""
import glob
import os
import tempfile

import numpy as np
import pytest

from oracle import dense_depth_oracle as O
from vggsfm_b200 import colmap_io, dense_depth
from vggsfm_b200.reconstruction import Camera, Reconstruction, Rigid3d, Rotation3d

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")
f32 = np.float32


def _frame(rng, n, ratio):
    X = rng.uniform(0.05, 2, n).astype(f32)
    y = 0.7 * X.astype(np.float64) + 0.1 + rng.normal(0, 1e-3, n)
    out = rng.uniform(size=n) > ratio
    y[out] = rng.uniform(0.05, 2, out.sum())
    return X, y


def test_oracle_equals_sklearn():
    sk = pytest.importorskip("sklearn.linear_model")
    rng = np.random.default_rng(0)
    for t in range(300):
        n = int(rng.choice([2, 3, 9, 50, 199, 200, 700]))
        X, y = _frame(rng, n, rng.uniform(0.05, 1))
        th = np.median(y) / 30
        seed = int(rng.integers(2**31))
        ref = sk.RANSACRegressor(sk.LinearRegression(), min_samples=2, residual_threshold=th, max_trials=20000,
                                 loss="squared_error", random_state=np.random.RandomState(seed)).fit(X[:, None], y)
        o = O.ransac_fit(X, y, th, seed)
        assert ref.n_trials_ == o["n_trials"]
        np.testing.assert_array_equal(ref.inlier_mask_, o["inlier_mask"])
        np.testing.assert_allclose(o["coef"], ref.estimator_.coef_[0], rtol=1e-12)
        np.testing.assert_allclose(o["intercept"], ref.estimator_.intercept_, rtol=1e-12, atol=1e-12)


@pytest.mark.parametrize("n", [2, 3, 50, 5000])
def test_sample_draws_match_sklearn(n):
    swr = pytest.importorskip("sklearn.utils.random").sample_without_replacement
    a, b = np.random.RandomState(5), np.random.RandomState(5)
    ref = np.stack([swr(n, 2, random_state=a) for _ in range(500)])
    np.testing.assert_array_equal(O.sample_pairs(b, n, 500), ref)
    stream = dense_depth._PairStream(n, 5)
    got = np.concatenate([stream.take(T) for T in (1, 7, 100, 392)])
    np.testing.assert_array_equal(got, ref)


def test_fit_two_is_sgelsd_bitwise():
    rng = np.random.default_rng(1)
    for _ in range(5000):
        x = rng.uniform(0.01, 10, 2).astype(f32)
        y = rng.uniform(0.01, 3, 2)
        assert O.fit_two(x[0], x[1], y[0], y[1]) == O.linear_regression(x, y)
    assert O.fit_two(1.5, 1.5, 0.2, 0.4) == O.linear_regression(np.array([1.5, 1.5], f32), np.array([0.2, 0.4]))
    c, b = O.fit_two(1.5, 1.5, 0.2, 0.4)             # equal x: the minimum-norm line
    assert c == 0 and b == f32(0.3)


def test_dynamic_max_trials():
    rt = pytest.importorskip("sklearn.linear_model._ransac")
    for n_in, n in ((0, 10), (10, 10), (1, 10), (5, 10), (3, 4096), (4000, 4096), (1, 2)):
        assert O.dynamic_max_trials(n_in, n) == rt._dynamic_max_trials(n_in, n, 2, 0.99)


def test_errors_of_the_reference():
    with pytest.raises(ValueError, match="Too few points"):
        O.frame_samples(np.ones((4, 4), f32), np.zeros((0, 3)))
    with pytest.raises(ValueError, match="min_samples"):
        O.ransac_fit(np.ones(1, f32), np.ones(1), 0.1, 0)
    X, y, th = O.frame_samples(np.ones((4, 4), f32), np.array([[1, 1, 2.0], [2, 2, 4.0]]))
    assert th == np.median(np.array([0.5, 0.25])) / 30 == (0.5 + 0.25) / 2 / 30


def _golden_frames(path):
    z = np.load(path)
    F = len(z["seeds"])
    return z, F


@pytest.mark.parametrize("path", sorted(glob.glob(os.path.join(GOLDEN, "dense_depth_*.npz"))))
def test_oracle_equals_reference_goldens(path):
    if path.endswith("write_array.npz"):
        pytest.skip("bytes golden")
    z, F = _golden_frames(path)
    for f in range(F):
        r = O.align_frame(z[f"disp_in_{f}"], z[f"uvd_{f}"], int(z["seeds"][f]))
        np.testing.assert_array_equal(r["depth"].view(np.uint32), z[f"depth_{f}"].view(np.uint32))
        np.testing.assert_array_equal(r["disp"].view(np.uint32), z[f"disp_out_{f}"].view(np.uint32))
        if bool(z["visual"]):
            cam = z[f"cam_{f}"]
            pose = z[f"pose_{f}"]
            pts = O.unproject(r["depth"], r["valid"], "SIMPLE_PINHOLE", cam, pose[:, :3], pose[:, 3], z[f"rgb_{f}"])
            np.testing.assert_array_equal(pts, z[f"points_{f}"])


def test_write_array_bytes():
    z = np.load(os.path.join(GOLDEN, "dense_depth_write_array.npz"))
    for c in (1, 3):
        with tempfile.TemporaryDirectory() as d:
            p = os.path.join(d, "m.bin")
            colmap_io.write_array(z[f"array_{c}"], p)
            assert open(p, "rb").read() == z[f"bytes_{c}"].tobytes()


def _reference_loop(rec):
    """runner.py:755-771 verbatim, rows re-sorted to ascending point id (pycolmap's order is unpinned)."""
    from collections import defaultdict
    sparse_depth, sparse_point = defaultdict(list), defaultdict(list)
    for point3D_idx in sorted(rec.points3D):
        pt3D = rec.points3D[point3D_idx]
        for track_element in pt3D.track.elements:
            pyimg = rec.images[track_element.image_id]
            pycam = rec.cameras[pyimg.camera_id]
            projection = pyimg.cam_from_world * pt3D.xyz
            depth = projection[-1]
            uv = pycam.img_from_cam(projection)
            sparse_depth[pyimg.name].append(np.append(uv, depth))
            sparse_point[pyimg.name].append(np.append(pt3D.xyz, point3D_idx))
    return sparse_depth, sparse_point


def _recon(camera_type, seed=0):
    from vggsfm_b200.synthetic import make_scene
    sc = make_scene(6, 80, camera_type, seed=seed)
    return lambda: Reconstruction.from_batch_matrix(sc.points3d, sc.extrinsics, sc.intrinsics, sc.tracks, sc.mask,
                                                    np.array([640, 480]), camera_type=camera_type,
                                                    extra_params=getattr(sc, "extra_params", None))


@pytest.mark.parametrize("camera_type", ["SIMPLE_PINHOLE", "SIMPLE_RADIAL"])
@pytest.mark.parametrize("form", ["arrays", "objects", "rescaled"])
def test_sparse_extraction_equals_reference_statements(camera_type, form):
    make = _recon(camera_type)
    rec = make()
    if form != "arrays":
        rec.images                                        # materialise the object graph
    if form == "rescaled":                                # what rename_colmap_recons_and_rescale_camera does
        for cam in rec.cameras.values():
            cam.params[:3] = cam.params[:3] * 2.5
            cam.width, cam.height = cam.width * 2.5, cam.height * 2.5
        for im in rec.images.values():
            im.name = "renamed_" + im.name
    got = dense_depth.extract_sparse_depth_and_point_from_reconstruction(None, {"reconstruction": rec})
    ref_rec = make() if form == "arrays" else rec
    ref_d, ref_p = _reference_loop(ref_rec)
    assert list(got["sparse_depth"]) == list(ref_d)
    for nm in ref_d:
        np.testing.assert_array_equal(got["sparse_depth"][nm], np.array(ref_d[nm]))
        np.testing.assert_array_equal(got["sparse_point"][nm], np.array(ref_p[nm]))


def test_camera_and_pose_methods():
    rng = np.random.default_rng(3)
    R = Rotation3d(np.concatenate([rng.normal(0, 0.2, 3), [1.0]])).matrix()
    T = Rigid3d(Rotation3d(R), rng.normal(size=3))
    p = rng.normal(size=(10, 3))
    np.testing.assert_allclose(T.inverse() * (T * p), p, atol=1e-14)
    for k in range(10):
        np.testing.assert_array_equal(T * p[k], (T * p)[k])
    for model, prm in (("SIMPLE_PINHOLE", [500.0, 320, 240]), ("SIMPLE_RADIAL", [500.0, 320, 240, -0.08])):
        cam = Camera(model, 640, 480, np.array(prm))
        xy = rng.uniform(0, 640, (50, 2))
        n = cam.cam_from_img(xy)
        np.testing.assert_allclose(n, O.cam_from_img(model, np.array(prm), xy), atol=1e-12)
        np.testing.assert_allclose(cam.img_from_cam(np.column_stack([n, np.ones(50)]) * 3.0), xy, atol=1e-6)
        np.testing.assert_array_equal(cam.img_from_cam(p[0]), O.img_from_cam(model, np.array(prm), p[0]))
