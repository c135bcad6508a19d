"""Golden vectors of the dense depth stage from the UNMODIFIED reference (run once; needs $VGGSFM_REFERENCE and
scikit-learn).  Writes tests/golden/dense_depth_*.npz.

Each frame runs the reference's own ``align_dense_depth_maps`` (vggsfm/utils/utils.py:635-770) alone, after
``np.random.seed(seed_f)``: sklearn then draws from the global RandomState seeded with seed_f, which is the
random-number pin of DESIGN §3.  The reconstruction handed to it is this project's stand-in ``Reconstruction``
(pycolmap is not needed), so the visual goldens pin everything but the camera model: SIMPLE_PINHOLE only.
``write_array`` goldens are the reference's bytes for a 1- and a 3-channel map.
"""
import importlib
import os
import sys
import tempfile

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from oracle import reference_shim  # noqa: E402
from vggsfm_b200.reconstruction import Camera, Image, Reconstruction, Rigid3d, Rotation3d  # noqa: E402

OUT = os.path.join(ROOT, "tests", "golden")


def import_reference_utils():
    reference_shim.install()
    for _ in range(30):
        try:
            return importlib.import_module("vggsfm.utils.utils")
        except ModuleNotFoundError as e:          # plotting / video packages the dense path never calls
            sys.modules[e.name] = reference_shim._Stub(e.name)
    raise RuntimeError("could not import vggsfm.utils.utils")


def scene(rng, shapes, n_samples, inlier_ratio, sky=0.1, pad=3):
    """Frames with a disparity map a / depth + b, sparse samples with outliers and zero 'sky' pixels."""
    rec = Reconstruction()
    sparse, disp, images = {}, {}, {}
    for f, (H, W) in enumerate(shapes):
        name = f"image_{f}"
        fl = 1.2 * max(H, W)
        cam = Camera("SIMPLE_PINHOLE", W, H, np.array([fl, W / 2 + rng.normal(), H / 2 + rng.normal()]), f)
        rec.add_camera(cam)
        ang = rng.normal(0, 0.1, 3)
        R = Rotation3d(np.concatenate([ang / 2, [1.0]])).matrix()
        im = Image(id=f, name=name, camera_id=f, cam_from_world=Rigid3d(Rotation3d(R), rng.normal(0, 1, 3)))
        rec.add_image(im)
        yy, xx = np.mgrid[0:H, 0:W]
        depth = 2.0 + 1.5 * np.sin(xx / W * 3) + yy / H
        a, b = rng.uniform(0.5, 2.0), rng.uniform(-0.05, 0.05)
        dm = (a / depth + b).astype(np.float32)
        dm[rng.uniform(size=(H, W)) < sky] = 0
        n = n_samples
        u = rng.uniform(-pad, W - 1 + pad, n)
        v = rng.uniform(-pad, H - 1 + pad, n)
        iu, iv = np.clip(np.round(u).astype(int), 0, W - 1), np.clip(np.round(v).astype(int), 0, H - 1)
        d = depth[iv, iu] * (1 + rng.normal(0, 1e-3, n))
        out = rng.uniform(size=n) > inlier_ratio
        d[out] = rng.uniform(0.5, 6, out.sum())
        sparse[name] = np.column_stack([u, v, d])
        disp[name] = dm
        images[name] = rng.integers(0, 256, (H, W, 3), dtype=np.uint8)
    return rec, sparse, disp, images


def run(U, name, shapes, n_samples, inlier_ratio, visual, seed, **kw):
    rng = np.random.default_rng(seed)
    rec, sparse, disp, images = scene(rng, shapes, n_samples, inlier_ratio, **kw)
    seeds = rng.integers(0, 2**31, len(shapes))
    arrays = dict(seeds=seeds, visual=np.array(visual))
    for f, nm in enumerate(sparse):
        arrays[f"uvd_{f}"] = sparse[nm]
        arrays[f"disp_in_{f}"] = disp[nm].copy()
        arrays[f"rgb_{f}"] = images[nm]
        cam = rec.cameras[f]
        arrays[f"cam_{f}"] = cam.params
        arrays[f"pose_{f}"] = rec.images[f].cam_from_world.matrix()
        np.random.seed(int(seeds[f]))
        one_disp = {nm: disp[nm]}
        depth, pts = U.align_dense_depth_maps(rec, {nm: sparse[nm]}, one_disp, images, visual)
        arrays[f"depth_{f}"] = depth[nm]
        arrays[f"disp_out_{f}"] = one_disp[nm]
        if visual:
            arrays[f"points_{f}"] = pts[nm]
    np.savez_compressed(os.path.join(OUT, f"dense_depth_{name}.npz"), **arrays)
    print(name, "frames", len(shapes))


def main():
    U = import_reference_utils()
    run(U, "mixed", [(48, 64), (37, 53), (64, 48), (30, 30)], 400, 0.9, False, 1)
    run(U, "low_inliers", [(40, 60), (41, 61)], 600, 0.3, False, 2)
    run(U, "noise", [(32, 40)], 300, 0.0, False, 3)
    run(U, "small", [(20, 24), (22, 26), (24, 20)], 3, 0.9, False, 4, sky=0.0, pad=0)
    run(U, "visual", [(36, 50), (27, 31)], 300, 0.8, True, 5)
    rng = np.random.default_rng(6)
    arrays = {}
    for c, shape in ((1, (5, 7)), (3, (4, 6, 3))):
        a = rng.normal(size=shape).astype(np.float32)
        with tempfile.TemporaryDirectory() as d:
            p = os.path.join(d, "m.bin")
            U.write_array(a, p)
            arrays[f"array_{c}"] = a
            arrays[f"bytes_{c}"] = np.frombuffer(open(p, "rb").read(), dtype=np.uint8)
    np.savez_compressed(os.path.join(OUT, "dense_depth_write_array.npz"), **arrays)


if __name__ == "__main__":
    main()
