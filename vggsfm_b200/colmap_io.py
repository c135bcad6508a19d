"""COLMAP binary model files for ``vggsfm_b200.reconstruction.Reconstruction`` -- the data format on the far side of the path.

The reference hands a live ``pycolmap.Reconstruction`` to its caller, which ends in ``reconstruction.write(dir)``
(``cameras.bin`` / ``images.bin`` / ``points3D.bin``; vggsfm/runners/runner.py:592-599).  pycolmap is not a dependency
of this path, so the three files are written directly from the plain-dict model ``Reconstruction.to_model()`` builds,
with the ids and ordering ``batch_matrix_to_pycolmap`` would have produced (vggsfm/utils/tensor_to_pycolmap.py:16-160):
  * point3D ids 1..P' in track order (tracks with >= 2 inlier observations), colour 0 unless ``points3D_rgb`` is set;
  * image ids = frame index, names ``image_{idx}``, one camera per frame (camera id = frame index) or camera 0 for
    ``shared_camera``; SIMPLE_PINHOLE params (f, cx, cy), SIMPLE_RADIAL (f, cx, cy, k);
  * an image's points2D are its inlier observations in point order; track elements are (image id, index in that list).
File layout: COLMAP's binary model format (src/colmap/scene/reconstruction_io.cc, mirrored by COLMAP's
scripts/python/read_write_model.py) [3P-memory]; the readers below exist for the round-trip tests.
Host-side I/O only: nothing here is on the GPU hot path.
"""
from __future__ import annotations

import os
import struct

import numpy as np

CAMERA_MODEL_IDS = {"SIMPLE_PINHOLE": 0, "PINHOLE": 1, "SIMPLE_RADIAL": 2}
CAMERA_MODEL_NUM_PARAMS = {0: 3, 1: 4, 2: 4}


def rotmat_to_qvec(R):
    """Rotation matrix -> (qw, qx, qy, qz), the branch structure of Eigen::Quaterniond(matrix) that pycolmap.Rotation3d uses."""
    m = np.asarray(R, dtype=np.float64)
    q = np.zeros(4)
    t = m[0, 0] + m[1, 1] + m[2, 2]
    if t > 0:
        t = np.sqrt(t + 1.0)
        q[0] = 0.5 * t
        t = 0.5 / t
        q[1] = (m[2, 1] - m[1, 2]) * t
        q[2] = (m[0, 2] - m[2, 0]) * t
        q[3] = (m[1, 0] - m[0, 1]) * t
    else:
        i = 0
        if m[1, 1] > m[0, 0]:
            i = 1
        if m[2, 2] > m[i, i]:
            i = 2
        j, k = (i + 1) % 3, (i + 2) % 3
        t = np.sqrt(m[i, i] - m[j, j] - m[k, k] + 1.0)
        q[1 + i] = 0.5 * t
        t = 0.5 / t
        q[0] = (m[k, j] - m[j, k]) * t
        q[1 + j] = (m[j, i] + m[i, j]) * t
        q[1 + k] = (m[k, i] + m[i, k]) * t
    return q / np.linalg.norm(q)


def qvec_to_rotmat(q):
    w, x, y, z = q
    return np.array([[1 - 2 * y * y - 2 * z * z, 2 * x * y - 2 * w * z, 2 * z * x + 2 * w * y],
                     [2 * x * y + 2 * w * z, 1 - 2 * x * x - 2 * z * z, 2 * y * z - 2 * w * x],
                     [2 * z * x - 2 * w * y, 2 * y * z + 2 * w * x, 1 - 2 * x * x - 2 * y * y]])


def _np(t):
    return t.detach().cpu().numpy() if hasattr(t, "detach") else np.asarray(t)


def write_model(model, path):
    """cameras.bin, images.bin, points3D.bin in COLMAP's binary layout (little endian)."""
    os.makedirs(path, exist_ok=True)
    with open(os.path.join(path, "cameras.bin"), "wb") as f:
        f.write(struct.pack("<Q", len(model["cameras"])))
        for cid, c in sorted(model["cameras"].items()):
            f.write(struct.pack("<iiQQ", cid, c["model_id"], c["width"], c["height"]))
            f.write(struct.pack("<%dd" % len(c["params"]), *c["params"]))
    with open(os.path.join(path, "images.bin"), "wb") as f:
        f.write(struct.pack("<Q", len(model["images"])))
        for iid, im in sorted(model["images"].items()):
            f.write(struct.pack("<idddddddi", iid, *im["qvec"], *im["tvec"], im["camera_id"]))
            f.write(im["name"].encode("utf-8") + b"\x00")
            n = len(im["point3D_ids"])
            f.write(struct.pack("<Q", n))
            rec = np.zeros(n, dtype=[("x", "<f8"), ("y", "<f8"), ("id", "<i8")])
            if n:
                rec["x"], rec["y"], rec["id"] = im["xys"][:, 0], im["xys"][:, 1], im["point3D_ids"]
            f.write(rec.tobytes())
    with open(os.path.join(path, "points3D.bin"), "wb") as f:
        f.write(struct.pack("<Q", len(model["points3D"])))
        for pid, p in sorted(model["points3D"].items()):
            f.write(struct.pack("<QdddBBBd", pid, *p["xyz"], *[int(v) for v in p["rgb"]], p["error"]))
            f.write(struct.pack("<Q", len(p["track"])))
            if p["track"]:
                f.write(np.asarray(p["track"], dtype="<i4").tobytes())


def read_model(path):
    """Inverse of write_model (used by the round-trip tests)."""
    cameras, images, points = {}, {}, {}
    with open(os.path.join(path, "cameras.bin"), "rb") as f:
        (n,) = struct.unpack("<Q", f.read(8))
        for _ in range(n):
            cid, mid, w, h = struct.unpack("<iiQQ", f.read(24))
            k = CAMERA_MODEL_NUM_PARAMS[mid]
            cameras[cid] = {"model_id": mid, "width": w, "height": h, "params": np.array(struct.unpack("<%dd" % k, f.read(8 * k)))}
    with open(os.path.join(path, "images.bin"), "rb") as f:
        (n,) = struct.unpack("<Q", f.read(8))
        for _ in range(n):
            vals = struct.unpack("<idddddddi", f.read(64))
            name = b""
            while True:
                ch = f.read(1)
                if ch == b"\x00":
                    break
                name += ch
            (m,) = struct.unpack("<Q", f.read(8))
            rec = np.frombuffer(f.read(24 * m), dtype=[("x", "<f8"), ("y", "<f8"), ("id", "<i8")])
            images[vals[0]] = {"qvec": np.array(vals[1:5]), "tvec": np.array(vals[5:8]), "camera_id": vals[8],
                               "name": name.decode("utf-8"), "xys": np.stack([rec["x"], rec["y"]], -1), "point3D_ids": rec["id"].copy()}
    with open(os.path.join(path, "points3D.bin"), "rb") as f:
        (n,) = struct.unpack("<Q", f.read(8))
        for _ in range(n):
            vals = struct.unpack("<QdddBBBd", f.read(43))
            (m,) = struct.unpack("<Q", f.read(8))
            tr = np.frombuffer(f.read(8 * m), dtype="<i4").reshape(m, 2)
            points[vals[0]] = {"xyz": np.array(vals[1:4]), "rgb": np.array(vals[4:7], dtype=np.uint8), "error": vals[7],
                               "track": [tuple(int(v) for v in t) for t in tr]}
    return {"cameras": cameras, "images": images, "points3D": points}


def write_array(array, path):
    """COLMAP's dense map format (``colmap::mvs::Mat<T>::Write``) as vggsfm/utils/utils.py:359-389 writes it, byte for
    byte: the ASCII header ``width&height&channels&``, then the float32 values little-endian in column-major order
    (x fastest within a row of the transposed map, channels slowest)."""
    assert array.dtype == np.float32
    if array.ndim == 2:
        height, width = array.shape
        channels = 1
        trans = array.T
    elif array.ndim == 3:
        height, width, channels = array.shape
        trans = np.transpose(array, (1, 0, 2))
    else:
        raise AssertionError("write_array takes a 2-D or 3-D array")
    with open(path, "wb") as fid:
        fid.write(f"{width}&{height}&{channels}&".encode())
        fid.write(trans.reshape(-1, order="F").astype("<f4", copy=False).tobytes())
