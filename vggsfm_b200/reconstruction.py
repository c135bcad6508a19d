"""pycolmap-shaped scene object for the far side of the bundle-adjustment path (SURVEY 8(b), 8(f) rank 1).

The reference hands a live ``pycolmap.Reconstruction`` back to its callers, which keep reading and mutating it
(vggsfm/runners/runner.py:555-559 ``add_point3D``, :575 ``deregister_image``, :592-631 ``images / cameras /
calibration_matrix``, :911 ``write``; vggsfm/utils/tensor_to_pycolmap.py:163-214 reads it back into tensors).
pycolmap is not a dependency of this path, so the object model those call sites touch is provided here with the
same attribute and method names:

    Reconstruction.cameras / .images / .points3D (dicts keyed by id), .point3D_ids(), .add_camera(), .add_image(),
    .add_point3D(xyz, track, color) -> id, .deregister_image(id), .normalize(extent, p0, p1, use_images),
    .write(dir), .num_points3D(), .num_images(), .num_reg_images(), .reg_image_ids()
    Camera(model, width, height, params, camera_id).calibration_matrix(); Image(id, name, camera_id, cam_from_world)
    with .points2D / .registered; Rigid3d(Rotation3d(R), t).matrix(); Point2D(xy, point3D_id); Track().add_element();
    Point3D.xyz / .color / .error / .track

A ``Reconstruction`` coming out of the CUDA bundle adjustment is created from tensors and stays a handful of numpy
arrays until somebody touches the object graph (``from_batch_matrix`` is the vectorised equivalent of the O(S*P) Python
loops of ``batch_matrix_to_pycolmap``, tensor_to_pycolmap.py:16-160: same ids, same point2D order, same 3000 clamp,
same camera sharing).  Host-side bookkeeping only: nothing here is on the GPU hot path, and nothing here computes BA.
"""
from __future__ import annotations

import numpy as np


def _np(t):
    return t.detach().cpu().numpy() if hasattr(t, "detach") else np.asarray(t)


class Rotation3d:
    """pycolmap.Rotation3d: built from a 3x3 matrix (tensor_to_pycolmap.py:115) or an xyzw quaternion."""

    def __init__(self, arg=None):
        a = np.eye(3) if arg is None else np.asarray(arg, dtype=np.float64)
        if a.shape == (4,):
            x, y, z, w = a / np.linalg.norm(a)
            a = np.array([[1 - 2 * (y * y + z * z), 2 * (x * y - w * z), 2 * (x * z + w * y)],
                          [2 * (x * y + w * z), 1 - 2 * (x * x + z * z), 2 * (y * z - w * x)],
                          [2 * (x * z - w * y), 2 * (y * z + w * x), 1 - 2 * (x * x + y * y)]])
        self._R = a.reshape(3, 3).copy()

    def matrix(self):
        return self._R.copy()

    @property
    def quat(self):
        """xyzw, like pycolmap."""
        from .colmap_io import rotmat_to_qvec
        w, x, y, z = rotmat_to_qvec(self._R)
        return np.array([x, y, z, w])


class Rigid3d:
    """pycolmap.Rigid3d(rotation, translation); ``matrix()`` is the 3x4 [R|t] (tensor_to_pycolmap.py:195)."""

    def __init__(self, rotation=None, translation=None):
        self.rotation = rotation if isinstance(rotation, Rotation3d) else Rotation3d(rotation)
        self.translation = np.zeros(3) if translation is None else np.asarray(translation, dtype=np.float64).copy()

    def matrix(self):
        return np.concatenate([self.rotation.matrix(), self.translation[:, None]], axis=1)

    def inverse(self):
        """pycolmap.Rigid3d.inverse(): rotation R^T, translation -R^T t."""
        Ri = self.rotation.matrix().T
        return Rigid3d(Rotation3d(Ri), -_apply(Ri, np.zeros(3), self.translation))

    def __mul__(self, x):
        """``Rigid3d * point`` for a 3-vector or an [N,3] array: R x + t (pycolmap 3.10)."""
        if isinstance(x, Rigid3d):
            R = self.rotation.matrix()
            return Rigid3d(Rotation3d(R @ x.rotation.matrix()), _apply(R, self.translation, x.translation))
        return _apply(self.rotation.matrix(), self.translation, np.asarray(x, dtype=np.float64))


def _apply(R, t, p):
    """R p + t with each row's terms added left to right, for p of shape [3] or [N,3] (the same rounding either way,
    which the vectorised dense-depth code relies on)."""
    return p[..., 0, None] * R[:, 0] + p[..., 1, None] * R[:, 1] + p[..., 2, None] * R[:, 2] + t


class Camera:
    """pycolmap.Camera for the two models the reference supports (tensor_to_pycolmap.py:78-110)."""

    def __init__(self, model="SIMPLE_PINHOLE", width=0, height=0, params=None, camera_id=0):
        if model not in ("SIMPLE_PINHOLE", "SIMPLE_RADIAL"):
            raise ValueError(f"Camera type {model} is not supported yet")
        self.model, self.width, self.height, self.camera_id = model, width, height, int(camera_id)
        self.params = np.asarray(params if params is not None else np.zeros(3 if model == "SIMPLE_PINHOLE" else 4),
                                 dtype=np.float64).copy()

    @property
    def model_name(self):
        return self.model

    @property
    def focal_length(self):
        return float(self.params[0])

    def calibration_matrix(self):
        f, cx, cy = self.params[:3]
        return np.array([[f, 0.0, cx], [0.0, f, cy], [0.0, 0.0, 1.0]])

    def img_from_cam(self, cam_points):
        """pycolmap 3.10 ``Camera.img_from_cam`` [3P-memory]: a 3-vector (or [N,3]) is divided by its z, then the
        model maps it to pixels (SIMPLE_RADIAL: f (u + u k r^2) + cx); a 2-vector (or [N,2]) is taken as already
        normalised.  runner.py:769 passes the 3-vector ``cam_from_world * xyz``."""
        p = np.asarray(cam_points, dtype=np.float64)
        if p.shape[-1] == 3:
            u, v = p[..., 0] / p[..., 2], p[..., 1] / p[..., 2]
        else:
            u, v = p[..., 0], p[..., 1]
        f, cx, cy = self.params[:3]
        if self.model == "SIMPLE_RADIAL":
            rad = self.params[3] * (u * u + v * v)
            u, v = u + u * rad, v + v * rad
        return np.stack([f * u + cx, f * v + cy], axis=-1)

    def cam_from_img(self, image_points):
        """pycolmap 3.10 ``Camera.cam_from_img``: pixels [N,2] (or a 2-vector) -> normalised [N,2].  SIMPLE_RADIAL
        inverts the distortion with COLMAP's iterative undistortion [3P-memory]."""
        xy = np.asarray(image_points, dtype=np.float64)
        f, cx, cy = self.params[:3]
        u, v = (xy[..., 0] - cx) / f, (xy[..., 1] - cy) / f
        if self.model == "SIMPLE_RADIAL":
            u, v = _iterative_undistortion(self.params[3], u, v)
        return np.stack([u, v], axis=-1)


def _iterative_undistortion(k, u, v):
    """COLMAP BaseCameraModel::IterativeUndistortion for SIMPLE_RADIAL (Newton, central-difference Jacobian with
    relative step 1e-6, at most 100 iterations, stop once the squared step is below 1e-10) [3P-memory]."""
    u, v = np.array(u, dtype=np.float64, ndmin=1), np.array(v, dtype=np.float64, ndmin=1)
    shape = np.shape(u)
    u, v = u.reshape(-1).copy(), v.reshape(-1).copy()
    x0, y0 = u.copy(), v.copy()
    eps = np.finfo(np.float64).eps
    for i in range(len(u)):
        x, y = u[i], v[i]
        for _ in range(100):
            s0, s1 = max(eps, abs(1e-6 * x)), max(eps, abs(1e-6 * y))
            d = [(a * k * (a * a + b * b), b * k * (a * a + b * b))
                 for a, b in ((x, y), (x - s0, y), (x + s0, y), (x, y - s1), (x, y + s1))]
            J00, J01 = 1 + (d[2][0] - d[1][0]) / (2 * s0), (d[4][0] - d[3][0]) / (2 * s1)
            J10, J11 = (d[2][1] - d[1][1]) / (2 * s0), 1 + (d[4][1] - d[3][1]) / (2 * s1)
            r0, r1 = x + d[0][0] - x0[i], y + d[0][1] - y0[i]
            det = J00 * J11 - J01 * J10
            st0, st1 = (J11 * r0 - J01 * r1) / det, (J00 * r1 - J10 * r0) / det
            x, y = x - st0, y - st1
            if st0 * st0 + st1 * st1 < 1e-10:
                break
        u[i], v[i] = x, y
    return u.reshape(shape), v.reshape(shape)


class Point2D:
    INVALID = 18446744073709551615           # colmap::kInvalidPoint3DId

    def __init__(self, xy=(0.0, 0.0), point3D_id=INVALID):
        self.xy = np.asarray(xy, dtype=np.float64).copy()
        self.point3D_id = int(point3D_id)

    def has_point3D(self):
        return self.point3D_id != Point2D.INVALID


class ListPoint2D(list):
    pass


class TrackElement:
    __slots__ = ("image_id", "point2D_idx")

    def __init__(self, image_id=0, point2D_idx=0):
        self.image_id, self.point2D_idx = int(image_id), int(point2D_idx)


class Track:
    def __init__(self, elements=None):
        self.elements = list(elements) if elements is not None else []

    def add_element(self, image_id, point2D_idx):
        self.elements.append(TrackElement(image_id, point2D_idx))

    def length(self):
        return len(self.elements)


class Point3D:
    def __init__(self, xyz, track=None, color=None, error=-1.0):
        self.xyz = np.asarray(xyz, dtype=np.float64).copy()
        self.track = track if track is not None else Track()
        self.color = np.zeros(3, dtype=np.uint8) if color is None else np.asarray(color).astype(np.uint8)
        self.error = float(error)


class Image:
    def __init__(self, id=0, name="", camera_id=0, cam_from_world=None, image_id=None):
        self.image_id = int(id if image_id is None else image_id)
        self.name, self.camera_id = name, int(camera_id)
        self.cam_from_world = cam_from_world if cam_from_world is not None else Rigid3d()
        self.registered = False
        self._points2D = ListPoint2D()
        self._lazy = None                      # (xys [n,2], point3D_ids [n]) until somebody asks for objects

    @property
    def points2D(self):
        if self._lazy is not None:
            xys, ids = self._lazy
            self._lazy = None
            self._points2D = ListPoint2D(Point2D(xys[i], ids[i]) for i in range(len(ids)))
        return self._points2D

    @points2D.setter
    def points2D(self, value):
        self._lazy = None
        self._points2D = value if isinstance(value, ListPoint2D) else ListPoint2D(value)

    def num_points2D(self):
        return len(self._lazy[1]) if self._lazy is not None else len(self._points2D)

    def _arrays(self):
        if self._lazy is not None:
            return self._lazy
        n = len(self._points2D)
        xys = np.array([p.xy for p in self._points2D], dtype=np.float64).reshape(n, 2)
        ids = np.array([p.point3D_id if p.has_point3D() else -1 for p in self._points2D], dtype=np.int64)
        return xys, ids

    def projection_center(self):
        return -self.cam_from_world.rotation.matrix().T @ self.cam_from_world.translation


class Reconstruction:
    """See the module docstring.  ``summary`` carries the LM report of the solve that produced it."""

    def __init__(self):
        self._cameras, self._images, self._points3D = {}, {}, {}
        self._next_point3D_id = 1
        self._pending = None                   # arrays of from_batch_matrix, until the object graph is touched
        self.summary = None
        self.camera_type, self.shared_camera = "SIMPLE_PINHOLE", False

    # ---- construction ---------------------------------------------------------------------------------------------
    @classmethod
    def from_batch_matrix(cls, points3d, extrinsics, intrinsics, tracks, masks, image_size, max_points3D_val=3000,
                          shared_camera=False, camera_type="SIMPLE_PINHOLE", extra_params=None, points3D_rgb=None,
                          summary=None, alive=None):
        """Vectorised ``batch_matrix_to_pycolmap`` (tensor_to_pycolmap.py:16-160), same arguments.  Point ids are
        1..P' over the tracks with >= 2 inliers in track order (:62-70); a point with any coordinate >=
        ``max_points3D_val`` exists but gets no observations (:131-133); image ids = frame index, names
        ``image_{idx}``; one camera per frame, or camera 0 when ``shared_camera`` (:78-110).  ``alive`` [P] marks
        points the solve deleted (negative-depth filter of the COLMAP controller): their ids stay allocated, the
        points and their observations are absent -- the state pycolmap leaves behind."""
        if camera_type not in ("SIMPLE_PINHOLE", "SIMPLE_RADIAL"):
            raise ValueError(f"Camera type {camera_type} is not supported yet")
        tracks = _np(tracks).astype(np.float64)
        N, P, _ = tracks.shape
        extrinsics, intrinsics = _np(extrinsics).astype(np.float64), _np(intrinsics).astype(np.float64)
        points3d, masks = _np(points3d).astype(np.float64), _np(masks).astype(bool)
        image_size = _np(image_size)
        assert len(extrinsics) == N and len(intrinsics) == N and len(points3d) == P and image_size.shape[0] == 2
        r = cls()
        r.camera_type, r.shared_camera, r.summary = camera_type, bool(shared_camera), summary
        r._pending = dict(points3d=points3d, extrinsics=extrinsics, intrinsics=intrinsics, tracks=tracks, masks=masks,
                          image_size=image_size, max_val=max_points3D_val,
                          extra=_np(extra_params).astype(np.float64) if extra_params is not None else None,
                          rgb=None if points3D_rgb is None else _np(points3D_rgb).astype(np.float64),
                          alive=None if alive is None else _np(alive).astype(bool))
        return r

    def set_point_colors(self, rgb01):
        """Colours in [0,1] for point ids 1..max id, rounded to uint8 like models/triangulator.py:333-340."""
        rgb01 = _np(rgb01).astype(np.float64)
        if self._pending is not None and self._pending["alive"] is None:
            full = np.zeros((self._pending["masks"].shape[1], 3))
            valid_idx = np.nonzero(self._pending["masks"].sum(0) >= 2)[0]
            if len(valid_idx) == rgb01.shape[0]:
                full[valid_idx] = rgb01
                self._pending["rgb"] = full
                return
        for pid, p in self.points3D.items():
            p.color = np.round(rgb01[pid - 1] * 255).astype(np.uint8)

    def _materialize(self):
        p = self._pending
        if p is None:
            return
        self._pending = None
        masks, pts = p["masks"], p["points3d"]
        N, P = masks.shape
        valid_idx = np.nonzero(masks.sum(0) >= 2)[0]
        ids = np.zeros(P, dtype=np.int64)
        ids[valid_idx] = np.arange(1, len(valid_idx) + 1)
        rgb = p["rgb"]
        alive = np.ones(P, dtype=bool) if p["alive"] is None else p["alive"]
        for k, v in enumerate(valid_idx):
            if alive[v]:
                col = np.zeros(3) if rgb is None else np.round(rgb[v] * 255)
                self._points3D[k + 1] = Point3D(pts[v], Track(), col)
        self._next_point3D_id = len(valid_idx) + 1
        small = np.zeros(P, dtype=bool)
        small[valid_idx] = (pts[valid_idx] < p["max_val"]).all(axis=1) & alive[valid_idx]
        camera = None
        for f in range(N):
            if camera is None or not self.shared_camera:
                prm = [p["intrinsics"][f, 0, 0], p["intrinsics"][f, 0, 2], p["intrinsics"][f, 1, 2]]
                if self.camera_type == "SIMPLE_RADIAL":
                    prm.append(p["extra"][f][0])
                camera = Camera(self.camera_type, p["image_size"][0], p["image_size"][1], np.array(prm), f)
                self.add_camera(camera)
            im = Image(id=f, name=f"image_{f}", camera_id=camera.camera_id,
                       cam_from_world=Rigid3d(Rotation3d(p["extrinsics"][f][:3, :3]), p["extrinsics"][f][:3, 3]))
            obs = np.nonzero(masks[f] & small)[0]
            im._lazy = (p["tracks"][f, obs], ids[obs])
            im.registered = True
            for k, o in enumerate(obs):
                self._points3D[int(ids[o])].track.add_element(f, k)
            self._images[f] = im

    @property
    def cameras(self):
        self._materialize()
        return self._cameras

    @property
    def images(self):
        self._materialize()
        return self._images

    @property
    def points3D(self):
        self._materialize()
        return self._points3D

    # ---- pycolmap.Reconstruction methods the reference calls ------------------------------------------------------------
    def add_camera(self, camera):
        self._materialize()
        self._cameras[camera.camera_id] = camera

    def add_image(self, image):
        self._materialize()
        self._images[image.image_id] = image

    def add_point3D(self, xyz, track, color=None):
        self._materialize()
        pid = self._next_point3D_id
        self._next_point3D_id += 1
        self._points3D[pid] = Point3D(xyz, track, color)
        return pid

    def point3D_ids(self):
        return set(self.points3D.keys())

    def num_points3D(self):
        return len(self.points3D)

    def num_images(self):
        return len(self.images)

    def num_cameras(self):
        return len(self.cameras)

    def reg_image_ids(self):
        return [i for i, im in sorted(self.images.items()) if im.registered]

    def num_reg_images(self):
        return len(self.reg_image_ids())

    def delete_point3D(self, point3D_id):
        pt = self.points3D.pop(point3D_id)
        for el in pt.track.elements:
            im = self._images.get(el.image_id)
            if im is not None:
                im.points2D[el.point2D_idx].point3D_id = Point2D.INVALID

    def deregister_image(self, image_id):
        """colmap::Reconstruction::DeRegisterImage: every observation of the image is deleted (a point whose track
        would drop to one element is deleted entirely), then the image is marked unregistered [3P-memory]."""
        im = self.images[image_id]
        for idx, p2 in enumerate(im.points2D):
            if not p2.has_point3D():
                continue
            pt = self._points3D.get(p2.point3D_id)
            if pt is None:
                p2.point3D_id = Point2D.INVALID
                continue
            if pt.track.length() <= 2:
                self.delete_point3D(p2.point3D_id)
            else:
                pt.track.elements = [e for e in pt.track.elements
                                     if not (e.image_id == image_id and e.point2D_idx == idx)]
                p2.point3D_id = Point2D.INVALID
        im.registered = False

    def normalize(self, extent=10.0, p0=0.1, p1=0.9, use_images=True):
        """colmap::Reconstruction::Normalize [3P-memory], the arithmetic of bundle_adjustment.normalize: similarity
        that maps the p0..p1 percentile box of the registered images' projection centres to ``extent``."""
        ims = [im for _, im in sorted(self.images.items()) if im.registered]
        if use_images:
            if len(ims) < 2:
                return
            coords = np.stack([im.projection_center() for im in ims])
        else:
            if len(self._points3D) < 2:
                return
            coords = np.stack([p.xyz for _, p in sorted(self._points3D.items())])
        n = len(coords)
        c32 = np.sort(coords.astype(np.float32), axis=0)
        P0 = int(p0 * (n - 1)) if n > 3 else 0
        P1 = int(p1 * (n - 1)) if n > 3 else n - 1
        bmin, bmax = c32[P0].astype(np.float64), c32[P1].astype(np.float64)
        mean = c32[P0:P1 + 1].astype(np.float64).sum(axis=0) / (P1 - P0 + 1)
        old = np.linalg.norm(bmax - bmin)
        scale = 1.0 if old < np.finfo(np.float64).eps else extent / old
        tr = -scale * mean
        for p in self._points3D.values():
            p.xyz = scale * p.xyz + tr
        for im in ims:
            R = im.cam_from_world.rotation.matrix()
            im.cam_from_world.translation = scale * im.cam_from_world.translation - R @ tr

    def write(self, path):
        """``pycolmap.Reconstruction.write(path)``: cameras.bin / images.bin / points3D.bin (runner.py:911)."""
        from . import colmap_io as cio
        cio.write_model(self.to_model(), path)

    # ---- tensor views -------------------------------------------------------------------------------------------------
    def to_model(self):
        """Plain-dict model in COLMAP ids (the layout colmap_io.write_model serialises); registered images only."""
        from .colmap_io import CAMERA_MODEL_IDS, rotmat_to_qvec
        cams = {cid: {"model_id": CAMERA_MODEL_IDS[c.model], "width": int(c.width), "height": int(c.height),
                      "params": np.asarray(c.params, dtype=np.float64)} for cid, c in self.cameras.items()}
        ims = {}
        for iid, im in self._images.items():
            if not im.registered:
                continue
            xys, ids = im._arrays()
            ims[iid] = {"qvec": rotmat_to_qvec(im.cam_from_world.rotation.matrix()), "tvec": im.cam_from_world.translation,
                        "camera_id": im.camera_id, "name": im.name, "xys": xys, "point3D_ids": ids}
        pts = {pid: {"xyz": p.xyz, "rgb": p.color, "error": p.error,
                     "track": [(e.image_id, e.point2D_idx) for e in p.track.elements]}
               for pid, p in self._points3D.items()}
        return {"cameras": cams, "images": ims, "points3D": pts}

    def to_batch_matrix(self, device="cuda", camera_type=None):
        """``pycolmap_to_batch_matrix`` (tensor_to_pycolmap.py:163-214): (points3D [max_id,3], extrinsics [S,3,4],
        intrinsics [S,3,3], extra_params [S,1]|None); deleted ids read back as zero rows."""
        import torch
        camera_type = camera_type or self.camera_type
        n = len(self.images)
        pts = np.zeros((max(self.point3D_ids()), 3))
        for pid, p in self._points3D.items():
            pts[pid - 1] = p.xyz
        E = np.stack([self._images[i].cam_from_world.matrix() for i in range(n)])
        K = np.stack([self._cameras[self._images[i].camera_id].calibration_matrix() for i in range(n)])
        extra = None
        if camera_type == "SIMPLE_RADIAL":
            extra = torch.from_numpy(np.array([self._cameras[self._images[i].camera_id].params[-1] for i in range(n)])).to(device)[:, None]
        return torch.from_numpy(pts).to(device), torch.from_numpy(E).to(device), torch.from_numpy(K).to(device), extra


def batch_matrix_to_pycolmap(points3d, extrinsics, intrinsics, tracks, masks, image_size, max_points3D_val=3000,
                             shared_camera=False, camera_type="SIMPLE_PINHOLE", extra_params=None):
    """Same name and arguments as vggsfm/utils/tensor_to_pycolmap.py:16-27."""
    return Reconstruction.from_batch_matrix(points3d, extrinsics, intrinsics, tracks, masks, image_size,
                                            max_points3D_val, shared_camera, camera_type, extra_params)


def pycolmap_to_batch_matrix(reconstruction, device="cuda", camera_type="SIMPLE_PINHOLE"):
    """Same name and arguments as vggsfm/utils/tensor_to_pycolmap.py:163-165."""
    return reconstruction.to_batch_matrix(device, camera_type)
