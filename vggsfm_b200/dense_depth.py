"""Dense depth stage of the runner (``dense_depth=True``, runners/runner.py:250-269) on the GPU.

* ``extract_sparse_depth_and_point_from_reconstruction(self, predictions)`` -- runner.py:744-774 vectorised: every
  observation of the reconstruction projected into its image.  Rows are pinned to ascending point3D id, then track
  order (pycolmap iterates an unordered_map, whose order cannot be reproduced).
* ``align_dense_depth_maps(reconstruction, sparse_depth, disp_dict, original_images, visual_dense_point_cloud=False)``
  -- vggsfm/utils/utils.py:635-770 with all frames in one batched RANSAC (csrc/dense_depth.cu) and the per-pixel work
  in one HBM pass per batch of frames.  Frame f's RANSAC draws from ``np.random.RandomState(seeds[f])``; the seeds are
  drawn in frame order from numpy's global generator unless given (DESIGN §3).

No CPU fallback: the kernels run on ``device`` (CUDA); a missing library raises.
"""
from __future__ import annotations

import ctypes
from collections import defaultdict

import numpy as np
import torch

from . import _lib
from .colmap_io import write_array  # noqa: F401  (the runner imports it from the same place as align_dense_depth_maps)

DISPARITY_MAX = 10000
DISPARITY_MIN = 0.0001
DEPTH_MAX = 1 / DISPARITY_MIN
DEPTH_MIN = 1 / DISPARITY_MAX
MAX_TRIALS = 20000
THRES_RATIO = 30
FIRST_CHUNK = 32
_CAMERA_MODELS = {"SIMPLE_PINHOLE": 0, "SIMPLE_RADIAL": 1}


def _ptr(t):
    return ctypes.c_void_p(t.data_ptr()) if t is not None else None


# ---------------------------------------------------------------------------------------------------------------------
# sparse depth
# ---------------------------------------------------------------------------------------------------------------------
def _frame_views(p, shared_camera, camera_type):
    """{image id: (name, cam_from_world, Camera)} of the array form, as _materialize would build them."""
    from .reconstruction import Camera, Rigid3d, Rotation3d
    out, cam = {}, None
    for f in range(p["masks"].shape[0]):
        if cam is None or not shared_camera:
            K = p["intrinsics"][f]
            prm = [K[0, 0], K[0, 2], K[1, 2]] + ([p["extra"][f][0]] if camera_type == "SIMPLE_RADIAL" else [])
            cam = Camera(camera_type, p["image_size"][0], p["image_size"][1], np.array(prm), f)
        E = p["extrinsics"][f]
        out[f] = (f"image_{f}", Rigid3d(Rotation3d(E[:3, :3]), E[:3, 3]), cam)
    return out


def _observations(reconstruction):
    """(xyz [n,3], point ids [n], image ids [n]) in ascending point id, then track order."""
    p = getattr(reconstruction, "_pending", None)
    if p is not None:
        masks, pts = p["masks"], p["points3d"]
        valid_idx = np.nonzero(masks.sum(0) >= 2)[0]
        alive = np.ones(masks.shape[1], dtype=bool) if p["alive"] is None else p["alive"]
        keep = valid_idx[(pts[valid_idx] < p["max_val"]).all(axis=1) & alive[valid_idx]]
        ids = np.zeros(masks.shape[1], dtype=np.int64)
        ids[valid_idx] = np.arange(1, len(valid_idx) + 1)
        obs = masks[:, keep].T                           # [points, frames], point-major = ascending id
        pi, fi = np.nonzero(obs)
        return pts[keep][pi], ids[keep][pi], fi.astype(np.int64)
    items = sorted(reconstruction.points3D.items())
    lens = np.array([len(pt.track.elements) for _, pt in items], dtype=np.int64)
    xyz = np.repeat(np.array([pt.xyz for _, pt in items]).reshape(-1, 3), lens, axis=0)
    pid = np.repeat(np.array([k for k, _ in items], dtype=np.int64), lens)
    img = np.array([e.image_id for _, pt in items for e in pt.track.elements], dtype=np.int64)
    return xyz, pid, img


def extract_sparse_depth_and_point_from_reconstruction(self, predictions):
    """runner.py:744-774, same keys and content: per image name, rows [u, v, depth] and [x, y, z, point3D_id]
    (numpy arrays instead of lists of rows).  ``self`` is unused (it is a runner method)."""
    rec = predictions["reconstruction"]
    xyz, pid, img = _observations(rec)
    sparse_depth, sparse_point = defaultdict(list), defaultdict(list)
    if len(img) == 0:
        predictions["sparse_depth"], predictions["sparse_point"] = sparse_depth, sparse_point
        return predictions
    p = getattr(rec, "_pending", None)
    if p is not None:                                    # array form: no object graph needed
        views = _frame_views(p, rec.shared_camera, rec.camera_type)
    else:
        views = {i: (im.name, im.cam_from_world, rec.cameras[im.camera_id]) for i, im in rec.images.items()}
    order = np.argsort(img, kind="stable")
    uniq, start = np.unique(img[order], return_index=True)
    bounds = dict(zip(uniq.tolist(), zip(start.tolist(), np.append(start[1:], len(img)).tolist())))
    _, first = np.unique(img, return_index=True)
    for iid in uniq[np.argsort(first)]:                  # images in order of first appearance, like the defaultdict
        a, b = bounds[int(iid)]
        sel = order[a:b]
        name, pose, cam = views[int(iid)]
        proj = pose * xyz[sel]
        uv = cam.img_from_cam(proj)
        sparse_depth[name] = np.column_stack([uv, proj[:, 2]])
        sparse_point[name] = np.column_stack([xyz[sel], pid[sel].astype(np.float64)])
    predictions["sparse_depth"], predictions["sparse_point"] = sparse_depth, sparse_point
    return predictions


# ---------------------------------------------------------------------------------------------------------------------
# RANSAC samples (host side of the random-number pin)
# ---------------------------------------------------------------------------------------------------------------------
class _PairStream:
    """``sample_without_replacement(n, 2, random_state=RandomState(seed))`` repeated, drawn a chunk at a time."""

    def __init__(self, n, seed):
        self.n, self.rs, self.buf = n, np.random.RandomState(seed), np.empty(0, dtype=np.int64)

    def _need(self, k):
        if len(self.buf) < k:
            self.buf = np.concatenate([self.buf, self.rs.randint(self.n, size=max(k - len(self.buf), 64))])

    def take(self, T):
        n = self.n
        if n == 2:                                       # reservoir sampling of 2 out of 2: no draw
            return np.tile(np.array([0, 1], dtype=np.int32), (T, 1))
        if 2 / n > 0.01:                                 # permutation(n)[:2]
            return np.stack([self.rs.permutation(n)[:2] for _ in range(T)]).astype(np.int32)
        out = []                                         # tracking selection: randint(n) until unseen
        left = T
        while left:
            self._need(2 * left)
            a, b = self.buf[0:2 * left:2], self.buf[1:2 * left:2]
            coll = np.nonzero(a == b)[0]
            k = left if len(coll) == 0 else int(coll[0])
            out.append(np.stack([a[:k], b[:k]], axis=1))
            self.buf, left = self.buf[2 * k:], left - k
            if left:
                j0, pos = self.buf[0], 1
                while True:
                    self._need(pos + 1)
                    if self.buf[pos] != j0:
                        break
                    pos += 1
                out.append(np.array([[j0, self.buf[pos]]]))
                self.buf, left = self.buf[pos + 1:], left - 1
        return np.concatenate(out).astype(np.int32)


def _ransac(offsets, x, y, thresh, seeds, device, max_trials=MAX_TRIALS):
    """Batched RANSACRegressor.fit -> (scale f32 [F], shift f32 [F], n_trials [F], n_inliers [F], mask [n])."""
    L = _lib.lib()
    F = len(seeds)
    counts = np.diff(offsets.cpu().numpy())
    streams = [_PairStream(int(counts[f]), int(seeds[f])) for f in range(F)]
    ws_bytes = ctypes.c_size_t()
    _lib.check(L.vgg_depth_ransac_workspace_bytes(F, ctypes.byref(ws_bytes)), "vgg_depth_ransac_workspace_bytes")
    ws = torch.empty(ws_bytes.value, dtype=torch.uint8, device=device)
    stream = ctypes.c_void_p(torch.cuda.current_stream(device).cuda_stream)
    _lib.check(L.vgg_depth_ransac_begin(F, max_trials, _ptr(ws), ws_bytes.value, stream), "vgg_depth_ransac_begin")
    running = torch.ones(F, dtype=torch.uint8, device=device)
    live = np.arange(F)
    T, cap = FIRST_CHUNK, L.vgg_depth_ransac_max_chunk()
    while len(live):
        samples = np.stack([streams[f].take(T) for f in live])
        frames_d = torch.from_numpy(live.astype(np.int32)).to(device)
        samples_d = torch.from_numpy(samples).to(device)
        _lib.check(L.vgg_depth_ransac_chunk(F, _ptr(offsets), _ptr(x), _ptr(y), _ptr(thresh), len(live),
                                            _ptr(frames_d), T, _ptr(samples_d), _ptr(running), _ptr(ws),
                                            ws_bytes.value, stream), "vgg_depth_ransac_chunk")
        run = running.cpu().numpy()
        live = live[run[live] != 0]
        T = min(2 * T, cap)
    scale = torch.empty(F, dtype=torch.float32, device=device)
    shift = torch.empty_like(scale)
    n_trials = torch.empty(F, dtype=torch.int32, device=device)
    n_inl = torch.empty_like(n_trials)
    mask = torch.empty(len(x), dtype=torch.uint8, device=device)
    _lib.check(L.vgg_depth_ransac_finish(F, _ptr(offsets), _ptr(x), _ptr(y), _ptr(thresh), _ptr(scale), _ptr(shift),
                                         _ptr(n_trials), _ptr(n_inl), _ptr(mask), _ptr(ws), ws_bytes.value, stream),
               "vgg_depth_ransac_finish")
    return scale, shift, n_trials, n_inl, mask


# ---------------------------------------------------------------------------------------------------------------------
# the whole stage
# ---------------------------------------------------------------------------------------------------------------------
def _batches(shapes, bytes_per_pixel, budget):
    out, cur, used = [], [], 0
    for i, (h, w) in enumerate(shapes):
        b = h * w * bytes_per_pixel
        if cur and used + b > budget:
            out.append(cur)
            cur, used = [], 0
        cur.append(i)
        used += b
    if cur:
        out.append(cur)
    return out


def _pinned(n, dtype):
    return torch.empty(n, dtype=dtype, pin_memory=True)


def align_dense_depth_maps(reconstruction, sparse_depth, disp_dict, original_images, visual_dense_point_cloud=False,
                           *, seeds=None, device="cuda", memory_budget=8 << 30, return_debug=False):
    """vggsfm/utils/utils.py:635-770, same arguments and return ``(depth_dict, unproj_dense_points3D)``.

    ``disp_dict[name]`` must be a float32 [H, W] numpy array; it is rescaled in place, as the reference does.
    ``seeds`` (one per frame of ``sparse_depth``, in its order) pins each frame's RANSAC draws; by default they are
    drawn from numpy's global generator.  ``memory_budget`` bounds the device bytes of one batch of frames.
    ``return_debug`` adds a third element with the per-frame RANSAC results (scale, shift, n_trials, n_inliers,
    inlier masks over the kept samples, samples x / y, thresholds)."""
    device = torch.device(device)
    if device.type != "cuda":
        raise ValueError("align_dense_depth_maps runs on a CUDA device")
    L = _lib.lib()
    names = list(sparse_depth)
    F = len(names)
    uvds = [np.asarray(sparse_depth[nm], dtype=np.float64).reshape(-1, 3) for nm in names]
    for u in uvds:
        if len(u) <= 0:
            raise ValueError("Too few points for depth alignment")
    maps = [disp_dict[nm] for nm in names]
    for nm, m in zip(names, maps):
        if not (isinstance(m, np.ndarray) and m.dtype == np.float32 and m.ndim == 2):
            raise TypeError(f"disp_dict[{nm!r}] must be a float32 [H, W] numpy array")
    if seeds is None:
        seeds = np.random.randint(0, 2**32, size=F, dtype=np.int64)
    seeds = np.asarray(seeds, dtype=np.int64)
    if len(seeds) != F:
        raise ValueError("seeds needs one entry per frame of sparse_depth")
    shapes = [m.shape for m in maps]
    stream = ctypes.c_void_p(torch.cuda.current_stream(device).cuda_stream)
    per_pixel = 4 + 4 + (3 + 48 if visual_dense_point_cloud else 0)
    batches = _batches(shapes, per_pixel, memory_budget)

    def upload(idx):
        npix = np.array([shapes[i][0] * shapes[i][1] for i in idx], dtype=np.int64)
        moff = np.concatenate([[0], np.cumsum(npix)])
        host = _pinned(int(moff[-1]), torch.float32)
        hn = host.numpy()
        for k, i in enumerate(idx):
            hn[moff[k]:moff[k + 1]] = maps[i].reshape(-1)
        disp = host.to(device, non_blocking=True)
        hw = torch.tensor([shapes[i] for i in idx], dtype=torch.int32).reshape(-1, 2).to(device)
        return disp, torch.from_numpy(moff).to(device), hw, moff

    # 1. sparse samples: nearest-pixel disparity, clipped target disparity (utils.py:669-690)
    xs, ys, fids, kept = [], [], [], []
    resident = None
    for idx in batches:
        disp, moff_d, hw, moff = upload(idx)
        if len(batches) == 1:
            resident = (disp, moff_d, hw, moff)
        uvd = np.concatenate([uvds[i] for i in idx])
        fid = np.repeat(np.arange(len(idx), dtype=np.int32), [len(uvds[i]) for i in idx])
        n = len(uvd)
        uvd_d = torch.from_numpy(uvd).to(device)
        fid_d = torch.from_numpy(fid).to(device)
        x = torch.empty(n, dtype=torch.float32, device=device)
        y = torch.empty(n, dtype=torch.float64, device=device)
        keep = torch.empty(n, dtype=torch.uint8, device=device)
        _lib.check(L.vgg_depth_sparse_samples(n, _ptr(fid_d), _ptr(uvd_d), DEPTH_MIN, DEPTH_MAX, _ptr(moff_d),
                                              _ptr(hw), _ptr(disp), _ptr(x), _ptr(y), _ptr(keep), stream),
                   "vgg_depth_sparse_samples")
        k = keep.bool()
        xs.append(x[k])
        ys.append(y[k])
        fids.append(fid_d[k].long() + int(idx[0]))
    x, y, fid = torch.cat(xs), torch.cat(ys), torch.cat(fids)
    counts = torch.bincount(fid, minlength=F)
    cnt_host = counts.cpu().numpy()
    for f in range(F):
        if cnt_host[f] < 2:
            raise ValueError("`min_samples` may not be larger than number of samples: n_samples = %d."
                             % cnt_host[f])
    offsets = torch.zeros(F + 1, dtype=torch.int32, device=device)
    offsets[1:] = torch.cumsum(counts, 0).to(torch.int32)

    # 2. threshold = np.median(y) / 30, then RANSAC on every frame at once
    thresh = torch.empty(F, dtype=torch.float64, device=device)
    _lib.check(L.vgg_depth_median(F, _ptr(offsets), _ptr(y), float(THRES_RATIO), _ptr(thresh), stream),
               "vgg_depth_median")
    if bool((thresh <= 0).any()):
        raise ValueError("Ill-posed scene for depth alignment")
    scale, shift, n_trials, n_inl, mask = _ransac(offsets, x, y, thresh, seeds, device)
    if bool((n_inl < 0).any()):
        raise ValueError("RANSAC could not find a valid consensus set. All `max_trials` iterations were skipped "
                         "because each randomly chosen sub-sample failed the passing criteria. See estimator "
                         "attributes for diagnostics (n_skips*).")

    # 3. rescale, clip, depth and (optionally) the coloured point cloud, one batch of frames at a time
    tile = L.vgg_depth_tile_pixels()
    depth_dict, points = {}, {}
    for idx in batches:
        disp, moff_d, hw, moff = resident if resident is not None else upload(idx)
        B = len(idx)
        npix = np.diff(moff)
        toff = np.concatenate([[0], np.cumsum((npix + tile - 1) // tile)]).astype(np.int64)
        n_tiles = int(toff[-1])
        toff_d = torch.from_numpy(toff).to(device)
        sel = torch.tensor(idx, dtype=torch.long, device=device)
        sc, sh = scale[sel].contiguous(), shift[sel].contiguous()
        depth = torch.empty_like(disp)
        tcount = torch.empty(n_tiles, dtype=torch.int32, device=device) if visual_dense_point_cloud else None
        _lib.check(L.vgg_depth_apply(B, n_tiles, _ptr(moff_d), _ptr(toff_d), _ptr(sc), _ptr(sh), _ptr(disp),
                                     _ptr(depth), _ptr(tcount), stream), "vgg_depth_apply")
        if visual_dense_point_cloud:
            tbase = torch.zeros(n_tiles + 1, dtype=torch.int64, device=device)
            tbase[1:] = torch.cumsum(tcount, 0)
            rgb_host = _pinned(int(moff[-1]) * 3, torch.uint8)
            rn = rgb_host.numpy()
            for k, i in enumerate(idx):
                img = np.asarray(original_images[names[i]], dtype=np.uint8)
                rn[3 * moff[k]:3 * moff[k + 1]] = img.reshape(-1)
            rgb = rgb_host.to(device, non_blocking=True)
            images = reconstruction.images
            fname_to_id = {images[i].name: i for i in images}
            model = np.zeros(B, dtype=np.int32)
            params = np.zeros((B, 4))
            wfc = np.zeros((B, 3, 4))
            for k, i in enumerate(idx):
                im = images[fname_to_id[names[i]]]
                cam = reconstruction.cameras[im.camera_id]
                model[k] = _CAMERA_MODELS[cam.model]
                params[k, :len(cam.params)] = cam.params
                wfc[k] = im.cam_from_world.inverse().matrix()
            M = int(tbase[-1].item())
            out = torch.empty(6 * M, dtype=torch.float64, device=device)
            model_d, params_d, wfc_d = (torch.from_numpy(a).to(device) for a in (model, params, wfc))
            _lib.check(L.vgg_depth_unproject(B, n_tiles, _ptr(moff_d), _ptr(hw), _ptr(toff_d), _ptr(tbase),
                                             _ptr(depth), _ptr(rgb), _ptr(model_d), _ptr(params_d), _ptr(wfc_d),
                                             _ptr(out), stream), "vgg_depth_unproject")
            out_host = _pinned(6 * M, torch.float64)
            out_host.copy_(out)
            on = out_host.numpy()
            fb = tbase[torch.from_numpy(toff).to(device)].cpu().numpy()
            for k, i in enumerate(idx):
                points[names[i]] = on[6 * fb[k]:6 * fb[k + 1]].reshape(2, -1, 3)
        dh = _pinned(int(moff[-1]), torch.float32)
        dh.copy_(depth)
        disp_h = _pinned(int(moff[-1]), torch.float32)
        disp_h.copy_(disp)
        dn, pn = dh.numpy(), disp_h.numpy()
        for k, i in enumerate(idx):
            depth_dict[names[i]] = dn[moff[k]:moff[k + 1]].reshape(shapes[i])
            maps[i][...] = pn[moff[k]:moff[k + 1]].reshape(shapes[i])      # the reference rescales in place
    result = (depth_dict, points if visual_dense_point_cloud else None)
    if return_debug:
        offs = offsets.cpu().numpy()
        m, xh, yh = mask.cpu().numpy().astype(bool), x.cpu().numpy(), y.cpu().numpy()
        dbg = dict(scale=scale.cpu().numpy(), shift=shift.cpu().numpy(), n_trials=n_trials.cpu().numpy(),
                   n_inliers=n_inl.cpu().numpy(), threshold=thresh.cpu().numpy(), seeds=seeds,
                   inlier_mask=[m[offs[f]:offs[f + 1]] for f in range(F)],
                   x=[xh[offs[f]:offs[f + 1]] for f in range(F)], y=[yh[offs[f]:offs[f + 1]] for f in range(F)])
        result = result + (dbg,)
    return result
