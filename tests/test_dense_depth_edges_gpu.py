"""GPU: the dense depth stage's entry points (csrc/dense_depth.cu through _lib) at their edges, against
oracle/dense_depth_oracle.py and the reference's numpy statements.

- vgg_depth_sparse_samples: x, y and keep bitwise per observation before compaction, at half-pixel and non-finite
  coordinates, clip-edge and non-finite depths, and zero / negative / NaN / +inf / subnormal / FLT_MAX disparities,
  on 1 x 1, 1 x W and H x 1 maps.
- vgg_depth_median: bitwise against np.median(y) / 30 over a CSR of frames, including chains of adjacent doubles that
  make the radix select decide in every byte, and an empty frame (NaN).
- RANSAC through begin / chunk / finish: n_trials, n_inliers and the mask equal the oracle's, and scale / shift within
  the bars of test_dense_depth_gpu.check_fit; all five outputs bitwise equal across chunk schedules (the host's
  doubling, T = 1, one maximal chunk, irregular T, live frames in a permuted non-contiguous order).  Offset-dominated
  disparities, the exact tie, the no-consensus path, perfect data, all-equal x, n = 2, max_trials around the chunk
  sizes, a 2e5-sample frame, and VGG_EINVAL with the outputs untouched.
- vgg_depth_apply / vgg_depth_unproject: bitwise against apply_scale and a restatement of the unprojection fed the
  same world_from_cam, tile counts, every output position written once in np.nonzero order, frames without pixels
  (an empty [2, 0, 3] block), and kept pixels whose depth 1 / disp overflowed to 0 (the reference keeps them).
- align_dense_depth_maps: the reference's errors for the first failing frame, and batching by memory_budget bitwise
  equal to one batch."""
import ctypes

import numpy as np
import pytest
import torch

from oracle import dense_depth_oracle as O
from tests.test_dense_depth_gpu import _scene, check_fit
from vggsfm_b200 import _lib, dense_depth

pytestmark = pytest.mark.gpu
f32 = np.float32


def _p(t):
    return ctypes.c_void_p(t.data_ptr()) if t is not None else None


_HELD = []


def _d(a, dev):
    """A device copy that stays alive until the test ends: a temporary passed as a raw pointer would go back to the
    caching allocator at once, and the next copy of the same call could reuse its memory before the kernel runs."""
    t = torch.from_numpy(np.ascontiguousarray(a)).to(dev)
    _HELD.append(t)
    return t


@pytest.fixture(autouse=True)
def _release_held():
    yield
    torch.cuda.synchronize()
    _HELD.clear()


def _bits_equal(a, b):
    a, b = np.asarray(a), np.asarray(b)
    assert a.shape == b.shape and a.dtype == b.dtype
    nan = np.isnan(a)
    np.testing.assert_array_equal(nan, np.isnan(b))
    u = np.uint32 if a.dtype == np.float32 else np.uint64
    np.testing.assert_array_equal(a[~nan].view(u), b[~nan].view(u))


# ---------------------------------------------------------------------------------------------------------------------
# sparse samples
# ---------------------------------------------------------------------------------------------------------------------
def _samples_reference(maps, uvd, fid):
    """utils.py:669-690 per observation, before compaction -> (x float32, y float64, keep)."""
    n = len(uvd)
    x, keep = np.zeros(n, f32), np.zeros(n, bool)
    with np.errstate(invalid="ignore"):
        iu = np.round(uvd[:, :2]).astype(int)          # NaN, inf and beyond int64 become INT64_MIN: out of bounds
        y = 1 / np.clip(uvd[:, 2], O.DEPTH_MIN, O.DEPTH_MAX)
    for i in range(n):
        m = maps[fid[i]]
        H, W = m.shape
        if 0 <= iu[i, 0] < W and 0 <= iu[i, 1] < H:
            x[i] = m[iu[i, 1], iu[i, 0]]
        with np.errstate(invalid="ignore"):
            keep[i] = x[i] > 0
    return x, y, keep


def test_sparse_samples_edges(cuda_dev):
    L = _lib.lib()
    sub, fmax = float(np.finfo(f32).smallest_subnormal), float(np.finfo(f32).max)
    dmin, dmax = O.DEPTH_MIN, O.DEPTH_MAX
    depths = [0.0, -0.0, -2.0, np.nan, np.inf, -np.inf, dmin, dmax, np.nextafter(dmin, 0), np.nextafter(dmax, np.inf),
              np.nextafter(dmin, 1), np.nextafter(dmax, 0), 0.37]
    rng = np.random.default_rng(0)
    maps = [rng.uniform(0.1, 2, (6, 9)).astype(f32), np.full((1, 1), 0.5, f32), rng.uniform(0.1, 2, (1, 7)).astype(f32),
            rng.uniform(0.1, 2, (5, 1)).astype(f32)]
    maps[0].reshape(-1)[:8] = [0.0, -0.0, -1.0, np.nan, np.inf, sub, fmax, -np.inf]
    rows, fid = [], []
    for f, m in enumerate(maps):
        H, W = m.shape
        coords = [-0.5, -0.5000001, 0.5, 1.5, 2.5, W - 0.5, H - 0.5, W - 1.5, np.nan, np.inf, -np.inf, 1e19, -1e19,
                  2.0 ** 31, 2.0 ** 53, 0.49999997, 3.5000002]
        for u in coords:
            for v in coords[:8] + [np.nan, 2.0 ** 31]:
                rows.append((u, v, depths[len(rows) % len(depths)]))
                fid.append(f)
        if f == 0:                                       # every special disparity with every special depth
            for k in range(8):
                for d in depths:
                    rows.append((k % 9, k // 9, d))
                    fid.append(0)
    uvd, fid = np.array(rows), np.array(fid, np.int32)
    moff = np.concatenate([[0], np.cumsum([m.size for m in maps])]).astype(np.int64)
    hw = np.array([m.shape for m in maps], np.int32)
    disp = np.concatenate([m.reshape(-1) for m in maps])
    n = len(uvd)
    x, y, keep = (torch.empty(n, dtype=t, device=cuda_dev) for t in (torch.float32, torch.float64, torch.uint8))
    _lib.check(L.vgg_depth_sparse_samples(n, _p(_d(fid, cuda_dev)), _p(_d(uvd, cuda_dev)), dmin, dmax,
                                          _p(_d(moff, cuda_dev)), _p(_d(hw, cuda_dev)), _p(_d(disp, cuda_dev)), _p(x),
                                          _p(y), _p(keep), None), "samples")
    torch.cuda.synchronize()
    xr, yr, kr = _samples_reference(maps, uvd, fid)
    _bits_equal(x.cpu().numpy(), xr)
    _bits_equal(y.cpu().numpy(), yr)
    np.testing.assert_array_equal(keep.cpu().numpy().astype(bool), kr)
    assert kr.sum() > 50 and (~kr).sum() > 50


# ---------------------------------------------------------------------------------------------------------------------
# median
# ---------------------------------------------------------------------------------------------------------------------
def test_median_bitwise(cuda_dev):
    L = _lib.lib()
    rng = np.random.default_rng(1)
    chain = lambda v, k: np.array([v] + [v := np.nextafter(v, np.inf) for _ in range(k - 1)])  # noqa: E731
    frames = [rng.uniform(0.1, 1, n) for n in (1, 2, 3, 255, 256, 257)]
    frames += [np.full(100, 0.3), np.full(101, 0.3), np.array([]), rng.uniform(0.1, 1, 10 ** 6)]
    frames += [rng.permutation(chain(0.7, 513)), rng.permutation(chain(1.0, 300)),
               rng.permutation(chain(2.0 ** -20, 64))]
    frames += [10.0 ** rng.uniform(-4, 4, 4001), np.array([]), np.array([0.5, 0.2, 0.2, 0.9]),
               np.array([0.1, 0.4, 0.4, 0.4, 0.9, 1.0])]
    # values whose bit patterns differ only in byte b, for each b: every radix step has to decide
    for b in range(8):
        base = np.float64(1.5).view(np.uint64)
        v = (base & ~np.uint64(0xff << (8 * b))) | (np.arange(1, 40, dtype=np.uint64) << np.uint64(8 * b))
        frames.append(rng.permutation(v.view(np.float64)[np.isfinite(v.view(np.float64))]))
    offs = np.concatenate([[0], np.cumsum([len(f) for f in frames])]).astype(np.int32)
    y = _d(np.concatenate(frames), cuda_dev)
    med = torch.empty(len(frames), dtype=torch.float64, device=cuda_dev)
    _lib.check(L.vgg_depth_median(len(frames), _p(_d(offs, cuda_dev)), _p(y), 30.0, _p(med), None), "median")
    got = med.cpu().numpy()
    with np.errstate(invalid="ignore"), pytest.warns(RuntimeWarning):
        ref = np.array([np.median(f) / 30 for f in frames])
    _bits_equal(got, ref)
    assert np.isnan(got[8]) and np.isnan(got[14])


# ---------------------------------------------------------------------------------------------------------------------
# RANSAC through begin / chunk / finish
# ---------------------------------------------------------------------------------------------------------------------
def _schedule(name, cap):
    if name == "double":
        return lambda k: min(32 << min(k, 20), cap)
    if name == "one":
        return lambda k: 1
    if name == "max":
        return lambda k: cap
    irregular = [3, 1, 4093, 4096, 4096, 4096, 3610, 7, 29, 4096, 2]
    return lambda k: irregular[k % len(irregular)]


def _ransac(frames, seeds, dev, schedule="double", max_trials=O.MAX_TRIALS, permute=False):
    """frames: [(X float32, y float64, threshold)] -> dict of scale, shift, n_trials, n_inliers, per-frame masks."""
    L = _lib.lib()
    F = len(frames)
    offs = np.concatenate([[0], np.cumsum([len(X) for X, _, _ in frames])]).astype(np.int32)
    offs_d = _d(offs, dev)
    x = _d(np.concatenate([X for X, _, _ in frames]).astype(f32), dev)
    y = _d(np.concatenate([yy for _, yy, _ in frames]).astype(np.float64), dev)
    th = _d(np.array([t for _, _, t in frames], np.float64), dev)
    wsb = ctypes.c_size_t()
    _lib.check(L.vgg_depth_ransac_workspace_bytes(F, ctypes.byref(wsb)), "ws")
    ws = torch.empty(wsb.value, dtype=torch.uint8, device=dev)
    _lib.check(L.vgg_depth_ransac_begin(F, max_trials, _p(ws), wsb.value, None), "begin")
    cap = L.vgg_depth_ransac_max_chunk()
    T_of = _schedule(schedule, cap)
    streams = [dense_depth._PairStream(len(X), int(s)) for (X, _, _), s in zip(frames, seeds)]
    running = torch.ones(F, dtype=torch.uint8, device=dev)
    live, k, rng = np.arange(F), 0, np.random.default_rng(0)
    while len(live):
        T = T_of(k)
        order = rng.permutation(live) if permute else live
        samples = np.stack([streams[f].take(T) for f in order])
        frames_d = _d(order.astype(np.int32), dev)
        _lib.check(L.vgg_depth_ransac_chunk(F, _p(offs_d), _p(x), _p(y), _p(th), len(order), _p(frames_d),
                                            T, _p(_d(samples, dev)), _p(running), _p(ws), wsb.value, None), "chunk")
        run = running.cpu().numpy()
        live = live[run[live] != 0]
        k += 1
    empty = lambda n, t: torch.empty(n, dtype=t, device=dev)  # noqa: E731
    out = dict(scale=empty(F, torch.float32), shift=empty(F, torch.float32), n_trials=empty(F, torch.int32),
               n_inliers=empty(F, torch.int32), mask=empty(len(x), torch.uint8))
    _lib.check(L.vgg_depth_ransac_finish(F, _p(offs_d), _p(x), _p(y), _p(th), _p(out["scale"]), _p(out["shift"]),
                                         _p(out["n_trials"]), _p(out["n_inliers"]), _p(out["mask"]), _p(ws), wsb.value,
                                         None), "finish")
    out = {key: v.cpu().numpy() for key, v in out.items()}
    out["mask"] = [out["mask"][offs[f]:offs[f + 1]].astype(bool) for f in range(F)]
    return out


def _line_frame(rng, n, x0, spread, ratio=0.8, noise=1e-4):
    """n samples: disparities x0 + U(0, spread), a fraction `ratio` on y = 0.5 (x - x0) / spread + 0.2 (+ noise)."""
    X = (x0 + rng.uniform(0, spread, n)).astype(f32)
    y = 0.5 * (X.astype(np.float64) - x0) / spread + 0.2 + rng.normal(0, noise, n)
    out = rng.uniform(size=n) > ratio
    y[out] = rng.uniform(1.0, 3.0, out.sum())
    return X, y, np.median(y) / O.THRES_RATIO


def _check_against_oracle(frames, seeds, got, max_trials=O.MAX_TRIALS, margins=True):
    worst = 0.0
    for f, ((X, y, th), s) in enumerate(zip(frames, seeds)):
        r = O.ransac_fit(X, y, th, int(s), max_trials, return_debug=True)
        if margins:
            assert r["debug"]["residual_margin"] > 1e-9 and r["debug"]["score_gap"] > 1e-12, f
        assert got["n_trials"][f] == r["n_trials"], (f, got["n_trials"][f], r["n_trials"])
        assert got["n_inliers"][f] == r["n_inliers"], f
        np.testing.assert_array_equal(got["mask"][f], r["inlier_mask"])
        worst = max(worst, check_fit(got["scale"][f], got["shift"][f], X, y, r, f"frame {f}"))
    print(f"largest shift error / bar: {worst:.3g}")


def _same(a, b):
    for key in ("scale", "shift"):
        np.testing.assert_array_equal(a[key].view(np.uint32), b[key].view(np.uint32))
    for key in ("n_trials", "n_inliers"):
        np.testing.assert_array_equal(a[key], b[key])
    for ma, mb in zip(a["mask"], b["mask"]):
        np.testing.assert_array_equal(ma, mb)


OFFSET_CASES = [(1000.0, 0.05, 300), (1000.0, 0.05, 100_000), (100.0, 0.01, 100_000), (1.0, 1e-4, 300)]


def test_offset_dominated_disparities(cuda_dev):
    """Inlier disparities with a large offset: the final fit's means must be numpy's float32 pairwise means."""
    rng = np.random.default_rng(2)
    frames, seeds = [], []
    for x0, spread, n in OFFSET_CASES:
        for _ in range(3):
            frames.append(_line_frame(rng, n, x0, spread))
            seeds.append(int(rng.integers(2 ** 31)))
    got = _ransac(frames, seeds, cuda_dev)
    _check_against_oracle(frames, seeds, got)


def _mixed_frames(rng):
    frames, seeds = [], []
    for n, ratio in ((2, 1.0), (3, 0.7), (9, 0.8), (200, 0.5), (700, 0.9), (4096, 0.3), (200_000, 0.6)):
        frames.append(_line_frame(rng, n, 0.5, 1.0, ratio, noise=1e-3))
        seeds.append(int(rng.integers(2 ** 31)))
    X = rng.uniform(0.2, 1, 3000).astype(f32)                                  # pure noise: runs to the cap
    y = rng.uniform(1, 1e4, 3000)
    frames.append((X, y, np.median(y) / O.THRES_RATIO))
    seeds.append(int(rng.integers(2 ** 31)))
    return frames, seeds


def test_chunk_schedules_are_bitwise_equal(cuda_dev):
    rng = np.random.default_rng(3)
    frames, seeds = _mixed_frames(rng)
    base = _ransac(frames, seeds, cuda_dev)
    _check_against_oracle(frames, seeds, base)
    assert base["n_trials"][-1] == O.MAX_TRIALS
    for schedule, permute in (("one", False), ("max", False), ("irregular", False), ("double", True),
                              ("irregular", True)):
        if schedule == "one":                                                  # early-stopping frames only
            sub = [i for i in range(len(frames)) if base["n_trials"][i] < 200]
            got = _ransac([frames[i] for i in sub], [seeds[i] for i in sub], cuda_dev, schedule, permute=permute)
            _same(got, {k: (v[sub] if k != "mask" else [v[i] for i in sub]) for k, v in base.items()})
        else:
            _same(_ransac(frames, seeds, cuda_dev, schedule, permute=permute), base)


@pytest.mark.parametrize("max_trials", [1, 2, 31, 32, 33, 4097])
def test_max_trials_on_noise(cuda_dev, max_trials):
    rng = np.random.default_rng(4)
    frames, seeds = [], []
    for n in (50, 400):
        X = rng.uniform(0.2, 1, n).astype(f32)
        y = rng.uniform(1, 1e4, n)                                             # targets far beyond the threshold
        frames.append((X, y, np.median(y) / O.THRES_RATIO))
        seeds.append(int(rng.integers(2 ** 31)))
    for schedule in ("double", "irregular"):
        got = _ransac(frames, seeds, cuda_dev, schedule, max_trials=max_trials)
        _check_against_oracle(frames, seeds, got, max_trials, margins=False)
        assert (got["n_trials"] <= max_trials).all()


def test_degenerate_frames(cuda_dev):
    rng = np.random.default_rng(5)
    Xp = rng.uniform(0.2, 1, 64).astype(f32)
    perfect = (Xp, Xp.astype(np.float64) * 0 + 0.25, 0.25 / 30)            # every trial fits all: 1 trial
    Xe = np.full(50, 0.75, f32)
    ye = 0.3 + rng.normal(0, 1e-4, 50)
    equal_x = (Xe, ye, np.median(ye) / 30)                                   # scale 0 in trial and final fit
    two = (np.array([0.3, 0.9], f32), np.array([0.2, 0.5]), np.median([0.2, 0.5]) / 30)
    frames = [perfect, equal_x, two]
    seeds = [11, 12, 13]
    got = _ransac(frames, seeds, cuda_dev)
    _check_against_oracle(frames, seeds, got, margins=False)
    assert got["n_trials"][0] == 1 and got["n_inliers"][0] == 64
    assert got["scale"][1] == 0 and got["n_trials"][2] == 1


def test_no_consensus_and_exact_tie(cuda_dev):
    """Threshold 0 with targets float32 does not represent: every trial has no inlier, so none is kept (n_inliers -1,
    n_trials = max_trials, scale and shift 0, where sklearn raises).  The exact tie: the later group wins."""
    rng = np.random.default_rng(6)
    Xn = rng.uniform(0.2, 1, 30).astype(f32)
    none = (Xn, np.full(30, 0.1), 0.0)
    Xt, yt, tht, group = O.tie_fixture(3)
    seeds = list(range(40))
    frames = [none] + [(Xt, yt, tht)] * len(seeds)
    for schedule in ("double", "one", "irregular"):
        got = _ransac(frames, [0] + seeds, cuda_dev, schedule, max_trials=50)
        assert got["n_inliers"][0] == -1 and got["n_trials"][0] == 50
        assert got["scale"][0] == 0 and got["shift"][0] == 0 and not got["mask"][0].any()
        for f, s in enumerate(seeds, 1):
            r = O.ransac_fit(Xt, yt, tht, s, 50, return_debug=True)
            assert got["n_trials"][f] == r["n_trials"] == 17
            np.testing.assert_array_equal(got["mask"][f], r["inlier_mask"])
            assert got["scale"][f] == 0 and got["shift"][f] == r["intercept"]
    with pytest.raises(ValueError, match="could not find a valid consensus"):
        O.ransac_fit(*none, 0, 50)


def test_invalid_arguments_touch_nothing(cuda_dev):
    L = _lib.lib()
    F = 3
    wsb = ctypes.c_size_t()
    _lib.check(L.vgg_depth_ransac_workspace_bytes(F, ctypes.byref(wsb)), "ws")
    ws = torch.zeros(wsb.value, dtype=torch.uint8, device=cuda_dev)
    offs = _d(np.array([0, 4, 8, 12], np.int32), cuda_dev)
    x = torch.rand(12, device=cuda_dev)
    y = torch.rand(12, dtype=torch.float64, device=cuda_dev)
    th = torch.full((F,), 0.1, dtype=torch.float64, device=cuda_dev)
    frames = _d(np.arange(F, dtype=np.int32), cuda_dev)
    cap = L.vgg_depth_ransac_max_chunk()
    samples = torch.zeros(F * (cap + 1) * 2, dtype=torch.int32, device=cuda_dev)
    running = torch.full((F,), 7, dtype=torch.uint8, device=cuda_dev)
    assert L.vgg_depth_ransac_begin(F, 100, _p(ws), wsb.value - 1, None) == -1
    assert L.vgg_depth_ransac_begin(F, 0, _p(ws), wsb.value, None) == -1
    for R, T, nbytes, FF in ((F, 0, wsb.value, F), (F, cap + 1, wsb.value, F), (F + 1, 1, wsb.value, F),
                             (65536, 1, 0, 65536), (F, 1, wsb.value - 1, F)):
        rc = L.vgg_depth_ransac_chunk(FF, _p(offs), _p(x), _p(y), _p(th), R, _p(frames), T, _p(samples), _p(running),
                                      _p(ws) if nbytes else None, nbytes, None)
        assert rc == -1, (R, T, nbytes)
        if R == 65536:
            assert "65535" in L.vgg_last_error().decode()
    outs = [torch.full((F,), 5, dtype=t, device=cuda_dev) for t in (torch.float32, torch.float32, torch.int32,
                                                                       torch.int32)]
    mask = torch.full((12,), 9, dtype=torch.uint8, device=cuda_dev)
    assert L.vgg_depth_ransac_finish(F, _p(offs), _p(x), _p(y), _p(th), *[_p(o) for o in outs], _p(mask), _p(ws),
                                     wsb.value - 1, None) == -1
    torch.cuda.synchronize()
    assert (running == 7).all() and (mask == 9).all() and all((o == 5).all() for o in outs)
    assert (ws == 0).all()


# ---------------------------------------------------------------------------------------------------------------------
# apply and unproject
# ---------------------------------------------------------------------------------------------------------------------
def _tiles(npix, tile):
    return np.concatenate([[0], np.cumsum((npix + tile - 1) // tile)]).astype(np.int64)


def test_apply_bitwise_and_tile_counts(cuda_dev):
    L = _lib.lib()
    tile = L.vgg_depth_tile_pixels()
    rng = np.random.default_rng(7)
    shapes = [(1, 1), (1, 2047), (2047, 1), (1, 2048), (7, 293), (1, 4097), (3, 2048), (0, 5), (1, 5000), (0, 0)]
    shapes += [(int(rng.integers(1, 40)), int(rng.integers(1, 90))) for _ in range(1000)]
    shapes.insert(500, (0, 17))
    sub = float(np.finfo(f32).smallest_subnormal)
    special = np.array([0.0, -0.0, np.nan, np.inf, -np.inf, sub, -sub, 1e30, -1e30, 3.0, -3.0], f32)
    maps, scales, shifts = [], [], []
    for k, (H, W) in enumerate(shapes):
        m = rng.uniform(-0.5, 2, (H, W)).astype(f32)
        flat = m.reshape(-1)
        flat[rng.uniform(size=flat.size) < 0.1] = 0
        sc, sh = f32(rng.choice([1.0, 0.7, -0.4, 3e37])), f32(rng.uniform(-0.2, 0.2))
        if flat.size >= 16:
            flat[:len(special)] = special
            # exactly 10000, the next float above, and d * sc == -sh (a result of exactly 0)
            flat[11] = (f32(10000) - sh) / sc if sc != 0 else 0
            flat[12] = f32(1.0)
            flat[13] = -sh / sc if sc != 0 else 0
        maps.append(m)
        scales.append(sc)
        shifts.append(sh)
    # frame 3: scale 1 and shift 0, so its values are the results themselves
    scales[3], shifts[3] = f32(1), f32(0)
    maps[3].reshape(-1)[:3] = [10000, np.nextafter(f32(10000), f32(np.inf)), np.nextafter(f32(10000), f32(0))]
    npix = np.array([m.size for m in maps], np.int64)
    moff = np.concatenate([[0], np.cumsum(npix)]).astype(np.int64)
    toff = _tiles(npix, tile)
    disp = _d(np.concatenate([m.reshape(-1) for m in maps]), cuda_dev)
    depth = torch.full_like(disp, np.nan)
    counts = torch.full((int(toff[-1]),), -1, dtype=torch.int32, device=cuda_dev)
    _lib.check(L.vgg_depth_apply(len(maps), int(toff[-1]), _p(_d(moff, cuda_dev)), _p(_d(toff, cuda_dev)),
                                 _p(_d(np.array(scales, f32), cuda_dev)), _p(_d(np.array(shifts, f32), cuda_dev)),
                                 _p(disp), _p(depth), _p(counts), None), "apply")
    dn, pn, cn = disp.cpu().numpy(), depth.cpu().numpy(), counts.cpu().numpy()
    with np.errstate(all="ignore"):
        for k, m in enumerate(maps):
            dref, depref, valid = O.apply_scale(m, scales[k], shifts[k])
            _bits_equal(dn[moff[k]:moff[k + 1]], dref.reshape(-1))
            _bits_equal(pn[moff[k]:moff[k + 1]], depref.reshape(-1))
            v = valid.reshape(-1)
            ref_counts = [int(v[t * tile:(t + 1) * tile].sum()) for t in range(int(toff[k + 1] - toff[k]))]
            np.testing.assert_array_equal(cn[toff[k]:toff[k + 1]], ref_counts)
    assert dn[moff[3]] == 10000 and dn[moff[3] + 1] == 0


def test_unproject_positions_and_values(cuda_dev):
    L = _lib.lib()
    tile = L.vgg_depth_tile_pixels()
    rng = np.random.default_rng(8)
    shapes = [(3, 5000), (5000, 1), (4, 4), (1, 1), (2, 3000), (9, 700)]
    models = [0, 1, 0, 0, 0, 1]
    depths, rgbs, params, wfc = [], [], [], []
    edges = [0, 1, 30, 31, 32, 255, 256, 257, 2047, 2048, 2049, 4095, 4096, 6143, 6144]
    for k, (H, W) in enumerate(shapes):
        n = H * W
        d = np.zeros(n, f32)
        if k not in (2, 3):                                                  # frames 2, 3: no valid pixel
            pos = [p for p in edges if p < n] + [p - 1 for p in range(tile, n + 1, tile)]
            d[np.array(sorted(set(pos)))] = rng.uniform(0.5, 4, len(set(pos))).astype(f32)
        depths.append(d.reshape(H, W))
        rgbs.append(rng.integers(0, 256, (H, W, 3), dtype=np.uint8))
        k_rad = -0.9 if k == 5 else -0.05                                    # frame 5: Newton does not converge
        params.append([0.8 * max(H, W), W / 2, H / 2, k_rad])
        R = np.linalg.qr(rng.normal(size=(3, 3)))[0]
        wfc.append(np.column_stack([R, rng.normal(size=3)]))
    npix = np.array([d.size for d in depths], np.int64)
    moff = np.concatenate([[0], np.cumsum(npix)]).astype(np.int64)
    toff = _tiles(npix, tile)
    flat = np.concatenate([d.reshape(-1) for d in depths])
    valid = (flat != 0).astype(f32)                   # the rescaled disparity: validity comes from it, not the depth
    valid[[moff[0] + 100, moff[0] + 2050]] = 1.0      # kept pixels whose 1 / disp overflowed: depth 0, still points
    counts = np.array([int((valid[moff[k] + t * tile: min(moff[k] + (t + 1) * tile, moff[k + 1])] != 0).sum())
                       for k in range(len(shapes)) for t in range(int(toff[k + 1] - toff[k]))])
    tbase = np.concatenate([[0], np.cumsum(counts)]).astype(np.int64)
    M = int(tbase[-1])
    out = torch.full((6 * M,), np.nan, dtype=torch.float64, device=cuda_dev)
    hw = np.array(shapes, np.int32)
    _lib.check(L.vgg_depth_unproject(len(shapes), int(toff[-1]), _p(_d(moff, cuda_dev)), _p(_d(hw, cuda_dev)),
                                     _p(_d(toff, cuda_dev)), _p(_d(tbase, cuda_dev)), _p(_d(flat, cuda_dev)),
                                     _p(_d(valid, cuda_dev)),
                                     _p(_d(np.concatenate([r.reshape(-1) for r in rgbs]), cuda_dev)),
                                     _p(_d(np.array(models, np.int32), cuda_dev)),
                                     _p(_d(np.array(params), cuda_dev)), _p(_d(np.array(wfc), cuda_dev)), _p(out),
                                     None), "unproject")
    on = out.cpu().numpy()
    assert not np.isnan(on).any()                                            # every position written
    fb = tbase[toff]
    for k, (H, W) in enumerate(shapes):
        blk = on[6 * fb[k]:6 * fb[k + 1]].reshape(2, -1, 3)
        nz = np.nonzero(valid[moff[k]:moff[k + 1]])[0]
        assert blk.shape[1] == len(nz)
        if len(nz) == 0:
            continue
        np.testing.assert_array_equal(blk[1], rgbs[k].reshape(-1, 3)[nz] / 255.0)
        z = depths[k].reshape(-1)[nz].astype(np.float64)
        px, py = (nz % W).astype(np.float64), (nz // W).astype(np.float64)
        fl, cx, cy, kr = params[k]
        u, v = (px - cx) / fl, (py - cy) / fl
        if models[k] == 1:
            u, v = O.colmap_undistort_radial(kr, u, v)
        X, Y = u * z, v * z
        P = wfc[k]
        ref = np.stack([((P[i, 0] * X + P[i, 1] * Y) + P[i, 2] * z) + P[i, 3] for i in range(3)], axis=1)
        if models[k] == 0:
            _bits_equal(blk[0], ref)
        else:
            np.testing.assert_allclose(blk[0], ref, rtol=0, atol=1e-9 * np.abs(ref).max())


# ---------------------------------------------------------------------------------------------------------------------
# the public call
# ---------------------------------------------------------------------------------------------------------------------
def _public_scene(seed, F=4):
    rng = np.random.default_rng(seed)
    return _scene(rng, [(30, 40)] * F, 60, 0.9, sky=0.0)


def _break(kind, sparse, disp, nm):
    s = sparse[nm]
    if kind == "nan target":
        s[5, :] = [10.2, 11.0, np.nan]
    elif kind == "inf disparity":
        s[5, :2] = [10.2, 11.0]
        disp[nm][11, 10] = np.inf
    elif kind == "no sample":
        s[:, 0] = -5
    elif kind == "no point":
        sparse[nm] = np.zeros((0, 3))


NAN_THRESHOLD = O.NAN_THRESHOLD_ERROR.format(np.float64(np.nan))         # the reference's threshold is np.float64
MESSAGES = {"nan target": NAN_THRESHOLD, "inf disparity": O.INF_X_ERROR, "no sample": NAN_THRESHOLD,
            "no point": "Too few points for depth alignment"}


@pytest.mark.parametrize("kind", ["nan target", "inf disparity", "no sample"])
def test_reference_errors(cuda_dev, kind):
    rec, sparse, disp, rgb = _public_scene(9)
    nm = list(sparse)[1]
    _break(kind, sparse, disp, nm)
    with pytest.raises(ValueError) as e:
        O.ransac_fit(*O.frame_samples(disp[nm], sparse[nm]), 0)
    assert str(e.value) == MESSAGES[kind]
    before = {k: v.copy() for k, v in disp.items()}
    with pytest.raises(ValueError) as e:
        dense_depth.align_dense_depth_maps(rec, sparse, disp, rgb, seeds=np.arange(4))
    assert str(e.value) == MESSAGES[kind]
    for k in disp:                                                           # raised before any frame is rescaled
        _bits_equal(disp[k], before[k])


def test_first_failing_frame_wins(cuda_dev):
    for kinds in (("inf disparity", "no point", "nan target"), ("no point", "no sample", "inf disparity"),
                  (None, "nan target", "no point"), (None, None, "inf disparity")):
        rec, sparse, disp, rgb = _public_scene(10)
        names = list(sparse)
        for nm, kind in zip(names, kinds):
            if kind:
                _break(kind, sparse, disp, nm)
        first = next(k for k in kinds if k)
        with pytest.raises(ValueError) as e:
            dense_depth.align_dense_depth_maps(rec, sparse, disp, rgb, seeds=np.arange(4))
        assert str(e.value) == MESSAGES[first], kinds


def test_memory_budget_is_bitwise_one_batch(cuda_dev):
    """A budget below one frame (one frame per batch) and one of exactly two frames give the single batch's maps,
    in-place disparities and points."""
    rng = np.random.default_rng(11)
    shapes = [(30, 40), (31, 41), (29, 39), (30, 40)]
    rec, sparse, disp, rgb = _scene(rng, shapes, 200, 0.9, sky=0.1)
    seeds = rng.integers(0, 2 ** 31, 4)
    orig = {k: v.copy() for k, v in disp.items()}
    per_pixel = 4 + 4 + 3 + 48
    runs = []
    for budget in (None, 100, per_pixel * (30 * 40 + 31 * 41)):
        d = {k: v.copy() for k, v in orig.items()}
        kw = {} if budget is None else dict(memory_budget=budget)
        depth, pts = dense_depth.align_dense_depth_maps(rec, sparse, d, rgb, True, seeds=seeds, **kw)
        runs.append((depth, pts, d))
    depth, pts, _ = runs[0]
    for depth_b, pts_b, d_b in runs[1:]:
        for nm in sparse:
            _bits_equal(depth_b[nm], depth[nm])
            _bits_equal(d_b[nm], runs[0][2][nm])
            assert pts_b[nm].shape == pts[nm].shape
            _bits_equal(pts_b[nm], pts[nm])
