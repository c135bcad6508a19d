"""numpy restatement of the dense depth stage (test infrastructure only -- never on the product path).

What it restates, and how:

* ``ransac_fit``: ``RANSACRegressor(LinearRegression(), min_samples=2, residual_threshold=t, max_trials=20000,
  loss="squared_error").fit(X, y)`` as vggsfm/utils/utils.py:700-707 calls it, with ``random_state`` pinned to
  ``np.random.RandomState(seed)`` (DESIGN §3).  The dtype path is sklearn's for a float32 ``X`` and a float64 ``y``:
  ``LinearRegression`` casts ``y`` to float32 (``_preprocess_data``: ``check_array(y, dtype=X.dtype)``), centres both in
  float32 by their float32 means and solves with ``scipy.linalg.lstsq`` (LAPACK sgelsd) in float32, so ``coef_`` and
  ``intercept_`` are float32.  ``predict`` is float32 (``X @ coef_ + intercept_``); the residual ``(y - y_pred)**2`` is
  float64 (``y`` is the caller's float64 target), as is the R^2 of ``score``.  Rules of ``fit``: ``n_inliers_best``
  starts at 1, a trial with fewer inliers is skipped, one with equal inliers and a lower R^2 is skipped,
  ``max_trials = min(max_trials, _dynamic_max_trials(n_best, n, 2, 0.99))`` after each kept trial, stop once
  ``n_trials_ >= max_trials``; the final model is LinearRegression on the best inlier set.
* ``pairwise_sum_f32`` / ``mean_f32``: numpy's float32 ``np.mean`` (``pairwise_sum`` of ``loops_utils.h``, then one
  float32 division by float32(n)), which ``_preprocess_data`` uses for the float32 offsets of ``LinearRegression``.
  This restatement is the rule ``dd_final_kernel`` follows for its means; ``test_dense_depth_oracle.py`` checks it
  bitwise against ``np.mean``.
* Errors: ``frame_samples`` and ``ransac_fit`` raise what the reference loop and sklearn 1.9 raise, in their order:
  "Too few points", "Ill-posed scene", the ``residual_threshold`` parameter error of a NaN threshold (an empty sample
  set or any NaN target), ``min_samples`` (one sample), then "Input X contains infinity" (a +inf disparity).
* ``sample_pairs``: ``sklearn.utils.random.sample_without_replacement(n, 2, random_state)``, whose method depends on
  the ratio 2 / n: n = 2 returns [0, 1] without a draw (reservoir sampling), 2 / n in (0.01, 0.99) is
  ``permutation(n)[:2]``, and 2 / n <= 0.01 is tracking selection (``randint(n)`` until unseen).
* ``fit_two``: the two-sample ``LinearRegression`` written out as the float32 operations LAPACK's sgelsd performs on a
  2 x 1 system (slarfg / slapy2 Householder, Q^T b, slalsd's scaling by 1 / R); ``test_dense_depth_oracle.py`` checks it
  bitwise against ``scipy.linalg.lstsq``.  This is what the CUDA trial kernel computes.
* ``align_frame``: one iteration of ``align_dense_depth_maps`` (utils.py:662-765).  The rescale is float32 (scale and
  shift are float32 scalars, so numpy 2 keeps ``disp * scale + shift`` in float32); depth = float32(1 / disp).
* ``cam_from_img`` / ``img_from_cam``: pycolmap 3.10 (COLMAP ``SimplePinholeCameraModel`` /
  ``SimpleRadialCameraModel``).  SIMPLE_RADIAL ``cam_from_img`` is COLMAP's ``IterativeUndistortion`` (Newton with a
  central-difference Jacobian, relative step 1e-6, 100 iterations, stop when the squared step is below 1e-10)
  [3P-memory]; its parity with COLMAP is unpinned.  ``img_from_cam`` of a 3-vector divides by its z first.
"""
from __future__ import annotations

import warnings

import numpy as np
import scipy.linalg

f32 = np.float32
DISPARITY_MAX = 10000
DISPARITY_MIN = 0.0001
DEPTH_MAX = 1 / DISPARITY_MIN
DEPTH_MIN = 1 / DISPARITY_MAX
THRES_RATIO = 30
MAX_TRIALS = 20000


NAN_THRESHOLD_ERROR = ("The 'residual_threshold' parameter of RANSACRegressor must be a float in the range [0.0, inf) "
                       "or None. Got {!r} instead.")
MIN_SAMPLES_ERROR = "`min_samples` may not be larger than number of samples: n_samples = %d."
INF_X_ERROR = "Input X contains infinity or a value too large for dtype('float32')."
PAIRWISE_BLOCK = 128                                  # numpy's PW_BLOCKSIZE


def pairwise_sum_f32(a):
    """numpy's float32 pairwise sum of a contiguous vector, operation by operation: below 8 elements, 0 plus each in
    order; up to 128, eight accumulators seeded with a[0..7] and stepped by 8 to n - n % 8, combined as
    ((r0+r1)+(r2+r3))+((r4+r5)+(r6+r7)), then the tail in order; above, split at n2 = n//2 - (n//2) % 8 and recurse."""
    a = np.asarray(a, dtype=f32).reshape(-1)
    n = len(a)
    if n < 8:
        s = f32(0)
        for v in a:
            s = f32(s + v)
        return s
    if n <= PAIRWISE_BLOCK:
        m = n - n % 8
        r = a[:m].reshape(-1, 8)
        acc = r[0].copy()
        for row in r[1:]:
            acc = acc + row
        s = ((acc[0] + acc[1]) + (acc[2] + acc[3])) + ((acc[4] + acc[5]) + (acc[6] + acc[7]))
        for v in a[m:]:
            s = f32(s + v)
        return f32(s)
    n2 = n // 2
    n2 -= n2 % 8
    return f32(pairwise_sum_f32(a[:n2]) + pairwise_sum_f32(a[n2:]))


def mean_f32(a):
    """np.mean of a float32 vector: the pairwise sum over float32(n), both float32."""
    a = np.asarray(a, dtype=f32).reshape(-1)
    return f32(pairwise_sum_f32(a) / f32(len(a)))


def dynamic_max_trials(n_inliers, n_samples, min_samples=2, probability=0.99):
    """sklearn.linear_model._ransac._dynamic_max_trials."""
    inlier_ratio = n_inliers / float(n_samples)
    nom = max(np.spacing(1), 1 - probability)
    denom = max(np.spacing(1), 1 - inlier_ratio ** min_samples)
    if nom == 1:
        return 0
    if denom == 1:
        return float("inf")
    return abs(float(np.ceil(np.log(nom) / np.log(denom))))


def sample_pairs(rs, n, count):
    """``count`` successive ``sample_without_replacement(n, 2, random_state=rs)`` draws, [count, 2] int64."""
    out = np.empty((count, 2), dtype=np.int64)
    for k in range(count):
        if n == 2:
            out[k] = (0, 1)
        elif 2 / n > 0.01:
            out[k] = rs.permutation(n)[:2]
        else:
            j0 = rs.randint(n)
            j1 = rs.randint(n)
            while j1 == j0:
                j1 = rs.randint(n)
            out[k] = (j0, j1)
    return out


def linear_regression(X, y):
    """LinearRegression().fit(X[:, None], y) for float32 X and float64 y -> (coef_ float32, intercept_ float32)."""
    X = np.asarray(X, dtype=f32).reshape(-1, 1)
    y = np.asarray(y).astype(f32)
    X_offset = X.mean(axis=0)
    y_offset = y.mean(axis=0)
    coef = scipy.linalg.lstsq(X - X_offset, y - y_offset, cond=1e-6)[0]
    return coef[0], y_offset - X_offset @ coef


def fit_two(x0, x1, y0, y1):
    """The two-sample LinearRegression as sgelsd's float32 operations (see the module docstring)."""
    x0, x1, y0, y1 = f32(x0), f32(x1), f32(y0), f32(y1)
    xm, ym = (x0 + x1) * f32(0.5), (y0 + y1) * f32(0.5)
    a0, a1, b0, b1 = x0 - xm, x1 - xm, y0 - ym, y1 - ym
    R, bb = a0, b0
    if a1 != 0:
        w, z = max(abs(a0), abs(a1)), min(abs(a0), abs(a1))
        nrm = w if z == 0 else w * np.sqrt(f32(1) + (z / w) * (z / w))
        beta = f32(-np.copysign(nrm, a0))
        tau = (beta - a0) / beta
        v1 = a1 * (f32(1) / (a0 - beta))
        bb = b0 + (-tau) * (b0 + b1 * v1)
        R = beta
    c = f32(0) if R == 0 else bb * (f32(1) / R)
    return c, ym - xm * c


def predict(X, c, b):
    return np.asarray(X, dtype=f32).reshape(-1, 1) @ np.array([c], dtype=f32) + b


def r2_score(y, y_pred):
    """sklearn.metrics.r2_score with force_finite=True, single output."""
    y_pred = y_pred.astype(np.float64)
    num = ((y - y_pred) ** 2).sum()
    den = ((y - np.average(y)) ** 2).sum()
    if den == 0:
        return 1.0 if num == 0 else 0.0
    return 1.0 - num / den


def ransac_fit(X, y, threshold, seed, max_trials=MAX_TRIALS, return_debug=False):
    """RANSACRegressor.fit (see the module docstring) -> dict(coef, intercept, n_trials, inlier_mask[, debug])."""
    X = np.asarray(X, dtype=f32)
    y = np.asarray(y, dtype=np.float64)
    n = len(X)
    if np.isnan(threshold):                           # parameter validation comes first in fit
        raise ValueError(NAN_THRESHOLD_ERROR.format(threshold))
    if 2 > n:
        raise ValueError(MIN_SAMPLES_ERROR % n)
    if np.isinf(X).any():                             # validate_data of the first trial's predict
        raise ValueError(INF_X_ERROR)
    rs = np.random.RandomState(seed)
    n_best, score_best, mask_best, c_best = 1, -np.inf, None, None
    n_trials, mt = 0, max_trials
    samples, res_margin, score_gap = [], np.inf, np.inf
    while n_trials < mt:
        n_trials += 1
        idx = sample_pairs(rs, n, 1)[0]
        samples.append(idx)
        c, b = linear_regression(X[idx], y[idx])
        res = (y - predict(X, c, b)) ** 2
        mask = res <= threshold
        k = int(mask.sum())
        if k < n_best:
            continue
        score = r2_score(y[mask], predict(X[mask], c, b))
        if k == n_best and mask_best is not None and k > 2:   # two-term sums do not depend on the order
            score_gap = min(score_gap, abs(score - score_best))
        if k == n_best and score < score_best:
            continue
        n_best, score_best, mask_best, c_best = k, score, mask, (c, b, res)
        mt = min(mt, dynamic_max_trials(n_best, n, 2, 0.99))
    if mask_best is None:
        raise ValueError("RANSAC could not find a valid consensus set. All `max_trials` iterations were skipped "
                         "because each randomly chosen sub-sample failed the passing criteria. See estimator "
                         "attributes for diagnostics (n_skips*).")
    coef, intercept = linear_regression(X[mask_best], y[mask_best])
    out = dict(coef=coef, intercept=intercept, n_trials=n_trials, inlier_mask=mask_best, n_inliers=n_best)
    if return_debug:
        res = c_best[2]
        res_margin = float(np.min(np.abs(res - threshold)) / threshold)
        out["debug"] = dict(samples=np.array(samples), residual_margin=res_margin, score_gap=score_gap,
                            best_model=c_best[:2])
    return out


def tie_fixture(k=3):
    """Two groups of k samples at interleaved, distinct float32 x (group 0 at 1, 3, 5, ..., group 1 at 2, 4, ...) with
    targets exactly 0.25 and 0.75 -> (X, y, threshold = median / 30, group [2k]).  A trial within a group fits the
    horizontal line through it with zero residuals, so its R^2 takes the SStot == 0 branch (1.0): the two groups tie in
    count and score, and RANSACRegressor keeps the later one.  Asserted here: every within-group pair has exactly its
    group as inliers and every mixed pair fewer than k inliers, so no other trial can take part in the tie."""
    X = np.concatenate([1 + 2 * np.arange(k), 2 + 2 * np.arange(k)]).astype(f32)
    y = np.repeat([0.25, 0.75], k)
    group = np.repeat([0, 1], k)
    th = np.median(y) / THRES_RATIO
    for i in range(2 * k):
        for j in range(i + 1, 2 * k):
            c, b = fit_two(X[i], X[j], y[i], y[j])
            res = (y - predict(X, c, b)) ** 2
            if group[i] == group[j]:
                assert (res[group == group[i]] == 0).all() and (res <= th).sum() == k
            else:
                assert (res <= th).sum() < k
    return X, y, th, group


def frame_samples(disp_map, sparse_uvd):
    """utils.py:662-695 -> (X float32, y float64, threshold).  Raises the reference's ValueErrors."""
    sparse_uvd = np.array(sparse_uvd)
    if len(sparse_uvd) <= 0:
        raise ValueError("Too few points for depth alignment")
    ww, hh = disp_map.shape
    int_uv = np.round(sparse_uvd[:, :2]).astype(int)
    mask = (int_uv[:, 0] >= 0) & (int_uv[:, 0] < hh) & (int_uv[:, 1] >= 0) & (int_uv[:, 1] < ww)
    sparse_uvd, int_uv = sparse_uvd[mask], int_uv[mask]
    sampled = disp_map[int_uv[:, 1], int_uv[:, 0]]
    pos = sampled > 0
    X = sampled[pos]
    y = 1 / np.clip(sparse_uvd[:, -1][pos], DEPTH_MIN, DEPTH_MAX)
    with np.errstate(invalid="ignore"), warnings.catch_warnings():
        warnings.simplefilter("ignore", RuntimeWarning)   # the median of no sample is NaN, which ransac_fit rejects
        threshold = np.median(y) / THRES_RATIO
    if threshold <= 0:
        raise ValueError("Ill-posed scene for depth alignment")
    return X, y, threshold


def apply_scale(disp_map, scale, shift):
    """utils.py:712-724 on a copy -> (rescaled disparity float32, depth float32, valid mask)."""
    disp = np.array(disp_map, dtype=np.float32)
    nz = disp != 0
    disp[nz] = disp[nz] * scale + shift
    valid = (disp > 0) & (disp <= DISPARITY_MAX)
    disp[~valid] = 0
    depth = np.full(disp.shape, np.inf)
    depth[disp != 0] = 1 / disp[disp != 0]
    depth[depth == np.inf] = 0
    return disp, depth.astype(np.float32), valid


def colmap_undistort_radial(k, u, v):
    """COLMAP IterativeUndistortion for SIMPLE_RADIAL, vectorised over points [3P-memory]."""
    u = np.array(u, dtype=np.float64, copy=True)
    v = np.array(v, dtype=np.float64, copy=True)
    x0, y0 = u.copy(), v.copy()
    active = np.ones(u.shape, dtype=bool)

    def dist(a, b):
        rad = k * (a * a + b * b)
        return a * rad, b * rad

    eps = np.finfo(np.float64).eps
    for _ in range(100):
        if not active.any():
            break
        x, y = u[active], v[active]
        s0, s1 = np.maximum(eps, np.abs(1e-6 * x)), np.maximum(eps, np.abs(1e-6 * y))
        dx, dy = dist(x, y)
        a0, a1 = dist(x - s0, y)
        b0, b1 = dist(x + s0, y)
        c0, c1 = dist(x, y - s1)
        e0, e1 = dist(x, y + s1)
        J00, J01 = 1 + (b0 - a0) / (2 * s0), (e0 - c0) / (2 * s1)
        J10, J11 = (b1 - a1) / (2 * s0), 1 + (e1 - c1) / (2 * s1)
        r0, r1 = x + dx - x0[active], y + dy - y0[active]
        det = J00 * J11 - J01 * J10
        st0, st1 = (J11 * r0 - J01 * r1) / det, (J00 * r1 - J10 * r0) / det
        u[active], v[active] = x - st0, y - st1
        idx = np.nonzero(active)[0]
        active[idx[st0 * st0 + st1 * st1 < 1e-10]] = False
    return u, v


def cam_from_img(model, params, xy):
    xy = np.asarray(xy, dtype=np.float64)
    f, cx, cy = params[:3]
    u, v = (xy[..., 0] - cx) / f, (xy[..., 1] - cy) / f
    if model == "SIMPLE_RADIAL":
        u, v = colmap_undistort_radial(params[3], u, v)
    return np.stack([u, v], axis=-1)


def img_from_cam(model, params, p):
    p = np.asarray(p, dtype=np.float64)
    u, v = p[..., 0] / p[..., 2], p[..., 1] / p[..., 2]
    f, cx, cy = params[:3]
    if model == "SIMPLE_RADIAL":
        rad = params[3] * (u * u + v * v)
        u, v = u + u * rad, v + v * rad
    return np.stack([f * u + cx, f * v + cy], axis=-1)


def unproject(depth, valid, model, params, R, t, rgb):
    """utils.py:733-765 with cam_from_world = [R | t] -> [2, M, 3] float64 (world points, colour / 255)."""
    H, W = depth.shape
    yy, xx = np.meshgrid(np.arange(H), np.arange(W), indexing="ij")
    v = valid.reshape(-1)
    pts = np.column_stack((xx.ravel(), yy.ravel()))[v]
    d = depth.reshape(-1)[v].astype(np.float64)
    uv = cam_from_img(model, params, pts)
    p = np.hstack((uv, np.ones((len(uv), 1)))) * d[:, None]
    Ri = R.T
    ti = -(Ri[:, 0] * t[0] + Ri[:, 1] * t[1] + Ri[:, 2] * t[2])
    world = p[:, 0:1] * Ri[:, 0] + p[:, 1:2] * Ri[:, 1] + p[:, 2:3] * Ri[:, 2] + ti
    return np.array([world, (rgb / 255.0).reshape(-1, 3)[v]])


def align_frame(disp_map, sparse_uvd, seed, max_trials=MAX_TRIALS):
    """One frame of align_dense_depth_maps -> dict(depth, disp, valid, X, y, threshold, ransac result)."""
    X, y, th = frame_samples(disp_map, sparse_uvd)
    r = ransac_fit(X, y, th, seed, max_trials, return_debug=True)
    disp, depth, valid = apply_scale(disp_map, r["coef"], r["intercept"])
    return dict(depth=depth, disp=disp, valid=valid, X=X, y=y, threshold=th, ransac=r)
