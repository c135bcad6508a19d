"""CPU oracle for the absolute-pose fall-back of ``refine_pose`` -- TEST INFRASTRUCTURE ONLY.

Restates what ``pycolmap.absolute_pose_estimation`` does for the reference's call sites
(vggsfm/utils/triangulation.py:404-433 with ``estimate_focal_length=True``, ``ransac.max_error=12``;
vggsfm/runners/video_runner.py:985-998 with the defaults): COLMAP 3.10 ``EstimateAbsolutePose``
[3P-memory] =
  * focal-length factors 0.2 + 4.8 (i/30)^2, i = 0..30, when ``estimate_focal_length`` (else the single factor 1);
  * per factor: image points -> normalised camera coordinates of the scaled camera (SIMPLE_RADIAL: true inverse of
    x(1 + k r^2) by Newton), threshold ``max_error / focal``, LO-RANSAC with a P3P minimal solver on squared
    reprojection error in the normalised plane, support = (inlier count, then smaller residual sum), local optimisation
    on all inliers, at most 10 rounds while the inlier count grows;
  * best factor wins on the same support order; ``None`` when fewer than 3 inliers.
PARITY UNPINNED and not pinnable: pycolmap is absent AND its RANSAC draws from COLMAP's internal Mersenne twister,
which no caller can seed per call; two deliberate, stated differences: (1) the minimal samples are drawn by the CALLER
(``u_samples`` [T,3] uniform numbers -> indices into the frame's usable points; the product path draws them with
torch's CPU generator, the way the triangulation pairs are drawn) for a FIXED number of trials T instead of COLMAP's
adaptive stopping rule; (2) the local estimator is a 4-step Gauss-Newton on the inliers' normalised reprojection error
instead of EPnP.  What is checked: the CUDA kernel reproduces this restatement on the same samples, and the restatement
recovers ground-truth poses / focal lengths on synthetic scenes with gross outliers (tests/test_pnp_oracle.py).
The P3P solver is Grunert's formulation: the quartic in v = s3/s1 derived symbolically (tools: sympy resultant of the
three law-of-cosines equations; coefficients below), real roots by Ferrari's method + Newton polishing.
"""
from __future__ import annotations

import numpy as np

SIMPLE_PINHOLE, SIMPLE_RADIAL = 0, 1
NUM_FOCAL_SAMPLES = 30
MIN_FOCAL_RATIO, MAX_FOCAL_RATIO = 0.2, 5.0
MAX_LOCAL_TRIALS = 10
GN_STEPS = 4


def focal_length_factors(estimate_focal_length: bool):
    if not estimate_focal_length:
        return np.array([1.0])
    i = np.arange(NUM_FOCAL_SAMPLES + 1) / float(NUM_FOCAL_SAMPLES)
    return MIN_FOCAL_RATIO + (MAX_FOCAL_RATIO - MIN_FOCAL_RATIO) * i * i


def _cbrt(x):
    return np.sign(x) * np.abs(x) ** (1.0 / 3.0)


def solve_quartic_real(A4, A3, A2, A1, A0):
    """Real roots of A4 x^4 + ... + A0 (Ferrari; the resolvent cubic's largest real root by Cardano / the trigonometric
    form, Newton-polished), each polished by 3 Newton steps on the quartic.  Returns a list (possibly empty)."""
    if not np.isfinite([A4, A3, A2, A1, A0]).all() or abs(A4) < 1e-300:
        return []
    b, c, d, e = A3 / A4, A2 / A4, A1 / A4, A0 / A4
    # depressed quartic y^4 + p y^2 + q y + r, x = y - b/4
    p = c - 3.0 * b * b / 8.0
    q = d - b * c / 2.0 + b * b * b / 8.0
    r = e - b * d / 4.0 + b * b * c / 16.0 - 3.0 * b ** 4 / 256.0
    # resolvent cubic m^3 + p m^2 + (p^2/4 - r) m - q^2/8 = 0 ; take the largest real root (>= 0)
    c2, c1, c0 = p, p * p / 4.0 - r, -q * q / 8.0
    # depressed cubic t^3 + P t + Q, m = t - c2/3
    P = c1 - c2 * c2 / 3.0
    Q = 2.0 * c2 ** 3 / 27.0 - c2 * c1 / 3.0 + c0
    disc = Q * Q / 4.0 + P ** 3 / 27.0
    if disc >= 0.0:
        s = np.sqrt(disc)
        t = _cbrt(-Q / 2.0 + s) + _cbrt(-Q / 2.0 - s)
    else:
        rr = 2.0 * np.sqrt(-P / 3.0)
        phi = np.arccos(np.clip(3.0 * Q / (P * rr), -1.0, 1.0))      # cos(3 theta) = 3Q/(P rr)
        t = rr * np.cos(phi / 3.0)                                      # the largest of the three real roots
    m = t - c2 / 3.0
    for _ in range(3):                                                  # Newton polish of the cubic root
        fm = ((m + c2) * m + c1) * m + c0
        dm = (3.0 * m + 2.0 * c2) * m + c1
        if dm != 0.0:
            m = m - fm / dm
    ys = []
    if m > 1e-14 * max(1.0, abs(p)):
        s2m = np.sqrt(2.0 * m)
        for sg in (1.0, -1.0):
            # y^2 - sg*s2m*y + (p/2 + m + sg*q/(2 s2m)) = 0
            bb, cc = -sg * s2m, p / 2.0 + m + sg * q / (2.0 * s2m)
            dd = bb * bb - 4.0 * cc
            if dd >= 0.0:
                sd = np.sqrt(dd)
                ys += [(-bb + sd) / 2.0, (-bb - sd) / 2.0]
    else:
        # biquadratic: y^4 + p y^2 + r = 0
        dd = p * p - 4.0 * r
        if dd >= 0.0:
            for z in ((-p + np.sqrt(dd)) / 2.0, (-p - np.sqrt(dd)) / 2.0):
                if z >= 0.0:
                    ys += [np.sqrt(z), -np.sqrt(z)]
    roots = []
    for y in ys:
        x = y - b / 4.0
        for _ in range(3):
            f = (((A4 * x + A3) * x + A2) * x + A1) * x + A0
            df = ((4.0 * A4 * x + 3.0 * A3) * x + 2.0 * A2) * x + A1
            if df != 0.0:
                x = x - f / df
        if np.isfinite(x):
            roots.append(x)
    return roots


def _frame(p0, p1, p2):
    e1 = p1 - p0
    e1 = e1 / np.linalg.norm(e1)
    e3 = np.cross(e1, p2 - p0)
    e3 = e3 / np.linalg.norm(e3)
    e2 = np.cross(e3, e1)
    return np.stack([e1, e2, e3], axis=1)


def p3p(f, X):
    """f [3,3] unit bearing vectors (rows), X [3,3] world points (rows) -> list of poses [3,4] with R X_i + t = s_i f_i."""
    a2 = np.sum((X[1] - X[2]) ** 2)
    b2 = np.sum((X[0] - X[2]) ** 2)
    c2 = np.sum((X[0] - X[1]) ** 2)
    ca, cb, cg = f[1] @ f[2], f[0] @ f[2], f[0] @ f[1]
    A4 = a2 * a2 - 2 * a2 * b2 - 2 * a2 * c2 + b2 * b2 - 4 * b2 * c2 * ca * ca + 2 * b2 * c2 + c2 * c2
    A3 = -4 * (a2 * a2 * cb - a2 * b2 * ca * cg - a2 * b2 * cb - 2 * a2 * c2 * cb + b2 * b2 * ca * cg
               - 2 * b2 * c2 * ca * ca * cb - b2 * c2 * ca * cg + b2 * c2 * cb + c2 * c2 * cb)
    A2 = 2 * (2 * a2 * a2 * cb * cb + a2 * a2 - 4 * a2 * b2 * ca * cb * cg - 2 * a2 * b2 * cg * cg - 4 * a2 * c2 * cb * cb
              - 2 * a2 * c2 + 2 * b2 * b2 * ca * ca + 2 * b2 * b2 * cg * cg - b2 * b2 - 2 * b2 * c2 * ca * ca
              - 4 * b2 * c2 * ca * cb * cg + 2 * c2 * c2 * cb * cb + c2 * c2)
    A1 = -4 * (a2 * a2 * cb - a2 * b2 * ca * cg - 2 * a2 * b2 * cb * cg * cg + a2 * b2 * cb - 2 * a2 * c2 * cb
               + b2 * b2 * ca * cg - b2 * c2 * ca * cg - b2 * c2 * cb + c2 * c2 * cb)
    A0 = a2 * a2 - 4 * a2 * b2 * cg * cg + 2 * a2 * b2 - 2 * a2 * c2 + b2 * b2 - 2 * b2 * c2 + c2 * c2
    out = []
    for v in solve_quartic_real(A4, A3, A2, A1, A0):
        if not (v > 0.0):
            continue
        den = 2.0 * b2 * (ca * v - cg)
        if abs(den) < 1e-300:
            continue
        u = (2 * a2 * cb * v - a2 * v * v - a2 + b2 * v * v - b2 - 2 * c2 * cb * v + c2 * v * v + c2) / den
        if not (u > 0.0):
            continue
        w = 1.0 + v * v - 2.0 * v * cb
        if not (w > 0.0):
            continue
        s1 = np.sqrt(b2 / w)
        Y = np.stack([s1 * f[0], u * s1 * f[1], v * s1 * f[2]])
        with np.errstate(all="ignore"):
            Ey, Ex = _frame(Y[0], Y[1], Y[2]), _frame(X[0], X[1], X[2])
        R = Ey @ Ex.T
        t = Y[0] - R @ X[0]
        P = np.concatenate([R, t[:, None]], axis=1)
        if np.isfinite(P).all():
            out.append(P)
    return out


def undistort_radial(xd, k, iters=20):
    """Inverse of x_d = x (1 + k |x|^2) by Newton on the radius (what COLMAP's CamFromImg computes)."""
    rd = np.linalg.norm(xd, axis=-1)
    r = rd.copy()
    for _ in range(iters):
        r = r - (r * (1.0 + k * r * r) - rd) / (1.0 + 3.0 * k * r * r)
    s = np.where(rd > 0, r / np.where(rd > 0, rd, 1.0), 1.0)
    return xd * s[:, None]


def residuals(P, X, xn):
    p = X @ P[:, :3].T + P[:, 3]
    z = p[:, 2]
    ok = z > 0
    zz = np.where(ok, z, 1.0)
    res = (p[:, 0] / zz - xn[:, 0]) ** 2 + (p[:, 1] / zz - xn[:, 1]) ** 2
    return np.where(ok, res, np.inf)


def _support(res, thr2):
    inl = res <= thr2
    return int(inl.sum()), float(res[inl].sum()), inl


def _better(n, s, bn, bs):
    return n > bn or (n == bn and s < bs)


def _exp_so3(w):
    th = np.linalg.norm(w)
    if th < 1e-12:
        return np.eye(3) + np.array([[0, -w[2], w[1]], [w[2], 0, -w[0]], [-w[1], w[0], 0]])
    a = w / th
    K = np.array([[0, -a[2], a[1]], [a[2], 0, -a[0]], [-a[1], a[0], 0]])
    return np.eye(3) + np.sin(th) * K + (1 - np.cos(th)) * (K @ K)


def gauss_newton(P, X, xn, steps=GN_STEPS):
    """Local estimator: `steps` Gauss-Newton iterations on sum |pi(R X + t) - x|^2 (left rotation update, 6 dof)."""
    P = P.copy()
    for _ in range(steps):
        R, t = P[:, :3], P[:, 3]
        p = X @ R.T + t
        iz = 1.0 / p[:, 2]
        u, v = p[:, 0] * iz, p[:, 1] * iz
        r = np.stack([u - xn[:, 0], v - xn[:, 1]], axis=1)
        # d pi / d p
        J = np.zeros((len(X), 2, 6))
        jp = np.zeros((len(X), 2, 3))
        jp[:, 0, 0], jp[:, 0, 2] = iz, -u * iz
        jp[:, 1, 1], jp[:, 1, 2] = iz, -v * iz
        a = p - t                                   # R X
        # d(R X)/d w = -[R X]_x  (left perturbation exp(w) R)
        sk = np.zeros((len(X), 3, 3))
        sk[:, 0, 1], sk[:, 0, 2] = a[:, 2], -a[:, 1]
        sk[:, 1, 0], sk[:, 1, 2] = -a[:, 2], a[:, 0]
        sk[:, 2, 0], sk[:, 2, 1] = a[:, 1], -a[:, 0]
        J[:, :, :3] = jp @ sk
        J[:, :, 3:] = jp
        H = np.einsum("nij,nik->jk", J, J)
        g = np.einsum("nij,ni->j", J, r)
        try:
            d = np.linalg.solve(H + 1e-12 * np.trace(H) * np.eye(6), -g)
        except np.linalg.LinAlgError:
            break
        if not np.isfinite(d).all():
            break
        P = np.concatenate([_exp_so3(d[:3]) @ R, (t + d[3:])[:, None]], axis=1)
    return P


def new_debug():
    """Decision record filled by ``lo_ransac(..., debug=d)``:
      nsol_hist [5]     trials by number of P3P solutions (0..4); trials with a repeated index are counted in ``skipped``;
      best_from_lo      the returned pose is a local-optimisation iterate (False: a raw P3P candidate);
      lo_not_last       local optimisations started from a candidate that was not the last of its trial (the kernel
                        must then restore the supports of the later candidates);
      thr_margin        smallest |res - thr2| / thr2 over the finite residuals of every scored pose (P3P candidates
                        and local-optimisation iterates), i.e. of every inlier decision the support depends on;
      tie_gap           smallest |s_a - s_b| / max(s_a, s_b) over the support comparisons with equal inlier counts of at
                        least 4 whose two poses differ by more than 1e-8 (closer poses are interchangeable at the 1e-8
                        bar).  With 3 inliers every candidate fits its own sample exactly, the sums are rounding noise,
                        and such a support never starts a local optimisation: any larger support replaces it, and a
                        final count of 3 leaves the pose ambiguous."""
    return {"nsol_hist": np.zeros(5, dtype=np.int64), "skipped": 0, "lo_not_last": 0, "thr_margin": np.inf,
            "tie_gap": np.inf, "best_from_lo": False}


def _note_margin(debug, res, thr2):
    if debug is not None:
        fin = res[np.isfinite(res)]
        if len(fin):
            debug["thr_margin"] = min(debug["thr_margin"], float(np.min(np.abs(fin - thr2))) / thr2)


def _note_tie(debug, Pa, cnt, rs, Pb, bcnt, bs):
    if debug is not None and Pb is not None and cnt == bcnt >= 4 and np.abs(Pa - Pb).max() > 1e-8:
        den = max(abs(rs), abs(bs))
        debug["tie_gap"] = min(debug["tie_gap"], abs(rs - bs) / den if den > 0 else 0.0)


def lo_ransac(X, xn, thr2, u_samples, debug=None):
    """LO-RANSAC over the host-drawn minimal samples.  X [n,3], xn [n,2] (usable points only).
    Returns (pose, num_inliers, residual_sum, inlier mask) or None.  ``debug``: a ``new_debug()`` dict to accumulate
    into."""
    n = len(X)
    if n < 3:
        return None
    best = (None, 0, np.inf, np.zeros(n, dtype=bool))
    from_lo = False
    for us in u_samples:
        idx = np.minimum((us * n).astype(np.int64), n - 1)
        if len(set(idx.tolist())) < 3:
            if debug is not None:
                debug["skipped"] += 1
            continue
        b = np.concatenate([xn[idx], np.ones((3, 1))], axis=1)
        b = b / np.linalg.norm(b, axis=1, keepdims=True)
        sols = p3p(b, X[idx])
        if debug is not None:
            debug["nsol_hist"][len(sols)] += 1
        for q, P in enumerate(sols):
            res = residuals(P, X, xn)
            _note_margin(debug, res, thr2)
            cnt, rs, inl = _support(res, thr2)
            _note_tie(debug, P, cnt, rs, best[0], best[1], best[2])
            if not _better(cnt, rs, best[1], best[2]):
                continue
            best = (P, cnt, rs, inl)
            from_lo = False
            if cnt >= 4:
                if debug is not None and q < len(sols) - 1:
                    debug["lo_not_last"] += 1
                for _ in range(MAX_LOCAL_TRIALS):
                    prev = best[1]
                    Pl = gauss_newton(best[0], X[best[3]], xn[best[3]])
                    res = residuals(Pl, X, xn)
                    _note_margin(debug, res, thr2)
                    c2, r2, i2 = _support(res, thr2)
                    _note_tie(debug, Pl, c2, r2, best[0], best[1], best[2])
                    if _better(c2, r2, best[1], best[2]):
                        best = (Pl, c2, r2, i2)
                        from_lo = True
                    if best[1] <= prev:
                        break
    if debug is not None:
        debug["best_from_lo"] = from_lo
    if best[0] is None or best[1] < 3:
        return None
    return best


def absolute_pose_estimation(points2D, points3D, intr4, model, u_samples, estimate_focal_length=False, max_error=12.0,
                             mask=None, return_debug=False):
    """-> dict(pose [3,4], focal, num_inliers, inliers [P] bool) before the non-linear refinement, or None.

    ``return_debug``: returns (result or None, debug) where debug is ``new_debug()`` accumulated over every factor plus
    ``factors``: per focal factor a dict(focal, num_inliers (0 when nothing was found), residual_sum, pose, inliers [P],
    from_lo); ``best_from_lo`` then refers to the winning factor."""
    P = len(points3D)
    mask = np.ones(P, dtype=bool) if mask is None else np.asarray(mask, dtype=bool)
    idx = np.nonzero(mask)[0]
    X = np.asarray(points3D, dtype=np.float64)[idx]
    uv = np.asarray(points2D, dtype=np.float64)[idx]
    f0, cx, cy, k = [float(v) for v in intr4]
    debug = new_debug() if return_debug else None
    if debug is not None:
        debug["factors"] = []
    best, best_f = None, f0
    for fac in focal_length_factors(estimate_focal_length):
        f = f0 * fac
        xn = (uv - np.array([cx, cy])) / f
        if model == SIMPLE_RADIAL:
            xn = undistort_radial(xn, k)
        r = lo_ransac(X, xn, (max_error / f) ** 2, u_samples, debug)
        if debug is not None:
            m = np.zeros(P, dtype=bool)
            if r is not None:
                m[idx[r[3]]] = True
            debug["factors"].append({"focal": f, "num_inliers": 0 if r is None else r[1],
                                     "residual_sum": np.inf if r is None else r[2],
                                     "pose": np.zeros((3, 4)) if r is None else r[0], "inliers": m,
                                     "from_lo": debug["best_from_lo"]})
        if r is not None and (best is None or r[1] > best[1]):        # across factors: inlier count only, first wins ties
            best, best_f = r, f
    out = None
    if debug is not None:
        debug["best_from_lo"] = best is not None and debug["factors"][int(np.argmax(
            [fc["num_inliers"] for fc in debug["factors"]]))]["from_lo"]
    if best is not None:
        inl = np.zeros(P, dtype=bool)
        inl[idx[best[3]]] = True
        out = {"pose": best[0], "focal": best_f, "num_inliers": best[1], "inliers": inl}
    return (out, debug) if return_debug else out
