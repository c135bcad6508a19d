"""Float64 restatement of PoseLib's ``estimate_fundamental`` as the reference calls it -- TEST INFRASTRUCTURE ONLY.

vggsfm/two_view_geo/estimate_preliminary.py:37-95 (estimate_preliminary_cameras_poselib, the two-view stage of both
shipped configurations, ``use_poselib: True``) calls, per (frame 0, frame s) pair, ``poselib.estimate_fundamental``
on the matches with ``vis >= 0.05`` with ``max_epipolar_error = max_error``, ``max_iterations = max_ransac_iters``,
``min_iterations = 1000``, ``real_focal_check = True``, ``progressive_sampling = False`` and default BundleOptions.
PoseLib's sources are not available here and it cannot be installed, so everything below is [3P-memory] of
PoseLib 2.0.x.  PARITY UNPINNED.  It is pinnable on a machine that has PoseLib: PoseLib seeds its sampler per call
(``RansacOptions.seed``, default 0), so its draws, and with them its result, are reproducible.  What the tests pin is
this restatement, and csrc/twoview_msac.cu reproduces it:

  1. Input: only the valid matches (``vis >= 0.05``); ``tracks_score`` is ignored.  The left points are
     ``tracks[0, 0]`` for every pair, also for the pairs of later batches (a reference quirk, kept).
  2. Normalisation: one uniform scale shared by both views, no translation (a translation would change the real-focal
     check); scale = mean point norm over both views / sqrt(2), points and threshold divided by it.  Choice: the mean
     runs over the matches whose four coordinates are finite (PoseLib would turn every point into NaN), and a scale
     that is not positive and finite is replaced by 1.
  3. Sampler: PoseLib's RandomSampler, state = seed, ``state = (state * 1103515245 + 12345) mod 2^31``, index =
     state mod n, a duplicate index within a sample is redrawn.  The state runs on across trials.
  4. Minimal solver: the 7-point solver with REAL ROOTS ONLY (1 or 3 candidates; a degenerate leading coefficient gives
     the quadratic's 0 or 2, or the linear case's 0 or 1), on the null space and cubic of oracle/twoview_oracle.py
     (the pinned basis of DESIGN.md section 3, which also fixes the candidate order within a trial).  Real focal check
     (Bougnoux, principal point at the origin of the scaled frame): f1^2 = -n1/d1, f2^2 = -n2/d2 with
     n1 = (e2 x (F02, F12, 0))_z F22, d1 = (e2 x (I~ F I~ F^T p))_z and the transposed expressions for the second
     view (e1, e2 the right / left epipoles, each the longest cross product of two columns / rows of F, I~ =
     diag(1, 1, 0), p = (0, 0, 1)).  Choice: a candidate is dropped when n1 d1 > 0 or n2 d2 > 0 (an imaginary focal
     length) or when F is not finite.
  5. Scoring: MSAC on the squared Sampson error r^2 = (x2^T F x1)^2 / (l0^2 + l1^2 + m0^2 + m1^2): add r^2 when
     r^2 < thr^2 (strict), else thr^2; the inlier count is the number of strict r^2 < thr^2.  A NaN r^2 is an outlier at
     full cost.
  6. ransac<FundamentalEstimator>: stop at the start of iteration ``it`` when ``it > min_iterations`` and
     ``it > dynamic_max_iter``, at most ``max_iterations`` iterations.  Candidates of a trial in order; one that beats
     the best minimal inlier count OR the best minimal MSAC score updates what it beats and becomes the trial's LO seed
     (the last one wins); if its score also beats the model score it becomes the best model at once.  A trial with a seed
     refines it (step 7), keeps the result if its score is better, and updates ``dynamic_max_iter`` from the inlier
     ratio of the best model (success probability 0.9999, multiplier 1, ratio >= 0.9999 -> min_iterations, ratio
     <= 0.0001 -> max_iterations; choice: a non-finite or larger value is clamped to max_iterations, which stops nothing
     earlier).  After the loop the best model is refined once more the same way.  The mask is r^2 < thr^2 under it.
  7. Local optimisation: refine_fundamental with a truncated loss at the threshold, 25 LM iterations, all matches.
     Parameterisation F = U diag(1, sigma, 0) V^T; an update is U <- exp([w]x) U, V <- exp([v]x) V, sigma <- sigma + ds
     (Rodrigues), so dF/dw_k = [e_k]x F, dF/dv_k = -F [e_k]x, dF/dsigma = u1 v1^T.  LM as in PoseLib's lm_impl: lambda
     1e-3 added to the diagonal, x10 on reject (max 1e10), /10 on accept (min 1e-10), accept when the new cost is
     strictly lower, stop when |J^T r| < 1e-10 or |step| < 1e-8; the Cholesky of the damped 7 x 7 system (choice: a
     non-positive pivot ends the refinement).  IRLS weights: 1 for r^2 < thr^2, else 0; cost = MSAC score.
  8. Final polish: if the inlier count is > 7, refine again on the inliers with default BundleOptions (Cauchy loss,
     scale 1 px -> 1 / scale, 100 iterations; weight 1 / (1 + r^2/s^2), cost s^2 log1p(r^2/s^2)).  Then F <- T^T F T
     with T = diag(1/scale, 1/scale, 1), F / |F|_F.  Sign pin: the entry of largest magnitude is positive.  The mask stays
     the one of step 6.
  9. Fewer than 7 valid matches: PoseLib returns no model and the reference then fails at the mask assignment.  Here
     (deliberately) F = 0, an all-false mask, 0 iterations.  The same F = 0 and empty mask (with the iterations run)
     when no candidate of any trial passed the real focal check.
"""
from __future__ import annotations

import numpy as np

from oracle import twoview_oracle as tvo

SUCCESS_PROB = 0.9999
MIN_ITERATIONS = 1000
LO_ITERATIONS = 25
POLISH_ITERATIONS = 100
GRADIENT_TOL = 1e-10
STEP_TOL = 1e-8
INITIAL_LAMBDA = 1e-3
MIN_LAMBDA = 1e-10
MAX_LAMBDA = 1e10
LCG_A, LCG_C, LCG_M = 1103515245, 12345, 1 << 31
TRIAL_BLOCK = 256          # trials whose minimal candidates are solved and scored at once


# ---------------------------------------------------------------------------------------------------------------------
# sampler, scale
# ---------------------------------------------------------------------------------------------------------------------
class RandomSampler:
    def __init__(self, n, seed=0):
        self.n = int(n)
        self.state = int(seed)

    def _next(self):
        self.state = (self.state * LCG_A + LCG_C) % LCG_M
        return self.state

    def sample(self, k=7):
        out = []
        while len(out) < k:
            i = self._next() % self.n
            if i not in out:
                out.append(i)
        return out


def shared_scale(x1, x2):
    fin = np.isfinite(x1).all(1) & np.isfinite(x2).all(1)
    nf = int(fin.sum())
    if nf == 0:
        return 1.0
    s = (np.sqrt((x1[fin] ** 2).sum(1)).sum() + np.sqrt((x2[fin] ** 2).sum(1)).sum()) / (2.0 * nf) / np.sqrt(2.0)
    return float(s) if (np.isfinite(s) and s > 0) else 1.0


# ---------------------------------------------------------------------------------------------------------------------
# 7-point with real roots only, real focal check
# ---------------------------------------------------------------------------------------------------------------------
def real_root_count(c):
    """Number of leading solve_cubic slots that hold real roots (its branch structure), and the relative margin of the
    branch decision (|D| / (|Q^3| + R^2) in the cubic case)."""
    a, b, cc, d = (float(v) for v in c)
    if a == 0.0:
        if b == 0.0:
            return (1 if cc != 0.0 else 0), np.inf
        delta = cc * cc - 4.0 * b * d
        return (2 if delta >= 0.0 else 0), (abs(delta) / (cc * cc + abs(4.0 * b * d)) if delta != 0 else np.inf)
    inv_a = 1.0 / a
    b_a = b * inv_a
    b_a2 = b_a * b_a
    c_a = cc * inv_a
    d_a = d * inv_a
    Q = (3.0 * c_a - b_a2) / 9.0
    R = (9.0 * b_a * c_a - 27.0 * d_a - 2.0 * b_a * b_a2) / 54.0
    Q3 = Q * Q * Q
    D = Q3 + R * R
    if Q == 0.0:
        return (1 if R != 0.0 else 3), np.inf
    den = abs(Q3) + R * R
    return (3 if D <= 0.0 else 1), (abs(D) / den if den > 0 else np.inf)


def seven_point_real(left, right):
    """left/right [M,7,2] -> (F [M,3,3,3] in the twoview_oracle parameterisation, nreal [M], branch margin [M])."""
    p1n, _ = tvo.normalize_points(left)
    p2n, _ = tvo.normalize_points(right)
    X = tvo._design_rows(p1n, p2n)
    v1, v2 = tvo.null_basis(X)
    f1, f2 = v1.reshape(-1, 3, 3), v2.reshape(-1, 3, 3)
    f1[np.linalg.det(f1) == 0] = np.eye(3)
    f2[np.linalg.det(f2) == 0] = np.eye(3)
    d1, d2 = np.linalg.det(f1), np.linalg.det(f2)
    with np.errstate(all="ignore"):
        coeffs = np.stack([d1, np.einsum("bii->b", f2 @ np.linalg.inv(f1)) * d1,
                           np.einsum("bii->b", f1 @ np.linalg.inv(f2)) * d2, d2], -1)
    cnt = np.zeros(len(left), np.int64)
    mar = np.zeros(len(left))
    for m in range(len(left)):
        cnt[m], mar[m] = real_root_count(coeffs[m])
    with np.errstate(all="ignore"):
        F = tvo.run_7point(left, right)
    return F, cnt, mar


def _epipole(M):
    """Longest cross product of two columns of M (orthogonal to its column space for rank 2)."""
    c = [np.cross(M[:, 0], M[:, 1]), np.cross(M[:, 0], M[:, 2]), np.cross(M[:, 1], M[:, 2])]
    n = [float(v @ v) for v in c]
    return c[int(np.argmax(n))]


def _cross_z(e, a):
    v = e[0] * a[1] - e[1] * a[0]
    s = abs(e[0] * a[1]) + abs(e[1] * a[0])
    return v, (abs(v) / s if s > 0 else np.inf)


def _bougnoux(F):
    """(n, d, margin) of f^2 = -n/d for the first view."""
    e2 = _epipole(F)                                   # F^T e2 = 0: orthogonal to the columns of F
    n0, m0 = _cross_z(e2, np.array([F[0, 2], F[1, 2]]))
    n = n0 * F[2, 2]
    b = np.array([F[0, 0] * F[2, 0] + F[0, 1] * F[2, 1], F[1, 0] * F[2, 0] + F[1, 1] * F[2, 1]])
    d, m1 = _cross_z(e2, b)
    mf = abs(F[2, 2]) / np.abs(F).max() if np.abs(F).max() > 0 else np.inf
    return n, d, min(m0, m1, mf)


def real_focal_check(F):
    """-> (keep, margin, (f1^2, f2^2))."""
    if not np.isfinite(F).all():
        return False, np.inf, (np.nan, np.nan)
    n1, d1, ma = _bougnoux(F)
    n2, d2, mb = _bougnoux(F.T)
    with np.errstate(all="ignore"):
        f = (-n1 / d1, -n2 / d2)
    return not (n1 * d1 > 0 or n2 * d2 > 0), min(ma, mb), f


# ---------------------------------------------------------------------------------------------------------------------
# Sampson, MSAC
# ---------------------------------------------------------------------------------------------------------------------
def _sampson_parts(F, x1, x2):
    """F [3,3], x [n,2] -> e (x2^T F x1), den, l = F x1 [n,3], m = F^T x2 [n,3]."""
    X1 = np.concatenate([x1, np.ones((len(x1), 1))], 1)
    X2 = np.concatenate([x2, np.ones((len(x2), 1))], 1)
    with np.errstate(all="ignore"):
        l = X1 @ F.T
        m = X2 @ F
        e = (X2 * l).sum(1)
        den = l[:, 0] ** 2 + l[:, 1] ** 2 + m[:, 0] ** 2 + m[:, 1] ** 2
    return e, den, l, m, X1, X2


def sampson_sq(F, x1, x2):
    """[K,3,3] or [3,3] -> r^2 [K,n] / [n]."""
    F = np.asarray(F, np.float64)
    single = F.ndim == 2
    Fs = F[None] if single else F
    x1h = np.concatenate([x1, np.ones((len(x1), 1))], 1)
    x2h = np.concatenate([x2, np.ones((len(x2), 1))], 1)
    with np.errstate(all="ignore"):
        l = np.einsum("kij,nj->kni", Fs, x1h)
        m = np.einsum("kij,ni->knj", Fs, x2h)
        e = (x2h[None] * l).sum(-1)
        r2 = e * e / (l[..., 0] ** 2 + l[..., 1] ** 2 + m[..., 0] ** 2 + m[..., 1] ** 2)
    return r2[0] if single else r2


def msac(r2, thr2):
    inl = r2 < thr2
    return inl.sum(-1), np.where(inl, r2, thr2).sum(-1), inl


def _thr_margin(r2, thr2):
    r = r2[np.isfinite(r2)]
    return float(np.min(np.abs(r - thr2)) / thr2) if r.size else np.inf


def _gap(a, b):
    """relative gap of a comparison between two scores; an exact tie (identical sums) counts as decided identically."""
    if a == b:
        return np.inf
    return abs(a - b) / max(abs(a), abs(b))


# ---------------------------------------------------------------------------------------------------------------------
# LM on the factorised fundamental matrix
# ---------------------------------------------------------------------------------------------------------------------
def _skew(w):
    return np.array([[0.0, -w[2], w[1]], [w[2], 0.0, -w[0]], [-w[1], w[0], 0.0]])


def rodrigues(w):
    t2 = float(w @ w)
    if t2 == 0.0:
        return np.eye(3)
    t = np.sqrt(t2)
    K = _skew(w)
    a = np.sin(t) / t
    h = np.sin(0.5 * t)
    b = 2.0 * h * h / t2
    return np.eye(3) + a * K + b * (K @ K)


def factorize(F):
    """F -> (A = u0 v0^T, Bm = u1 v1^T, sigma = s1 / s0); None when s1 is not positive."""
    U, S, Vt = np.linalg.svd(F)
    if not (S[1] > 0 and np.isfinite(S).all()):
        return None
    return np.outer(U[:, 0], Vt[0]), np.outer(U[:, 1], Vt[1]), S[1] / S[0]


_E = [_skew(np.eye(3)[k]) for k in range(3)]


def _eval(A, Bm, sig, x1, x2, loss, c2):
    """cost, JtJ [7,7], Jtr [7], r^2 at F = A + sig Bm."""
    F = A + sig * Bm
    e, den, l, m, X1, X2 = _sampson_parts(F, x1, x2)
    with np.errstate(all="ignore"):
        r2 = e * e / den
    if loss == "truncated":
        w = (r2 < c2).astype(np.float64)
        cost = np.where(r2 < c2, r2, c2).sum()
    else:
        w = 1.0 / (1.0 + r2 / c2)
        cost = (c2 * np.log1p(r2 / c2)).sum()
    use = w > 0
    e, den, l, m, X1, X2, w = e[use], den[use], l[use], m[use], X1[use], X2[use], w[use]
    sq = np.sqrt(den)
    r = e / sq
    # dr/dF_ij = (x2_i x1_j - (e / den) (l_i x1_j [i < 2] + m_j x2_i [j < 2])) / sqrt(den)
    l2 = l.copy()
    l2[:, 2] = 0.0
    m2 = m.copy()
    m2[:, 2] = 0.0
    k = (e / den)[:, None, None]
    dF = (X2[:, :, None] * X1[:, None, :] - k * (l2[:, :, None] * X1[:, None, :] + X2[:, :, None] * m2[:, None, :]))
    dF = dF / sq[:, None, None]
    G = [Ek @ F for Ek in _E] + [-(F @ Ek) for Ek in _E] + [Bm]
    J = np.stack([(dF * g).sum((1, 2)) for g in G], 1)
    JtJ = (J * w[:, None]).T @ J
    Jtr = (J * (w * r)[:, None]).sum(0)
    return float(cost), JtJ, Jtr


def lm_refine(F, x1, x2, loss, c2, max_iter, dbg=None):
    """PoseLib's lm_impl on the factorised F; returns the refined F (scale |s0| = 1), the cost history in dbg."""
    fz = factorize(F)
    if fz is None:
        return F
    A, Bm, sig = fz
    cost, JtJ, Jtr = _eval(A, Bm, sig, x1, x2, loss, c2)
    lam = INITIAL_LAMBDA
    costs = [cost]
    for _ in range(max_iter):
        g = float(np.linalg.norm(Jtr))
        if dbg is not None:
            dbg["grad"].append(abs(g - GRADIENT_TOL) / GRADIENT_TOL)
        if g < GRADIENT_TOL:
            break
        H = JtJ + lam * np.eye(7)
        try:
            L = np.linalg.cholesky(H)
        except np.linalg.LinAlgError:
            break
        sol = -np.linalg.solve(L.T, np.linalg.solve(L, Jtr))
        st = float(np.linalg.norm(sol))
        if dbg is not None:
            dbg["step"].append(abs(st - STEP_TOL) / STEP_TOL)
        if st < STEP_TOL:
            break
        Rw, Rv = rodrigues(sol[0:3]), rodrigues(sol[3:6])
        An, Bn, sn = Rw @ A @ Rv.T, Rw @ Bm @ Rv.T, sig + sol[6]
        cn, Jn, jn = _eval(An, Bn, sn, x1, x2, loss, c2)
        if dbg is not None:
            dbg["accept"].append(_gap(cn, cost))
        if cn < cost:
            A, Bm, sig, cost, JtJ, Jtr = An, Bn, sn, cn, Jn, jn
            lam = max(MIN_LAMBDA, lam / 10.0)
            costs.append(cost)
        else:
            lam = min(MAX_LAMBDA, lam * 10.0)
    if dbg is not None:
        dbg["costs"].append(costs)
    return A + sig * Bm


def _lm_dbg():
    return {"grad": [], "step": [], "accept": [], "costs": []}


# ---------------------------------------------------------------------------------------------------------------------
# RANSAC
# ---------------------------------------------------------------------------------------------------------------------
def dynamic_max_iter(num_inliers, n, min_iterations, max_iterations):
    """-> (value, margin of the ceil: distance of its argument to the nearest integer, relative)."""
    ratio = num_inliers / n
    if ratio >= 0.9999:
        return min_iterations, np.inf
    if ratio <= 0.0001:
        return max_iterations, np.inf
    prob_outlier = 1.0 - ratio ** 7
    with np.errstate(all="ignore"):
        v = np.log(1.0 - SUCCESS_PROB) / np.log(prob_outlier)
    if not np.isfinite(v) or v >= max_iterations:
        return max_iterations, np.inf
    fr = abs(v - np.round(v)) / max(abs(v), 1.0)
    return int(np.ceil(v)), fr


def ransac_pair(x1, x2, thr, max_iterations, min_iterations=MIN_ITERATIONS, seed=0, debug=None):
    """x1/x2 [n,2] scaled points, thr the scaled threshold.  -> (F scaled frame, mask [n], iterations)."""
    n = len(x1)
    thr2 = thr * thr
    smp = RandomSampler(n, seed)
    best_min_cnt, best_min_score = 0, np.finfo(np.float64).max
    model_score, model_cnt, model = np.finfo(np.float64).max, 0, None
    model_src = None
    dyn = max_iterations
    d = debug
    it = 0
    F_blk = cnt_blk = sc_blk = None
    blk0 = -1
    while it < max_iterations:
        if it > min_iterations and it > dyn:
            break
        if blk0 < 0 or it >= blk0 + TRIAL_BLOCK:
            blk0 = it
            nb = min(TRIAL_BLOCK, max_iterations - it)
            S = np.array([smp.sample() for _ in range(nb)])
            Fc, nreal, bm = seven_point_real(x1[S], x2[S])
            keep = np.zeros((nb, 3), bool)
            for t in range(nb):
                for k in range(nreal[t]):
                    kp, mg, _ = real_focal_check(Fc[t, k])
                    keep[t, k] = kp
                    if d is not None:
                        d["rfc"] = min(d["rfc"], mg)
            if d is not None:
                d["roots"] = min(d["roots"], float(bm.min()))
            r2 = sampson_sq(Fc.reshape(-1, 3, 3), x1, x2)
            c, s, _ = msac(r2, thr2)
            F_blk, cnt_blk, sc_blk, keep_blk = Fc, c.reshape(nb, 3), s.reshape(nb, 3), keep
            if d is not None:
                kk = keep.reshape(-1)
                if kk.any():
                    d["thr"] = min(d["thr"], _thr_margin(r2[kk], thr2))
        t = it - blk0
        seed_k = -1
        for k in range(3):
            if not keep_blk[t, k]:
                continue
            c, s = int(cnt_blk[t, k]), float(sc_blk[t, k])
            more, better = c > best_min_cnt, s < best_min_score
            if d is not None:
                d["score"] = min(d["score"], _gap(s, best_min_score))
            if more or better:
                if more:
                    best_min_cnt = c
                if better:
                    best_min_score = s
                seed_k = k
                if d is not None:
                    _model_cmp(d, s, model_score, c, model_cnt, F_blk[t, k], model)
                if s < model_score:
                    model_score, model_cnt, model = s, c, F_blk[t, k]
                    model_src = ("min", it, k)
        if seed_k < 0:
            it += 1
            continue
        lo_dbg = _lm_dbg() if d is not None else None
        Fr = lm_refine(F_blk[t, seed_k], x1, x2, "truncated", thr2, LO_ITERATIONS, lo_dbg)
        r2 = sampson_sq(Fr, x1, x2)
        c, s, _ = msac(r2, thr2)
        if d is not None:
            d["lo_trials"].append(it)
            d["thr"] = min(d["thr"], _thr_margin(r2, thr2))
            _model_cmp(d, float(s), model_score, int(c), model_cnt, Fr, model)
            _merge_lm(d, lo_dbg)
        if s < model_score:
            model_score, model_cnt, model = float(s), int(c), Fr
            model_src = ("lo", it, seed_k)
        dyn, fm = dynamic_max_iter(model_cnt, n, min_iterations, max_iterations)
        if d is not None:
            d["ceil"] = min(d["ceil"], fm)
            d["dyn"].append((it, model_cnt, dyn))
        it += 1
    iterations = it
    if model is None:                  # no candidate passed the real focal check in any trial
        if d is not None:
            d["win"] = None
        return None, np.zeros(n, bool), iterations
    # final refinement
    lo_dbg = _lm_dbg() if d is not None else None
    Fr = lm_refine(model, x1, x2, "truncated", thr2, LO_ITERATIONS, lo_dbg)
    r2 = sampson_sq(Fr, x1, x2)
    c, s, _ = msac(r2, thr2)
    if d is not None:
        d["thr"] = min(d["thr"], _thr_margin(r2, thr2))
        _model_cmp(d, float(s), model_score, int(c), model_cnt, Fr, model)
        _merge_lm(d, lo_dbg)
        d["win"] = model_src
        d["final_lo_taken"] = bool(s < model_score)
    if s < model_score:
        model = Fr
    r2 = sampson_sq(model, x1, x2)
    mask = r2 < thr2
    if d is not None:
        d["thr"] = min(d["thr"], _thr_margin(r2, thr2))
    return model, mask, iterations


TIE_GAP = 1e-10


def _same_model(F, G):
    a, b = F / np.linalg.norm(F), G / np.linalg.norm(G)
    return min(np.abs(a - b).max(), np.abs(a + b).max()) <= 1e-8


def _model_cmp(d, s, model_score, c, model_cnt, F, model):
    """A comparison with the model score.  Two local optimisations that converge to the same model tie to roundoff;
    such a near-tie (gap < TIE_GAP, equal counts, the same matrix to 1e-8) is recorded in `ties` and kept out of the
    `score` margin: either outcome gives the same model, but the winning trial is then not determined."""
    g = _gap(s, model_score)
    if g < TIE_GAP and model is not None and c == model_cnt and _same_model(F, model):
        d["ties"] += 1
        return
    d["score"] = min(d["score"], g)


def _merge_lm(d, lo):
    for key in ("grad", "step", "accept"):
        if lo[key]:
            d["lm_" + key] = min(d["lm_" + key], min(lo[key]))
    d["lm_costs"].extend(lo["costs"])


def _new_debug():
    return {"iterations": 0, "lo_trials": [], "win": None, "thr": np.inf, "score": np.inf, "rfc": np.inf,
            "roots": np.inf, "ceil": np.inf, "lm_grad": np.inf, "lm_step": np.inf, "lm_accept": np.inf,
            "lm_costs": [], "dyn": [], "ties": 0, "n": 0, "scale": 1.0, "num": 0, "polished": False}


def sign_pin(F):
    i = int(np.argmax(np.abs(F).reshape(-1)))
    return -F if F.reshape(-1)[i] < 0 else F


def estimate_fundamental_pair(x1, x2, max_error, max_iterations, min_iterations=MIN_ITERATIONS, seed=0, debug=None):
    """x1/x2 [n,2] pixel coordinates of the valid matches -> (F [3,3] pixel frame, mask [n], iterations)."""
    x1 = np.asarray(x1, np.float64)
    x2 = np.asarray(x2, np.float64)
    n = len(x1)
    if debug is not None:
        debug["n"] = n
    if n < 7:
        return np.zeros((3, 3)), np.zeros(n, bool), 0
    s = shared_scale(x1, x2)
    y1, y2 = x1 / s, x2 / s
    thr = max_error / s
    F, mask, iters = ransac_pair(y1, y2, thr, max_iterations, min_iterations, seed, debug)
    if F is None:
        if debug is not None:
            debug.update(iterations=iters, scale=s)
        return np.zeros((3, 3)), mask, iters
    num = int(mask.sum())
    if num > 7:
        pd = _lm_dbg() if debug is not None else None
        F = lm_refine(F, y1[mask], y2[mask], "cauchy", (1.0 / s) ** 2, POLISH_ITERATIONS, pd)
        if debug is not None:
            _merge_lm(debug, pd)
    t = np.array([1.0 / s, 1.0 / s, 1.0])
    F = F * t[:, None] * t[None, :]
    F = sign_pin(F / np.linalg.norm(F))
    if debug is not None:
        debug.update(iterations=iters, scale=s, num=num, polished=num > 7)
    return F, mask, iters


def estimate_fundamental_msac(points1, points2, valid_mask, max_error, max_iterations, min_iterations=MIN_ITERATIONS,
                              seed=0, pairs=None, return_debug=False):
    """points1/points2 [B,N,2], valid_mask [B,N] bool or None.  -> dict fmat [B',3,3], inlier_num [B'], inlier_mask
    [B',N], iterations [B'] (B' = the selected `pairs`, all by default), and per-pair debug records."""
    points1 = np.asarray(points1, np.float64)
    points2 = np.asarray(points2, np.float64)
    B, N, _ = points1.shape
    rows = range(B) if pairs is None else pairs
    out = dict(fmat=[], inlier_num=[], inlier_mask=[], iterations=[], debug=[])
    for b in rows:
        v = np.ones(N, bool) if valid_mask is None else np.asarray(valid_mask[b], bool)
        dbg = _new_debug() if return_debug else None
        F, m, iters = estimate_fundamental_pair(points1[b][v], points2[b][v], max_error, max_iterations,
                                                min_iterations, seed, dbg)
        full = np.zeros(N, bool)
        full[np.nonzero(v)[0]] = m
        out["fmat"].append(F)
        out["inlier_num"].append(int(full.sum()))
        out["inlier_mask"].append(full)
        out["iterations"].append(iters)
        out["debug"].append(dbg)
    for k in ("fmat", "inlier_num", "inlier_mask", "iterations"):
        out[k] = np.array(out[k])
    return out


def estimate_preliminary_cameras_poselib(tracks, tracks_vis, width, height, max_error=0.5, max_ransac_iters=20000,
                                         min_iterations=MIN_ITERATIONS, seed=0, pairs=None, return_debug=False):
    """estimate_preliminary.py:37-95 on numpy arrays: tracks [B,S,N,2], tracks_vis [B,S,N].  Left points are
    tracks[0, 0] for every pair (the reference's query_points[0])."""
    tracks = np.asarray(tracks, np.float64)
    B, S, N, _ = tracks.shape
    left = np.broadcast_to(tracks[0, 0], (B * (S - 1), N, 2))
    right = tracks[:, 1:].reshape(B * (S - 1), N, 2)
    valid = (np.asarray(tracks_vis) >= 0.05)[:, 1:].reshape(B * (S - 1), N)
    return estimate_fundamental_msac(left, right, valid, max_error, max_ransac_iters, min_iterations, seed, pairs,
                                     return_debug)
