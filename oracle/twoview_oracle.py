"""Float64 restatement of the reference's batched two-view stage -- TEST INFRASTRUCTURE ONLY.

vggsfm/two_view_geo/estimate_preliminary.py:98-241 (estimate_preliminary_cameras) over fundamental.py:43-183
(estimate_fundamental: 7-point minimal solves, Sampson scoring, two rounds of 8-point local refinement, residual
indicator) and essential.py:36-83 / utils.py:325-448 (decomposition of E = K2^T F K1 and the cheirality vote), statement
for statement in numpy float64.  kornia is absent; its helpers (normalize_points, normalize_transformation,
solve_cubic, transform_points) are restated from memory and marked [3P-memory].

Two pins where the reference's result depends on LAPACK's choice of basis (DESIGN.md section 3), shared with
csrc/twoview.cu:
  * the 7-point null space is built by Gaussian elimination with partial pivoting over the columns in order, the last
    two free columns set to unit values (f1: second to last, f2: last);
  * the sign of the 8-point eigenvector is chosen so that the denormalised F_22 is >= 0, and the SVD of E is
    oriented so that t = U[:, 2] has its largest-magnitude entry positive.
"""
from __future__ import annotations

import numpy as np

HOM = 1.0 / (1.0 + 1e-8)                    # kornia convert_points_from_homogeneous on z = 1 (eps 1e-8)
SQRT2_F32 = float(np.sqrt(np.float32(2.0)))  # torch.sqrt(torch.tensor(2.0)) in both normalisations
K_MIN_DEPTH = float(np.finfo(np.float32).eps)   # torch.finfo(R.dtype).eps: the reference runs this in float32
INVALID_RESIDUAL = 1e6


# ---------------------------------------------------------------------------------------------------------------------
# sampling (utils.py:39-60)
# ---------------------------------------------------------------------------------------------------------------------
def generate_samples(N, target_num, sample_num=7, expand_ratio=2):
    """np.random.randint draws of the reference; raises where the reference would fail at `.view`."""
    sample_idx = np.random.randint(0, N, size=(target_num * expand_ratio, sample_num))
    sorted_array = np.sort(sample_idx, axis=1)
    has_duplicates = (np.diff(sorted_array, axis=1) == 0).any(axis=1)
    safe = sample_idx[np.where(~has_duplicates)[0]][:target_num]
    if len(safe) < target_num:
        raise ValueError(f"only {len(safe)} of {target_num} duplicate-free {sample_num}-point samples drawn from "
                         f"{N} points")
    return safe


# ---------------------------------------------------------------------------------------------------------------------
# kornia helpers [3P-memory]
# ---------------------------------------------------------------------------------------------------------------------
def normalize_transformation(M, eps=1e-8):
    n = M[..., 2:3, 2:3]
    return np.where(np.abs(n) > eps, M / (n + eps), M)


def _transform(scale, mx, my):
    T = np.zeros(scale.shape + (3, 3))
    T[..., 0, 0] = scale
    T[..., 0, 2] = -scale * mx
    T[..., 1, 1] = scale
    T[..., 1, 2] = -scale * my
    T[..., 2, 2] = 1.0
    return T


def _apply(T, p):
    """transform_points(T, p) with kornia's homogeneous division (z = 1 -> factor 1/(1+eps))."""
    x = (T[..., None, 0, 0] * p[..., 0] + T[..., None, 0, 2]) * HOM
    y = (T[..., None, 1, 1] * p[..., 1] + T[..., None, 1, 2]) * HOM
    return np.stack([x, y], -1)


def normalize_points(p, eps=1e-8):
    """kornia.geometry.epipolar.normalize_points: p [M,n,2] -> (normalised points, T [M,3,3])."""
    mean = p.sum(axis=1) / p.shape[1]
    d = np.sqrt(((p - mean[:, None]) ** 2).sum(-1))
    scale = SQRT2_F32 / (d.sum(-1) / p.shape[1] + eps)
    T = _transform(scale, mean[:, 0], mean[:, 1])
    return _apply(T, p), T


def normalize_points_masked(p, mask, eps=1e-8):
    """utils.py:175-253, non-COLMAP branch: p [M,N,2], mask [M,N] bool."""
    m = mask.astype(np.float64)
    cnt = m.sum(-1)
    mean = (p * m[..., None]).sum(1) / (cnt + eps)[:, None]
    d = np.sqrt(((p * m[..., None] - mean[:, None]) ** 2).sum(-1))
    scale = (d * m).sum(-1) / (cnt + eps)
    scale = SQRT2_F32 / (scale + eps)
    T = _transform(scale, mean[:, 0], mean[:, 1])
    return _apply(T, p), T


def solve_quadratic(c):
    a, b, cc = c[:, 0], c[:, 1], c[:, 2]
    out = np.zeros((len(c), 2))
    delta = b * b - 4 * a * cc
    with np.errstate(divide="ignore", invalid="ignore"):
        inv_2a = 0.5 / a
        z = delta == 0
        out[z, 0] = -b[z] * inv_2a[z]
        out[z, 1] = out[z, 0]
        pos = delta > 0
        sd = np.sqrt(delta[pos])
        out[pos, 0] = (-b[pos] + sd) * inv_2a[pos]
        out[pos, 1] = (-b[pos] - sd) * inv_2a[pos]
    return out


def solve_cubic(coeffs):
    """kornia.geometry.solvers.solve_cubic [3P-memory]: real roots of c0 x^3 + c1 x^2 + c2 x + c3, non-real (and
    unsolved zero-order) slots left at 0.  The acos argument is clamped to [-1, 1] (NaN-free at D ~ 0)."""
    c = np.asarray(coeffs, dtype=np.float64)
    a, b, cc, d = c[:, 0], c[:, 1], c[:, 2], c[:, 3]
    out = np.zeros((len(c), 3))
    az, bz, cz = a == 0, b == 0, cc == 0
    first = az & bz & ~cz
    out[first, 0] = -d[first] / cc[first]
    second = az & ~bz
    if second.any():
        out[second, 0:2] = solve_quadratic(c[second, 1:])
    third = ~az
    if third.any():
        inv_a = 1.0 / a[third]
        b_a = b[third] * inv_a
        b_a2 = b_a * b_a
        c_a = cc[third] * inv_a
        d_a = d[third] * inv_a
        Q = (3 * c_a - b_a2) / 9
        R = (9 * b_a * c_a - 27 * d_a - 2 * b_a * b_a2) / 54
        Q3 = Q * Q * Q
        D = Q3 + R * R
        b_a_3 = (1.0 / 3.0) * b_a
        sol = np.zeros((int(third.sum()), 3))
        qz = (Q == 0) & (R != 0)
        sol[qz, 0] = np.cbrt(2 * R[qz]) - b_a_3[qz]
        qrz = (Q == 0) & (R == 0)
        sol[qrz] = -b_a_3[qrz, None]
        three = (D <= 0) & (Q != 0)
        if three.any():
            arg = np.clip(R[three] / np.sqrt(-Q3[three]), -1.0, 1.0)
            th = np.arccos(arg)
            sq = 2 * np.sqrt(-Q[three])
            for k in range(3):
                sol[three, k] = sq * np.cos((th + 2 * k * np.pi) / 3.0) - b_a_3[three]
        one = (D > 0) & (Q != 0)
        if one.any():
            Rp = R[one]
            AD = np.where(Rp >= 0, 1.0, -1.0) * np.cbrt(np.abs(Rp) + np.sqrt(D[one]))
            with np.errstate(divide="ignore", invalid="ignore"):
                BD = np.where(AD == 0, 0.0, -Q[one] / AD)
            sol[one, 0] = AD + BD - b_a_3[one]
        out[third] = sol
    return out


# ---------------------------------------------------------------------------------------------------------------------
# 7-point (fundamental.py:341-469)
# ---------------------------------------------------------------------------------------------------------------------
def null_basis(A):
    """Pinned basis (f1, f2) [M,9] of the null space of A [M,7,9]: row echelon form by partial pivoting over the columns
    in order (an exactly zero column below the current row makes that column free), the last two free columns set to
    (1, 0) for f1 and (0, 1) for f2, the pivot variables by back substitution."""
    A = A.copy()
    M = A.shape[0]
    ar = np.arange(M)
    rank = np.zeros(M, dtype=np.int64)
    pcol = np.full((M, 7), -1, dtype=np.int64)
    rows = np.arange(7)
    for c in range(9):
        col = np.abs(A[:, :, c])
        col = np.where(rows[None] >= rank[:, None], col, -1.0)
        p = np.argmax(col, axis=1)
        has = (col[ar, p] > 0) & (rank < 7)
        idx = np.nonzero(has)[0]
        if len(idx) == 0:
            continue
        r0, pp = rank[idx], p[idx]
        tmp = A[idx, r0].copy()
        A[idx, r0] = A[idx, pp]
        A[idx, pp] = tmp
        piv = A[idx, r0, c]
        for r in range(7):
            below = r > r0
            if not below.any():
                continue
            j = idx[below]
            f = A[j, r, c] / piv[below]
            A[j, r, c:] -= f[:, None] * A[j, r0[below], c:]
            A[j, r, c] = 0.0
        pcol[idx, r0] = c
        rank[idx] += 1
    out = []
    for which in (0, 1):
        x = np.zeros((M, 9))
        for m in range(M):
            free = [c for c in range(9) if c not in set(pcol[m, :rank[m]].tolist())]
            x[m, free[-2 + which]] = 1.0
            for i in range(rank[m] - 1, -1, -1):
                pc = pcol[m, i]
                s = 0.0
                for j in range(pc + 1, 9):
                    s += A[m, i, j] * x[m, j]
                x[m, pc] = -s / A[m, i, pc]
        out.append(x)
    return out[0], out[1]


def _design_rows(p1n, p2n):
    x1, y1 = p1n[..., 0], p1n[..., 1]
    x2, y2 = p2n[..., 0], p2n[..., 1]
    return np.stack([x2 * x1, x2 * y1, x2, y2 * x1, y2 * y1, y2, x1, y1, np.ones_like(x1)], -1)


def run_7point(left, right):
    """left/right [M,7,2] -> F [M,3,3,3] (three candidates per sample)."""
    p1n, T1 = normalize_points(left)
    p2n, T2 = normalize_points(right)
    X = _design_rows(p1n, p2n)
    v1, v2 = null_basis(X)
    f1, f2 = v1.reshape(-1, 3, 3), v2.reshape(-1, 3, 3)
    d1, d2 = np.linalg.det(f1), np.linalg.det(f2)
    f1[d1 == 0] = np.eye(3)
    f2[d2 == 0] = np.eye(3)
    d1, d2 = np.linalg.det(f1), np.linalg.det(f2)
    coeffs = np.stack([d1, np.einsum("bii->b", f2 @ np.linalg.inv(f1)) * d1,
                       np.einsum("bii->b", f1 @ np.linalg.inv(f2)) * d2, d2], -1)
    roots = solve_cubic(coeffs)
    s = f1[:, 2, 2, None] * roots + f2[:, 2, 2, None]
    nz = ~(np.abs(s) <= 1e-8)                         # ~torch.isclose(s, 0)
    mu = np.ones_like(roots)
    lam = roots.copy()
    mu[nz] = 1.0 / s[nz]
    lam[nz] = lam[nz] * mu[nz]
    F = f1[:, None] * lam[..., None, None] + f2[:, None] * mu[..., None, None]
    F[..., 2, 2] = np.where(nz, 1.0, 0.0)
    F = np.swapaxes(T2, -1, -2)[:, None] @ (F @ T1[:, None])
    return normalize_transformation(F)


# ---------------------------------------------------------------------------------------------------------------------
# 8-point (fundamental.py:254-333) and local refinement (utils.py:256-297)
# ---------------------------------------------------------------------------------------------------------------------
def _smallest_eigvec(M):
    _, _, Vh = np.linalg.svd(M)
    return Vh[..., -1, :]


def run_8point(p1, p2, mask):
    """p1/p2 [M,N,2], mask [M,N] bool -> F [M,3,3] (sign pin: denormalised F_22 >= 0)."""
    p1n, T1 = normalize_points_masked(p1, mask)
    p2n, T2 = normalize_points_masked(p2, mask)
    X = _design_rows(p1n, p2n) * mask[..., None]
    Mn = np.swapaxes(X, -1, -2) @ X
    F = _smallest_eigvec(Mn).reshape(-1, 3, 3)
    U, S, Vh = np.linalg.svd(F)
    S[:, 2] = 0.0
    Fp = U @ (S[:, :, None] * Vh)
    Fe = np.swapaxes(T2, -1, -2) @ (Fp @ T1)
    Fe = np.where(Fe[:, 2:3, 2:3] < 0, -Fe, Fe)
    return normalize_transformation(Fe)


def sampson(p1, p2, F, squared=True, eps=1e-8):
    """p1/p2 [N,2], F [K,3,3] -> [K,N] (utils.py:90-172)."""
    x1, y1, x2, y2 = p1[:, 0], p1[:, 1], p2[:, 0], p2[:, 1]
    F = F.reshape(-1, 9)[:, :, None]
    with np.errstate(divide="ignore", invalid="ignore", over="ignore"):
        l0 = F[:, 0] * x1 + F[:, 1] * y1 + F[:, 2]
        l1 = F[:, 3] * x1 + F[:, 4] * y1 + F[:, 5]
        l2 = F[:, 6] * x1 + F[:, 7] * y1 + F[:, 8]
        m0 = F[:, 0] * x2 + F[:, 3] * y2 + F[:, 6]
        m1 = F[:, 1] * x2 + F[:, 4] * y2 + F[:, 7]
        num = x2 * l0 + y2 * l1 + l2
        num = num * num
        den = l0 * l0 + l1 * l1 + m0 * m0 + m1 * m1
        r = num / den
        return r if squared else np.sqrt(r + eps)


def _lo_points(p, masks):
    """local_refinement's lo_points (utils.py:280-283): the seed's inliers scattered into zeros, so that a NaN or inf
    match outside the mask does not reach the normal matrix."""
    return np.where(masks[..., None], p[None], 0.0)


def _stable_desc(counts):
    return np.argsort(-counts, axis=-1, kind="stable")


def _indicator_mean(res, thr):
    inl = res <= thr
    cnt = inl.sum(-1)
    with np.errstate(invalid="ignore", divide="ignore", over="ignore"):
        mean = (inl * res).sum(-1) / cnt
    return np.where(np.isfinite(mean), mean, 1e6), cnt


# ---------------------------------------------------------------------------------------------------------------------
# estimate_fundamental (fundamental.py:43-183), one pair at a time; the batch-wide `thres` is applied by the caller
# ---------------------------------------------------------------------------------------------------------------------
def score_pair(p1, p2, valid, samples, thr, lo_num, squared=True, second_refine=True):
    """Everything of estimate_fundamental for one pair that does not depend on other pairs.  Returns a dict with the
    candidate matrices F [K,3,3] (3T minimal, lo, lo//2 refined), inlier counts [K], indicator means [K]
    (NaN/inf -> 1e6), and the seeds of both refinement rounds."""
    N = p1.shape[0]
    valid = np.ones(N, bool) if valid is None else valid.astype(bool)
    T = samples.shape[0]
    Fm = run_7point(p1[samples], p2[samples]).reshape(T * 3, 3, 3)

    def scored(F, apply_valid=True):
        r = sampson(p1, p2, F, squared)
        if apply_valid:
            r = np.where(valid[None], r, INVALID_RESIDUAL)
        return r

    res = scored(Fm)
    inl = res <= thr
    seeds1 = _stable_desc(inl.sum(-1))[:lo_num]
    Flo = run_8point(_lo_points(p1, inl[seeds1]), _lo_points(p2, inl[seeds1]), inl[seeds1])
    F_all = [Fm, Flo]
    seeds2 = np.zeros(0, np.int64)
    if second_refine:
        lo2 = lo_num // 2
        raw = scored(Flo, apply_valid=False) <= thr           # fundamental.py:131: before the valid-mask overwrite
        seeds2 = _stable_desc(raw.sum(-1))[:lo2]
        if lo2 > 0:
            m2 = raw[seeds2]
            F_all.append(run_8point(_lo_points(p1, m2), _lo_points(p2, m2), m2))
    F = np.concatenate(F_all, 0)
    res_all = np.concatenate([res, scored(np.concatenate(F_all[1:], 0))], 0)
    mean, cnt = _indicator_mean(res_all, thr)
    return dict(F=F, cnt=cnt, mean=mean, seeds1=seeds1, seeds2=seeds2, res=res_all)


def select(pairs, thr):
    """calculate_residual_indicator over the batch (utils.py:63-87) + first argmax per pair."""
    thres = max(float(p["mean"].max()) for p in pairs) + 1e-6
    out = []
    for p in pairs:
        ind = (thres - p["mean"]) / thres + p["cnt"].astype(np.float64)
        b = int(np.argmax(ind))
        r = p["res"][b]
        out.append(dict(best=b, F=p["F"][b], num=int(p["cnt"][b]), mask=r <= thr, residuals=r, indicator=ind))
    return out, thres


def estimate_fundamental(points1, points2, samples, max_error=1.0, lo_num=300, valid_mask=None, squared=True,
                         second_refine=True):
    """points1/points2 [B,N,2], samples [T,7] -> dict of fmat [B,3,3], inlier_num [B], inlier_mask [B,N],
    residuals [B,N], best [B], thres, per-pair details."""
    thr = max_error ** 2 if squared else max_error
    B = points1.shape[0]
    pairs = [score_pair(np.asarray(points1[b], np.float64), np.asarray(points2[b], np.float64),
                        None if valid_mask is None else valid_mask[b], samples, thr, lo_num, squared, second_refine)
             for b in range(B)]
    sel, thres = select(pairs, thr)
    return dict(fmat=np.stack([s["F"] for s in sel]), inlier_num=np.array([s["num"] for s in sel]),
                inlier_mask=np.stack([s["mask"] for s in sel]), residuals=np.stack([s["residuals"] for s in sel]),
                best=np.array([s["best"] for s in sel]), thres=thres, pairs=pairs, sel=sel)


# ---------------------------------------------------------------------------------------------------------------------
# relative pose (estimate_preliminary.py:148-164, essential.py:36-83, utils.py:325-448)
# ---------------------------------------------------------------------------------------------------------------------
def default_kmat(width, height):
    f = float(max(width, height))
    return np.array([[f, 0.0, width / 2], [0.0, f, height / 2], [0.0, 0.0, 1.0]])


def decompose_essential_matrix(E):
    """E [B,3,3] -> Rs [B,4,3,3], ts [B,4,3] (order R1 t, R1 -t, R2 t, R2 -t; orientation pin on t)."""
    U, _, Vt = np.linalg.svd(E)
    U = np.where((np.linalg.det(U) < 0)[:, None, None], U * np.array([1.0, 1.0, -1.0]), U)
    Vt = np.where((np.linalg.det(Vt) < 0)[:, None, None], Vt * np.array([1.0, 1.0, -1.0])[:, None], Vt)
    t = U[:, :, 2]
    flip = t[np.arange(len(t)), np.argmax(np.abs(t), axis=1)] < 0
    P = np.array([-1.0, 1.0, -1.0])
    U = np.where(flip[:, None, None], U * P, U)
    Vt = np.where(flip[:, None, None], Vt * P[:, None], Vt)
    W = np.array([[0.0, -1.0, 0.0], [1.0, 0.0, 0.0], [0.0, 0.0, 1.0]])
    R1 = U @ W @ Vt
    R2 = U @ W.T @ Vt
    T = U[:, :, 2]
    return np.stack([R1, R1, R2, R2], 1), np.stack([T, -T, T, -T], 1)


def cheirality_counts(R, t, x1, x2, return_margin=False):
    """R [3,3], t [3], x1/x2 [N,2] normalised -> number of points in front of both cameras inside the depth window.
    With return_margin: (count, margin), margin = the smallest relative distance of a finite depth (either camera) to
    K_MIN_DEPTH or to the window 1000 |R^T t|."""
    N = x1.shape[0]
    P1 = np.eye(3, 4)
    P2 = np.concatenate([R, t[:, None]], 1)
    A = np.zeros((N, 4, 4))
    A[:, 0] = x1[:, 0, None] * P1[2] - P1[0]
    A[:, 1] = x1[:, 1, None] * P1[2] - P1[1]
    A[:, 2] = x2[:, 0, None] * P2[2] - P2[0]
    A[:, 3] = x2[:, 1, None] * P2[2] - P2[1]
    with np.errstate(invalid="ignore", divide="ignore"):
        ok = np.isfinite(A).all(axis=(1, 2))
        Vh = np.full((N, 4, 4), np.nan)
        if ok.any():
            Vh[ok] = np.linalg.svd(A[ok])[2]
        X = Vh[:, -1, :3] / Vh[:, -1, 3:4]
        d1 = X[:, 2]
        d2 = X @ R[2] + t[2]
    max_depth = 1000.0 * np.linalg.norm(R.T @ t)
    cnt = int(((d1 > K_MIN_DEPTH) & (d1 < max_depth) & (d2 > K_MIN_DEPTH) & (d2 < max_depth)).sum())
    if not return_margin:
        return cnt
    d = np.concatenate([d1, d2])
    d = d[np.isfinite(d)]
    margin = np.inf
    if d.size:
        margin = float(np.min(np.abs(d - K_MIN_DEPTH)) / K_MIN_DEPTH)
        if max_depth > 0:
            margin = min(margin, float(np.min(np.abs(d - max_depth)) / max_depth))
    return cnt, margin


def relative_pose(fmat, points1, points2, width, height, return_debug=False):
    """fmat [B,3,3], points [B,N,2] -> (R [B,3,3], t [B,3], E [B,3,3], counts [B,4]).  With return_debug a fifth
    element: per pair a dict with the candidates (Rs [4,3,3], ts [4,3]), the chosen index `k` (first maximum), the
    singular values `sigma` of E, `depth_margin` (the smallest relative distance of any finite triangulated depth, over
    the four candidates and both cameras, to K_MIN_DEPTH or to the depth window) and `count_gap` (the smallest count
    difference between the winner and a candidate with a different (R, t); inf when there is none)."""
    K = default_kmat(width, height)
    E = K.T @ fmat @ K
    Rs, ts = decompose_essential_matrix(E)
    f = float(max(width, height))
    pp = np.array([width / 2, height / 2])
    B = fmat.shape[0]
    R = np.zeros((B, 3, 3))
    t = np.zeros((B, 3))
    counts = np.zeros((B, 4), np.int64)
    debug = []
    for b in range(B):
        x1 = (np.asarray(points1[b], np.float64) - pp) / f
        x2 = (np.asarray(points2[b], np.float64) - pp) / f
        cm = [cheirality_counts(Rs[b, k], ts[b, k], x1, x2, return_margin=True) for k in range(4)]
        counts[b] = [c for c, _ in cm]
        k = int(np.argmax(counts[b]))
        R[b], t[b] = Rs[b, k], ts[b, k]
        if return_debug:
            gap = np.inf
            for j in range(4):
                same = np.abs(Rs[b, j] - Rs[b, k]).max() <= 1e-12 and np.abs(ts[b, j] - ts[b, k]).max() <= 1e-12
                if j != k and not same:
                    gap = min(gap, float(counts[b, k] - counts[b, j]))
            debug.append(dict(Rs=Rs[b], ts=ts[b], k=k, sigma=np.linalg.svd(E[b], compute_uv=False),
                              depth_margin=min(m for _, m in cm), count_gap=gap))
    if return_debug:
        return R, t, E, counts, debug
    return R, t, E, counts


# ---------------------------------------------------------------------------------------------------------------------
# conditioning of the decomposition
# ---------------------------------------------------------------------------------------------------------------------
EPS = 2.0 ** -52
POSE_BAR_C = 96.0


def pose_bar(sigma):
    """Bar on max |R - R_ref| and max |t - t_ref| between two float64 decompositions of the same F:
    POSE_BAR_C * eps * sigma_1 / sigma_2 (eps = 2^-52; inf when sigma_2 = 0).

    Derivation, with u = 2^-53 the unit roundoff and sigma_3 << sigma_2 (E is within rounding of rank 2):
      * forming E = K^T F K takes two length-3 inner products per entry, so |dE| <= 6u |K^T| |F| |K|.  With the default
        K (c_x, c_y <= f / 2) the entries of |K^T| |K^-T| and |K^-1| |K| are at most 2 and their 2-norms below 1.9,
        and F = K^-T E K^-1, so || |K^T| |F| |K| ||_2 <= 1.9^2 ||E||_F <= 3.7 sqrt(2) sigma_1: ||dE|| <= 32u sigma_1;
      * a backward-stable 3 x 3 SVD (LAPACK's, or a few sweeps of one-sided Jacobi, each rotation exact to a few u)
        returns the exact SVD of E + dE' with ||dE'|| <= 16u sigma_1;
      * R = U W V^T is the orthogonal factor of the rank-2 part of E, and t its left null vector: to first order both
        move by at most 2 ||dE|| / sigma_2 (polar-factor and singular-subspace perturbation with the gap
        sigma_2 - sigma_3 ~ sigma_2; the gap sigma_1 - sigma_2 does not enter, since R is the same for every
        rotation of the leading singular pair);
      * two independent decompositions differ by the sum: 2 * 2 (32 + 16) u sigma_1 / sigma_2 = 192 u sigma_1 / sigma_2
        = 96 eps sigma_1 / sigma_2.
    A decomposition through the normal matrix E^T E instead loses eps sigma_1^2 / sigma_2^2 (the eigenvector gap of
    E^T E is sigma_2^2 while its rounding is eps sigma_1^2), which exceeds this bar once sigma_2 / sigma_1 <~ 1e-3."""
    s = np.asarray(sigma, np.float64)
    return POSE_BAR_C * EPS * s[0] / s[1] if s[1] > 0 else np.inf


def random_rotation(rng):
    Q, Rr = np.linalg.qr(rng.normal(size=(3, 3)))
    Q = Q * np.sign(np.diag(Rr))
    return Q if np.linalg.det(Q) > 0 else -Q


def fundamental_with_singular_values(sigma, width, height, rng):
    """F = K^-T E K^-1 for E = U diag(sigma) V^T with random rotations U, V and the default K of (width, height).
    -> (F [3,3], E [3,3], U, V).  sigma = (1, r, 0) plants an E whose second singular value is r."""
    U, V = random_rotation(rng), random_rotation(rng)
    E = U @ np.diag(np.asarray(sigma, np.float64)) @ V.T
    Ki = np.linalg.inv(default_kmat(width, height))
    return Ki.T @ E @ Ki, E, U, V
