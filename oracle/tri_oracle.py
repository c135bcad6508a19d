"""CPU oracle for the triangulation half of the hot path -- TEST INFRASTRUCTURE ONLY.

numpy float64 restatement of the reference's pure-torch geometry functions.  PINNED: checked against
the reference itself (imported in the build container through oracle/reference_shim.py) by
tests/test_tri_oracle.py and through the committed fixtures in tests/golden/.

Follows (all in the reference):
  triangulate_tracks_single_chunk     vggsfm/utils/triangulation.py:776-956
  local_refine_and_compute_error      vggsfm/utils/triangulation.py:959-1017
  local_refinement_tri                vggsfm/utils/triangulation_helpers.py:648-725
  triangulate_multi_view_point_batched  triangulation_helpers.py:27-131   (DLT)
  calculate_normalized_angular_error_batched  triangulation_helpers.py:431-472
  calculate_triangulation_angle_batched / _exhaustive / calculate_triangulation_angle  :475-587
  calculate_residual_indicator        vggsfm/two_view_geo/utils.py:63-87
  filter_all_points3D_single_chunk    triangulation_helpers.py:215-307
  project_3D_points / img_from_cam    triangulation_helpers.py:311-395
  cam_from_img                        triangulation_helpers.py:398-428
  iterative_undistortion / apply_distortion  vggsfm/utils/distortion.py:27-159
  triangulate_by_pair                 vggsfm/utils/triangulation.py:45-135
  generate_combinations               triangulation_helpers.py:638-645

One deliberate pin: the reference ranks hypotheses with ``torch.sort(descending=True)`` which is NOT
stable, so the order among equal inlier counts is implementation-defined (it differs between torch's
CPU and CUDA sorts).  This oracle -- and the CUDA path -- use the stable order (lower hypothesis index
first).  The golden fixtures are generated from the reference with torch.sort forced stable, and a
second unpinned fixture bounds the effect (tests/test_triangulation_gpu.py).
"""
from __future__ import annotations

import itertools
import numpy as np

PI = float(np.pi)


# ----------------------------------------------------------------------------------------------
# camera model helpers
# ----------------------------------------------------------------------------------------------

def apply_distortion(k, u, v):
    """SIMPLE_RADIAL branch of distortion.py:119-128: x + x*k*r^2.  k [S], u/v [S,N]."""
    r2 = u * u + v * v
    radial = k[:, None] * r2
    return u + u * radial, v + v * radial


def iterative_undistortion(k, tn, max_iterations=100, max_step_norm=1e-10, rel_step_size=1e-6):
    """distortion.py:27-99 including its quirks: central-difference Jacobian of the FULL distorted
    coordinate with the identity added again (J ~ 2I + ...), 2x2 solve, and a GLOBAL stop when the
    largest squared step over all observations drops below max_step_norm."""
    u = tn[..., 0].copy()
    v = tn[..., 1].copy()
    ou, ov = u.copy(), v.copy()
    eps = np.finfo(u.dtype).eps
    iters = 0
    for _ in range(max_iterations):
        iters += 1
        ud, vd = apply_distortion(k, u, v)
        dx = ou - ud
        dy = ov - vd
        su = np.maximum(np.abs(u) * rel_step_size, eps)
        sv = np.maximum(np.abs(v) * rel_step_size, eps)
        pu = apply_distortion(k, u + su, v)
        mu = apply_distortion(k, u - su, v)
        pv = apply_distortion(k, u, v + sv)
        mv = apply_distortion(k, u, v - sv)
        J00 = (pu[0] - mu[0]) / (2 * su) + 1
        J01 = (pv[0] - mv[0]) / (2 * sv)
        J10 = (pu[1] - mu[1]) / (2 * su)
        J11 = (pv[1] - mv[1]) / (2 * sv) + 1
        # torch.linalg.solve on 2x2 = LU with partial pivoting; Cramer differs by rounding only
        det = J00 * J11 - J01 * J10
        d0 = (J11 * dx - J01 * dy) / det
        d1 = (-J10 * dx + J00 * dy) / det
        u = u + d0
        v = v + d1
        if np.max(d0 * d0 + d1 * d1) < max_step_norm:
            break
    return np.stack([u, v], axis=-1), iters


def cam_from_img(tracks, intrinsics, extra_params=None):
    """triangulation_helpers.py:398-428.  tracks [S,N,2], intrinsics [S,3,3], extra_params [S,1]|None."""
    pp = np.stack([intrinsics[:, 0, 2], intrinsics[:, 1, 2]], -1)[:, None, :]
    fl = np.stack([intrinsics[:, 0, 0], intrinsics[:, 1, 1]], -1)[:, None, :]
    tn = (tracks - pp) / fl
    if extra_params is not None:
        tn, _ = iterative_undistortion(extra_params[:, 0], tn)
    return tn


def project_3D_points(points3D, extrinsics, intrinsics, extra_params=None):
    """triangulation_helpers.py:311-395: returns (points2D [S,P,2], points_cam [S,3,P])."""
    Xh = np.concatenate([points3D, np.ones_like(points3D[:, :1])], axis=1)
    pc = np.einsum("sij,pj->sip", extrinsics, Xh)
    with np.errstate(divide="ignore", invalid="ignore"):
        q = pc / pc[:, 2:3, :]
        u, v = q[:, 0], q[:, 1]
        if extra_params is not None:
            u, v = apply_distortion(extra_params[:, 0], u, v)
        x = intrinsics[:, 0, 0][:, None] * u + intrinsics[:, 0, 1][:, None] * v + intrinsics[:, 0, 2][:, None]
        y = intrinsics[:, 1, 0][:, None] * u + intrinsics[:, 1, 1][:, None] * v + intrinsics[:, 1, 2][:, None]
    p2 = np.stack([x, y], axis=-1)
    p2 = np.where(np.isnan(p2), 0.0, p2)
    big = np.finfo(np.float64).max
    p2 = np.clip(p2, -big, big)          # torch.nan_to_num maps +-inf to the largest finite value
    return p2, pc


# ----------------------------------------------------------------------------------------------
# DLT, angular error, triangulation angle
# ----------------------------------------------------------------------------------------------

def dlt(cams, pts, mask=None):
    """triangulation_helpers.py:27-98.  cams [B,n,3,4], pts [B,n,2], mask [B,n]|None -> X [B,3]."""
    B, n, _ = pts.shape
    ph = np.concatenate([pts, np.ones((B, n, 1))], axis=-1)
    pn = ph / np.linalg.norm(ph, axis=-1, keepdims=True)
    proj = np.einsum("bni,bnik->bnk", pn, cams)                 # x^T P  [B,n,4]
    terms = cams - pn[..., :, None] * proj[..., None, :]
    if mask is not None:
        terms = terms * mask[:, :, None, None]
    A = np.einsum("bnij,bnik->bjk", terms, terms)
    _, vecs = np.linalg.eigh(A)
    v = vecs[:, :, 0]
    with np.errstate(divide="ignore", invalid="ignore"):
        return v[:, :3] / v[:, 3:4]


def angular_error(tn, X, cams):
    """triangulation_helpers.py:431-472.  tn [S,N,2], X [P,N,3], cams [S,3,4] -> [P,S,N] radians."""
    ray1 = np.concatenate([tn, np.ones_like(tn[..., :1])], axis=-1)
    ray1 = ray1 / np.maximum(np.linalg.norm(ray1, axis=-1, keepdims=True), 1e-12)
    ray2 = np.einsum("sij,pnj->psni", cams[:, :, :3], X) + cams[None, :, None, :, 3]
    with np.errstate(invalid="ignore"):
        ray2 = ray2 / np.maximum(np.linalg.norm(ray2, axis=-1, keepdims=True), 1e-12)
        cosv = np.clip(np.sum(ray1[None] * ray2, axis=-1), -1.0, 1.0)
        return np.arccos(cosv)


def proj_centers(cams):
    return -np.einsum("sji,sj->si", cams[:, :, :3], cams[:, :, 3])


def tri_angle_deg(c1, c2, X, eps=1e-12):
    """triangulation_helpers.py:547-587 (law of cosines, min(t, pi-t), degrees).  Broadcasts."""
    base2 = np.sum((c1 - c2) ** 2, axis=-1)
    r1 = np.sum((X - c1) ** 2, axis=-1)
    r2 = np.sum((X - c2) ** 2, axis=-1)
    with np.errstate(invalid="ignore", divide="ignore"):
        den = 2.0 * np.sqrt(r1 * r2)
        num = r1 + r2 - base2
        bad = den <= eps
        num = np.where(bad, 1.0, num)
        den = np.where(bad, 1.0, den)
        cosv = np.clip(num / den, -1.0, 1.0)
        t = np.abs(np.arccos(cosv))
        t = np.minimum(t, PI - t)
    return t * (180.0 / PI)


def any_pair_tri_angle_exhaustive(centers, X, min_deg, inl=None):
    """exists (a,b) [both flagged by inl if given] with triangulation angle >= min_deg.
    centers [S,3], X [P,3], inl [S,P]|None -> [P] bool.  NaN angles compare False like torch.
    The reference's full S x S table; kept as the definition any_pair_tri_angle is tested against."""
    S = centers.shape[0]
    out = np.zeros(X.shape[0], dtype=bool)
    for a in range(S):
        ang = tri_angle_deg(centers[a][None, None, :], centers[:, None, :], X[None, :, :])   # [S,P]
        with np.errstate(invalid="ignore"):
            ok = ang >= min_deg
        if inl is not None:
            ok = ok & inl[a][None, :] & inl
        out |= ok.any(axis=0)
    return out


def separation_order(S):
    """Frame-index separations d of the pairs (a, a+d), wide baselines first as the kernels visit them:
    S/2, ..., S-1, S/2-1, ..., 1, then 0 (the self pairs, which only pass when min_deg <= 0)."""
    mid = max(S // 2, 1)
    return list(range(mid, S)) + list(range(mid - 1, 0, -1)) + [0]


def any_pair_tri_angle(centers, X, min_deg, inl=None, margin=0.0, return_best=False):
    """Same answer as any_pair_tri_angle_exhaustive, found faster: pairs are visited by separation, wide first,
    vectorised over the points still undecided, and a point leaves the search as soon as one of its pairs reaches
    min_deg + margin.  The points that never do (the False answers, and the True ones whose best pair lies in
    [min_deg, min_deg + margin)) run through every pair.  tri_angle_deg is symmetric in its two centres and gives
    exactly 0 for a self pair, so the unordered pairs plus the self pairs are the whole S x S table.

    With return_best also returns, per point, the largest angle over the pairs visited (ignoring NaN, -inf if
    none): the exact maximum when it is below min_deg + margin, a lower bound at or above it otherwise."""
    S = centers.shape[0]
    P = X.shape[0]
    out = np.zeros(P, dtype=bool)
    best = np.full(P, -np.inf)
    block = max(1, (1 << 21) // max(S, 1))
    for p0 in range(0, P, block):
        live = np.arange(p0, min(P, p0 + block))
        for d in separation_order(S):
            if live.size == 0:
                break
            a = np.arange(S - d)
            ang = tri_angle_deg(centers[a][:, None, :], centers[a + d][:, None, :], X[live][None, :, :])   # [S-d,U]
            with np.errstate(invalid="ignore"):
                ok = ang >= min_deg
            if inl is not None:
                pair_inl = inl[a][:, live] & inl[a + d][:, live]
                ok &= pair_inl
                ang = np.where(pair_inl, ang, -np.inf)
            out[live] |= ok.any(axis=0)
            best[live] = np.maximum(best[live], np.where(np.isnan(ang), -np.inf, ang).max(axis=0))
            live = live[best[live] < min_deg + margin]
    if return_best:
        return out, best
    return out


# ----------------------------------------------------------------------------------------------
# LORANSAC triangulation
# ----------------------------------------------------------------------------------------------

def generate_combinations(S):
    return np.array(list(itertools.combinations(range(S), 2)), dtype=np.int64)


def draw_pairs(S, max_ransac_iters=256):
    """Pair list exactly as triangulation.py:804-813 draws it (CPU global torch RNG)."""
    import torch
    comb = generate_combinations(S)
    if max_ransac_iters > len(comb):
        return comb
    perm = torch.randperm(len(comb))[:max_ransac_iters].numpy()
    return comb[perm]


def residual_indicator(err, thr, nanvalue):
    """two_view_geo/utils.py:63-87 on err [N,H,S]: (score, inlier_num, inlier_mask)."""
    with np.errstate(invalid="ignore", divide="ignore"):
        inl = err <= thr
        cnt = inl.sum(axis=-1)
        m = (inl.astype(np.float32).astype(np.float64) * err).sum(axis=-1) / cnt
    m = np.where(np.isfinite(m), m, nanvalue)
    thres = m.max() + 1e-6
    return (thres - m) / thres + cnt.astype(np.float64), cnt, inl


# A refined hypothesis whose best camera pair lies within this many degrees above min_tri_angle keeps searching, so
# that its reported best pair angle is exact there (see any_pair_tri_angle); the answer itself does not depend on it.
TRI_TIE_DEG = 1e-6


def _refine(tn_t, cams, centers, inl, order, lo, min_tri_angle, invalid_vis, thr):
    """local_refine_and_compute_error for the top-`lo` hypotheses.  tn_t [N,S,2], inl [N,H,S] bool,
    order [N,H] ranking -> (X [N,lo,3], err [N,lo,S], best pair angle - min_tri_angle [N,lo])."""
    N, S, _ = tn_t.shape
    X = np.zeros((N, lo, 3))
    camsB = np.broadcast_to(cams[None], (N, S, 3, 4))
    for j in range(lo):
        mk = inl[np.arange(N), order[:, j]]                       # [N,S]
        pts = np.where(mk[..., None], tn_t, 0.0)                  # masked-out observations are zeroed (:670-672)
        X[:, j] = dlt(camsB, pts, mk.astype(np.float64))
    with np.errstate(invalid="ignore"):
        z = np.einsum("sj,nlj->nls", cams[:, 2, :3], X) + cams[None, None, :, 2, 3]
        bad_che = (z <= 0).any(axis=2)                            # all S cameras (:100-115)
    ok_tri, best = any_pair_tri_angle(centers, X.reshape(-1, 3), min_tri_angle, margin=TRI_TIE_DEG,
                                      return_best=True)           # all S^2 camera pairs (:117-120)
    invalid = (~ok_tri.reshape(N, lo)) | bad_che
    err = angular_error(np.transpose(tn_t, (1, 0, 2)), np.transpose(X, (1, 0, 2)), cams)   # [lo,S,N]
    err = np.transpose(err, (2, 0, 1))
    err = np.where(np.isfinite(err), err, 100 * PI)               # nan_to_num(100*pi) (:1001-1006)
    err = err + PI * invalid[:, :, None] + PI * invalid_vis[:, None, :]
    return X, err, best.reshape(N, lo) - min_tri_angle


def triangulate_tracks(extrinsics, tn, pairs, track_vis, track_score=None, lo_num=50, max_angular_error=2.0,
                       min_tri_angle=1.5, return_debug=False):
    """triangulate_tracks_single_chunk (triangulation.py:776-956) with the hypothesis pair list given.
    extrinsics [S,3,4], tn [S,N,2], pairs [H0,2], track_vis/track_score [S,N].
    Returns points [N,3] f64, inlier_num [N] int64, inlier_mask [N,S] bool."""
    extrinsics = np.asarray(extrinsics, dtype=np.float64)
    tn = np.asarray(tn, dtype=np.float64)
    thr = max_angular_error * (PI / 180.0)
    S, N, _ = tn.shape
    tn_t = np.transpose(tn, (1, 0, 2))                            # [N,S,2]
    H0 = len(pairs)
    lo = lo_num if H0 >= lo_num else H0
    centers = proj_centers(extrinsics)
    # -- two-view hypotheses
    pts2 = tn_t[:, pairs].reshape(N * H0, 2, 2)
    cams2 = np.broadcast_to(extrinsics[pairs][None], (N, H0, 2, 3, 4)).reshape(N * H0, 2, 3, 4)
    X0 = dlt(cams2, pts2)
    with np.errstate(invalid="ignore"):
        z = np.einsum("bnj,bj->bn", cams2[:, :, 2, :3], X0) + cams2[:, :, 2, 3]
        bad_che = (z <= 0).any(axis=1)
        ang = tri_angle_deg(np.broadcast_to(centers[pairs[:, 0]][None], (N, H0, 3)).reshape(-1, 3),
                            np.broadcast_to(centers[pairs[:, 1]][None], (N, H0, 3)).reshape(-1, 3), X0)
        bad_tri = ~(ang >= min_tri_angle)       # the self pairs of the 2x2 table give 0 deg and never pass
    invalid = (bad_tri | bad_che).reshape(N, H0)
    X0 = X0.reshape(N, H0, 3)
    err = np.transpose(angular_error(tn, np.transpose(X0, (1, 0, 2)), extrinsics), (2, 0, 1))   # [N,H0,S]
    if track_score is not None:
        invalid_vis = (np.asarray(track_vis) <= 0.05) | (np.asarray(track_score) <= 0.5)
    else:
        invalid_vis = np.asarray(track_vis) <= 0.05
    invalid_vis = invalid_vis.T                                   # [N,S]
    err = err + PI * invalid[:, :, None] + PI * invalid_vis[:, None, :]
    with np.errstate(invalid="ignore"):
        inl = err <= thr
    # -- local refinement, two rounds
    order = np.argsort(-inl.sum(axis=-1), axis=1, kind="stable")
    X1, err1, tri1 = _refine(tn_t, extrinsics, centers, inl, order, lo, min_tri_angle, invalid_vis, thr)
    lo2 = 10 if lo > 10 else lo
    inl1 = err1 <= thr
    order1 = np.argsort(-inl1.sum(axis=-1), axis=1, kind="stable")
    X2, err2, tri2 = _refine(tn_t, extrinsics, centers, inl1, order1, lo2, min_tri_angle, invalid_vis, thr)
    allX = np.concatenate([X0, X1, X2], axis=1)
    allE = np.concatenate([err, err1, err2], axis=1)
    score, cnt, mask = residual_indicator(allE, thr, 2 * PI)
    best = np.argmax(score, axis=1)
    ar = np.arange(N)
    out = allX[ar, best], cnt[ar, best].astype(np.int64), mask[ar, best]
    if return_debug:
        # near-tie information: how far each decision that selects or counts something is from flipping
        Xb = allX[ar, best][:, None, :]
        with np.errstate(invalid="ignore"):
            same_point = np.all(np.abs(allX - Xb) <= 1e-9 * (1.0 + np.abs(Xb)), axis=-1)   # NaN -> different
            gate = np.abs(allE - thr)
        gate = np.where(np.isnan(gate), np.inf, gate)                # a NaN error is never an inlier
        other = np.where(same_point, -np.inf, score).max(axis=1)
        return out + (dict(allX=allX, allE=allE, score=score, best=best, order=order, order1=order1, cnt=cnt,
                           mask=mask,
                           # best score minus the best score of a hypothesis with a different point (inf if none)
                           score_margin=score[ar, best] - other,
                           # |angular error - gate| of the chosen hypothesis per observation [N,S], and the
                           # smallest such distance over every hypothesis of the track [N]
                           gate_dist=gate[ar, best], gate_dist_min=gate.min(axis=(1, 2)),
                           # triangulation angle of the two-view pair [N,H0], and of the best camera pair of each
                           # refined hypothesis [N,lo+lo2], minus min_tri_angle (exact within TRI_TIE_DEG of 0)
                           tri_dist0=ang.reshape(N, H0) - min_tri_angle,
                           tri_dist=np.concatenate([tri1, tri2], axis=1)),)
    return out


def triangulate_by_pair(extrinsics, tn):
    """triangulation.py:45-135 on the non-batched inputs: pairs (0, s) for s = 1..S-1.
    Returns points [S-1,N,3], cheirality_mask [S-1,N] (True = in front of both cameras), tri_angle_deg [S-1,N]."""
    S, N, _ = tn.shape
    centers = proj_centers(extrinsics)
    pts = np.stack([np.broadcast_to(tn[0][None], (S - 1, N, 2)), tn[1:]], axis=2).reshape(-1, 2, 2)
    cams = np.stack([np.broadcast_to(extrinsics[0][None], (S - 1, 3, 4)), extrinsics[1:]], axis=1)
    cams = np.broadcast_to(cams[:, None], (S - 1, N, 2, 3, 4)).reshape(-1, 2, 3, 4)
    X = dlt(cams, pts)
    with np.errstate(invalid="ignore"):
        z = np.einsum("bnj,bj->bn", cams[:, :, 2, :3], X) + cams[:, :, 2, 3]
        bad = (z <= 0).any(axis=1)
    c0 = np.broadcast_to(centers[0][None, None], (S - 1, N, 3)).reshape(-1, 3)
    c1 = np.broadcast_to(centers[1:][:, None], (S - 1, N, 3)).reshape(-1, 3)
    ang = tri_angle_deg(c0, c1, X)
    return X.reshape(S - 1, N, 3), ~bad.reshape(S - 1, N), ang.reshape(S - 1, N)


# ----------------------------------------------------------------------------------------------
# reprojection / triangulation-angle filter
# ----------------------------------------------------------------------------------------------

def filter_all_points3D(points3D, points2D, extrinsics, intrinsics, extra_params=None, max_reproj_error=4,
                        min_tri_angle=1.5, check_triangle=True, return_detail=False, hard_max=300):
    """triangulation_helpers.py:215-307.  points3D [P,3], points2D [S,P,2] -> (valid [P], detail [S,P]|None)."""
    p2, pc = project_3D_points(points3D, extrinsics, intrinsics, extra_params)
    with np.errstate(invalid="ignore", over="ignore"):
        e2 = np.sum((p2 - points2D) ** 2, axis=-1)
        e2 = np.where(pc[:, 2, :] <= 0, 1e6, e2)
        inl = e2 <= max_reproj_error ** 2
    valid = inl.sum(axis=0) >= 2
    if hard_max > 0:
        with np.errstate(invalid="ignore"):
            valid = valid & (np.abs(points3D) <= hard_max).all(axis=-1)
    tri_ok_full = None
    if check_triangle:
        idx = np.nonzero(valid)[0]
        tri_ok = any_pair_tri_angle(proj_centers(extrinsics), points3D[idx], min_tri_angle, inl[:, idx])
        tri_ok_full = np.zeros_like(valid)
        tri_ok_full[idx] = tri_ok
        ret = tri_ok_full & valid
    else:
        ret = valid
    detail = None
    if return_detail:
        detail = inl.copy()
        if check_triangle:
            detail = detail & tri_ok_full[None]
    return ret, detail
