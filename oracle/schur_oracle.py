"""Float64 references, with error bars, for the four stages that build the reduced camera system of one LM iteration
(csrc/ba_blocks.cu ba_blocks_kernel, csrc/ba_schur.cu point_prep / z_build / syrk_f64) -- TEST INFRASTRUCTURE ONLY.

Every reference comes with its absolute companion: the same sum taken over bounds of |term|.  A bar is
    (m + c) u A,    u = 2^-53,
where A is the companion, m the number of roundings a sum of the kernel can chain (its terms) and c the roundings
before the sum.  The derivations:

* Observation Jacobians (obs_terms).  ba_obs.h obs_math evaluates r, J_c and J_p as chains of at most C_J = 32
  roundings (rotated point 3, depth / inverse depth 2, normalised coordinates 1, distortion 5, projection derivatives
  4, the rotation columns' cross products 2, the point columns' 3-term products 3, plus slack for FMA contraction
  choices).  Each rounding contributes at most u relative to the companion of its operands: the same formula
  evaluated on |inputs| with every subtraction turned into an addition.  The one division, by the depth pz = a3 + t_z,
  turns the depth's error relative to |a3| + |t_z| into a relative error of 1/pz; the companions are therefore scaled
  by kappa_z = (|a3| + |t_z|) / |pz| (1 for a point well in front of the camera).  So
  |J_kernel - J| <= C_J u J_comp, and the float64 oracle's own J obeys the same bound.
* Products and sums (blocks_ref).  A term x y of an accumulated block differs between kernel and oracle by at most
  2 C_J u (x_c |y| + |x| y_c) + u |x y|; its companion is A_term = x_c |y| + |x| y_c (>= 2 |x y|).  The kernel adds m
  terms (two residual rows per observation; FMA chains, warp trees and f64 REDs are all at most m - 1 additions
  deep); the oracle sums in extended precision (numpy longdouble: 2^-64 on x86), which is below the bar's slack.
  Bar: (m + C0) u A, m = 2 x observations in the sum, C0 = 4 C_J.
* point_prep.  dpp = clip((h s) s) has no addition, so it is exact: compared bitwise (FMA contraction cannot apply).
  M = Dp L^-T with L the 3x3 Cholesky factor of V = Dp H Dp + diag(dpp)/radius: the backward check is
  ||L^-1 V L^-T - I||_max <= C_P u kappa_2(V) with L^-T = Dp^-1 M (Cholesky's backward error (n+1) u |L||L^T| and the
  triangular inverse's n u each turn into kappa_2(V) after the two-sided scaling; C_P = 64 covers n = 3 with room for
  the scale products).  q = M^T g is a sum of at most 3 products: |q - M^T g| <= 3 u |M|^T |g|.
* z_build (zt_ref).  Zt[3n+c, s dc+i] = sum_j W_sn[i, j] M_n[j, c], W_sn = J_c^T J_p of one observation (2-term sum)
  times a 3-term column of M: bar (C_Z) u (W_comp |M|)[i, c], W_comp = J_c,comp^T J_p,comp, C_Z = 4 C_J + 10.  The
  shared-intrinsics columns sum W over the track's observations: bar (m + C_Z) u, m = 2 x observations.  rhs[row] =
  -g[row] + sum_{n,c} Z q over all tracks (zq per lane, one f64 RED per 8-track CTA): bar
  (3 m + N/8 + C_Z + 8) u (|g| + sum Z_comp |q|), m = observations of the frame (all observations for a shared row).
* Written set (written_set).  z_build writes the three Zt rows of track n in the columns of frame group g (32 frames)
  iff some frame of g has a valid observation of n -- and, with a band table, iff the CTA's 8-track tile meets the
  group's track range -- and the shared-intrinsics columns of every track.  Columns [D, Dpad) and rows [3N, Kpad) are
  never written.
* SYRK work list (check_work_list).  The cover contract: every (upper tile, k block) inside the tile's clipped band
  range appears in exactly one item and nothing outside appears; no tile is cut into more than 16 items; no item is
  longer than max_item_kb or empty; items are sorted longest first.
* SYRK NaN set (syrk_nan_set).  A NaN at Zt[k, i] enters every product of the items that read k block k // 64 in a
  tile holding column i: row and column i of exactly those tiles' lower-triangle footprint (0 * NaN is NaN on the
  tensor cores; syrk_red_upper adds every non-zero, and NaN is not zero).
"""
from __future__ import annotations

import numpy as np

from oracle import ba_oracle as bo

U = 2.0 ** -53
C_J = 32
C0 = 4 * C_J
C_P = 64
C_Z = 4 * C_J + 10
MAX_PARTS = 16


# ----------------------------------------------------------------------------------------------
# observation Jacobians with companions
# ----------------------------------------------------------------------------------------------

def _obs(poses, intr, points, uv, mask, model, absmode):
    """(res [S,N,2], Jc [S,N,2,8], Jp [S,N,2,3]) as ba_obs.h obs_math computes them; absmode: the companions (|inputs|,
    subtractions as additions, the true |pz| as divisor)."""
    S, N = mask.shape
    A = np.abs if absmode else (lambda x: x)
    sg = 1.0 if absmode else -1.0
    R, t = A(poses[:, :, :3]), A(poses[:, :, 3])
    X = A(points)
    RX = np.einsum("sij,nj->sni", R, X)
    p = RX + t[:, None, :]
    pz_true = np.einsum("sj,nj->sn", poses[:, 2, :3], points) + poses[:, 2, 3][:, None]
    pz = np.where(mask, np.abs(pz_true) if absmode else pz_true, 1.0)
    iz = 1.0 / pz
    u, v = p[..., 0] * iz, p[..., 1] * iz
    f, cx, cy = A(intr[:, 0])[:, None], A(intr[:, 1])[:, None], A(intr[:, 2])[:, None]
    k = A(intr[:, 3])[:, None] if model == bo.SIMPLE_RADIAL else np.zeros((S, 1))
    r2 = u * u + v * v
    d = 1.0 + k * r2
    uvo = A(uv)
    res = np.stack([f * d * u + cx + sg * uvo[..., 0], f * d * v + cy + sg * uvo[..., 1]], axis=-1)
    if model == bo.SIMPLE_RADIAL:
        a00, a01, a11 = f * (d + 2.0 * k * u * u), f * (2.0 * k * u * v), f * (d + 2.0 * k * v * v)
    else:
        a00, a01, a11 = f + 0 * u, 0 * u, f + 0 * u
    Jproj = np.zeros((S, N, 2, 3))
    Jproj[..., 0, 0], Jproj[..., 0, 1] = a00 * iz, a01 * iz
    Jproj[..., 0, 2] = sg * (a00 * u + a01 * v) * iz
    Jproj[..., 1, 0], Jproj[..., 1, 1] = a01 * iz, a11 * iz
    Jproj[..., 1, 2] = sg * (a01 * u + a11 * v) * iz
    Jp = np.einsum("snij,sjk->snik", Jproj, R)
    Jc = np.zeros((S, N, 2, 8))
    a1, a2, a3 = RX[..., 0], RX[..., 1], RX[..., 2]
    Jc[..., 0] = 2.0 * (a2[..., None] * Jproj[..., 2] + sg * a3[..., None] * Jproj[..., 1])
    Jc[..., 1] = 2.0 * (a3[..., None] * Jproj[..., 0] + sg * a1[..., None] * Jproj[..., 2])
    Jc[..., 2] = 2.0 * (a1[..., None] * Jproj[..., 1] + sg * a2[..., None] * Jproj[..., 0])
    Jc[..., 3:6] = Jproj
    Jc[..., 0, 6], Jc[..., 1, 6] = d * u, d * v
    if model == bo.SIMPLE_RADIAL:
        Jc[..., 0, 7], Jc[..., 1, 7] = f * u * r2, f * v * r2
    if absmode:
        kz = np.where(mask, (np.abs(np.einsum("sj,nj->sn", poses[:, 2, :3], points)) + np.abs(poses[:, 2, 3])[:, None])
                      * np.abs(iz), 0.0)
        res, Jc, Jp = res * kz[..., None], Jc * kz[..., None, None], Jp * kz[..., None, None]
    keep = mask[..., None, None]
    return np.where(mask[..., None], res, 0.0), np.where(keep, Jc, 0.0), np.where(keep, Jp, 0.0)


def obs_terms(c, point_const=None):
    """dict(res, Jc, Jp, res_c, Jc_c, Jp_c): the observation terms of case c (poses, intr, points, uv, mask, model) and
    their companions; a constant point has no point columns (obs_math's vp)."""
    args = (c["poses"], c["intr"], c["points"], np.asarray(c["uv"], dtype=np.float64), np.asarray(c["mask"], bool),
            c["model"])
    with np.errstate(all="ignore"):
        res, Jc, Jp = _obs(*args, absmode=False)
        res_c, Jc_c, Jp_c = _obs(*args, absmode=True)
    if point_const is not None:
        pc = np.asarray(point_const, bool)[None, :, None, None]
        Jp, Jp_c = np.where(pc, 0.0, Jp), np.where(pc, 0.0, Jp_c)
    return dict(res=res, Jc=Jc, Jp=Jp, res_c=res_c, Jc_c=Jc_c, Jp_c=Jp_c)


# ----------------------------------------------------------------------------------------------
# normal-equation blocks
# ----------------------------------------------------------------------------------------------

def _prod_sum(spec, x, xc, y, yc):
    """(sum x y in longdouble -> float64, companion sum (x_c |y| + |x| y_c))"""
    L = np.longdouble
    val = np.einsum(spec, x.astype(L), y.astype(L)).astype(np.float64)
    comp = np.einsum(spec, xc, np.abs(y)) + np.einsum(spec, np.abs(x), yc)
    return val, comp


def blocks_ref(c, point_const=None, terms=None):
    """Reference of everything ba_blocks_kernel accumulates, in the kernel's output layout: dict name -> (ref, bar)
    for cost [1], camrec [S,KR] (g_c | H_cc upper-packed | H_cs[6][ns]), g_p [N,3], H_pp [N,6] (xx,xy,xz,yy,yz,zz) and
    shared [5] (g_s[2], H_ss xx,xy,yy; zeros beyond ns)."""
    t = obs_terms(c, point_const) if terms is None else terms
    mask = np.asarray(c["mask"], bool)
    S, N = mask.shape
    dc, ns = bo.dims(c["model"], c["mode"])
    r, rc = t["res"], t["res_c"]
    Jc, Jcc = t["Jc"][..., :dc], t["Jc_c"][..., :dc]
    Js, Jsc = t["Jc"][..., 6:6 + ns], t["Jc_c"][..., 6:6 + ns]
    Jp, Jpc = t["Jp"], t["Jp_c"]
    m_s = 2.0 * mask.sum(1)                     # terms per frame sum
    m_n = 2.0 * mask.sum(0)                     # terms per point sum
    m_all = 2.0 * mask.sum()
    bar = lambda m, comp: (m + C0) * U * comp
    out = {}
    cost = 0.5 * float(np.sum((r.astype(np.longdouble) ** 2)))
    out["cost"] = (np.array([cost]), bar(m_all, np.array([np.sum(rc * np.abs(r))])))
    g_c, g_cc = _prod_sum("snri,snr->si", Jc, Jcc, r, rc)
    H, Hc = _prod_sum("snri,snrj->sij", Jc, Jcc, Jc, Jcc)
    iu = np.triu_indices(dc)
    parts, comps = [g_c, H[:, iu[0], iu[1]]], [g_cc, Hc[:, iu[0], iu[1]]]
    if ns:
        Hcs, Hcsc = _prod_sum("snri,snrj->sij", Jc[..., :6], Jcc[..., :6], Js, Jsc)
        parts.append(Hcs.reshape(S, 6 * ns))
        comps.append(Hcsc.reshape(S, 6 * ns))
    out["camrec"] = (np.concatenate(parts, 1), bar(m_s[:, None], np.concatenate(comps, 1)))
    g_p, g_pc = _prod_sum("snri,snr->ni", Jp, Jpc, r, rc)
    out["g_p"] = (g_p, bar(m_n[:, None], g_pc))
    Hp, Hpc = _prod_sum("snri,snrj->nij", Jp, Jpc, Jp, Jpc)
    pk = ([0, 0, 0, 1, 1, 2], [0, 1, 2, 1, 2, 2])
    out["H_pp"] = (Hp[:, pk[0], pk[1]], bar(m_n[:, None], Hpc[:, pk[0], pk[1]]))
    sh, shc = np.zeros(5), np.zeros(5)
    if ns:
        gs, gsc = _prod_sum("snri,snr->i", Js, Jsc, r, rc)
        Hs, Hsc = _prod_sum("snri,snrj->ij", Js, Jsc, Js, Jsc)
        sh[:ns], shc[:ns] = gs, gsc
        sh[2], shc[2] = Hs[0, 0], Hsc[0, 0]
        if ns > 1:
            sh[3:5], shc[3:5] = [Hs[0, 1], Hs[1, 1]], [Hsc[0, 1], Hsc[1, 1]]
    out["shared"] = (sh, bar(m_all, shc))
    return out


def check_blocks(got, ref):
    """{name: max |got - ref| / bar} over the entries of blocks_ref; a ratio > 1 is a failure.  got: dict of arrays in
    the kernel's layout (shared may be the 8-double record)."""
    ratios = {}
    for k, (r, b) in ref.items():
        g = np.asarray(got[k], dtype=np.float64).reshape(-1)[:r.size].reshape(r.shape)
        err = np.abs(g - r)
        with np.errstate(invalid="ignore", divide="ignore"):
            q = np.where(err == 0, 0.0, err / b)
        ratios[k] = float(np.max(np.where(np.isnan(q), np.inf, q), initial=0.0))
    return ratios


# ----------------------------------------------------------------------------------------------
# point_prep
# ----------------------------------------------------------------------------------------------

def point_prep_ref(H_pp, sc_p, radius, min_diag, max_diag):
    """(dpp [N,3] as the kernel must produce it bit for bit, V [N,3,3] the damped scaled point block, in float64 with the
    kernel's operation order)"""
    h = np.asarray(H_pp, np.float64)
    s = np.asarray(sc_p, np.float64)
    with np.errstate(all="ignore"):
        diag = np.stack([(h[:, 0] * s[:, 0]) * s[:, 0], (h[:, 3] * s[:, 1]) * s[:, 1], (h[:, 5] * s[:, 2]) * s[:, 2]], 1)
        dpp = np.fmin(np.fmax(diag, min_diag), max_diag)
        off = [(h[:, 1] * s[:, 0]) * s[:, 1], (h[:, 2] * s[:, 0]) * s[:, 2], (h[:, 4] * s[:, 1]) * s[:, 2]]
        V = np.zeros((h.shape[0], 3, 3))
        for i in range(3):
            V[:, i, i] = diag[:, i] + dpp[:, i] / radius
        for (i, j), o in zip(((0, 1), (0, 2), (1, 2)), off):
            V[:, i, j] = V[:, j, i] = o
    return dpp, V


def point_prep_backward(M, V, sc_p):
    """(||L^-1 V L^-T - I||_max, its bar C_P u kappa_2(V)) per point, L^-T = Dp^-1 M, evaluated in extended precision"""
    L = np.longdouble
    Linv_T = M.reshape(-1, 3, 3).astype(L) / np.asarray(sc_p, np.float64).astype(L)[:, :, None]
    E = np.einsum("nji,njk,nkl->nil", Linv_T, V.astype(L), Linv_T) - np.eye(3, dtype=L)
    err = np.abs(E).max(axis=(1, 2)).astype(np.float64)
    with np.errstate(all="ignore"):
        kappa = np.linalg.cond(V)
    return err, C_P * U * kappa


def q_bar(M, g_p):
    """(M^T g in extended precision, 3 u |M|^T |g|) per point"""
    Mm = M.reshape(-1, 3, 3)
    ref = np.einsum("nji,nj->ni", Mm.astype(np.longdouble), np.asarray(g_p).astype(np.longdouble)).astype(np.float64)
    return ref, 3.0 * U * np.einsum("nji,nj->ni", np.abs(Mm), np.abs(g_p))


# ----------------------------------------------------------------------------------------------
# z_build
# ----------------------------------------------------------------------------------------------

def zt_ref(c, M, q, g, Kpad, Dpad, point_const=None, terms=None):
    """(Zt ref [Kpad,Dpad], Zt bar, Zt companion, rhs ref [D], rhs bar) of z_build given the kernel's own M [N,9] and
    q [N,3]; g [D] = the camera gradient assemble_hc put (with the opposite sign) into rhs."""
    t = obs_terms(c, point_const) if terms is None else terms
    mask = np.asarray(c["mask"], bool)
    S, N = mask.shape
    dc, ns = bo.dims(c["model"], c["mode"])
    D = S * dc + ns
    Mm = np.asarray(M, np.float64).reshape(N, 3, 3)
    Ma = np.abs(Mm)
    Jc, Jcc = t["Jc"], t["Jc_c"]
    Jp, Jpc = t["Jp"], t["Jp_c"]
    W = np.einsum("snri,snrj->snij", Jc[..., :dc], Jp)                  # [S,N,dc,3]
    Wc = np.einsum("snri,snrj->snij", Jcc[..., :dc], Jpc)
    Z = np.zeros((Kpad, Dpad))
    Zc = np.zeros((Kpad, Dpad))
    # Zt[3n+c, s dc+i] = sum_j W[s,n,i,j] M[n,j,c]
    Zf = np.einsum("snij,njc->ncsi", W, Mm).reshape(3 * N, S * dc)
    Zfc = np.einsum("snij,njc->ncsi", Wc, Ma).reshape(3 * N, S * dc)
    Z[:3 * N, :S * dc], Zc[:3 * N, :S * dc] = Zf, Zfc
    bar = np.zeros((Kpad, Dpad))
    bar[:3 * N, :S * dc] = C_Z * U * Zfc
    if ns:
        Ws = np.einsum("snri,snrj->nij", Jc[..., 6:6 + ns].astype(np.longdouble), Jp.astype(np.longdouble)).astype(np.float64)
        Wsc = np.einsum("snri,snrj->nij", Jcc[..., 6:6 + ns], Jpc)
        Zs = np.einsum("nij,njc->nci", Ws, Mm).reshape(3 * N, ns)
        Zsc = np.einsum("nij,njc->nci", Wsc, Ma).reshape(3 * N, ns)
        Z[:3 * N, S * dc:D], Zc[:3 * N, S * dc:D] = Zs, Zsc
        m_n = np.repeat(2.0 * mask.sum(0), 3)[:, None]
        bar[:3 * N, S * dc:D] = (m_n + C_Z) * U * Zsc
    qa = np.asarray(q, np.float64).reshape(-1)
    rhs = (-np.asarray(g, np.float64)[:D].astype(np.longdouble) +
           (Z[:3 * N, :D].astype(np.longdouble) * qa[:, None].astype(np.longdouble)).sum(0)).astype(np.float64)
    comp = np.abs(g[:D]) + (Zc[:3 * N, :D] * np.abs(qa)[:, None]).sum(0)
    m = np.concatenate([np.repeat(mask.sum(1), dc), np.full(ns, mask.sum())]).astype(np.float64)
    rhs_bar = (3.0 * m + N / 8.0 + C_Z + 8) * U * comp
    return Z, bar, Zc, rhs, rhs_bar


def written_set(mask, dc, ns, Kpad, Dpad, fg_tracks=None):
    """[Kpad, Dpad] bool: the entries of Zt z_build writes (module docstring)"""
    mask = np.asarray(mask, bool)
    S, N = mask.shape
    ng = (S + 31) // 32
    out = np.zeros((Kpad, Dpad), bool)
    for g in range(ng):
        s0, s1 = 32 * g, min(S, 32 * g + 32)
        reach = mask[s0:s1].any(0)
        if fg_tracks is not None:
            lo, hi = fg_tracks[g]
            n0 = np.arange(N) // 8 * 8
            nt = np.minimum(8, N - n0)
            reach &= ~((n0 + nt <= lo) | (n0 >= hi))
        rows = np.repeat(reach, 3)
        out[:3 * N][rows, s0 * dc:s1 * dc] = True
    out[:3 * N, S * dc:S * dc + ns] = True
    return out


def written_set_brute(mask, dc, ns, Kpad, Dpad, fg_tracks=None):
    """written_set by walking the kernel's loops (CTA of 8 tracks, frame groups, the any-valid test) one by one"""
    mask = np.asarray(mask, bool)
    S, N = mask.shape
    out = np.zeros((Kpad, Dpad), bool)
    for n0 in range(0, N, 8):
        nt = min(8, N - n0)
        for g in range((S + 31) // 32):
            if fg_tracks is not None and (n0 + nt <= fg_tracks[g][0] or n0 >= fg_tracks[g][1]):
                continue
            cnt = min(32, S - 32 * g) * dc
            for tt in range(nt):
                if any(mask[s, n0 + tt] for s in range(32 * g, min(S, 32 * g + 32))):
                    out[3 * (n0 + tt):3 * (n0 + tt) + 3, 32 * g * dc:32 * g * dc + cnt] = True
        out[3 * n0:3 * (n0 + nt), S * dc:S * dc + ns] = True
    return out


# ----------------------------------------------------------------------------------------------
# SYRK work list and NaN propagation
# ----------------------------------------------------------------------------------------------

def tile_ranges(Kpad, Dpad, ranges=None):
    """{(bi, bj): (kb0, kb1)} of the upper tiles the SYRK must cover (bi <= bj), clipped to the band hint"""
    nb, KB = Dpad // 128, (Kpad + 63) // 64
    banded = ranges is not None and len(ranges) == 2 * nb
    out = {}
    for bj in range(nb):
        for bi in range(bj + 1):
            if banded:
                k0, k1 = max(ranges[2 * bi], ranges[2 * bj]), min(ranges[2 * bi + 1], ranges[2 * bj + 1])
                if k1 <= k0:
                    continue
            else:
                k0, k1 = 0, KB
            out[(bi, bj)] = (k0, k1)
    return out


def check_work_list(items, Kpad, Dpad, ranges=None, max_item_kb=None):
    """violations of the cover contract (module docstring) by items [nwork, 4] = (bi, bj, kb0, kb1); empty = none"""
    KB = (Kpad + 63) // 64
    max_item_kb = KB if max_item_kb is None else max_item_kb
    want = tile_ranges(Kpad, Dpad, ranges)
    seen, parts, bad = {}, {}, []
    prev = None
    for w, (bi, bj, k0, k1) in enumerate(np.asarray(items).reshape(-1, 4).tolist()):
        if not k0 < k1:
            bad.append(f"item {w} empty ({k0}, {k1})")
        if k1 - k0 > max_item_kb:
            bad.append(f"item {w} spans {k1 - k0} > {max_item_kb} k blocks")
        if prev is not None and k1 - k0 > prev:
            bad.append(f"item {w} longer than item {w - 1}")
        prev = k1 - k0
        if (bi, bj) not in want:
            bad.append(f"item {w}: tile ({bi}, {bj}) is not to be computed")
            continue
        parts[(bi, bj)] = parts.get((bi, bj), 0) + 1
        for kb in range(k0, k1):
            seen[(bi, bj, kb)] = seen.get((bi, bj, kb), 0) + 1
    for tile, (k0, k1) in want.items():
        if parts.get(tile, 0) > MAX_PARTS:
            bad.append(f"tile {tile} cut into {parts[tile]} > {MAX_PARTS} items")
        for kb in range(k0, k1):
            if seen.get((*tile, kb), 0) != 1:
                bad.append(f"tile {tile} k block {kb} covered {seen.get((*tile, kb), 0)} times")
    for (bi, bj, kb), n in seen.items():
        k0, k1 = want[(bi, bj)]
        if not k0 <= kb < k1:
            bad.append(f"tile ({bi}, {bj}) k block {kb} outside its range [{k0}, {k1})")
    return bad


def syrk_nan_set(items, Dpad, k, i):
    """[Dpad, Dpad] bool: the lower-triangle entries of Cmat that a NaN at Zt[k, i] makes NaN (module docstring)"""
    kb, b = k // 64, i // 128
    out = np.zeros((Dpad, Dpad), bool)
    for bi, bj, k0, k1 in np.asarray(items).reshape(-1, 4).tolist():
        if not (k0 <= kb < k1 and b in (bi, bj)):
            continue
        # tile (bi, bj) lands at Cmat rows of block bj, columns of block bi (lower triangle)
        rows, cols = slice(bj * 128, bj * 128 + 128), slice(bi * 128, bi * 128 + 128)
        blk = np.zeros((128, 128), bool)
        if bj == b:
            blk[i - bj * 128, :] = True
        if bi == b:
            blk[:, i - bi * 128] = True
        out[rows, cols] |= blk
    return np.tril(out)


def check_sentinel(Zt, written):
    """(written entries that still hold a NaN, unwritten entries that are not the all-ones NaN sentinel) of a Zt that
    z_build filled over the sentinel"""
    bits = np.ascontiguousarray(Zt, np.float64).view(np.uint64)
    sentinel = bits == np.uint64(0xFFFFFFFFFFFFFFFF)
    return int((written & np.isnan(Zt)).sum()), int((~written & ~sentinel).sum())
