"""Shared test helpers: scene -> oracle/CUDA argument sets."""
import numpy as np

from oracle import ba_oracle as bo
from vggsfm_b200.synthetic import make_scene, perturb


def ba_case(S, N, camera_type, mode, seed=0, invisible_frac=0.2, noise_px=0.3):
    sc = make_scene(S, N, camera_type, seed=seed, invisible_frac=invisible_frac, noise_px=noise_px)
    model = bo.SIMPLE_RADIAL if camera_type == "SIMPLE_RADIAL" else bo.SIMPLE_PINHOLE
    extr, K, extra, pts = perturb(sc, seed=seed + 1)
    intr = np.zeros((S, 4))
    intr[:, 0] = K[:, 0, 0]
    intr[:, 1] = K[:, 0, 2]
    intr[:, 2] = K[:, 1, 2]
    if extra is not None:
        intr[:, 3] = extra[:, 0]
    if mode == bo.INTR_SHARED:
        intr[:] = intr[0]
    return dict(scene=sc, model=model, mode=mode, poses=extr, intr=intr, points=pts,
                uv=sc.tracks.astype(np.float64), mask=sc.mask, K=K, extra=extra)


def banded_mask(S, N, life, seed, holes=0.2):
    """Sequential (video-like) visibility: point n is born in a frame (births sorted, so storage order = creation
    order) and seen for `life` to 1.5 `life` frames, with a fraction `holes` of those observations missing."""
    rng = np.random.default_rng(seed)
    m = np.zeros((S, N), dtype=bool)
    births = np.sort(rng.integers(0, max(1, S - life // 2), size=N))        # creation order = storage order
    for n, b in enumerate(births):
        m[b:min(S, b + life + rng.integers(0, life // 2 + 1)), n] = True
    m &= rng.uniform(size=m.shape) > holes
    return m


def banded_ba_case(S, N, camera_type, mode, life, seed=0, mask_seed=0):
    """ba_case with a banded visibility mask: the scene's observations stay, only which of them are used changes."""
    c = ba_case(S, N, camera_type, mode, seed=seed, invisible_frac=0.0)
    c["mask"] = banded_mask(S, N, life, mask_seed)
    return c


def far_points_first_case():
    """ba_case(8, 128, SIMPLE_PINHOLE, INTR_CONST, seed=2) with the tracks sorted by descending |X|: over 2 track shards
    the first holds the far points, and each shard's own points give an |x| well below the true one"""
    c = ba_case(8, 128, "SIMPLE_PINHOLE", bo.INTR_CONST, seed=2)
    order = np.argsort(-np.linalg.norm(c["points"], axis=1), kind="stable")
    return dict(c, points=c["points"][order].copy(), uv=c["uv"][:, order].copy(), mask=c["mask"][:, order].copy())


def shuffled_twin(c, seed=0):
    """c with its points in a fixed random order: the same problem, but every frame's visible points span the whole
    track axis, so the band detection of vgg_ba_solve finds nothing to skip and the solve takes its dense path"""
    perm = np.random.default_rng(seed).permutation(c["mask"].shape[1])
    return dict(c, points=c["points"][perm].copy(), uv=c["uv"][:, perm].copy(), mask=c["mask"][:, perm].copy())


def hidden_case(S, N, cam, mode, seed, point_value, uv_value, n_hidden=3, hidden_frame=None, case=None):
    """(problem with hidden values, its clean twin, hidden point indices).  The hidden points' columns are masked out
    entirely; a third of the other masked slots get uv_value; hidden_frame (if given) loses every observation and gets a
    NaN pose.  case: start from this ba_case / banded_ba_case instead of a new ba_case (S, N, cam, mode unused)."""
    c = ba_case(S, N, cam, mode, seed=seed) if case is None else case
    mask = c["mask"].copy()
    rng = np.random.default_rng(seed)
    hidden = rng.choice(N, size=n_hidden, replace=False)
    mask[:, hidden] = False
    if hidden_frame is not None:
        mask[hidden_frame] = False
    clean = dict(c, mask=mask, uv=np.where(mask[..., None], c["uv"], 0.0), points=c["points"].copy())
    clean["points"][hidden] = [0.0, 0.0, 1.0]
    dirty = dict(clean, uv=clean["uv"].copy(), points=clean["points"].copy(), poses=c["poses"].copy())
    dirty["points"][hidden] = point_value
    off = np.argwhere(~mask)
    pick = off[rng.uniform(size=len(off)) < 1.0 / 3.0]
    dirty["uv"][pick[:, 0], pick[:, 1]] = uv_value
    if hidden_frame is not None:
        dirty["poses"][hidden_frame] = np.nan
    return dirty, clean, hidden


def to_dev(a, dev, dtype=None):
    import torch
    t = torch.from_numpy(np.ascontiguousarray(a))
    if dtype is not None:
        t = t.to(dtype)
    return t.to(dev).contiguous()


def unpack_camrec(camrec, shared, S, dc, ns):
    """camrec[S,KR] -> g_c[S,dc], H_cc[S,dc,dc], H_cs[S,6,ns]; shared[8] -> g_s[ns], H_ss[ns,ns]."""
    g_c = camrec[:, :dc]
    H = np.zeros((S, dc, dc))
    idx = dc
    for i in range(dc):
        for j in range(i, dc):
            H[:, i, j] = camrec[:, idx]
            H[:, j, i] = camrec[:, idx]
            idx += 1
    H_cs = camrec[:, idx:idx + 6 * ns].reshape(S, 6, ns) if ns else None
    g_s = shared[:ns]
    H_ss = None
    if ns:
        full = np.array([[shared[2], shared[3]], [shared[3], shared[4]]])
        H_ss = full[:ns, :ns]
    return g_c, H, H_cs, g_s, H_ss


def rotation_angle_deg(R1, R2):
    """Geodesic rotation distance in degrees (the quantity of vggsfm/utils/metric.py:305-318), evaluated as
    2*asin(|R1-R2|_F / (2*sqrt(2))) so that it stays accurate near zero (acos((tr-1)/2) bottoms out at ~1e-6 deg)."""
    d = np.linalg.norm((R1 - R2).reshape(R1.shape[0], -1), axis=1)
    return np.degrees(2.0 * np.arcsin(np.clip(d / (2.0 * np.sqrt(2.0)), 0.0, 1.0)))


# One LM step of vgg_ba_solve against the oracle's damped system (tests/test_lm_step_gpu.py, tests/test_ba_lm_edges_gpu.py)

EPS = 2.0 ** -52


def so3_log(R):
    """rotation vectors of [..., 3, 3] rotations, accurate for small angles"""
    w = 0.5 * np.stack([R[..., 2, 1] - R[..., 1, 2], R[..., 0, 2] - R[..., 2, 0], R[..., 1, 0] - R[..., 0, 1]], -1)
    s = np.linalg.norm(w, axis=-1)
    th = np.arctan2(s, 0.5 * (np.trace(R, axis1=-2, axis2=-1) - 1.0))
    return w * np.where(s > 0, th / np.where(s > 0, s, 1.0), 1.0)[..., None]


def recovered_step(old, new, S, dc, ns, model, mode):
    """(camera step [D], its uncertainty [D], point step [N,3], its uncertainty [N,3]) from the parameters before and after
    the iteration: R_new = Exp(2 delta) R_old, everything else additive."""
    (p0, i0, x0), (p1, i1, x1) = old, new
    D = S * dc + ns
    d, u = np.zeros(D), np.zeros(D)
    dcam, ucam = d[:S * dc].reshape(S, dc), u[:S * dc].reshape(S, dc)
    R0, R1 = p0[:, :, :3], p1[:, :, :3]
    dcam[:, 0:3] = 0.5 * so3_log(R1 @ R0.transpose(0, 2, 1))
    ucam[:, 0:3] = EPS * np.maximum(np.abs(R0).max(axis=(1, 2)), np.abs(R1).max(axis=(1, 2)))[:, None]
    dcam[:, 3:6] = p1[:, :, 3] - p0[:, :, 3]
    ucam[:, 3:6] = EPS * np.maximum(np.abs(p0[:, :, 3]), np.abs(p1[:, :, 3]))
    for j, col in enumerate([0, 3][:bo.n_intr(model)]):
        if mode == bo.INTR_PER_FRAME:
            dcam[:, 6 + j] = i1[:, col] - i0[:, col]
            ucam[:, 6 + j] = EPS * np.maximum(np.abs(i0[:, col]), np.abs(i1[:, col]))
        elif mode == bo.INTR_SHARED:
            d[S * dc + j] = i1[0, col] - i0[0, col]
            u[S * dc + j] = EPS * max(abs(i0[0, col]), abs(i1[0, col]))
    return d, u, x1 - x0, EPS * np.maximum(np.abs(x0), np.abs(x1))


def reference_system(c, param_const, point_const, radius=1e4, min_diag=1e-6, max_diag=1e32):
    """The damped system of the first iteration in scaled variables (oracle/ba_oracle.py lm_solve) at trust-region
    radius `radius`: camera block A [D,D], coupling B [D,N,3], point blocks V [N,3,3], gradients; rows and columns of
    constant parameters / points zeroed."""
    S, N = c["mask"].shape
    model, mode = c["model"], c["mode"]
    dc, ns = bo.dims(model, mode)
    blocks = bo.build_blocks_c if bo._load_c() is not None else bo.build_blocks
    blk = blocks(c["poses"], c["intr"], c["points"], c["uv"], c["mask"], model, mode, point_const)
    Hc, gc = bo._assemble_camera_system(blk, S, dc, ns)
    W = bo._full_W(blk, S, dc, ns)
    fc, fp = ~param_const, ~point_const
    sc_c = 1.0 / (1.0 + np.sqrt(np.diag(Hc)))
    sc_p = 1.0 / (1.0 + np.sqrt(np.einsum("nii->ni", blk["H_pp"])))
    dcc = np.clip(np.diag(Hc) * sc_c * sc_c, min_diag, max_diag)
    Hps = blk["H_pp"] * sc_p[:, :, None] * sc_p[:, None, :]
    dpp = np.clip(np.einsum("nii->ni", Hps), min_diag, max_diag)
    A = (Hc * np.outer(sc_c, sc_c) + np.diag(dcc / radius)) * np.outer(fc, fc)
    B = W * (sc_c * fc)[:, None, None] * (sc_p * fp[:, None])[None]
    V = Hps + dpp[:, :, None] * np.eye(3) / radius
    return dict(cost=blk["cost"], gc=gc, gp=blk["g_p"], sc_c=sc_c, sc_p=sc_p, dcc=dcc, dpp=dpp, fc=fc, fp=fp, A=A,
                B=B.reshape(A.shape[0], 3 * N), V=V, gcs=gc * sc_c * fc, gps=blk["g_p"] * sc_p * fp[:, None])


def backward_error(ref, dcs, ucs, dps, ups):
    """normwise backward error of the scaled step (dcs [D], dps [N,3]) in the full damped system, evaluated blockwise"""
    A, B, V, fc, fp = ref["A"], ref["B"], ref["V"], ref["fc"], ref["fp"]
    N = V.shape[0]
    rc = A @ dcs + B @ dps.reshape(-1) + ref["gcs"]
    rp = (B.T @ dcs).reshape(N, 3) + np.einsum("nij,nj->ni", V, dps) + ref["gps"]
    absB = np.abs(B)
    row_c = np.abs(A).sum(1) + absB.sum(1)
    row_p = absB.sum(0).reshape(N, 3) + np.abs(V).sum(2)
    res = max(np.abs(rc[fc]).max(initial=0.0), np.abs(rp[fp]).max(initial=0.0))
    normH = max(row_c[fc].max(initial=0.0), row_p[fp].max(initial=0.0))
    nd = max(np.abs(dcs[fc]).max(initial=0.0), np.abs(dps[fp]).max(initial=0.0))
    nu = max(np.abs(ucs[fc]).max(initial=0.0), np.abs(ups[fp]).max(initial=0.0))
    ng = max(np.abs(ref["gcs"]).max(initial=0.0), np.abs(ref["gps"]).max(initial=0.0))
    return res / (normH * (nd + nu) + ng)


def tiny_former(in_dim, out_dim, seed):
    """Deterministic stand-in for the tracker's EfficientUpdateFormer (a learned module outside the hot path) used by
    the tracker host-loop goldens: token-wise + time-mixed + track-mixed linear maps, so that a wrong permutation of the
    (track, frame) axes or a wrong input layout changes the output."""
    import torch
    import torch.nn as nn

    class TinyFormer(nn.Module):
        def __init__(self):
            super().__init__()
            self.a = nn.Linear(in_dim, out_dim)
            self.b = nn.Linear(in_dim, out_dim)

        def forward(self, x):                       # [B, N, S, D] -> [B, N, S, out]
            # coordinate outputs (first two channels) small, feature outputs O(1): the loop then stays a contraction
            # (GroupNorm re-normalises the feature delta, so a tiny delta would amplify float32 rounding differences
            # between two correct correlation implementations ~20x per iteration and the golden would pin nothing)
            y = (torch.tanh(self.a(x)) + 0.5 * torch.tanh(self.b(x.mean(dim=2, keepdim=True)))
                 + 0.25 * torch.tanh(self.b(x.mean(dim=1, keepdim=True))))
            scale = torch.ones(y.shape[-1], device=y.device, dtype=y.dtype)
            scale[:2] = 0.08
            return y * scale

    g = torch.Generator().manual_seed(seed)
    m = TinyFormer()
    with torch.no_grad():
        for p in m.parameters():
            p.copy_(torch.randn(p.shape, generator=g) * 0.05)
    return m
