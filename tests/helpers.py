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
