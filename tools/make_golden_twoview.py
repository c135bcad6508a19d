#!/usr/bin/env python
"""Golden fixtures for the two-view stage (tests/golden/twoview_*.npz): the UNMODIFIED reference
``estimate_fundamental`` (vggsfm/two_view_geo/fundamental.py:43-183) and ``estimate_preliminary_cameras``
(estimate_preliminary.py:98-241) on CPU, float32 tracks (with float64 tracks the reference fails inside run_7point).
kornia is absent: the helpers it provides (normalize_points, normalize_transformation, solve_cubic, transform_points,
the homogeneous conversions and two checks) are restated here [3P-memory].  ``generate_samples`` and ``solve_cubic``
are wrapped to record the sample indices and the roots; no reference file is edited.

Every golden has one dead pair (no valid match), which pins the indicator threshold to 1e6 + 1e-6.  The tool asserts
that no candidate built from a zero-filled root slot (whose matrix depends on LAPACK's null-space basis, DESIGN.md
section 3) reaches a top-lo set or the winner.  Needs $VGGSFM_REFERENCE:   python tools/make_golden_twoview.py"""
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from oracle import reference_shim  # noqa: E402
from vggsfm_b200.synthetic import make_scene  # noqa: E402


def to_h(p):
    return torch.cat([p, torch.ones_like(p[..., :1])], -1)


def from_h(p, eps=1e-8):
    z = p[..., -1:]
    s = torch.where(z.abs() > eps, 1.0 / (z + eps), torch.ones_like(z))
    return s * p[..., :-1]


def transform_points(T, p):
    return from_h(to_h(p) @ T.transpose(-2, -1))


def normalize_points(points, eps=1e-8):
    x_mean = points.mean(dim=1, keepdim=True)
    scale = (points - x_mean).norm(dim=-1, p=2).mean(dim=-1)
    scale = torch.sqrt(torch.tensor(2.0)) / (scale + eps)
    o, z = torch.ones_like(scale), torch.zeros_like(scale)
    T = torch.stack([scale, z, -scale * x_mean[..., 0, 0], z, scale, -scale * x_mean[..., 0, 1], z, z, o], -1)
    T = T.view(-1, 3, 3)
    return transform_points(T, points), T


def normalize_transformation(M, eps=1e-8):
    n = M[..., -1:, -1:]
    return torch.where(n.abs() > eps, M / (n + eps), M)


ROOTS = []


def solve_cubic(coeffs):
    from oracle import twoview_oracle as tvo
    r = torch.from_numpy(tvo.solve_cubic(coeffs.double().numpy())).to(coeffs.dtype)
    ROOTS.append(r.clone())
    return r


def install():
    reference_shim.install()
    kc = sys.modules["kornia.core"]
    kc.concatenate, kc.ones_like, kc.stack, kc.where, kc.zeros = torch.cat, torch.ones_like, torch.stack, torch.where, torch.zeros
    kc.eye = torch.eye
    sys.modules["kornia.core.check"].KORNIA_CHECK_SHAPE = lambda *a, **k: None
    sys.modules["kornia.core.check"].KORNIA_CHECK_IS_TENSOR = lambda *a, **k: None
    sys.modules["kornia.core.check"].KORNIA_CHECK = lambda *a, **k: None
    sys.modules["kornia.core.check"].KORNIA_CHECK_SAME_SHAPE = lambda *a, **k: None
    sys.modules["kornia.utils._compat"].torch_version_ge = lambda *a: True
    sys.modules["kornia.geometry.conversions"].convert_points_to_homogeneous = to_h
    sys.modules["kornia.geometry.conversions"].convert_points_from_homogeneous = from_h
    sys.modules["kornia.geometry.linalg"].transform_points = transform_points
    sys.modules["kornia.geometry.solvers"].solve_cubic = solve_cubic
    sys.modules["kornia.geometry.epipolar.fundamental"].normalize_points = normalize_points
    sys.modules["kornia.geometry.epipolar.fundamental"].normalize_transformation = normalize_transformation


def main():
    install()
    from vggsfm.two_view_geo import fundamental as fm
    from vggsfm.two_view_geo import estimate_preliminary as ep
    recorded = []
    gen = fm.generate_samples

    def recording(*a, **k):
        s = gen(*a, **k)
        recorded.append(np.array(s))
        return s
    fm.generate_samples = recording
    out = os.path.join(ROOT, "tests", "golden")
    for name, seed, B, N, T, lo, max_error in [("twoview_5x256", 0, 5, 256, 256, 30, 2.0),
                                                ("twoview_4x300", 1, 4, 300, 256, 40, 1.0)]:
        sc = make_scene(B + 1, N, seed=seed, noise_px=0.3, outlier_frac=0.05, invisible_frac=0.3)
        tracks = torch.from_numpy(sc.tracks)[None]
        vis = torch.from_numpy(sc.vis)[None].clone()
        vis[0, -1] = 0.0                                                  # the dead pair
        recorded.clear()
        ROOTS.clear()
        np.random.seed(seed)
        torch.manual_seed(seed)
        cams, pd = ep.estimate_preliminary_cameras(tracks, vis, 1024, 1024, max_error=max_error, lo_num=lo,
                                                   max_ransac_iters=T)
        samples = recorded[0]
        roots = ROOTS[0].reshape(B, T, 3).numpy()
        # replay the selection of the reference to check the zero-slot candidates stay out of it
        q = tracks[:, 0:1].expand(-1, B, -1, -1).reshape(B, N, 2)
        r = tracks[:, 1:].reshape(B, N, 2)
        valid = (vis >= 0.05)[:, 1:].reshape(B, N)
        from oracle import twoview_oracle as tvo
        o = tvo.estimate_fundamental(q.numpy(), r.numpy(), samples, max_error=max_error, lo_num=lo,
                                     valid_mask=valid.numpy())
        zero_slot = (roots.reshape(B, 3 * T) == 0)
        for b, p in enumerate(o["pairs"]):
            if b == B - 1:
                continue
            assert not zero_slot[b][p["seeds1"]].any(), ("zero-slot candidate in the top-lo set", name, b)
            assert not (o["best"][b] < 3 * T and zero_slot[b][o["best"][b]]), ("zero-slot winner", name, b)
        fmat = pd["fmat"][0].numpy()
        mask = pd["fmat_inlier_mask"][0].numpy()
        np.savez_compressed(os.path.join(out, name + ".npz"), points1=q.numpy(), points2=r.numpy(),
                            valid=valid.numpy(), samples=samples.astype(np.int32), max_error=max_error, lo_num=lo,
                            width=1024, height=1024, fmat=fmat, inlier_mask=mask, inlier_num=mask.sum(-1),
                            residuals=pd["fmat_residuals"][0].numpy(),
                            R=pd["R_opencv"][0, 1:].numpy(), t=pd["t_opencv"][0, 1:].numpy())
        print(name, mask.sum(-1))


if __name__ == "__main__":
    main()
