"""CPU: correlation oracle vs the goldens produced by the reference CorrBlock / EfficientCorrBlock."""
import glob
import os

import numpy as np
import pytest
import torch

from oracle import corr_oracle as co

GOLDEN = sorted(glob.glob(os.path.join(os.path.dirname(__file__), "golden", "corr_*.npz")))


@pytest.mark.parametrize("path", GOLDEN, ids=[os.path.basename(p)[:-4] for p in GOLDEN])
def test_corr_oracle_matches_reference_golden(path):
    g = np.load(path)
    f, t, c = (torch.from_numpy(g[k]) for k in ("fmaps", "targets", "coords"))
    L, r = int(g["num_levels"]), int(g["radius"])
    out = co.corr_sample(f, t, c, L, r, border=False).numpy()
    # float32 volume + float32 normalise/unnormalise round trip in grid_sample: 1e-4 of the value range
    tol = 2e-4 * np.abs(g["out_zeros"]).max()
    assert np.abs(out - g["out_zeros"]).max() < tol
    outb = co.corr_sample(f, t, c, L, r, border=True).numpy()
    assert np.abs(outb - g["out_border"]).max() < 2e-4 * np.abs(g["out_border"]).max()


@pytest.mark.parametrize("border", [False, True])
def test_float64_reference_matches_float32_oracle(border):
    """corr_reference (float64, the yardstick of the CUDA kernels) against corr_sample (float32) on the same float
    pyramid, with taps across every border, and the bound is an upper bound of |out|."""
    g = torch.Generator().manual_seed(5)
    B, S, C, H, W, N, L, r = 2, 3, 32, 19, 24, 11, 3, 3
    f = torch.randn(B, S, C, H, W, generator=g)
    t = torch.randn(B, S, N, C, generator=g)
    c = torch.rand(B, S, N, 2, generator=g) * torch.tensor([W + 12.0, H + 12.0]) - 6.0
    ref32 = co.corr_sample(f, t, c, L, r, border=border).double()
    out, bound = co.corr_reference(co.build_pyramid(f, L), t, c, r, border=border)
    assert out.shape == ref32.shape and out.dtype == torch.float64
    assert torch.all((out - ref32).abs() <= 2.0 ** -18 * bound + 1e-30)
    assert torch.all(out.abs() <= bound * (1 + 2.0 ** -40))
    assert bound.max() > 0


@pytest.mark.parametrize("path", GOLDEN, ids=[os.path.basename(p)[:-4] for p in GOLDEN])
def test_float64_reference_matches_reference_golden(path):
    g = np.load(path)
    f, t, c = (torch.from_numpy(g[k]) for k in ("fmaps", "targets", "coords"))
    L, r = int(g["num_levels"]), int(g["radius"])
    lv = co.build_pyramid(f, L)
    for key, border in (("out_zeros", False), ("out_border", True)):
        out, bound = co.corr_reference(lv, t, c, r, border=border)
        assert np.abs(out.numpy() - g[key]).max() < 2e-4 * np.abs(g[key]).max()


@pytest.mark.parametrize("H,W,L", [(32, 32, 6), (40, 16, 4), (31, 31, 3), (7, 13, 3)])
def test_kernel_pyramid_matches_build_pyramid(H, W, L):
    """The bit-exact pyramid of the kernels: float levels equal avg_pool2d's, half levels are their fp16 roundings."""
    f = torch.randn(2, 2, 8, H, W, generator=torch.Generator().manual_seed(H * W))
    ref = co.build_pyramid(f, L)
    lv32 = co.kernel_pyramid(f, L, half=False)
    lv16 = co.kernel_pyramid(f, L, half=True)
    for a, b, h in zip(ref, lv32, lv16):
        assert a.shape == b.shape == h.shape
        assert torch.allclose(a, b, rtol=2.0 ** -22, atol=0)
        assert torch.equal(h, b.half().float())
    assert lv32[-1].shape[-2:] == (H >> (L - 1), W >> (L - 1))
