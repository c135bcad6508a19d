"""CPU: correlation oracle vs the goldens produced by the reference CorrBlock / EfficientCorrBlock."""
import glob
import math
import os

import numpy as np
import pytest
import torch
import torch.nn.functional as F

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


EDGE = [float("nan"), float("inf"), float("-inf"), 3e9, -3e9, 2.0 ** 31, -2.0 ** 31]


def _grid_sample_taps(vol, x, y, mode):
    """CPU F.grid_sample of vol [1,1,H,W] at pixel coordinates x, y [T] (align_corners=True) -> [T] float64"""
    H, W = vol.shape[-2:]
    g = torch.stack([x * (2.0 / (W - 1)) - 1.0, y * (2.0 / (H - 1)) - 1.0], dim=-1).reshape(1, 1, -1, 2)
    return F.grid_sample(vol, g.float(), align_corners=True, padding_mode=mode).reshape(-1).double()


def test_coordinate_rule_matches_grid_sample_border():
    """Border padding: the oracle's coordinate rule (NaN -> 0, -inf / -3e9 / -2^31 -> 0, +inf / 3e9 / 2^31 -> W - 1)
    equals CPU grid_sample on every pairing of an edge value with an edge or in-map value."""
    H, W = 5, 7
    vol = torch.randn(1, 1, H, W, generator=torch.Generator().manual_seed(1))
    vals = EDGE + [0.0, 2.0, W - 1.0]
    x = torch.tensor([a for a in vals for b in vals], dtype=torch.float32)
    y = torch.tensor([b for a in vals for b in vals], dtype=torch.float32)
    edge = ~(torch.isin(x, torch.tensor(vals[-3:])) & torch.isin(y, torch.tensor(vals[-3:])))
    got = co._bilinear_gather(vol.double().reshape(1, H, W), x[None].double(), y[None].double(), True)[0]
    want = _grid_sample_taps(vol, x, y, "border")
    assert torch.isfinite(got).all()
    assert edge.sum() == len(vals) ** 2 - 9
    assert torch.allclose(got, want, rtol=1e-6, atol=0), (got - want).abs().max()


def test_coordinate_rule_zeros_differs_from_cpu_grid_sample():
    """Zeros padding: a non-finite coordinate contributes nothing in the oracle (grid_sample on CUDA maps it to -100,
    outside the map), while CPU grid_sample returns NaN there.  Finite coordinates beyond the int range read 0 on both."""
    H, W = 5, 7
    vol = torch.randn(1, 1, H, W, generator=torch.Generator().manual_seed(2))
    for v in EDGE:
        for other in (2.0, v):
            for x, y in ((v, other), (other, v)):
                xt, yt = torch.tensor([x]), torch.tensor([y])
                got = co._bilinear_gather(vol.double().reshape(1, H, W), xt[None].double(), yt[None].double(), False)
                cpu = _grid_sample_taps(vol, xt, yt, "zeros")
                assert got.item() == 0.0, (x, y, got)
                if math.isfinite(x) and math.isfinite(y):
                    assert cpu.item() == 0.0, (x, y, cpu)
                else:
                    assert math.isnan(cpu.item()), (x, y, cpu)


@pytest.mark.parametrize("border", [False, True], ids=["zeros", "border"])
def test_float64_reference_on_edge_coordinates(border):
    """corr_reference on queries at NaN, ±inf and beyond the int range: every output finite; exact zeros with zeros
    padding; with border padding NaN, -inf, -3e9 and -2^31 read what -1e6 reads (the first row / column) and +inf, 3e9,
    2^31 and 1e38 what +1e6 reads (the last)."""
    g = torch.Generator().manual_seed(6)
    B, S, C, H, W, L, r = 1, 2, 16, 12, 10, 2, 3
    f = torch.randn(B, S, C, H, W, generator=g)
    lv = co.build_pyramid(f, L)
    edge = torch.tensor([[math.nan, 3.0], [math.inf, -math.inf], [-3e9, 2.0 ** 31], [1e38, math.nan], [-2.0 ** 31, 3e9]])
    same = torch.tensor([[-1e6, 3.0], [1e6, -1e6], [-1e6, 1e6], [1e6, -1e6], [-1e6, 1e6]])
    N = edge.shape[0]
    t = torch.randn(B, S, N, C, generator=g)
    out, bound = co.corr_reference(lv, t, edge.expand(B, S, N, 2).contiguous(), r, border=border)
    assert torch.isfinite(out).all() and torch.isfinite(bound).all()
    if not border:
        assert (out == 0).all() and (bound == 0).all()
        return
    ref, ref_bound = co.corr_reference(lv, t, same.expand(B, S, N, 2).contiguous(), r, border=True)
    assert torch.equal(out, ref) and torch.equal(bound, ref_bound)
    assert (bound > 0).all()


def test_sample_features4d_reference():
    """The float64 sample_features4d against CPU grid_sample (border, align_corners=True) through the reference's
    float32 normalisation, on in-map, border-crossing and edge coordinates, W = 1 and H = 1 included."""
    g = torch.Generator().manual_seed(8)
    for B, C, H, W in [(2, 3, 9, 13), (1, 5, 1, 7), (1, 4, 6, 1), (1, 2, 1, 1)]:
        inp = torch.randn(B, C, H, W, generator=g)
        R = 64
        c = torch.rand(B, R, 2, generator=g) * torch.tensor([W + 4.0, H + 4.0]) - 2.0
        c[:, :len(EDGE), 0] = torch.tensor(EDGE)
        c[:, len(EDGE):2 * len(EDGE), 1] = torch.tensor(EDGE)
        out, bound = co.sample_features4d_reference(inp, c)
        assert out.shape == bound.shape == (B, R, C) and out.dtype == torch.float64
        assert torch.isfinite(out).all() and (out.abs() <= bound * (1 + 2.0 ** -40)).all()
        # the reference's own statement: bilinear_sampler + grid_sample (CPU border mode clips NaN to 0 as CUDA does)
        s = torch.tensor([2 / max(W - 1, 1), 2 / max(H - 1, 1)])
        grid = (c * s - 1).unsqueeze(2)
        want = F.grid_sample(inp, grid, align_corners=True, padding_mode="border").permute(0, 2, 1, 3).reshape(B, R, C)
        assert (out - want.double()).abs().max() <= 2.0 ** -20 * bound.max(), (B, C, H, W)
        err = (out - want.double()).abs()
        assert (err <= 2.0 ** -20 * bound + 1e-30).all(), (B, C, H, W, (err / bound.clamp_min(1e-300)).max())
