"""GPU parity of the correlation kernels: reference goldens, the float32 torch oracle on fresh inputs, linearity in
the targets at the BASELINE C4 shape, and -- per output -- the float64 reference of oracle/corr_oracle.py on the
kernels' own pyramid and rounded targets: |out - ref| <= tau * bound, bound = the bilinear combination of
sum_c |t_c f_c| / sqrt(C).  tau = 2^-16 for the wgmma kernel (csrc/corr_tc.cu: fp32 accumulation of 128 fp16
products), 2^-18 for the CUDA-core kernels (csrc/corr.cu).  Largest err / bound observed on an H100 80GB HBM3 (700 W
limit): 2.6e-7 for the wgmma kernel (C4 shape), 2.1e-7 for the CUDA-core kernels; each check prints its own."""
import glob
import math
import os

import numpy as np
import pytest
import torch

from oracle import corr_oracle as co

pytestmark = pytest.mark.gpu
TAU_TC = 2.0 ** -16
TAU_CC = 2.0 ** -18
GOLDEN = sorted(glob.glob(os.path.join(os.path.dirname(__file__), "golden", "corr_*.npz")))


@pytest.mark.parametrize("path", GOLDEN, ids=[os.path.basename(p)[:-4] for p in GOLDEN])
def test_against_reference_golden(cuda_dev, path):
    from vggsfm_b200.corr import CorrBlock, EfficientCorrBlock
    g = np.load(path)
    f, t, c = (torch.from_numpy(g[k]).to(cuda_dev) for k in ("fmaps", "targets", "coords"))
    L, r = int(g["num_levels"]), int(g["radius"])
    cb = CorrBlock(f, num_levels=L, radius=r, half=False)
    cb.corr(t)
    out = cb.sample(c).cpu().numpy()
    assert out.shape == g["out_zeros"].shape
    assert np.abs(out - g["out_zeros"]).max() < 2e-4 * np.abs(g["out_zeros"]).max()
    eb = EfficientCorrBlock(f, num_levels=L, radius=r, half=False)
    outb = eb.sample(c, t).cpu().numpy()
    assert np.abs(outb - g["out_border"]).max() < 2e-4 * np.abs(g["out_border"]).max()


@pytest.mark.parametrize("B,S,C,H,W,N,L,r", [(1, 4, 128, 64, 64, 50, 5, 4), (7, 3, 32, 31, 31, 1, 3, 3), (2, 2, 64, 24, 40, 9, 3, 4)])
def test_against_oracle_float_and_half(cuda_dev, B, S, C, H, W, N, L, r):
    from vggsfm_b200.corr import CorrBlock
    g = torch.Generator().manual_seed(B * 100 + S)
    f = torch.randn(B, S, C, H, W, generator=g)
    t = torch.randn(B, S, N, C, generator=g)
    c = torch.rand(B, S, N, 2, generator=g) * torch.tensor([W + 8.0, H + 8.0]) - 4.0     # crosses every border
    ref = co.corr_sample(f, t, c, L, r).numpy()
    rng = np.abs(ref).max()
    cb = CorrBlock(f.to(cuda_dev), num_levels=L, radius=r, half=False)
    cb.corr(t.to(cuda_dev))
    out = cb.sample(c.to(cuda_dev)).cpu().numpy()
    assert np.abs(out - ref).max() < 2e-4 * rng
    cbh = CorrBlock(f.to(cuda_dev), num_levels=L, radius=r, half=True)
    cbh.corr(t.to(cuda_dev))
    outh = cbh.sample(c.to(cuda_dev))
    ref64, bound = co.corr_reference(co.kernel_pyramid(f, L), t.half().float(), c, r)
    _assert_within(outh.cpu(), ref64, bound, TAU_TC if cbh._pyr.tc_tiles is not None else TAU_CC, "half")


def test_c4_shape_linearity(cuda_dev):
    """BASELINE C4 coarse shape per chunk is [1,128,128,128,128] x 1024 queries; run 16 frames of it at full
    spatial size and check linearity in the targets and zero response far outside the map."""
    from vggsfm_b200.corr import CorrBlock
    g = torch.Generator().manual_seed(0)
    f = torch.randn(1, 16, 128, 128, 128, generator=g).to(cuda_dev)
    t1 = torch.randn(1, 16, 1024, 128, generator=g).to(cuda_dev)
    t2 = torch.randn(1, 16, 1024, 128, generator=g).to(cuda_dev)
    c = (torch.rand(1, 16, 1024, 2, generator=g) * 119 + 4).to(cuda_dev)
    cb = CorrBlock(f, num_levels=5, radius=4, half=False)
    outs = []
    for t in (t1, t2, t1 + 2 * t2):
        cb.corr(t)
        outs.append(cb.sample(c))
    assert outs[0].shape == (1, 16, 1024, 405)
    err = (outs[2] - (outs[0] + 2 * outs[1])).abs().max().item()
    assert err < 1e-3 * outs[2].abs().max().item()
    cb.corr(t1)
    far = cb.sample(torch.full_like(c, -1000.0))
    assert far.abs().max().item() == 0.0


@pytest.mark.parametrize("H,W,N,L,r", [(32, 32, 130, 3, 4), (24, 64, 256, 4, 3), (128, 128, 128, 5, 4)])
def test_tensor_core_path_matches_cuda_core_path(cuda_dev, H, W, N, L, r):
    """csrc/corr_tc.cu (wgmma f16, footprint extraction from the register accumulators) against csrc/corr.cu on the same half
    pyramid: both round targets and features to fp16 and accumulate in fp32, only the summation order differs (1e-3 of
    the value range); queries on, near and beyond the border, a ragged last 128-query tile, non-square maps."""
    import torch
    from vggsfm_b200.corr import CorrBlock
    g = torch.Generator(device=cuda_dev).manual_seed(H + N)
    B, S, C = 1, 3, 128
    fm = torch.randn(B, S, C, H, W, device=cuda_dev, generator=g)
    tg = torch.randn(B, S, N, C, device=cuda_dev, generator=g)
    co = torch.rand(B, S, N, 2, device=cuda_dev, generator=g) * torch.tensor([W + 10.0, H + 10.0], device=cuda_dev) - 5.0
    co[0, 0, 0] = torch.tensor([0.0, 0.0], device=cuda_dev)
    co[0, 0, 1] = torch.tensor([W - 1.0, H - 1.0], device=cuda_dev)
    co[0, 1, 2] = torch.tensor([3.5, 7.25], device=cuda_dev)
    a = CorrBlock(fm, num_levels=L, radius=r, half=True, tc=True)
    assert a._pyr.tc_tiles is not None
    b = CorrBlock(fm, num_levels=L, radius=r, half=True, tc=False)
    assert b._pyr.tc_tiles is None
    a.corr(tg)
    b.corr(tg)
    ya, yb = a.sample(co), b.sample(co)
    torch.cuda.synchronize()
    scale = yb.abs().max().item()
    assert scale > 1.0
    assert (ya - yb).abs().max().item() <= 1e-3 * scale, (ya - yb).abs().max().item() / scale


def _assert_within(out, ref, bound, tau, what=""):
    """|out - ref| <= tau * bound for every output (a zero bound demands an exact zero; a NaN output fails)."""
    err = (out.double() - ref).abs()
    ratio = torch.nan_to_num(err / bound.clamp_min(1e-300), nan=math.inf).max().item()
    print(f"corr {what}: max err/bound = {ratio:.3g} (tau {tau:.3g})")
    bad = ~(err <= tau * bound)
    assert not bad.any(), (what, ratio, bad.nonzero()[:5].tolist())


def _coords(B, S, N, H, W, dev, seed):
    """Uniform over [-6, W+6] x [-6, H+6], with every 8th query on an exact integer, (W-1, H-1), a half-integer or
    at -1000 (whose taps must all read exactly 0)."""
    g = torch.Generator(device=dev).manual_seed(seed)
    c = torch.rand(B, S, N, 2, device=dev, generator=g) * torch.tensor([W + 12.0, H + 12.0], device=dev) - 6.0
    flat = c.view(-1, 2)
    m = torch.arange(flat.shape[0], device=dev) % 8
    flat[m == 1] = torch.floor(flat[m == 1])
    flat[m == 2] = torch.tensor([W - 1.0, H - 1.0], device=dev)
    flat[m == 3] = torch.floor(flat[m == 3]) + 0.5
    flat[m == 4] = -1000.0
    return c


def _check_tc(dev, B, S, N, H, W, L, r, seed, what, cb=None, f=None):
    from vggsfm_b200.corr import CorrBlock
    g = torch.Generator(device=dev).manual_seed(seed)
    if cb is None:
        f = torch.randn(B, S, 128, H, W, device=dev, generator=g)
        cb = CorrBlock(f, num_levels=L, radius=r, half=True)
    assert cb._pyr.tc_tiles is not None
    t = torch.randn(B, S, N, 128, device=dev, generator=g)
    c = _coords(B, S, N, H, W, dev, seed + 1)
    cb.corr(t)
    out = cb.sample(c)
    far = (c == -1000.0).all(dim=-1)
    assert (out[far] == 0).all()
    ref, bound = co.corr_reference(co.kernel_pyramid(f, L), t.half().float(), c, r)
    _assert_within(out, ref, bound, TAU_TC, what)


def test_half_pyramid_is_bit_exact(cuda_dev):
    """The NHWC fp16 levels of CorrBlock._pyr.pyr (at align_up(BS h w C 2, 256) offsets, csrc/corr.cu) equal
    kernel_pyramid bit for bit, odd heights at the deep levels included."""
    from vggsfm_b200.corr import CorrBlock
    g = torch.Generator(device=cuda_dev).manual_seed(7)
    for (B, S, C, H, W, L) in [(1, 3, 128, 40, 16, 4), (2, 2, 32, 32, 32, 6), (1, 2, 64, 27, 22, 3)]:
        f = torch.randn(B, S, C, H, W, device=cuda_dev, generator=g) * 3
        cb = CorrBlock(f, num_levels=L, radius=4, half=True)
        raw = cb._pyr.pyr
        off = 0
        for lv in co.kernel_pyramid(f, L):
            h, w = lv.shape[-2:]
            n = B * S * h * w * C
            got = raw[off:off + 2 * n].view(torch.float16).view(B * S, h, w, C)
            want = lv.reshape(B * S, C, h, w).permute(0, 2, 3, 1).half()
            assert torch.equal(got.view(torch.int16), want.contiguous().view(torch.int16)), (H, W, L, h, w)
            off += (2 * n + 255) // 256 * 256
        assert off == raw.numel()


def test_tensor_core_c4_shape_against_float64(cuda_dev):
    """The C4 coarse shape as benched (128 frames x 1024 queries, 128 x 128, 5 levels, r = 4): 1024 work items, every
    CTA runs 7-8 of them, so the A-tile reuse and the B-ring stage/phase carried across items are exercised.
    Every frame is checked."""
    _check_tc(cuda_dev, 1, 128, 1024, 128, 128, 5, 4, 0, "C4")


@pytest.mark.parametrize("B,S,N,H,W,L,r", [
    (1, 200, 200, 128, 128, 4, 3),        # 85 position tiles per item: the ring phase flips between items
    (1, 140, 1, 32, 32, 3, 4),            # query tails, > 132 items each
    (1, 140, 64, 32, 32, 3, 4),           # the second warpgroup has no query
    (1, 140, 65, 32, 32, 3, 3),           # ... exactly one
    (1, 140, 127, 32, 32, 3, 4),
    (1, 70, 129, 32, 32, 3, 4),
    (2, 70, 130, 64, 64, 4, 4),           # B = 2
    (1, 6, 300, 32, 32, 6, 4),            # deep levels narrower than the footprint, the last one 1 x 1
    (1, 6, 300, 40, 16, 4, 3),            # odd height (5) at the last level
])
def test_tensor_core_shapes_against_float64(cuda_dev, B, S, N, H, W, L, r):
    _check_tc(cuda_dev, B, S, N, H, W, L, r, S + N, f"{B}x{S}x{N} {H}x{W} L{L} r{r}")


def test_tensor_core_scratch_reuse(cuda_dev):
    """One CorrBlock sampled with a growing, then shrinking, number of queries and fresh targets every call: the target
    tile scratch is reused and must never leak an earlier call's targets."""
    from vggsfm_b200.corr import CorrBlock
    g = torch.Generator(device=cuda_dev).manual_seed(3)
    f = torch.randn(1, 3, 128, 64, 64, device=cuda_dev, generator=g)
    cb = CorrBlock(f, num_levels=4, radius=4, half=True)
    for i, N in enumerate([200, 500, 129, 1, 300]):
        _check_tc(cuda_dev, 1, 3, N, 64, 64, 4, 4, 100 + i, f"reuse N={N}", cb=cb, f=f)


def test_tensor_core_path_selection(cuda_dev):
    """The wgmma kernel is used iff C = 128, the pyramid is half, the map width is a power of two, r in {3, 4} and the
    padding is zeros -- including half=None under fp16 autocast, which is how the coarse tracker runs."""
    from vggsfm_b200.corr import CorrBlock
    g = torch.Generator(device=cuda_dev).manual_seed(4)
    f = torch.randn(1, 2, 128, 32, 32, device=cuda_dev, generator=g)
    tc = lambda cb: cb._pyr.tc_tiles is not None
    assert tc(CorrBlock(f, num_levels=3, radius=4, half=True))
    assert tc(CorrBlock(f, num_levels=3, radius=3, half=True))
    assert not tc(CorrBlock(f, num_levels=3, radius=2, half=True))
    assert not tc(CorrBlock(f, num_levels=3, radius=4, half=False))
    assert not tc(CorrBlock(f, num_levels=3, radius=4, half=True, padding_mode="border"))
    assert not tc(CorrBlock(f[:, :, :64], num_levels=3, radius=4, half=True))
    assert not tc(CorrBlock(torch.randn(1, 2, 128, 32, 48, device=cuda_dev, generator=g), num_levels=3, radius=4, half=True))
    assert not tc(CorrBlock(f, num_levels=3, radius=4))                     # float32 maps, no autocast
    assert tc(CorrBlock(f.half(), num_levels=3, radius=4))
    with torch.autocast("cuda", dtype=torch.float16):
        cb = CorrBlock(f, num_levels=3, radius=4)
    assert cb._pyr.elem == 2 and tc(cb)
    _check_tc(cuda_dev, 1, 2, 150, 32, 32, 3, 4, 9, "autocast", cb=cb, f=f)


@pytest.mark.parametrize("border", [False, True], ids=["zeros", "border"])
@pytest.mark.parametrize("half", [False, True], ids=["float", "half"])
@pytest.mark.parametrize("C,r", [(32, 3), (32, 4), (64, 4), (128, 4), (128, 3)])
def test_cuda_core_path_against_float64(cuda_dev, C, r, half, border):
    """csrc/corr.cu (channel-per-lane kernel, and the position-per-lane one for C = 32) against the float64 reference,
    so the tensor-core and CUDA-core paths no longer vouch for each other."""
    from vggsfm_b200.corr import CorrBlock
    B, S, N, H, W, L = 2, 3, 45, 24, 20, 3
    g = torch.Generator(device=cuda_dev).manual_seed(C + r + 2 * half + border)
    f = torch.randn(B, S, C, H, W, device=cuda_dev, generator=g)
    t = torch.randn(B, S, N, C, device=cuda_dev, generator=g)
    c = _coords(B, S, N, H, W, cuda_dev, C + r)
    cb = CorrBlock(f, num_levels=L, radius=r, half=half, tc=False, padding_mode="border" if border else "zeros")
    assert cb._pyr.tc_tiles is None
    cb.corr(t)
    out = cb.sample(c)
    ref, bound = co.corr_reference(co.kernel_pyramid(f, L, half=half), t.half().float() if half else t, c, r, border=border)
    _assert_within(out, ref, bound, TAU_CC, f"cuda-core C={C} r={r} half={half} border={border}")
