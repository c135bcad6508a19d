"""GPU: the correlation and sampling kernels at their edges, per output against the float64 references of
oracle/corr_oracle.py under the bars of tests/test_corr_gpu.py (|out - ref| <= tau * bound, a zero bound demands an
exact 0, a NaN fails; tau = 2^-16 for the wgmma kernel, 2^-18 for the CUDA-core kernels).

- Coordinates: every kernel gets each x crossed with each y from NaN, ±inf, ±2^31, ±3e9, 1e38, -0.0, -1e-30 and, per
  level l (scaled by 2^l), W_l - 1, the next float above it, an in-map value, and both ends of the clamp window
  [-(r+2), W_l + r + 1] with the next float beyond each.  The edge queries share 128-query tiles and warp rows
  (q0, q0 + 8 of csrc/corr_tc.cu) with random in-map ones, which must come out unchanged.  The non-finite and
  beyond-int-range queries are also checked against live F.grid_sample on the device (ATen's CUDA kernel), which tests
  the oracle's rule.
- Empty and tiny query sets: N = 0 through every entry point (null pointers at the C ABI), then a normal call on the same
  block; N = 1, 7, 8, 9 around the 8-queries-per-CTA grid of csrc/corr.cu.
- Production shapes: the fine tracker as bench.py runs it (131 072 images of 31 x 31, C = 32) with the half pyramid, and
  at B = 256 with the float one; EfficientCorrBlock at the C4 coarse shape (border padding, channel-per-lane kernel);
  sample_features4d at the triangulator's colour read-back (400 x 4096 points on 1024 x 1024 images).
- The C = 32 scalar-load fallback, reached only through a target pointer that is not 16-byte aligned.
Each check prints its largest error-to-bound ratio."""
import ctypes
import math

import numpy as np
import pytest
import torch

from oracle import corr_oracle as co
from tests.test_corr_gpu import TAU_CC, TAU_TC, _assert_within, _coords

pytestmark = pytest.mark.gpu

SPECIAL = [math.nan, math.inf, -math.inf, 2.0 ** 31, -2.0 ** 31, 3e9, -3e9, 1e38, -0.0, -1e-30]


def _f32_next(v, direction):
    return float(np.nextafter(np.float32(v), np.float32(direction)))


def _axis_values(size, L, r):
    """level-0 coordinates that put some level's coordinate on an edge of a map axis of `size` positions"""
    vals = list(SPECIAL)
    for l in range(L):
        s, k = size >> l, 2.0 ** l
        lo, hi = -(r + 2.0), s + r + 1.0
        for v in (s - 1.0, _f32_next(s - 1.0, math.inf), 0.37 * s, lo, _f32_next(lo, -math.inf), hi,
                  _f32_next(hi, math.inf)):
            vals.append(float(np.float32(v)) * k)
    out, seen = [], set()
    for v in vals:
        key = "nan" if math.isnan(v) else (v, math.copysign(1.0, v))
        if key not in seen:
            seen.add(key)
            out.append(v)
    return out


def _edge_queries(xs, ys, H, W, dev, seed):
    """[N,2] float32 coordinates holding every (x, y) pair, and the mask of those slots.  Queries come in blocks of 8
    that alternate between edge pairs and random in-map queries; the order flips every 128 queries, so an edge query
    is the q0 of a good q0 + 8 in one tile and the other way round in the next."""
    pairs = torch.tensor([(x, y) for x in xs for y in ys], dtype=torch.float32)
    P = pairs.shape[0]
    N = -(-P // 8) * 16
    n = torch.arange(N)
    edge = ((n // 8) + (n // 128)) % 2 == 0
    g = torch.Generator().manual_seed(seed)
    c = torch.rand(N, 2, generator=g) * torch.tensor([W + 4.0, H + 4.0]) - 2.0
    slots = edge.nonzero().flatten()[:P]
    c[slots] = pairs
    mask = torch.zeros(N, dtype=torch.bool)
    mask[slots] = True
    return c.to(dev), mask.to(dev)


def _ratio(out, ref, bound):
    return torch.nan_to_num((out.double() - ref).abs() / bound.clamp_min(1e-300), nan=math.inf).max().item()


def _corr_case(dev, C, H, W, L, r, half, border, tc, seed, S=2):
    from vggsfm_b200.corr import CorrBlock
    g = torch.Generator(device=dev).manual_seed(seed)
    f = torch.randn(1, S, C, H, W, device=dev, generator=g)
    c, mask = _edge_queries(_axis_values(W, L, r), _axis_values(H, L, r), H, W, dev, seed)
    N = c.shape[0]
    c = c.expand(1, S, N, 2).contiguous()
    t = torch.randn(1, S, N, C, device=dev, generator=g)
    cb = CorrBlock(f, num_levels=L, radius=r, half=half, tc=tc, padding_mode="border" if border else "zeros")
    assert (cb._pyr.tc_tiles is not None) == bool(tc)
    cb.corr(t)
    out = cb.sample(c)
    ref, bound = co.corr_reference(co.kernel_pyramid(f, L, half=half), t.half().float() if half else t, c, r,
                                   border=border, frames=S)
    what = f"{'wgmma' if tc else 'cuda-core'} C={C} {H}x{W} L{L} r{r} half={half} border={border}"
    print(f"{what}: edge queries max err/bound = {_ratio(out[:, :, mask], ref[:, :, mask], bound[:, :, mask]):.3g}, "
          f"their neighbours {_ratio(out[:, :, ~mask], ref[:, :, ~mask], bound[:, :, ~mask]):.3g}")
    _assert_within(out, ref, bound, TAU_TC if tc else TAU_CC, what)
    if not border:
        nonfinite = ~torch.isfinite(c).all(dim=-1)
        assert (out[nonfinite] == 0).all()


@pytest.mark.parametrize("r", [3, 4])
def test_tensor_core_edge_coordinates(cuda_dev, r):
    _corr_case(cuda_dev, 128, 40, 32, 3, r, True, False, True, 10 + r)


@pytest.mark.parametrize("border", [False, True], ids=["zeros", "border"])
@pytest.mark.parametrize("half", [False, True], ids=["float", "half"])
@pytest.mark.parametrize("C", [64, 128])
def test_channel_per_lane_edge_coordinates(cuda_dev, C, half, border):
    _corr_case(cuda_dev, C, 24, 20, 3, 4, half, border, False, C + 2 * half + border)


@pytest.mark.parametrize("border", [False, True], ids=["zeros", "border"])
@pytest.mark.parametrize("half", [False, True], ids=["float", "half"])
def test_position_per_lane_edge_coordinates(cuda_dev, half, border):
    """corr_sample_c32_kernel: the fine tracker's C = 32, 31 x 31, r = 3"""
    _corr_case(cuda_dev, 32, 31, 31, 3, 3, half, border, False, 40 + 2 * half + border)


@pytest.mark.parametrize("border", [False, True], ids=["zeros", "border"])
def test_edge_rule_matches_grid_sample_on_device(cuda_dev, border):
    """The oracle's coordinate rule against live F.grid_sample on CUDA (oracle.TorchCorrBlock, float32 volume): every query
    with a non-finite coordinate reads exactly 0 with zeros padding on both (ATen's kernel; the cuDNN sampler torch uses
    by default returns NaN at a NaN coordinate, asserted so that the difference stays documented); with border padding, where both coordinates
    are non-finite or beyond the int range, every tap reads a clamped corner or edge, the same on both up to the float32
    matmul (2^-14 of the bound)."""
    C, H, W, L, r, S = 32, 24, 20, 3, 4, 2
    g = torch.Generator(device=cuda_dev).manual_seed(5)
    f = torch.randn(1, S, C, H, W, device=cuda_dev, generator=g)
    c, _ = _edge_queries(_axis_values(W, L, r), _axis_values(H, L, r), H, W, cuda_dev, 5)
    N = c.shape[0]
    c = c.expand(1, S, N, 2).contiguous()
    t = torch.randn(1, S, N, C, device=cuda_dev, generator=g)
    tb = co.TorchCorrBlock(f, num_levels=L, radius=r, padding_mode="border" if border else "zeros")
    tb.corr(t)
    live = tb.sample(c)
    ref, bound = co.corr_reference(co.build_pyramid(f, L), t, c, r, border=border, frames=S)
    nonfinite = ~torch.isfinite(c).all(dim=-1)
    assert nonfinite.sum() > 100
    if not border:
        # torch sends zeros / bilinear / align_corners=True on CUDA to cudnn_grid_sampler while cuDNN is enabled (the
        # default); cuDNN returns NaN at a NaN coordinate, as CPU grid_sample does.  The rule is ATen's own CUDA kernel.
        with torch.backends.cudnn.flags(enabled=False):
            native = tb.sample(c)
        assert (native[nonfinite] == 0).all() and (ref[nonfinite] == 0).all() and (bound[nonfinite] == 0).all()
        assert torch.isnan(live[torch.isnan(c).any(dim=-1)]).all()
        return
    clamped = (~torch.isfinite(c) | (c.abs() >= 2.0 ** 31)).all(dim=-1)
    assert clamped.sum() > 50
    err = (live[clamped].double() - ref[clamped]).abs()
    print(f"grid_sample border, clamped queries: max err/bound = {(err / bound[clamped]).max().item():.3g}")
    assert (err <= 2.0 ** -14 * bound[clamped]).all()


@pytest.mark.parametrize("C", [3, 128, 130])
def test_sample_features4d_edge_coordinates(cuda_dev, C):
    """sample_features_kernel on the same crossing of edge values (W - 1, the next float, an in-map value), with the
    edge points in the same warps' neighbourhood as random ones."""
    from vggsfm_b200.corr import sample_features4d
    B, H, W = 2, 23, 17
    g = torch.Generator(device=cuda_dev).manual_seed(C)
    inp = torch.randn(B, C, H, W, device=cuda_dev, generator=g)
    c, mask = _edge_queries(_axis_values(W, 1, 0), _axis_values(H, 1, 0), H, W, cuda_dev, C)
    c = c.expand(B, -1, 2).contiguous()
    out = sample_features4d(inp, c)
    ref, bound = co.sample_features4d_reference(inp, c)
    assert torch.isfinite(out).all()
    _assert_within(out, ref, bound, TAU_CC, f"sample_features4d C={C} edge coordinates")


def test_empty_query_sets(cuda_dev):
    """N = 0 returns the empty [B,S,0,L*K*K] tensor on the wgmma path, the CUDA-core path and EfficientCorrBlock; the
    C ABI accepts it with null pointers and launches nothing.  The same blocks then sample a normal query set."""
    from vggsfm_b200 import _lib
    from vggsfm_b200.corr import CorrBlock, EfficientCorrBlock
    g = torch.Generator(device=cuda_dev).manual_seed(11)
    B, S, C, H, W, L, r = 1, 3, 128, 32, 32, 3, 4
    f = torch.randn(B, S, C, H, W, device=cuda_dev, generator=g)
    lib = _lib.lib()
    assert lib.vgg_corr_sample(S, 0, C, H, W, L, r, None, 2, None, None, 0, None, None) == 0
    assert lib.vgg_corr_sample(0, 5, C, H, W, L, r, None, 4, None, None, 1, None, None) == 0
    assert lib.vgg_corr_tc_sample(S, 0, C, H, W, L, r, None, None, None, None, None, None) == 0
    assert lib.vgg_corr_tc_sample(0, 5, C, H, W, L, r, None, None, None, None, None, None) == 0
    assert lib.vgg_sample_features4d(0, 3, H, W, 5, None, None, None, None) == 0
    assert lib.vgg_sample_features4d(2, 3, H, W, 0, None, None, None, None) == 0
    blocks = {"wgmma": CorrBlock(f, num_levels=L, radius=r, half=True),
              "cuda-core": CorrBlock(f, num_levels=L, radius=r, half=True, tc=False),
              "efficient": EfficientCorrBlock(f, num_levels=L, radius=r, half=True)}
    assert blocks["wgmma"]._pyr.tc_tiles is not None and blocks["cuda-core"]._pyr.tc_tiles is None
    lv = co.kernel_pyramid(f, L)
    for name, cb in blocks.items():
        border = name == "efficient"
        for N in (0, 37, 0, 5):
            t = torch.randn(B, S, N, C, device=cuda_dev, generator=g)
            c = _coords(B, S, N, H, W, cuda_dev, N + 1)
            if border:
                out = cb.sample(c, t)
            else:
                cb.corr(t)
                out = cb.sample(c)
            torch.cuda.synchronize()
            assert out.shape == (B, S, N, L * (2 * r + 1) ** 2) and out.dtype == torch.float32
            if N:
                ref, bound = co.corr_reference(lv, t.half().float(), c, r, border=border)
                _assert_within(out, ref, bound, TAU_TC if name == "wgmma" else TAU_CC, f"{name} N={N} after N=0")
    from vggsfm_b200.corr import sample_features4d
    assert sample_features4d(f[0], torch.zeros(S, 0, 2, device=cuda_dev)).shape == (S, 0, C)


@pytest.mark.parametrize("N", [1, 7, 8, 9])
@pytest.mark.parametrize("C,tc", [(32, False), (64, False), (128, False), (128, True)], ids=["c32", "c64", "c128", "wgmma"])
def test_tiny_query_sets(cuda_dev, C, tc, N):
    """BS * N = 3, 21, 24, 27 queries: the last 8-query CTA of csrc/corr.cu partly empty, full, or one query over"""
    from vggsfm_b200.corr import CorrBlock
    B, S, H, W, L, r = 1, 3, 32, 32, 3, 4 if C == 128 else 3
    g = torch.Generator(device=cuda_dev).manual_seed(C + N)
    f = torch.randn(B, S, C, H, W, device=cuda_dev, generator=g)
    t = torch.randn(B, S, N, C, device=cuda_dev, generator=g)
    c = _coords(B, S, N, H, W, cuda_dev, N)
    cb = CorrBlock(f, num_levels=L, radius=r, half=True, tc=tc)
    assert (cb._pyr.tc_tiles is not None) == tc
    cb.corr(t)
    out = cb.sample(c)
    ref, bound = co.corr_reference(co.kernel_pyramid(f, L), t.half().float(), c, r)
    _assert_within(out, ref, bound, TAU_TC if tc else TAU_CC, f"C={C} tc={tc} N={N}")


@pytest.mark.parametrize("B,half", [(1024, True), (256, False)], ids=["half-B1024", "float-B256"])
def test_fine_tracker_as_benched(cuda_dev, B, half):
    """bench.py's fine section: [B,128,32,31,31] patches, one query each, 3 levels, r = 3, on the position-per-lane
    kernel; every output is checked (the oracle runs 64 patches at a time on the kernel's own pyramid)."""
    from vggsfm_b200.corr import CorrBlock
    S, C, H, W, N, L, r = 128, 32, 31, 31, 1, 3, 3
    g = torch.Generator(device=cuda_dev).manual_seed(B)
    f = torch.randn(B, S, C, H, W, device=cuda_dev, dtype=torch.float16 if half else torch.float32, generator=g)
    t = torch.randn(B, S, N, C, device=cuda_dev, generator=g)
    c = _coords(B, S, N, H, W, cuda_dev, B + 1)
    cb = CorrBlock(f, num_levels=L, radius=r, half=half)
    assert cb._pyr.elem == (2 if half else 4)
    cb.corr(t)
    out = cb.sample(c)
    del cb
    torch.cuda.synchronize()
    worst = 0.0
    for b0 in range(0, B, 64):
        sl = slice(b0, b0 + 64)
        tt = t[sl].half().float() if half else t[sl]
        ref, bound = co.corr_reference(co.kernel_pyramid(f[sl], L, half=half), tt, c[sl], r, frames=S)
        worst = max(worst, _ratio(out[sl], ref, bound))
        _assert_within(out[sl], ref, bound, TAU_CC, f"fine B={B} half={half} patches {b0}..{b0 + 63}")
    print(f"fine tracker B={B} half={half}: max err/bound = {worst:.3g}")


def test_efficient_corr_block_c4_shape(cuda_dev):
    """EfficientCorrBlock (border padding, channel-per-lane kernel) at the C4 coarse shape: 128 frames x 1024 queries,
    128 x 128, 5 levels, r = 4, half pyramid; every frame is checked."""
    from vggsfm_b200.corr import EfficientCorrBlock
    B, S, C, H, W, N, L, r = 1, 128, 128, 128, 128, 1024, 5, 4
    g = torch.Generator(device=cuda_dev).manual_seed(12)
    f = torch.randn(B, S, C, H, W, device=cuda_dev, generator=g)
    t = torch.randn(B, S, N, C, device=cuda_dev, generator=g)
    c = _coords(B, S, N, H, W, cuda_dev, 13)
    eb = EfficientCorrBlock(f, num_levels=L, radius=r, half=True)
    out = eb.sample(c, t)
    ref, bound = co.corr_reference(co.kernel_pyramid(f, L), t.half().float(), c, r, border=True)
    _assert_within(out, ref, bound, TAU_CC, "EfficientCorrBlock C4")


@pytest.mark.parametrize("border", [False, True], ids=["zeros", "border"])
@pytest.mark.parametrize("half", [False, True], ids=["float", "half"])
def test_c32_unaligned_targets_fallback(cuda_dev, half, border):
    """C = 32 with a targets pointer 4 bytes past a 16-byte boundary: launch_corr falls back from the position-per-lane
    kernel (16-byte loads) to the channel-per-lane one with scalar loads.  Edge and random queries."""
    from vggsfm_b200 import _lib
    from vggsfm_b200.corr import CorrBlock
    B, S, C, H, W, L, r = 1, 2, 32, 31, 31, 3, 3
    g = torch.Generator(device=cuda_dev).manual_seed(20 + 2 * half + border)
    f = torch.randn(B, S, C, H, W, device=cuda_dev, generator=g)
    c, _ = _edge_queries(_axis_values(W, L, r), _axis_values(H, L, r), H, W, cuda_dev, 21)
    N = c.shape[0]
    c = c.expand(B, S, N, 2).contiguous()
    t = torch.randn(B, S, N, C, device=cuda_dev, generator=g)
    cb = CorrBlock(f, num_levels=L, radius=r, half=half, tc=False)
    buf = torch.empty(B * S * N * C + 4, device=cuda_dev)
    tv = buf[1:1 + B * S * N * C]
    tv.copy_(t.reshape(-1))
    assert tv.data_ptr() % 16 == 4
    K2 = (2 * r + 1) ** 2
    out = torch.full((B, S, N, L * K2), math.nan, device=cuda_dev)
    stream = torch.cuda.current_stream(cuda_dev).cuda_stream
    _lib.check(_lib.lib().vgg_corr_sample(B * S, N, C, H, W, L, r, ctypes.c_void_p(cb._pyr.pyr.data_ptr()), cb._pyr.elem,
                                          ctypes.c_void_p(tv.data_ptr()), ctypes.c_void_p(c.data_ptr()), int(border),
                                          ctypes.c_void_p(out.data_ptr()), ctypes.c_void_p(stream)), "vgg_corr_sample")
    ref, bound = co.corr_reference(co.kernel_pyramid(f, L, half=half), t.half().float() if half else t, c, r,
                                   border=border, frames=S)
    _assert_within(out, ref, bound, TAU_CC, f"C=32 unaligned targets half={half} border={border}")


@pytest.mark.parametrize("B,C,H,W,R", [
    (400, 3, 1024, 1024, 4096),           # the triangulator's colour read-back
    (3, 128, 1, 40, 300),                 # one row
    (3, 130, 40, 1, 300),                 # one column
    (2, 3, 1, 1, 77),                     # one pixel
])
def test_sample_features4d_shapes(cuda_dev, B, C, H, W, R):
    """sample_features4d against its float64 reference (border, the reference's float32 normalisation): random points
    over [-2, W + 1] x [-2, H + 1], every 16th on the last row / column or just beyond it."""
    from vggsfm_b200.corr import sample_features4d
    g = torch.Generator(device=cuda_dev).manual_seed(B + C + H)
    inp = torch.rand(B, C, H, W, device=cuda_dev, generator=g)
    c = torch.rand(B, R, 2, device=cuda_dev, generator=g) * torch.tensor([W + 3.0, H + 3.0], device=cuda_dev) - 2.0
    c[:, ::16] = torch.tensor([W - 1.0, H - 1.0], device=cuda_dev)
    c[:, 1::16, 0] = _f32_next(W - 1.0, math.inf)
    out = sample_features4d(inp, c)
    worst = 0.0
    for b0 in range(0, B, 40):
        sl = slice(b0, b0 + 40)
        ref, bound = co.sample_features4d_reference(inp[sl], c[sl])
        worst = max(worst, _ratio(out[sl], ref, bound))
        _assert_within(out[sl], ref, bound, TAU_CC, f"sample_features4d {B}x{R} C={C} {H}x{W} frames {b0}..")
    print(f"sample_features4d {B}x{R} C={C} {H}x{W}: max err/bound = {worst:.3g}")
