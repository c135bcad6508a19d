"""CPU oracle for the tracker's correlation inner loop -- TEST INFRASTRUCTURE ONLY.

torch-CPU float32 restatement of CorrBlock (vggsfm/models/track_modules/blocks.py:338-416):
pyramid by repeated avg_pool2d(2,2) (:352-361), full correlation volume per level divided by sqrt(C)
(:396-416), then (2r+1)^2 bilinear taps per level with align_corners=True semantics and zero padding
(:363-394 via models/utils.py:347-412); and of EfficientCorrBlock.sample (:433-471, border padding).
The bilinear gather is written out by hand (no grid_sample) so it is an independent statement.
PINNED against the reference through tests/golden/corr_*.npz (tools/make_golden_corr.py).

corr_reference is the float64 statement the CUDA kernels are checked against: it takes the pyramid levels and targets
already rounded to the kernel's precision (kernel_pyramid rebuilds the kernels' pyramid bit for bit), and returns with
every output the same bilinear combination of sum_c |t_c f_c| / sqrt(C), the scale of the kernel's rounding error.
sample_features4d_reference is the float64 statement of sample_features4d, with the same kind of bound.  Both follow
grid_sample's coordinate rule on CUDA for non-finite and far-away coordinates (_source_coordinate).
"""
import math

import torch
import torch.nn.functional as F


def build_pyramid(fmaps, num_levels):
    B, S, C, H, W = fmaps.shape
    pyr = [fmaps]
    for _ in range(num_levels - 1):
        f = F.avg_pool2d(fmaps.reshape(B * S, C, H, W), 2, stride=2)
        _, _, H, W = f.shape
        fmaps = f.reshape(B, S, C, H, W)
        pyr.append(fmaps)
    return pyr


def _source_coordinate(x, size, border):
    """grid_sample's coordinate rule on CUDA (ATen/native/cuda/GridSampler.cuh compute_coordinates): border padding clips
    with fmaxf semantics (NaN -> 0, -inf -> 0, +inf -> size - 1); then a non-finite coordinate, or one beyond INT_MAX - 1
    or below INT_MIN, becomes -100 (safe_downgrade_to_int_range), outside the map, so with zeros padding it contributes
    nothing.  CPU grid_sample, and on CUDA the cuDNN sampler that torch uses by default for zeros / bilinear /
    align_corners=True, return NaN at a NaN coordinate with zeros padding; ATen's CUDA kernel is the rule here."""
    if border:
        x = torch.nan_to_num(x, nan=0.0, posinf=float(size - 1), neginf=0.0).clamp(0, size - 1)
    bad = ~torch.isfinite(x) | (x > 2.0 ** 31 - 2) | (x < -2.0 ** 31)
    return torch.where(bad, torch.full_like(x, -100.0), x)


def _bilinear_gather(vol, x, y, border):
    """vol [Q,H,W,...]; x,y [Q,T] pixel coords -> [Q,T,...]."""
    Q, H, W = vol.shape[:3]
    x = _source_coordinate(x, W, border)
    y = _source_coordinate(y, H, border)
    x0 = torch.floor(x)
    y0 = torch.floor(y)
    wx = x - x0
    wy = y - y0
    x0 = x0.long()
    y0 = y0.long()
    out = torch.zeros(x.shape + vol.shape[3:], dtype=vol.dtype, device=vol.device)
    qi = torch.arange(Q, device=vol.device)[:, None].expand_as(x0)
    for dy, wyv in ((0, 1 - wy), (1, wy)):
        for dx, wxv in ((0, 1 - wx), (1, wx)):
            xi = x0 + dx
            yi = y0 + dy
            if border:
                xi = xi.clamp(0, W - 1)
                yi = yi.clamp(0, H - 1)
                inside = torch.ones_like(xi, dtype=torch.bool)
            else:
                inside = (xi >= 0) & (xi < W) & (yi >= 0) & (yi < H)
            v = vol[qi, yi.clamp(0, H - 1), xi.clamp(0, W - 1)]
            w = torch.where(inside, wxv * wyv, torch.zeros_like(wxv)).to(vol.dtype)
            out = out + v * w.reshape(w.shape + (1,) * (vol.dim() - 3))
    return out


def corr_sample(fmaps, targets, coords, num_levels, radius, border=False):
    """fmaps [B,S,C,H,W], targets [B,S,N,C], coords [B,S,N,2] -> [B,S,N,L*(2r+1)^2] float32."""
    B, S, N, C = targets.shape
    r = radius
    K = 2 * r + 1
    outs = []
    d = torch.arange(-r, r + 1, dtype=torch.float32)
    for i, fm in enumerate(build_pyramid(fmaps.float(), num_levels)):
        H, W = fm.shape[-2:]
        vol = torch.einsum("bsnc,bschw->bsnhw", targets.float(), fm) / torch.sqrt(torch.tensor(float(C)))
        c = coords.float().reshape(B * S * N, 2) / 2 ** i
        # tap (a, b): x = cx + d[a], y = cy + d[b]   (blocks.py:374-382: the row-varying grid goes to x)
        x = (c[:, 0:1, None] + d[None, :, None]).expand(-1, K, K).reshape(-1, K * K)
        y = (c[:, 1:2, None] + d[None, None, :]).expand(-1, K, K).reshape(-1, K * K)
        outs.append(_bilinear_gather(vol.reshape(B * S * N, H, W), x, y, border).reshape(B, S, N, K * K))
    return torch.cat(outs, dim=-1)


class TorchCorrBlock:
    """Stock-PyTorch statement of CorrBlock on ANY device (blocks.py:338-416): per level one torch.matmul of the targets
    with every spatial position (fp16 under autocast on a GPU, as the reference runs it, runners/runner.py:418), the
    [B,S,N,H,W] volume in memory, then F.grid_sample (align_corners=True, zeros padding) at the (2r+1)^2 taps.  This is
    what the reference executes on a GPU; bench.py times it as the C4 baseline (kind "port": written from the reference's
    description, not imported from it)."""

    def __init__(self, fmaps, num_levels=4, radius=4, padding_mode="zeros"):
        B, S, C, H, W = fmaps.shape
        self.S, self.C, self.num_levels, self.radius, self.padding_mode = S, C, num_levels, radius, padding_mode
        self.pyr = [fmaps]
        for _ in range(num_levels - 1):
            f = F.avg_pool2d(fmaps.reshape(B * S, C, H, W), 2, stride=2)
            _, _, H, W = f.shape
            fmaps = f.reshape(B, S, C, H, W)
            self.pyr.append(fmaps)

    def corr(self, targets):
        B, S, N, C = targets.shape
        self.vols = []
        for fm in self.pyr:
            H, W = fm.shape[-2:]
            v = torch.matmul(targets, fm.reshape(B, S, C, H * W)).reshape(B, S, N, H, W)
            self.vols.append(v / torch.sqrt(torch.tensor(float(C))))

    def sample(self, coords):
        r = self.radius
        B, S, N, _ = coords.shape
        d = torch.linspace(-r, r, 2 * r + 1, device=coords.device)
        delta = torch.stack(torch.meshgrid(d, d, indexing="ij"), dim=-1)           # (..., 0) = row-varying -> added to x
        out = []
        for i, v in enumerate(self.vols):
            H, W = v.shape[-2:]
            c = coords.reshape(B * S * N, 1, 1, 2) / 2 ** i + delta[None]
            g = torch.stack([c[..., 0] * (2.0 / max(W - 1, 1)) - 1.0, c[..., 1] * (2.0 / max(H - 1, 1)) - 1.0], dim=-1)
            s = F.grid_sample(v.reshape(B * S * N, 1, H, W), g.to(v.dtype), align_corners=True, padding_mode=self.padding_mode)
            out.append(s.reshape(B, S, N, -1))
        return torch.cat(out, dim=-1).contiguous()


def kernel_pyramid(fmaps, num_levels, half=True):
    """The pyramid csrc/corr.cu builds, bit for bit: float32 levels pooled as ((a + b) + c) + d then * 0.25 from the
    float32 level above (odd sizes floored), each rounded to float16 round-to-nearest-even when `half`.
    fmaps [B,S,C,H,W] (any device) -> list of [B,S,C,h,w] float32 (half-valued when `half`)."""
    f = fmaps.float()
    levels = [f.half().float() if half else f]
    for _ in range(num_levels - 1):
        h, w = f.shape[-2] // 2, f.shape[-1] // 2
        a, b = f[..., 0:2 * h:2, 0:2 * w:2], f[..., 0:2 * h:2, 1:2 * w:2]
        c, d = f[..., 1:2 * h:2, 0:2 * w:2], f[..., 1:2 * h:2, 1:2 * w:2]
        f = (((a + b) + c) + d) * 0.25
        levels.append(f.half().float() if half else f)
    return levels


def corr_reference(levels, targets, coords, radius, border=False, frames=4):
    """float64 correlation + sampling: levels [B,S,C,h,w] per level, targets [B,S,N,C] and coords [B,S,N,2] float32, all
    on one device.  Returns (out, bound) [B,S,N,L*(2r+1)^2] float64, bound = the bilinear combination of
    sum_c |t_c f_c| / sqrt(C).  Tap positions as the kernels form them: for zeros padding floor(c) + d plus the
    float32 fraction c - floor(c), once per query (c = coords / 2^l); for border padding c + d rounded to float32,
    then clamped."""
    B, S, N, C = targets.shape
    r = radius
    K = 2 * r + 1
    dev = targets.device
    out = torch.empty(B, S, N, len(levels) * K * K, dtype=torch.float64, device=dev)
    bound = torch.empty_like(out)
    d = torch.arange(-r, r + 1, dtype=torch.float64, device=dev)
    for s0 in range(0, S, frames):
        s1 = min(S, s0 + frames)
        t = targets[:, s0:s1].double()
        for i, fm in enumerate(levels):
            H, W = fm.shape[-2:]
            f = fm[:, s0:s1].double()
            vol = torch.stack([torch.einsum("bsnc,bschw->bsnhw", t, f), torch.einsum("bsnc,bschw->bsnhw", t.abs(), f.abs())],
                              dim=-1) / math.sqrt(C)
            c = coords[:, s0:s1].float().reshape(-1, 2) / 2 ** i
            if border:
                x = (c[:, 0:1, None] + d.float()[None, :, None]).double()
                y = (c[:, 1:2, None] + d.float()[None, None, :]).double()
            else:
                fl = torch.floor(c)
                pos = fl.double() + (c - fl).double()          # the float32 fraction: inexact for c in (-0.5, 0)
                x = pos[:, 0:1, None] + d[None, :, None]
                y = pos[:, 1:2, None] + d[None, None, :]
            x = x.expand(-1, K, K).reshape(-1, K * K)
            y = y.expand(-1, K, K).reshape(-1, K * K)
            g = _bilinear_gather(vol.reshape(-1, H, W, 2), x, y, border).reshape(B, s1 - s0, N, K * K, 2)
            out[:, s0:s1, :, i * K * K:(i + 1) * K * K] = g[..., 0]
            bound[:, s0:s1, :, i * K * K:(i + 1) * K * K] = g[..., 1]
    return out, bound


def sample_features4d_reference(inp, coords):
    """float64 sample_features4d (models/utils.py:415-447: bilinear_sampler, align_corners=True, border padding):
    inp [B,C,H,W], coords [B,R,2] (x, y) float32, on one device -> (out, bound) [B,R,C] float64.  The sample position is
    the reference's float32 round trip, x * float32(2 / max(W - 1, 1)) - 1, then ((g + 1) / 2) * (W - 1), each step
    rounded; it is clipped by grid_sample's CUDA rule (_source_coordinate) and interpolated in float64.
    bound = sum_i w_i |v_i|, the scale of a float32 kernel's rounding error."""
    B, C, H, W = inp.shape
    c = coords.float()
    pos = []
    for k, size in ((0, W), (1, H)):
        s = torch.tensor(2 / max(size - 1, 1), dtype=torch.float32, device=c.device)
        g = c[..., k] * s - 1
        pos.append(_source_coordinate((((g + 1) / 2) * (size - 1)).double(), size, True))
    x, y = pos
    x0, y0 = torch.floor(x), torch.floor(y)
    wx, wy = (x - x0)[..., None], (y - y0)[..., None]
    x0, y0 = x0.long(), y0.long()
    x1, y1 = (x0 + 1).clamp(max=W - 1), (y0 + 1).clamp(max=H - 1)
    v = inp.double().permute(0, 2, 3, 1)
    bi = torch.arange(B, device=inp.device)[:, None]
    out = torch.zeros(B, x.shape[1], C, dtype=torch.float64, device=inp.device)
    bound = torch.zeros_like(out)
    for yi, wyv in ((y0, 1 - wy), (y1, wy)):
        for xi, wxv in ((x0, 1 - wx), (x1, wx)):
            t = v[bi, yi, xi]
            out = out + wxv * wyv * t
            bound = bound + wxv * wyv * t.abs()
    return out, bound
