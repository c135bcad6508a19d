"""CPU oracle for the tracker's correlation inner loop -- TEST INFRASTRUCTURE ONLY.

torch-CPU float32 restatement of CorrBlock (vggsfm/models/track_modules/blocks.py:338-416):
pyramid by repeated avg_pool2d(2,2) (:352-361), full correlation volume per level divided by sqrt(C)
(:396-416), then (2r+1)^2 bilinear taps per level with align_corners=True semantics and zero padding
(:363-394 via models/utils.py:347-412); and of EfficientCorrBlock.sample (:433-471, border padding).
The bilinear gather is written out by hand (no grid_sample) so it is an independent statement.
PINNED against the reference through tests/golden/corr_*.npz (tools/make_golden_corr.py).
"""
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


def _bilinear_gather(vol, x, y, border):
    """vol [Q,H,W]; x,y [Q,T] pixel coords -> [Q,T]."""
    Q, H, W = vol.shape
    if border:
        x = x.clamp(0, W - 1)
        y = y.clamp(0, H - 1)
    x0 = torch.floor(x)
    y0 = torch.floor(y)
    wx = x - x0
    wy = y - y0
    x0 = x0.long()
    y0 = y0.long()
    out = torch.zeros_like(x)
    qi = torch.arange(Q)[:, None].expand_as(x0)
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
            out = out + torch.where(inside, v, torch.zeros_like(v)) * wxv * wyv
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
