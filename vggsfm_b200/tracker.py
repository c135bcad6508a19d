"""Host loops around the correlation kernel: the track predictor's iterative refinement and the fine-track stage.

``track_predictor_forward`` is ``BaseTrackerPredictor.forward`` (vggsfm/models/track_modules/base_track_predictor.py:81-238)
and ``refine_track`` / ``compute_score_fn`` are vggsfm/models/track_modules/refine_track.py:24-187 / :190-294, with the
reference's arguments and return values.  The learned modules stay the caller's (``predictor.updateformer``, ``.norm``,
``.ffeat_updater``, ``.vis_predictor``, ``fine_fnet``: stock PyTorch layers holding the reference's checkpoints); what
moves onto the CUDA kernels is everything between them:

  * correlation + local sampling: ``vggsfm_b200.corr.CorrBlock`` / ``EfficientCorrBlock`` (csrc/corr.cu, fused; the
    [B,S,N,H,W] volume of blocks.py:396-416 is never built);
  * query-feature and positional-embedding lookups: ``vgg_sample_features4d``; the positional embedding of the query
    points does not change over the iterations (coords[:, 0] is pinned to the query, :219) and is sampled once, not
    ``iters`` times;
  * the fine stage gathers its 31x31 patches by index instead of materialising the (H-30)x(W-30)x31x31 unfold view.

Drop-in: ``install(vggsfm.models.track_modules)`` rebinds the two symbols on the reference's modules.
"""
from __future__ import annotations

import math

import torch

from .corr import CorrBlock, EfficientCorrBlock, sample_features4d


def get_2d_embedding(xy, C, cat_coords=True):
    """models/utils.py:313-344: per coordinate C values, sin at even / cos at odd slots of x * (1000/C) * [0,2,4,...]."""
    B, N, D = xy.shape
    assert D == 2
    div = (torch.arange(0, C, 2, device=xy.device, dtype=torch.float32) * (1000.0 / C)).reshape(1, 1, C // 2)
    pe = torch.empty(B, N, 2, C // 2, 2, device=xy.device, dtype=torch.float32)
    ang = xy.float().unsqueeze(-1) * div.unsqueeze(2)                 # [B,N,2,C/2]
    pe[..., 0] = torch.sin(ang)
    pe[..., 1] = torch.cos(ang)
    pe = pe.reshape(B, N, 2 * C)
    return torch.cat([xy, pe], dim=2) if cat_coords else pe


def get_2d_sincos_pos_embed(embed_dim, grid_size, device=None):
    """models/utils.py:229-310: [1, embed_dim, H, W]; the first half of the channels encodes the column index (the
    reference's ``grid[0]`` of a meshgrid(w, h, indexing="xy")), the second half the row index; sin block then cos block,
    frequencies 1/10000^(2i/(D/2)) evaluated in float64 and rounded to float32."""
    gh, gw = grid_size if isinstance(grid_size, tuple) else (grid_size, grid_size)
    assert embed_dim % 4 == 0 or embed_dim % 2 == 0
    half = embed_dim // 2
    assert half % 2 == 0, "embed_dim/2 must be even (models/utils.py:287)"
    omega = torch.arange(half // 2, dtype=torch.float64, device=device) / (half / 2.0)
    omega = 1.0 / 10000 ** omega
    xs = torch.arange(gw, dtype=torch.float32, device=device).double()
    ys = torch.arange(gh, dtype=torch.float32, device=device).double()
    ex = torch.cat([torch.sin(xs[:, None] * omega), torch.cos(xs[:, None] * omega)], dim=1).float()      # [W, half]
    ey = torch.cat([torch.sin(ys[:, None] * omega), torch.cos(ys[:, None] * omega)], dim=1).float()      # [H, half]
    emb = torch.cat([ex[None].expand(gh, gw, half), ey[:, None].expand(gh, gw, half)], dim=2)            # [H,W,D]
    return emb.permute(2, 0, 1)[None].contiguous()


@torch.no_grad()
def track_predictor_forward(predictor, query_points, fmaps=None, iters=4, return_feat=False, down_ratio=1):
    """``BaseTrackerPredictor.forward`` with ``predictor`` in the place of ``self`` (so it can be bound as a method).

    query_points [B,N,2] pixels, fmaps [B,S,C,HH,WW] -> (coord_preds: list of [B,S,N,2], vis_e [B,S,N] | None
    [, track_feats [B,S,N,C], query_track_feat [B,N,C]])."""
    B, N, D = query_points.shape
    B, S, C, HH, WW = fmaps.shape
    assert D == 2
    if not fmaps.is_cuda:
        raise RuntimeError("vggsfm_b200.tracker needs CUDA tensors (no CPU fallback)")
    stride, latent = predictor.stride, predictor.latent_dim
    tdim = predictor.transformer_dim
    if down_ratio > 1:
        query_points = query_points / float(down_ratio)
    query_points = query_points / float(stride)
    coords = query_points.clone().reshape(B, 1, N, 2).repeat(1, S, 1, 1)
    query_track_feat = sample_features4d(fmaps[:, 0], coords[:, 0])                       # [B,N,C]
    track_feats = query_track_feat.unsqueeze(1).repeat(1, S, 1, 1)
    coords_backup = coords.clone()
    efficient = bool(getattr(predictor, "efficient_corr", False))
    if efficient:
        fcorr_fn = EfficientCorrBlock(fmaps, num_levels=predictor.corr_levels, radius=predictor.corr_radius)
    else:
        fcorr_fn = CorrBlock(fmaps, num_levels=predictor.corr_levels, radius=predictor.corr_radius)
    # positional embedding of the query positions: iteration-invariant (:219 pins coords[:, 0])
    pos_embed = get_2d_sincos_pos_embed(tdim, (HH, WW), device=fmaps.device)
    sampled_pos_emb = sample_features4d(pos_embed.expand(B, -1, -1, -1), coords[:, 0]).reshape(B * N, 1, tdim)
    coord_preds = []
    for _ in range(iters):
        if efficient:
            fcorrs = fcorr_fn.sample(coords, track_feats)
        else:
            fcorr_fn.corr(track_feats)
            fcorrs = fcorr_fn.sample(coords)                                              # [B,S,N,L*(2r+1)^2]
        corrdim = fcorrs.shape[3]
        fcorrs_ = fcorrs.permute(0, 2, 1, 3).reshape(B * N, S, corrdim)
        flows = (coords - coords[:, 0:1]).permute(0, 2, 1, 3).reshape(B * N, S, 2)
        flows_emb = torch.cat([get_2d_embedding(flows, predictor.flows_emb_dim, cat_coords=False), flows], dim=-1)
        track_feats_ = track_feats.permute(0, 2, 1, 3).reshape(B * N, S, latent)
        x = torch.cat([flows_emb, fcorrs_.to(flows_emb.dtype), track_feats_.to(flows_emb.dtype)], dim=2)
        if x.shape[2] < tdim:
            x = torch.cat([x, x.new_zeros(B * N, S, tdim - x.shape[2])], dim=2)
        x = (x + sampled_pos_emb).reshape(B, N, S, tdim)
        delta = predictor.updateformer(x).reshape(B * N, S, latent + 2)
        delta_coords_ = delta[:, :, :2]
        delta_feats_ = delta[:, :, 2:].reshape(B * N * S, latent)
        track_feats_ = track_feats_.reshape(B * N * S, latent)
        track_feats_ = predictor.ffeat_updater(predictor.norm(delta_feats_)) + track_feats_
        track_feats = track_feats_.reshape(B, N, S, latent).permute(0, 2, 1, 3)
        coords = coords + delta_coords_.reshape(B, N, S, 2).permute(0, 2, 1, 3)
        coords[:, 0] = coords_backup[:, 0]
        coord_preds.append(coords * stride * down_ratio if down_ratio > 1 else coords * stride)
    if not predictor.fine:
        vis_e = torch.sigmoid(predictor.vis_predictor(track_feats.reshape(B * S * N, latent)).reshape(B, S, N))
    else:
        vis_e = None
    if return_feat:
        return coord_preds, vis_e, track_feats, query_track_feat
    return coord_preds, vis_e


def _call_tracker(fine_tracker, **kw):
    """A reference ``BaseTrackerPredictor`` (or anything exposing its attributes) runs through the loop above; any other
    callable is called as is."""
    if all(hasattr(fine_tracker, a) for a in ("updateformer", "ffeat_updater", "norm", "corr_levels", "corr_radius")):
        return track_predictor_forward(fine_tracker, **kw)
    return fine_tracker(**kw)


@torch.no_grad()
def refine_track(images, fine_fnet, fine_tracker, coarse_pred, compute_score=False, pradius=15, sradius=2, fine_iters=6,
                 cfg=None):
    """refine_track.py:24-187: 31x31 patches around the floored coarse tracks -> ``fine_fnet`` -> fine tracker with one
    query per patch -> tracks back in image coordinates (and the heat-map score).  images [B,S,3,H,W] with H == W (the
    reference clamps x and y with H, :108-111), coarse_pred [B,S,N,2]."""
    B, S, N, _ = coarse_pred.shape
    _, _, C_in, H, W = images.shape
    psize = pradius * 2 + 1
    query_points = coarse_pred[:, 0]
    track_int = coarse_pred.floor().int()
    track_frac = coarse_pred - track_int
    topleft_BSN = (track_int - pradius).clone()
    topleft = (track_int - pradius).clamp(0, H - psize).reshape(B * S, N, 2).long()
    # patch gather by index: rows y0..y0+30, columns x0..x0+30 of image (b,s)
    ar = torch.arange(psize, device=images.device)
    yy = (topleft[..., 1, None] + ar)[:, :, :, None].expand(B * S, N, psize, psize)
    xx = (topleft[..., 0, None] + ar)[:, :, None, :].expand(B * S, N, psize, psize)
    img = images.reshape(B * S, C_in, H, W)
    bidx = torch.arange(B * S, device=images.device)[:, None, None, None].expand(B * S, N, psize, psize)
    extracted = img.permute(0, 2, 3, 1)[bidx, yy, xx].permute(0, 1, 4, 2, 3)          # [(B S), N, C_in, p, p]
    patch_feat = fine_fnet(extracted.reshape(B * S * N, C_in, psize, psize))
    C_out = patch_feat.shape[1]
    patch_feat = patch_feat.reshape(B, S, N, C_out, psize, psize).permute(0, 2, 1, 3, 4, 5).reshape(B * N, S, C_out, psize, psize)
    patch_query_points = (track_frac[:, 0] + pradius).reshape(B * N, 2).unsqueeze(1)
    fine_lists, _, _, query_point_feat = _call_tracker(fine_tracker, query_points=patch_query_points, fmaps=patch_feat,
                                                       iters=fine_iters, return_feat=True)
    fine_pred_track = fine_lists[-1].clone()                                          # [(B N), S, 1, 2], patch frame
    for idx in range(len(fine_lists)):
        lvl = fine_lists[idx].reshape(B, N, S, 1, 2).permute(0, 2, 1, 3, 4).squeeze(-2)
        fine_lists[idx] = lvl + topleft_BSN
    refined_tracks = fine_lists[-1].clone()
    refined_tracks[:, 0] = query_points
    score = None
    if compute_score:
        score = compute_score_fn(query_point_feat, patch_feat, fine_pred_track, sradius, psize, B, N, S, C_out)
    return refined_tracks, score


def compute_score_fn(query_point_feat, patch_feat, fine_pred_track, sradius, psize, B, N, S, C_out):
    """refine_track.py:190-294: spread (sum over x,y of the standard deviation, in normalised [-1,1] patch coordinates)
    of the soft-max similarity between the query feature and a (2 sradius+1)^2 neighbourhood; 1 for the query frame.

    Reference behaviour kept bit for bit, including two indexing quirks of :256-276 that a drop-in must reproduce
    because the score feeds ``pred_score`` downstream: (1) ``batch_indices_score`` holds the BATCH index b, yet indexes
    the (b s n)-flattened patch table, so every entry reads its neighbourhood from patch row b (for B = 1: the patch of
    frame 0 / track 0); (2) the neighbourhood offsets are flattened in (b n) s order while the result is reshaped as
    b s n.  The offset's y addresses the patch rows and its x the patch columns."""
    ssize = sradius * 2 + 1
    q = query_point_feat.reshape(B, N, C_out)
    pf = patch_feat.reshape(B, N, S, C_out, psize, psize).permute(0, 2, 1, 3, 4, 5)      # b s n c p q
    ref = pf.reshape(B * S * N, C_out, psize, psize)
    flat = (fine_pred_track.floor().int() - sradius).clamp(0, psize - ssize).squeeze(2).reshape(B * N * S, 2).long()
    ar = torch.arange(ssize, device=patch_feat.device)
    rows = (flat[:, 1, None] + ar)[:, :, None].expand(-1, ssize, ssize)                   # y -> patch rows
    cols = (flat[:, 0, None] + ar)[:, None, :].expand(-1, ssize, ssize)                   # x -> patch columns
    k = torch.arange(B, device=patch_feat.device)[:, None, None].expand(B, S, N).reshape(-1)[:, None, None]
    nb = ref.permute(0, 2, 3, 1)[k.expand(-1, ssize, ssize), rows, cols].permute(0, 3, 1, 2)   # [(B S N), C, ss, ss]
    nb = nb.reshape(B, S, N, C_out, ssize * ssize)[:, 1:].reshape(B * (S - 1) * N, C_out, ssize * ssize)
    qq = q.unsqueeze(1).expand(-1, S - 1, -1, -1).reshape(B * (S - 1) * N, C_out)
    sim = torch.einsum("mc,mcr->mr", qq, nb)
    heat = torch.softmax(sim / math.sqrt(C_out), dim=1)                                  # [(B (S-1) N), ss*ss]
    lin = torch.linspace(-1.0, 1.0, ssize, device=heat.device, dtype=heat.dtype)
    gx = lin[None, :].expand(ssize, ssize).reshape(-1)                                    # x varies along the last axis
    gy = lin[:, None].expand(ssize, ssize).reshape(-1)
    grid = torch.stack([gx, gy], dim=-1)                                                  # [ss*ss, 2]
    mean = heat @ grid
    var = heat @ (grid ** 2) - mean ** 2
    std = torch.sqrt(torch.clamp(var, min=1e-10)).sum(-1)
    score = std.reshape(B, S - 1, N)
    return torch.cat([torch.ones_like(score[:, 0:1]), score], dim=1)


def install(track_modules_pkg):
    """Rebind the reference's symbols: ``install(vggsfm.models.track_modules)``."""
    bp = track_modules_pkg.base_track_predictor
    bp.BaseTrackerPredictor.forward = track_predictor_forward
    bp.CorrBlock, bp.EfficientCorrBlock = CorrBlock, EfficientCorrBlock
    track_modules_pkg.refine_track.refine_track = refine_track
    track_modules_pkg.refine_track.compute_score_fn = compute_score_fn
