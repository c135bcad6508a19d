"""Host-side pieces of the tracker loops (vggsfm_b200/tracker.py) that run without a GPU: the two embeddings against
goldens produced by the reference (tools/make_golden_tracker.py), and compute_score_fn against the reference's output on
the same seeded inputs (tools/make_golden_live.py)."""
import os

import numpy as np
import torch

from vggsfm_b200 import tracker as tk

GOLD = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")


def test_embeddings_match_reference_goldens():
    g = np.load(os.path.join(GOLD, "tracker_embed.npz"))
    xy = torch.from_numpy(g["xy"])
    assert np.abs(tk.get_2d_embedding(xy, 16, cat_coords=False).numpy() - g["e16"]).max() < 1e-6
    assert np.abs(tk.get_2d_embedding(xy, 64, cat_coords=True).numpy() - g["e64c"]).max() < 1e-6
    assert np.abs(tk.get_2d_sincos_pos_embed(216, (31, 31)).numpy() - g["pos216"]).max() < 1e-6
    assert np.abs(tk.get_2d_sincos_pos_embed(664, (6, 9)).numpy() - g["pos664"]).max() < 1e-6


def test_compute_score_fn_equals_live_reference():
    """Including the reference's two indexing quirks (refine_track.py:256-276), which a drop-in has to reproduce."""
    gold = np.load(os.path.join(GOLD, "tracker_score.npz"))
    g = torch.Generator().manual_seed(0)
    for i, (B, N, S) in enumerate(((1, 5, 4), (2, 3, 3))):
        C, psize, sr = 8, 31, 2
        qf = torch.randn(B, N, C, generator=g)
        pf = torch.randn(B * N, S, C, psize, psize, generator=g)
        trk = torch.rand(B * N, S, 1, 2, generator=g) * 34 - 2        # some neighbourhoods get clamped
        ref = torch.from_numpy(gold[f"score{i}"])
        got = tk.compute_score_fn(qf, pf, trk, sr, psize, B, N, S, C)
        assert got.shape == ref.shape == (B, S, N)
        assert (got - ref).abs().max().item() < 1e-6
