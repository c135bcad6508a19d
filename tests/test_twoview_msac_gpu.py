"""GPU parity of the batched LO-MSAC fundamental matrix (csrc/twoview_msac.cu, `estimate_preliminary_cameras_poselib`)
against oracle/poselib_oracle.py.

Exact: iterations run, the trials that ran local optimisation (LO), inlier counts and masks.  The winning trial is
exact unless the oracle saw two LO results converge to the same model (a near-tie recorded in `ties`: either choice
gives that model).  F: 1e-7 relative to its largest entry: the LM stops once a step is below 1e-8 in the scaled frame,
so two float64 evaluations that round differently can stop one such step apart (3.4e-8 seen at 400 x 4096).
Margin asserts on the oracle side guard every comparison: no r^2 within 1e-9 (relative) of thr^2, no MSAC-score
comparison between different models within 1e-10, no real-focal decision within 1e-9, no cubic-branch decision
(|D| / (|Q^3| + R^2)) within 1e-11 (2.2e-10 seen at 400 x 4096, decided alike), no ceil of dynamic_max_iter within
1e-9 of an integer, and no LM gradient / step test within 1e-6 of its tolerance."""
import ctypes

import numpy as np
import pytest

from oracle import poselib_oracle as po
from tests.helpers import to_dev
from vggsfm_b200.synthetic import make_scene

pytestmark = pytest.mark.gpu


def _pairs(B, N, seed, noise_px=0.3, outlier_frac=0.05, invisible_frac=0.3):
    sc = make_scene(B + 1, N, seed=seed, noise_px=noise_px, outlier_frac=outlier_frac, invisible_frac=invisible_frac)
    p1 = np.ascontiguousarray(np.broadcast_to(sc.tracks[:1], (B, N, 2)))
    return p1, np.ascontiguousarray(sc.tracks[1:]), sc.mask[1:].copy()


def _run(dev, p1, p2, valid, max_error, max_it, min_it, dtype=None, seed=0):
    import torch
    from vggsfm_b200 import _lib
    from vggsfm_b200 import two_view as tv
    dt = dtype or torch.float32
    B, N, _ = p1.shape
    nb = ctypes.c_size_t()
    _lib.check(_lib.lib().vgg_msac_fundamental_workspace_bytes(B, N, max_it, min_it, ctypes.byref(nb)), "ws")
    ws = torch.empty(max(nb.value, 256), dtype=torch.uint8, device=dev)
    out = tv.estimate_fundamental_msac(to_dev(p1, dev, dt), to_dev(p2, dev, dt),
                                       None if valid is None else to_dev(valid, dev), max_error=max_error,
                                       max_iterations=max_it, min_iterations=min_it, seed=seed, workspace=ws)
    torch.cuda.synchronize()
    cap = 64
    runs = np.zeros(B, np.int32)
    win = np.zeros(B, np.int32)
    trials = np.zeros((B, cap), np.int32)
    _lib.check(_lib.lib().vgg_dev_msac_trace(B, N, max_it, min_it, ws.data_ptr(), cap, runs.ctypes.data,
                                             win.ctypes.data, trials.ctypes.data), "trace")
    return [o.cpu().numpy() for o in out] + [runs, win, trials]


def _oracle(p1, p2, valid, max_error, max_it, min_it, rows, dtype=np.float32, seed=0):
    return po.estimate_fundamental_msac(p1.astype(dtype), p2.astype(dtype), valid, max_error, max_it, min_it, seed,
                                        pairs=rows, return_debug=True)


def _compare(out, ref, rows):
    F, num, mask, iters, runs, win, trials = out
    for i, b in enumerate(rows):
        d = ref["debug"][i]
        assert iters[b] == ref["iterations"][i], (b, iters[b], ref["iterations"][i])
        assert num[b] == ref["inlier_num"][i] == mask[b].sum(), (b, num[b], ref["inlier_num"][i])
        assert np.array_equal(mask[b], ref["inlier_mask"][i]), b
        G = ref["fmat"][i]
        if not G.any():
            assert not F[b].any(), b
        else:
            err = min(np.abs(F[b] - G).max(), np.abs(F[b] + G).max())
            assert err <= 1e-7 * np.abs(G).max(), (b, err)
        lo = d["lo_trials"]
        assert runs[b] == len(lo), (b, runs[b], len(lo))
        m = min(len(lo), trials.shape[1])
        assert np.array_equal(trials[b, :m], lo[:m]), b
        if d["ties"] == 0:
            assert win[b] == (-1 if d["win"] is None else d["win"][1]), (b, win[b], d["win"])
        assert d["thr"] > 1e-9 and d["score"] > 1e-10 and d["rfc"] > 1e-9 and d["roots"] > 1e-11, d
        assert d["ceil"] > 1e-9 and d["lm_grad"] > 1e-6 and d["lm_step"] > 1e-6, d


def test_production_shape_400x4096(cuda_dev):
    B, N = 400, 4096
    p1, p2, valid = _pairs(B, N, seed=0)
    out = _run(cuda_dev, p1, p2, valid, 4.0, 20000, 1000)
    F, num, mask, iters = out[:4]
    assert np.array_equal(num, mask.sum(1))
    rows = sorted(set(np.linspace(0, B - 1, 16).astype(int).tolist()))
    assert rows[0] == 0 and rows[-1] == B - 1
    _compare(out, _oracle(p1, p2, valid, 4.0, 20000, 1000, rows), rows)


def test_stop_in_first_chunk_later_chunk_and_at_max(cuda_dev):
    # min_iterations 100 -> chunks of 101 trials; pair 0 all inliers (stops at 101), pair 1 ~45 % outliers (stops in a
    # later chunk), pair 2 pure noise (runs max_iterations)
    N = 512
    p1, p2, valid = _pairs(3, N, seed=3, outlier_frac=0.0, invisible_frac=0.0)
    rng = np.random.default_rng(4)
    bad = rng.uniform(size=N) < 0.45
    p2[1, bad] = rng.uniform(0, 1024, size=(int(bad.sum()), 2))
    p2[2] = rng.uniform(0, 1024, size=(N, 2))
    out = _run(cuda_dev, p1, p2, valid, 1.0, 700, 100)
    ref = _oracle(p1, p2, valid, 1.0, 700, 100, [0, 1, 2])
    assert ref["iterations"][0] == 101 and 202 < ref["iterations"][1] < 700 and ref["iterations"][2] == 700, \
        ref["iterations"]
    _compare(out, ref, [0, 1, 2])


@pytest.mark.parametrize("N", [1, 7, 255, 256, 257, 4099, 65536])
def test_match_counts(cuda_dev, N):
    p1, p2, valid = _pairs(2, N, seed=10 + N % 97, invisible_frac=0.0 if N < 300 else 0.3)
    max_it, min_it = (300, 100) if N < 60000 else (120, 50)
    out = _run(cuda_dev, p1, p2, valid, 2.0, max_it, min_it)
    ref = _oracle(p1, p2, valid, 2.0, max_it, min_it, [0, 1])
    if N < 7:
        F, num, mask, iters = out[:4]
        assert not F.any() and not num.any() and not mask.any() and not iters.any()
        return
    if N == 7:
        # every trial draws the same seven matches: all candidates tie to roundoff, so only the outcome is compared
        F, num, mask, iters = out[:4]
        assert np.array_equal(iters, ref["iterations"]) and np.array_equal(num, ref["inlier_num"])
        assert np.array_equal(mask, ref["inlier_mask"])
        return
    _compare(out, ref, [0, 1])


def test_float64_tracks(cuda_dev):
    import torch
    p1, p2, valid = _pairs(3, 1024, seed=21)
    p1, p2 = p1.astype(np.float64) + 0.123456789, p2.astype(np.float64) - 0.987654321
    out = _run(cuda_dev, p1, p2, valid, 1.5, 500, 150, dtype=torch.float64)
    _compare(out, _oracle(p1, p2, valid, 1.5, 500, 150, [0, 1, 2], dtype=np.float64), [0, 1, 2])


def test_nan_in_a_valid_match(cuda_dev):
    p1, p2, valid = _pairs(2, 1024, seed=31, invisible_frac=0.0)
    p2[0, 5, 0] = np.nan          # sampled or not, an outlier at full cost; the scale skips it
    p1[:, 77, 1] = np.nan
    out = _run(cuda_dev, p1, p2, valid, 1.0, 400, 120)
    ref = _oracle(p1, p2, valid, 1.0, 400, 120, [0, 1])
    assert not ref["inlier_mask"][0, 5] and not ref["inlier_mask"][:, 77].any()
    _compare(out, ref, [0, 1])


def test_batch_quirk_and_ignored_score(cuda_dev):
    """B = 2: the pairs of batch 1 also use batch 0's query frame; tracks_score does not change anything."""
    import torch
    from vggsfm_b200 import two_view as tv
    S, N = 4, 600
    a = make_scene(S, N, seed=41, invisible_frac=0.2, outlier_frac=0.05)
    b = make_scene(S, N, seed=42, invisible_frac=0.2, outlier_frac=0.05)
    tracks = np.stack([a.tracks, b.tracks])
    vis = np.stack([a.vis, b.vis])
    t = to_dev(tracks, cuda_dev)
    v = to_dev(vis, cuda_dev)
    cams, pd = tv.estimate_preliminary_cameras_poselib(t, v, 1024, 1024, max_error=1.0, max_ransac_iters=1200)
    score = torch.rand(2, S, N, device=cuda_dev)
    _, pd2 = tv.estimate_preliminary_cameras_poselib(t, v, 1024, 1024, tracks_score=score, max_error=1.0,
                                                     max_ransac_iters=1200)
    assert cams is None and pd["fmat"].shape == (1, 2 * (S - 1), 3, 3) and pd["fmat"].dtype == torch.float64
    assert pd["fmat_inlier_mask"].shape == (1, 2 * (S - 1), N) and pd["fmat_inlier_mask"].dtype == torch.bool
    assert torch.equal(pd["fmat"], pd2["fmat"]) and torch.equal(pd["fmat_inlier_mask"], pd2["fmat_inlier_mask"])
    rows = [0, S - 1, 2 * (S - 1) - 1]           # batch 0's first pair, batch 1's first and last
    ref = po.estimate_preliminary_cameras_poselib(tracks, vis, 1024, 1024, max_error=1.0, max_ransac_iters=1200,
                                                  pairs=rows, return_debug=True)
    F = pd["fmat"][0].cpu().numpy()
    M = pd["fmat_inlier_mask"][0].cpu().numpy()
    for i, r in enumerate(rows):
        assert np.array_equal(M[r], ref["inlier_mask"][i]), r
        G = ref["fmat"][i]
        assert min(np.abs(F[r] - G).max(), np.abs(F[r] + G).max()) <= 1e-7 * np.abs(G).max(), r
    # batch 1 with its own query frame would be a different problem
    own = po.estimate_fundamental_msac(tracks[1, :1].astype(np.float64), tracks[1, 1:2], (vis[1, 1:2] >= 0.05),
                                       1.0, 1200)
    assert not np.array_equal(own["inlier_mask"][0], M[S - 1])


def test_einval(cuda_dev):
    import torch
    from vggsfm_b200 import _lib
    L = _lib.lib()
    x = torch.zeros(2, 16, 2, device=cuda_dev)
    f = torch.zeros(2, 9, dtype=torch.float64, device=cuda_dev)
    i = torch.zeros(2, dtype=torch.int32, device=cuda_dev)
    m = torch.zeros(2, 16, dtype=torch.uint8, device=cuda_dev)
    ws = torch.zeros(1 << 20, dtype=torch.uint8, device=cuda_dev)
    args = lambda B, N, err, mx, mn: (B, N, x.data_ptr(), x.data_ptr(), 0, None, err, mx, mn, 0, f.data_ptr(),
                                      i.data_ptr(), m.data_ptr(), i.data_ptr(), ws.data_ptr(), ws.numel(), None)
    for bad in [(-1, 16, 1.0, 10, 5), (2, -1, 1.0, 10, 5), (2, 16, 0.0, 10, 5), (2, 16, float("nan"), 10, 5),
                (2, 16, 1.0, 0, 5), (2, 16, 1.0, 10, -1), (1 << 16, 1 << 15, 1.0, 10, 5)]:
        assert L.vgg_estimate_fundamental_msac(*args(*bad)) == -1, bad
    nb = ctypes.c_size_t()
    assert L.vgg_msac_fundamental_workspace_bytes(2, 16, 0, 5, ctypes.byref(nb)) == -1
    assert L.vgg_msac_fundamental_workspace_bytes(2, 16, 10, 5, ctypes.byref(nb)) == 0


def test_cpu_tensors_raise():
    import torch
    from vggsfm_b200 import two_view as tv
    with pytest.raises(RuntimeError):
        tv.estimate_preliminary_cameras_poselib(torch.zeros(1, 2, 8, 2), torch.ones(1, 2, 8), 64, 64)
