"""GPU parity of the batched fundamental-matrix LO-RANSAC and relative pose (csrc/twoview.cu) against
oracle/twoview_oracle.py on the same host-drawn samples.

Bars: inlier counts and masks exact; F, residuals, R and t to 1e-9 relative.  Every launch carries one dead pair (no
valid match), which pins the batch-wide indicator threshold to 1e6 + 1e-6, so the oracle can be run on a subset of the
pairs and still select exactly what the kernel selects.  The comparisons are guarded by margin asserts on the oracle
side: no winner residual within 1e-9 (relative) of the threshold, and no other candidate with the winner's count and a
mean inlier residual within 1e-9 of its own unless it is the same matrix.  Degenerate inputs (planar scene, pure
rotation, identical points, pairs with 0 / 7 / 8 valid matches) have no unique answer to compare against -- the null
space of the 8-point system is more than one-dimensional there -- so they are checked for internal consistency
instead."""
import numpy as np
import pytest

from oracle import twoview_oracle as tvo
from tests.helpers import to_dev
from vggsfm_b200.synthetic import make_scene

pytestmark = pytest.mark.gpu


def _pairs(B, N, seed, noise_px=0.3, outlier_frac=0.05, invisible_frac=0.3, dead=True):
    sc = make_scene(B + 1, N, seed=seed, noise_px=noise_px, outlier_frac=outlier_frac, invisible_frac=invisible_frac)
    p1 = np.ascontiguousarray(np.broadcast_to(sc.tracks[:1], (B, N, 2)))
    p2 = np.ascontiguousarray(sc.tracks[1:])
    valid = sc.mask[1:].copy()
    if dead:
        valid[-1] = False
    return p1, p2, valid, sc


def _run(dev, p1, p2, valid, samples, max_error, lo, squared=True, dtype=None, second_refine=True):
    import torch
    from vggsfm_b200 import two_view as tv
    dt = dtype or torch.float32
    out = tv.estimate_fundamental(to_dev(p1, dev, dt), to_dev(p2, dev, dt), max_error=max_error, lo_num=lo,
                                  valid_mask=None if valid is None else to_dev(valid, dev), squared=squared,
                                  second_refine=second_refine, return_residuals=True, samples=samples)
    return [o.cpu().numpy() for o in out]


def _margins(ref, thr):
    for p, s in zip(ref["pairs"], ref["sel"]):
        r = s["residuals"]
        fin = np.isfinite(r)
        assert not (np.abs(r[fin] - thr) <= 1e-9 * thr).any(), "a winner residual sits on the threshold"
        # the indicator orders candidates of equal count by their mean inlier residual; a dead pair's candidates all
        # tie exactly (count 0, mean 1e6) and both sides take the first
        # (so does every candidate of a pair with a valid NaN match: any NaN residual makes the mean 1e6)
        b = s["best"]
        m = p["mean"]
        if p["cnt"][b] == 0 or m[b] == 1e6:
            continue
        close = np.nonzero((p["cnt"] == p["cnt"][b]) & (np.abs(m - m[b]) <= 1e-9 * m[b]) & (np.arange(len(m)) != b))[0]
        for k in close:
            assert np.abs(p["F"][k] - p["F"][b]).max() <= 1e-9 * np.abs(p["F"][b]).max(), "near-tie between matrices"


def _compare(out, ref, rows, thr):
    F, num, mask, res = out
    for i, b in enumerate(rows):
        assert num[b] == ref["inlier_num"][i], (b, num[b], ref["inlier_num"][i])
        assert np.array_equal(mask[b], ref["inlier_mask"][i]), b
        scale = np.abs(ref["fmat"][i]).max()
        assert np.abs(F[b] - ref["fmat"][i]).max() <= 1e-9 * scale, (b, np.abs(F[b] - ref["fmat"][i]).max(), scale)
        rr = ref["residuals"][i]
        fin = np.isfinite(rr)
        assert np.array_equal(np.isfinite(res[b]), fin)
        assert np.all(np.abs(res[b][fin] - rr[fin]) <= 1e-9 * np.maximum(np.abs(rr[fin]), thr))
    _margins(ref, thr)


def _consistent(out, p1, p2, valid, thr, squared=True):
    F, num, mask, res = out
    for b in range(F.shape[0]):
        r = tvo.sampson(p1[b].astype(np.float64), p2[b].astype(np.float64), F[b][None], squared)[0]
        if valid is not None:
            r = np.where(valid[b], r, 1e6)
        fin = np.isfinite(r)
        assert np.array_equal(np.isfinite(res[b]), fin)
        assert np.all(np.abs(res[b][fin] - r[fin]) <= 1e-9 * np.maximum(np.abs(r[fin]), thr))
        assert np.array_equal(mask[b], res[b] <= thr)
        assert num[b] == mask[b].sum()


@pytest.mark.parametrize("B,N,T,lo,squared,f64", [
    (5, 256, 256, 30, True, False),
    (4, 255, 128, 40, True, True),
    (4, 257, 128, 20, False, False),
    (3, 4099, 256, 30, True, False),
    (3, 12288, 256, 30, True, False),       # 3 query frames x 4096 tracks, as the runner's predict_tracks builds them
    (2, 190000, 64, 10, True, False),       # the largest N vgg_estimate_fundamental accepts
])
def test_matches_oracle(cuda_dev, B, N, T, lo, squared, f64):
    import torch
    p1, p2, valid, _ = _pairs(B, N, seed=N + B)
    np.random.seed(B * 7 + N)
    smp = tvo.generate_samples(N, T)
    max_error = 2.0 if squared else 1.5
    thr = max_error ** 2 if squared else max_error
    out = _run(cuda_dev, p1, p2, valid, smp, max_error, lo, squared, torch.float64 if f64 else torch.float32)
    ref = tvo.estimate_fundamental(p1, p2, smp, max_error=max_error, lo_num=lo, valid_mask=valid, squared=squared)
    assert ref["thres"] == 1e6 + 1e-6
    _compare(out, ref, list(range(B)), thr)
    assert out[1][-1] == 0 and not out[3][-1][np.isfinite(out[3][-1])].min() < 1e6


def test_single_pair_and_no_second_round(cuda_dev):
    p1, p2, valid, _ = _pairs(1, 300, seed=5, dead=False)
    np.random.seed(1)
    smp = tvo.generate_samples(300, 200)
    out = _run(cuda_dev, p1, p2, valid, smp, 2.0, 25)
    ref = tvo.estimate_fundamental(p1, p2, smp, max_error=2.0, lo_num=25, valid_mask=valid)
    _compare(out, ref, [0], 4.0)
    p1, p2, valid, _ = _pairs(3, 300, seed=6)
    out = _run(cuda_dev, p1, p2, valid, smp, 2.0, 25, second_refine=False)
    ref = tvo.estimate_fundamental(p1, p2, smp, max_error=2.0, lo_num=25, valid_mask=valid, second_refine=False)
    _compare(out, ref, [0, 1, 2], 4.0)


@pytest.mark.parametrize("N", [7, 8, 9])
def test_tiny_pairs(cuda_dev, N):
    """N = 7, 8, 9 with explicit permutation samples (too few points for the reference's draw to succeed)."""
    p1, p2, _, sc = _pairs(3, N, seed=20 + N, outlier_frac=0.0, invisible_frac=0.0)
    valid = np.ones((3, N), bool)
    valid[-1] = False
    rng = np.random.default_rng(N)
    smp = np.stack([rng.permutation(N)[:7] for _ in range(16)])
    out = _run(cuda_dev, p1, p2, valid, smp, 2.0, 10)
    _consistent(out, p1, p2, valid, 4.0)
    assert out[1][0] == N and out[1][1] == N and out[1][2] == 0


def test_large_batch_against_oracle_subset(cuda_dev):
    """400 pairs x 4096 matches, T = 4096, lo = 300 in one launch; first, last and a spread of pairs against the
    oracle (the last pair is the dead one)."""
    B, N, T, lo = 400, 4096, 4096, 300
    p1, p2, valid, _ = _pairs(B, N, seed=400)
    np.random.seed(0)
    smp = tvo.generate_samples(N, T)
    out = _run(cuda_dev, p1, p2, valid, smp, 4.0, lo)
    rows = [0, 133, 266, B - 2, B - 1]
    ref = tvo.estimate_fundamental(p1[rows], p2[rows], smp, max_error=4.0, lo_num=lo, valid_mask=valid[rows])
    assert ref["thres"] == 1e6 + 1e-6
    _compare(out, ref, rows, 16.0)
    assert (out[1][:-1] > 0.5 * valid[:-1].sum(1)).all()


def test_few_inliers_in_lo_seeds(cuda_dev):
    """Heavy contamination (about 16 % of the matches are clean in both frames, ~10 of 64): more than a third of the
    150 first-round seeds have fewer than 8 inliers, so their 8-point systems are rank-deficient."""
    p1, p2, valid, _ = _pairs(4, 64, seed=31, outlier_frac=0.6, invisible_frac=0.0)
    np.random.seed(2)
    smp = tvo.generate_samples(64, 64)
    ref = tvo.estimate_fundamental(p1, p2, smp, max_error=2.0, lo_num=150, valid_mask=valid)
    small = [(p["cnt"][p["seeds1"]] < 8).sum() for p in ref["pairs"][:-1]]
    assert min(small) > 150 / 3, small
    out = _run(cuda_dev, p1, p2, valid, smp, 2.0, 150)
    _consistent(out, p1, p2, valid, 4.0)
    assert (out[1][:-1] >= 9).all(), out[1]


def test_nan_tracks_match_oracle(cuda_dev):
    """A pair with NaN tracks among valid matches, next to live pairs and the dead one.  Any NaN coordinate in a
    7-point sample makes its whole normalised design matrix NaN (the mean spreads it), so both sides take the same
    all-free null-space basis; the NaN residuals make every candidate's mean 1e6 and the pair's winner is the first
    candidate of highest count on both sides."""
    p1, p2, valid, _ = _pairs(4, 300, seed=61)
    p2[1, ::5] = np.nan
    p1[2, 7] = np.inf
    np.random.seed(6)
    smp = tvo.generate_samples(300, 128)
    out = _run(cuda_dev, p1, p2, valid, smp, 2.0, 30)
    ref = tvo.estimate_fundamental(p1, p2, smp, max_error=2.0, lo_num=30, valid_mask=valid)
    _compare(out, ref, [0, 1, 2, 3], 4.0)
    assert out[1][1] > 0 and not out[2][1][::5].any()


def test_inlier_by_fundamental(cuda_dev):
    import torch
    from vggsfm_b200 import two_view as tv
    S, N = 5, 700
    sc = make_scene(S, N, seed=70, outlier_frac=0.1)
    p1 = np.ascontiguousarray(np.broadcast_to(sc.tracks[:1], (S - 1, N, 2)))
    np.random.seed(7)
    smp = tvo.generate_samples(N, 128)
    F, _, _, _ = _run(cuda_dev, p1, sc.tracks[1:], None, smp, 1.0, 30)
    mask = tv.inlier_by_fundamental(torch.from_numpy(F).to(cuda_dev)[None], to_dev(sc.tracks, cuda_dev)[None],
                                    max_error=1.0).cpu().numpy()
    assert mask.shape == (1, S - 1, N)
    for b in range(S - 1):
        r = tvo.sampson(p1[b].astype(np.float64), sc.tracks[b + 1].astype(np.float64), F[b][None])[0]
        assert not (np.abs(r - 1.0) <= 1e-9).any()
        assert np.array_equal(mask[0, b], r <= 1.0)
        assert mask[0, b].sum() > 0.7 * N           # ~81 % of the matches are clean in both frames


def test_degenerate_inputs(cuda_dev):
    """Planar scene, pure rotation, identical points, NaN tracks and pairs with 0, 7 and 8 valid matches in one
    launch: outputs are self-consistent (mask = residual <= threshold, count = mask sum, residuals = Sampson of the
    returned F), the identical-point and NaN pairs find no inlier."""
    N = 200
    rng = np.random.default_rng(3)
    p1, p2, valid, sc = _pairs(8, N, seed=41, outlier_frac=0.0, invisible_frac=0.0, dead=False)
    Xp = np.stack([rng.uniform(-1, 1, N), rng.uniform(-1, 1, N), np.full(N, 4.0)], -1)       # plane z = 4
    def proj(R, t, X):
        Y = X @ R.T + t
        return (1000.0 * Y[:, :2] / Y[:, 2:] + 512.0).astype(np.float32)
    a = 0.2
    Ry = np.array([[np.cos(a), 0, np.sin(a)], [0, 1, 0], [-np.sin(a), 0, np.cos(a)]])
    p1[0], p2[0] = proj(np.eye(3), np.zeros(3), Xp), proj(Ry, np.array([-0.5, 0.1, 0.0]), Xp)   # planar
    X = sc.points3d
    p1[1], p2[1] = proj(np.eye(3), np.zeros(3), X), proj(Ry, np.zeros(3), X)                      # pure rotation
    p1[2], p2[2] = 100.0, 300.0                                                                    # identical points
    p2[3, ::3] = np.nan                                                                            # NaN tracks
    valid[4] = False                                                                               # no valid match
    valid[5] = False
    valid[5, :7] = True                                                                            # 7 valid
    valid[6] = False
    valid[6, :8] = True                                                                            # 8 valid
    np.random.seed(4)
    smp = tvo.generate_samples(N, 128)
    out = _run(cuda_dev, p1, p2, valid, smp, 2.0, 40)
    _consistent(out, p1, p2, valid, 4.0)
    assert out[1][2] == 0 and out[1][4] == 0
    assert out[1][3] <= N - len(range(0, N, 3))
    assert out[1][5] <= 7 and out[1][6] <= 8
    assert out[1][0] >= 0.9 * N and out[1][1] >= 0.9 * N and out[1][7] >= 0.9 * N


def test_relative_pose_matches_oracle(cuda_dev):
    import torch
    from vggsfm_b200 import two_view as tv
    p1, p2, valid, sc = _pairs(6, 512, seed=50, noise_px=0.2)
    np.random.seed(5)
    smp = tvo.generate_samples(512, 256)
    F, _, _, _ = _run(cuda_dev, p1, p2, valid, smp, 2.0, 30)
    for dt in (torch.float32, torch.float64):
        R, t, E = (x.cpu().numpy() for x in tv.relative_pose_from_fundamental(
            torch.from_numpy(F).to(cuda_dev), to_dev(p1, cuda_dev, dt), to_dev(p2, cuda_dev, dt), 1024, 1024))
        Rr, tr, Er, counts = tvo.relative_pose(F, p1, p2, 1024, 1024)
        assert np.abs(E - Er).max() <= 1e-9 * np.abs(Er).max()
        for b in range(5):                                  # the dead pair's F is an arbitrary candidate
            top = np.sort(counts[b])[::-1]
            assert top[0] > top[1], counts[b]
            assert np.abs(R[b] - Rr[b]).max() < 1e-9 and np.abs(t[b] - tr[b]).max() < 1e-9, (b, R[b], Rr[b])
            Rg = sc.extrinsics[b + 1, :, :3]
            assert np.degrees(np.arccos(np.clip((np.trace(R[b].T @ Rg) - 1) / 2, -1, 1))) < 1.0
