"""Both two-view stages at their edges, against their float64 oracles.

Relative pose (csrc/twoview.cu `tv_pose_kernel` through `vgg_dev_relative_pose_counts`, which also returns the four
candidates' cheirality counts) against `oracle/twoview_oracle.relative_pose`:
  * counts of every candidate and the chosen candidate exact;
  * E = K^T F K within 8 eps of |K^T| |F| |K| per entry (two length-3 inner products on each side);
  * R and t within `pose_bar` = 96 eps sigma_1 / sigma_2 (derived in the oracle), and the largest error / bar ratio of
    every check printed;
  * the oracle's margins asserted: no finite depth within 1e-9 (relative) of K_MIN_DEPTH or of the depth window, and no
    count gap of 0 between the winner and a candidate with a different (R, t).
  Where sigma_1 / sigma_2 >= 1e8 (a rank-1 E) the basis of the decomposition is not unique, so the kernel's answer is
  checked on its own terms: R a rotation, t a unit left null vector of E, and the kernel's four counts equal to the
  oracle's cheirality counts of the kernel's own four candidates (rebuilt from R, t and the chosen index).  F = 0 has
  the unique completion U = V = I on both sides and is compared in full.

LO-MSAC (csrc/twoview_msac.cu) against `oracle/poselib_oracle.py` with the semantics of tests/test_twoview_msac_gpu.py:
iterations, LO trials, winning trial, counts and masks exact, F to 1e-7, the oracle's margins asserted.  Degenerate
pairs whose margins do not hold are checked for self-consistency instead: count = mask sum, no inlier among invalid
matches, and mask = (r^2 < thr^2) under the returned F where no polish moved F after the mask was taken.
"""
import numpy as np
import pytest

from oracle import poselib_oracle as po
from oracle import twoview_oracle as tvo
from tests.helpers import to_dev
from tests.test_twoview_msac_gpu import _compare as _msac_compare
from tests.test_twoview_msac_gpu import _oracle as _msac_oracle
from tests.test_twoview_msac_gpu import _run as _msac_run

pytestmark = pytest.mark.gpu

EPS = 2.0 ** -52
W_IMG, H_IMG = 1024, 768


# ---------------------------------------------------------------------------------------------------------------------
# relative pose: fixtures
# ---------------------------------------------------------------------------------------------------------------------
def _rot(axis, angle):
    a = np.asarray(axis, np.float64)
    a = a / np.linalg.norm(a)
    K = np.array([[0, -a[2], a[1]], [a[2], 0, -a[0]], [-a[1], a[0], 0]])
    return np.eye(3) + np.sin(angle) * K + (1 - np.cos(angle)) * K @ K


def _skew(t):
    return np.array([[0, -t[2], t[1]], [t[2], 0, -t[0]], [-t[1], t[0], 0]])


def _pix(X, R, t):
    """Pixels of world points X [N,3] in the camera (R, t) under the default K of W_IMG x H_IMG."""
    K = tvo.default_kmat(W_IMG, H_IMG)
    Y = X @ R.T + t
    return Y[:, :2] / Y[:, 2:] * K[0, 0] + K[:2, 2]


def _geometry(rng, N, angle=0.2, baseline=1.0, noise_px=0.3, depth=(4.0, 12.0), t=None):
    """A two-view pair: camera 1 at the origin, camera 2 = (R, t) with |t| = baseline; points in front of both."""
    R = _rot(rng.normal(size=3), angle)
    t = rng.normal(size=3) if t is None else np.asarray(t, np.float64)
    t = baseline * t / np.linalg.norm(t)
    X = np.stack([rng.uniform(-2, 2, N), rng.uniform(-1.5, 1.5, N), rng.uniform(*depth, N)], -1)
    p1 = _pix(X, np.eye(3), np.zeros(3)) + rng.normal(scale=noise_px, size=(N, 2))
    p2 = _pix(X, R, t) + rng.normal(scale=noise_px, size=(N, 2))
    return R, t, p1, p2


def _f_from_e(E):
    Ki = np.linalg.inv(tvo.default_kmat(W_IMG, H_IMG))
    return Ki.T @ E @ Ki


def _sigma_f(R, t, r):
    """F whose E = K^T F K has singular values (1, r, ~0) and the singular vectors of [t]x R: R_true stays a candidate
    for every r, so the vote has a clear winner."""
    U, _, Vt = np.linalg.svd(_skew(t) @ R)
    return _f_from_e(U @ np.diag([1.0, r, 0.0]) @ Vt)


def _rank1_f(R, t):
    U, _, Vt = np.linalg.svd(_skew(t) @ R)
    return _f_from_e(np.outer(U[:, 0], Vt[0]))


# ---------------------------------------------------------------------------------------------------------------------
# relative pose: launch and comparison
# ---------------------------------------------------------------------------------------------------------------------
def _pose(dev, F, p1, p2, dtype):
    import torch
    from vggsfm_b200 import _lib
    B, N, _ = p1.shape
    f64 = dtype == torch.float64
    P1, P2 = to_dev(p1, dev, dtype), to_dev(p2, dev, dtype)
    Fd = torch.from_numpy(np.ascontiguousarray(F, np.float64)).to(dev)
    R = torch.empty(B, 3, 3, dtype=torch.float64, device=dev)
    t = torch.empty(B, 3, dtype=torch.float64, device=dev)
    E = torch.empty(B, 3, 3, dtype=torch.float64, device=dev)
    counts = torch.full((B, 4), -1, dtype=torch.int32, device=dev)
    stream = torch.cuda.current_stream(dev).cuda_stream
    _lib.check(_lib.lib().vgg_dev_relative_pose_counts(B, N, P1.data_ptr(), P2.data_ptr(), int(f64), Fd.data_ptr(),
                                                        float(W_IMG), float(H_IMG), R.data_ptr(), t.data_ptr(),
                                                        E.data_ptr(), counts.data_ptr(), stream), "pose counts")
    # the product entry point is the same kernel without the counts
    from vggsfm_b200 import two_view as tv
    R2, t2, E2 = tv.relative_pose_from_fundamental(Fd, P1, P2, W_IMG, H_IMG)
    torch.cuda.synchronize()
    out = [x.cpu().numpy() for x in (R, t, E, counts)]
    for a, b in zip(out, (R2, t2, E2)):
        assert np.array_equal(a, b.cpu().numpy(), equal_nan=True)
    return out


def _own_candidates(R, t, k):
    """The kernel's four candidates from its chosen (R, t) and index k: R2 = (2 u2 u2^T - I) R1, t = +-u2."""
    u2 = t if k % 2 == 0 else -t
    H = 2.0 * np.outer(u2, u2) - np.eye(3)
    R1 = R if k < 2 else H @ R
    R2 = H @ R1
    return [R1, R1, R2, R2], [u2, -u2, u2, -u2]


def _check_pose(label, out, F, p1, p2, rows=None):
    """-> largest error / bar ratio over the rows compared against the oracle's (R, t)."""
    R, t, E, counts = out
    rows = list(range(F.shape[0])) if rows is None else rows
    p1o = p1[rows].astype(np.float64)
    p2o = p2[rows].astype(np.float64)
    Rr, tr, Er, cr, dbg = tvo.relative_pose(F[rows], p1o, p2o, W_IMG, H_IMG, return_debug=True)
    K = tvo.default_kmat(W_IMG, H_IMG)
    worst = 0.0
    for i, b in enumerate(rows):
        d = dbg[i]
        absE = np.abs(K.T) @ np.abs(F[b]) @ np.abs(K)
        assert np.all(np.abs(E[b] - Er[i]) <= 8 * EPS * absE), (label, b)
        kb = int(np.argmax(counts[b]))
        s = d["sigma"]
        if s[1] > 1e-12 * s[0]:
            assert d["depth_margin"] > 1e-9, (label, b, d["depth_margin"])
            assert d["count_gap"] > 0, (label, b, cr[i])
            assert np.array_equal(counts[b], cr[i]), (label, b, counts[b], cr[i])
            assert kb == d["k"], (label, b)
            if s[0] < 0.999e8 * s[1]:            # beyond sigma_1 / sigma_2 = 1e8 only the vote is compared
                bar = tvo.pose_bar(s)
                err = max(np.abs(R[b] - Rr[i]).max(), np.abs(t[b] - tr[i]).max())
                assert err <= bar, (label, b, err, bar)
                worst = max(worst, err / bar)
            continue
        # rank-deficient E: the kernel's own decomposition, checked on its own terms
        assert np.isfinite(R[b]).all() and np.isfinite(t[b]).all(), (label, b, R[b], t[b])
        assert np.abs(R[b].T @ R[b] - np.eye(3)).max() < 1e-14 and abs(np.linalg.det(R[b]) - 1) < 1e-14, (label, b)
        assert abs(np.linalg.norm(t[b]) - 1) < 1e-14, (label, b)
        assert np.abs(Er[i].T @ t[b]).max() <= 64 * EPS * max(s[0], np.abs(Er[i]).max()), (label, b)
        f = float(max(W_IMG, H_IMG))
        x1 = (p1o[i] - [W_IMG / 2, H_IMG / 2]) / f
        x2 = (p2o[i] - [W_IMG / 2, H_IMG / 2]) / f
        Rs, ts = _own_candidates(R[b], t[b], kb)
        cm = [tvo.cheirality_counts(Rs[k], ts[k], x1, x2, return_margin=True) for k in range(4)]
        assert min(m for _, m in cm) > 1e-9, (label, b)
        assert np.array_equal(counts[b], [c for c, _ in cm]), (label, b, counts[b], cm)
        if not F[b].any():                       # F = 0: U = V = I on both sides, so the oracle's answer is unique
            assert np.array_equal(counts[b], cr[i]) and kb == d["k"], (label, b, counts[b], cr[i])
            assert np.abs(R[b] - Rr[i]).max() <= 4 * EPS and np.abs(t[b] - tr[i]).max() <= 4 * EPS, (label, b)
    print(f"{label}: largest error / pose_bar = {worst:.3g}")
    return worst


# ---------------------------------------------------------------------------------------------------------------------
# relative pose: cases
# ---------------------------------------------------------------------------------------------------------------------
SIGMA_RATIOS = [1.0, 1 - 1e-12, 1e-2, 1e-4, 1e-6, 1e-8]


@pytest.mark.parametrize("f64", [False, True])
def test_pose_singular_value_sweep_and_rank_deficient(cuda_dev, f64):
    """sigma_2 / sigma_1 from 1 to 1e-8 on one geometry per row, then a rank-1 F and F = 0 (what LO-MSAC returns for a
    pair with fewer than 7 valid matches); without the completion of the basis these two gave NaN rotations."""
    import torch
    rng = np.random.default_rng(11)
    Fs, P1, P2 = [], [], []
    for r in SIGMA_RATIOS + ["rank1", "zero"]:
        R, t, p1, p2 = _geometry(rng, 512)
        Fs.append(np.zeros((3, 3)) if r == "zero" else _rank1_f(R, t) if r == "rank1" else _sigma_f(R, t, r))
        P1.append(p1)
        P2.append(p2)
    F, p1, p2 = np.stack(Fs), np.stack(P1), np.stack(P2)
    dt = torch.float64 if f64 else torch.float32
    if not f64:
        p1, p2 = p1.astype(np.float32), p2.astype(np.float32)
    out = _pose(cuda_dev, F, p1, p2, dt)
    _check_pose(f"sigma sweep ({'f64' if f64 else 'f32'})", out, F, p1, p2)
    for b in range(len(SIGMA_RATIOS)):                       # the planted geometry wins at every conditioning
        assert out[3][b].max() >= 500, (b, out[3][b])


def test_pose_depth_window_and_special_points(cuda_dev):
    """Points planted at depth 1000 |t| (1 +- 1e-8 ... 1e-6) in either camera, a point behind the second camera, points
    at infinity (x1 = x2 under R = I), NaN and +-inf tracks, next to the ordinary points of the pair."""
    import torch
    rng = np.random.default_rng(21)
    R, t, p1, p2 = _geometry(rng, 300, angle=0.1, noise_px=0.0, t=[0.5, 0.2, -0.8])
    tn = np.linalg.norm(R.T @ t)
    win = 1000.0 * tn
    extra = []
    for delta in (1e-8, -1e-8, 3e-8, -3e-8, 1e-7, -1e-7, 1e-6, -1e-6):
        x, y = rng.uniform(-0.3, 0.3, 2)
        extra.append(np.array([x * win, y * win, win * (1 + delta)]))          # camera-1 depth on the window
        Y = np.array([x * win, y * win, win * (1 + delta)])                     # camera-2 depth on the window
        X = R.T @ (Y - t)
        extra.append(X)
    X = np.stack(extra)
    q1 = _pix(X, np.eye(3), np.zeros(3))
    q2 = _pix(X, R, t)
    # a point in front of camera 1 and behind camera 2
    Xb = R.T @ (np.array([0.05, 0.05, -0.2]) - t)
    assert Xb[2] > 0.3 and (R @ Xb + t)[2] < 0
    q1 = np.concatenate([q1, _pix(Xb[None], np.eye(3), np.zeros(3))])
    q2 = np.concatenate([q2, _pix(Xb[None], R, t)])
    a1 = np.concatenate([p1, q1])
    a2 = np.concatenate([p2, q2])
    # second pair: pure translation with points at infinity (x1 = x2), NaN and +-inf tracks
    t2 = np.array([1.0, 0.2, 0.1])
    Xg =np.stack([rng.uniform(-2, 2, a1.shape[0]), rng.uniform(-1.5, 1.5, a1.shape[0]),
                   rng.uniform(4, 12, a1.shape[0])], -1)
    b1 = _pix(Xg, np.eye(3), np.zeros(3))
    b2 = _pix(Xg, np.eye(3), t2)
    b2[:20] = b1[:20]                                      # at infinity
    b1[20, 0] = np.nan
    b2[21, 1] = np.nan
    b1[22, 0] = np.inf
    b2[23, 1] = -np.inf
    F = np.stack([_f_from_e(_skew(t) @ R), _f_from_e(_skew(t2))])
    p1s, p2s = np.stack([a1, b1]), np.stack([a2, b2])
    for dt in (torch.float64, torch.float32):
        q1s = p1s if dt == torch.float64 else p1s.astype(np.float32)
        q2s = p2s if dt == torch.float64 else p2s.astype(np.float32)
        out = _pose(cuda_dev, F, q1s, q2s, dt)
        _check_pose(f"depth window ({dt})", out, F, q1s, q2s)
    # float64 tracks: the planted geometry wins and the planted depths keep their distance to the window
    Rr, tr, _, cr, dbg = tvo.relative_pose(F[:1], p1s[:1], p2s[:1], W_IMG, H_IMG, return_debug=True)
    assert np.abs(Rr[0] - R).max() < 1e-9 and cr[0].max() >= 300 and 5e-9 < dbg[0]["depth_margin"] < 2e-8


@pytest.mark.parametrize("N", [1, 190000])
def test_pose_match_counts(cuda_dev, N):
    import torch
    rng = np.random.default_rng(31 + N)
    Fs, P1, P2 = [], [], []
    for _ in range(2):
        R, t, p1, p2 = _geometry(rng, N)
        Fs.append(_f_from_e(_skew(t) @ R))
        P1.append(p1)
        P2.append(p2)
    F, p1, p2 = np.stack(Fs), np.stack(P1).astype(np.float32), np.stack(P2).astype(np.float32)
    out = _pose(cuda_dev, F, p1, p2, torch.float32)
    _check_pose(f"N = {N}", out, F, p1, p2)
    assert (out[3].max(1) >= (1 if N == 1 else 0.99 * N)).all()


def test_pose_near_pure_rotation(cuda_dev):
    """Baseline 1e-3 of the scene depth and 0.1 - 1 px noise: the four candidates' counts come close and the depths of
    many points sit near the window; the F is the exact one of the pair."""
    import torch
    rng = np.random.default_rng(41)
    Fs, P1, P2 = [], [], []
    for noise in (0.1, 0.3, 0.6, 1.0):
        R, t, p1, p2 = _geometry(rng, 2000, angle=0.15, baseline=0.01, noise_px=noise)
        Fs.append(_f_from_e(_skew(t / np.linalg.norm(t)) @ R))
        P1.append(p1)
        P2.append(p2)
    F, p1, p2 = np.stack(Fs), np.stack(P1), np.stack(P2)
    out = _pose(cuda_dev, F, p1, p2, torch.float64)
    _check_pose("near pure rotation", out, F, p1, p2)


def test_pose_large_batch(cuda_dev):
    """B = 400 x 4096 in one launch, sigma_2 / sigma_1 log-uniform in [1e-6, 1], every 25th pair F = 0 and every 40th
    rank 1; 16 spread rows and every planted row against the oracle."""
    import torch
    B, N = 400, 4096
    rng = np.random.default_rng(51)
    Fs, P1, P2 = [], [], []
    for b in range(B):
        R, t, p1, p2 = _geometry(rng, N)
        if b % 25 == 3:
            Fs.append(np.zeros((3, 3)))
        elif b % 40 == 7:
            Fs.append(_rank1_f(R, t))
        else:
            Fs.append(_sigma_f(R, t, 10.0 ** rng.uniform(-6, 0)))
        P1.append(p1)
        P2.append(p2)
    F, p1, p2 = np.stack(Fs), np.stack(P1).astype(np.float32), np.stack(P2).astype(np.float32)
    out = _pose(cuda_dev, F, p1, p2, torch.float32)
    rows = sorted(set(np.linspace(0, B - 1, 16).astype(int).tolist()) | {3, 7, 28, 47, 378, 399})
    _check_pose("400 x 4096", out, F, p1, p2, rows)
    assert np.isfinite(out[0]).all() and np.isfinite(out[1]).all()


# ---------------------------------------------------------------------------------------------------------------------
# LO-MSAC
# ---------------------------------------------------------------------------------------------------------------------
def _msac_pairs(N, seed, outliers=(0.0, 0.45, 1.0), noise_px=0.3):
    """One pair per outlier fraction on a shared left view; 1.0 = pure noise."""
    rng = np.random.default_rng(seed)
    P1, P2 = [], []
    for frac in outliers:
        _, _, p1, p2 = _geometry(rng, N, noise_px=noise_px)
        bad = rng.uniform(size=N) < frac
        p2[bad] = rng.uniform(0, [W_IMG, H_IMG], size=(int(bad.sum()), 2))
        P1.append(p1)
        P2.append(p2)
    return np.stack(P1).astype(np.float32), np.stack(P2).astype(np.float32)


def _self_consistent(out, p1, p2, valid, max_error, rows):
    """count = mask sum, no inlier among invalid matches, F = 0 has no inlier; and where no polish ran (count <= 7)
    the mask is r^2 < thr^2 under the returned F (the polish moves F after the mask is taken)."""
    F, num, mask, iters = out[:4]
    for b in rows:
        v = np.ones(p1.shape[1], bool) if valid is None else valid[b]
        assert num[b] == mask[b].sum() and not mask[b][~v].any(), b
        if not F[b].any():
            assert num[b] == 0, b
            continue
        if num[b] > 7 or not np.isfinite(F[b]).all():
            continue
        r2 = po.sampson_sq(F[b], p1[b].astype(np.float64), p2[b].astype(np.float64))
        inl = (r2 < max_error ** 2) & v
        fin = np.isfinite(r2)
        near = fin & (np.abs(r2 - max_error ** 2) <= 1e-6 * max_error ** 2)
        assert np.array_equal(mask[b][~near], inl[~near]), b


@pytest.mark.parametrize("max_it,min_it", [(300, 0), (1, 0), (1, 50), (120, 400), (2400, 2047), (2400, 2048),
                                           (3300, 3000)])
def test_msac_chunk_schedule(cuda_dev, max_it, min_it):
    """Chunk length C = min(max_iterations, min_iterations + 1, 2048): C = 1 (min 0; and max 1), C = max < min + 1, the
    last chunk length below the cap, the cap itself, and 3000 > 2048 where a clean pair stops inside the second chunk.
    A clean, a 45 %-outlier and a pure-noise pair."""
    p1, p2 = _msac_pairs(400, seed=min_it + 7 * max_it)
    out = _msac_run(cuda_dev, p1, p2, None, 1.0, max_it, min_it)
    ref = _msac_oracle(p1, p2, None, 1.0, max_it, min_it, [0, 1, 2])
    if min_it >= 2048:
        assert ref["iterations"][0] == min_it + 1, ref["iterations"]
    _msac_compare(out, ref, [0, 1, 2])


@pytest.mark.parametrize("n_valid", [6, 7, 8])
@pytest.mark.parametrize("where", ["tile", "warp"])
def test_msac_few_valid_scattered(cuda_dev, n_valid, where):
    """Exactly 6 / 7 / 8 valid matches among N = 4096, at the 256-match tile boundaries (255, 256, 257, ...) or at warp
    boundaries (31, 32, 63, 64, ...); the mask must stay 0 at every invalid match."""
    N = 4096
    p1, p2 = _msac_pairs(N, seed=60 + n_valid, outliers=(0.0, 0.0))
    pos = {"tile": [255, 256, 257, 511, 512, 2047, 2048, 4095], "warp": [31, 32, 63, 64, 95, 96, 1023, 1024]}[where]
    valid = np.zeros((2, N), bool)
    valid[0, pos[:n_valid]] = True
    valid[1, pos[-n_valid:]] = True
    out = _msac_run(cuda_dev, p1, p2, valid, 2.0, 200, 50)
    ref = _msac_oracle(p1, p2, valid, 2.0, 200, 50, [0, 1])
    F, num, mask, iters = out[:4]
    assert not mask[~valid].any()
    if n_valid < 7:
        assert not F.any() and not num.any() and not iters.any()
        assert np.array_equal(ref["iterations"], [0, 0])
        return
    # n = 7 and 8: the trials draw the same few matches over and over, so the MSAC scores of different candidates tie
    # to roundoff (the oracle's score margin is ~1e-13 there); the outcome is compared
    assert np.array_equal(iters, ref["iterations"]) and np.array_equal(mask, ref["inlier_mask"])
    assert np.array_equal(num, ref["inlier_num"])
    _self_consistent(out, p1, p2, valid, 2.0, [0, 1])


@pytest.mark.parametrize("want,seed,max_error", [(7, 0, 0.05), (8, 8031, 0.5)])
def test_msac_final_count_seven_and_eight(cuda_dev, want, seed, max_error):
    """Pure noise, 320 matches: a final inlier count of exactly 7 (the winner's own sample; no polish) and exactly 8
    (polish on the inliers), as the oracle's `polished` confirms.  At 7 the winning sample's MSAC score ties other
    samples' to ~1e-12 (every candidate fits its own 7 matches exactly), so the outcome is compared: iterations, count,
    mask, and the mask under the returned F.  At 8 everything is compared."""
    rng = np.random.default_rng(seed)
    p1 = rng.uniform(0, [W_IMG, H_IMG], size=(1, 320, 2)).astype(np.float32)
    p2 = rng.uniform(0, [W_IMG, H_IMG], size=(1, 320, 2)).astype(np.float32)
    ref = _msac_oracle(p1, p2, None, max_error, 60, 20, [0])
    assert ref["inlier_num"][0] == want and ref["debug"][0]["polished"] == (want > 7)
    out = _msac_run(cuda_dev, p1, p2, None, max_error, 60, 20)
    if want == 8:
        _msac_compare(out, ref, [0])
        return
    F, num, mask, iters = out[:4]
    assert iters[0] == ref["iterations"][0] and num[0] == 7
    _self_consistent(out, p1, p2, None, max_error, [0])


def test_msac_nan_offset_and_seeds(cuda_dev):
    """All valid matches NaN (scale falls back to 1, no model), coordinates offset by 1e4 px (the shared scale), and
    seeds 2^31 + 5 and 2^64 - 1 (the sampler state is taken mod 2^31 after the first draw)."""
    import torch
    p1, p2 = _msac_pairs(600, seed=71, outliers=(0.0, 0.2))
    q1, q2 = p1.copy(), p2.copy()
    q1[0, ::2] = np.nan
    valid = np.zeros((2, 600), bool)
    valid[0, ::2] = True                   # pair 0: every valid match NaN
    valid[1] = True
    out = _msac_run(cuda_dev, q1, q2, valid, 1.0, 150, 40)
    ref = _msac_oracle(q1, q2, valid, 1.0, 150, 40, [0, 1])
    assert ref["debug"][0]["scale"] == 1.0 and ref["inlier_num"][0] == 0 and not ref["fmat"][0].any()
    _msac_compare(out, ref, [0, 1])
    o1, o2 = p1.astype(np.float64) + 1e4, p2.astype(np.float64) + 1e4
    out = _msac_run(cuda_dev, o1, o2, None, 1.0, 300, 100, dtype=torch.float64)
    _msac_compare(out, _msac_oracle(o1, o2, None, 1.0, 300, 100, [0, 1], dtype=np.float64), [0, 1])
    for seed in (2 ** 31 + 5, 2 ** 64 - 1):
        out = _msac_run(cuda_dev, p1, p2, None, 1.0, 300, 100, seed=seed)
        ref = _msac_oracle(p1, p2, None, 1.0, 300, 100, [0, 1], seed=seed)
        _msac_compare(out, ref, [0, 1])


def _degenerate_pairs(N, rng):
    """Planar, pure-rotation, identical-point and collinear pairs (pixels, float32)."""
    Rr = _rot([0.2, 1.0, 0.1], 0.2)
    tt = np.array([-0.5, 0.1, 0.05])
    Xp = np.stack([rng.uniform(-1, 1, N), rng.uniform(-1, 1, N), np.full(N, 4.0)], -1)
    Xg = np.stack([rng.uniform(-2, 2, N), rng.uniform(-1.5, 1.5, N), rng.uniform(4, 12, N)], -1)
    Xl = np.stack([np.linspace(-1, 1, N), 0.5 * np.linspace(-1, 1, N), 5 + np.linspace(-1, 1, N)], -1)
    pairs = [(_pix(Xp, np.eye(3), np.zeros(3)), _pix(Xp, Rr, tt)),                  # planar
             (_pix(Xg, np.eye(3), np.zeros(3)), _pix(Xg, Rr, np.zeros(3))),         # pure rotation
             (np.full((N, 2), 100.0), np.full((N, 2), 300.0)),                      # identical points
             (_pix(Xl, np.eye(3), np.zeros(3)), _pix(Xl, Rr, tt))]                  # collinear
    noise = [rng.normal(scale=0.2, size=(N, 2)) if k in (0, 1) else 0.0 for k in range(4)]
    P1 = np.stack([a + n for (a, _), n in zip(pairs, noise)]).astype(np.float32)
    P2 = np.stack([b + n for (_, b), n in zip(pairs, noise)]).astype(np.float32)
    return P1, P2


def _margins_hold(d):
    return (d["thr"] > 1e-9 and d["score"] > 1e-10 and d["rfc"] > 1e-9 and d["roots"] > 1e-11 and d["ceil"] > 1e-9
            and d["lm_grad"] > 1e-6 and d["lm_step"] > 1e-6)


def _compare_row(out, ref, i, b, f_tol=None):
    """_msac_compare of oracle row i against kernel row b; a non-finite F (a degenerate pair whose final F has zero
    norm, F / |F|) must be non-finite in the same entries on both sides, the rest is compared as usual.  `f_tol`
    replaces the 1e-7 bar on F (every decision is still compared exactly)."""
    one = {k: (v[i:i + 1] if k != "debug" else [v[i]]) for k, v in ref.items()}
    G = one["fmat"][0]
    out = list(out)
    if not np.isfinite(G).all():
        assert np.array_equal(np.isfinite(out[0][b]), np.isfinite(G)), (b, out[0][b], G)
        out[0] = np.where(np.isfinite(out[0]), out[0], 0.0)
        one["fmat"] = np.where(np.isfinite(one["fmat"]), one["fmat"], 0.0)
    elif f_tol is not None:
        err = min(np.abs(out[0][b] - G).max(), np.abs(out[0][b] + G).max())
        assert err <= f_tol * np.abs(G).max(), (b, err)
        out[0] = out[0].copy()
        out[0][b] = G
    _msac_compare(out, one, [b])


# collinear matches leave the Cauchy polish's 7 x 7 normal equations singular along the directions that move the
# epipoles along the line, so where LM stops there depends on rounding (2e-6 seen on an H100 with every decision equal)
COLLINEAR_F_TOL = 1e-4


def test_msac_degenerate_pairs(cuda_dev):
    N = 300
    rng = np.random.default_rng(81)
    p1, p2 = _degenerate_pairs(N, rng)
    out = _msac_run(cuda_dev, p1, p2, None, 1.0, 200, 60)
    ref = _msac_oracle(p1, p2, None, 1.0, 200, 60, [0, 1, 2, 3])
    _self_consistent(out, p1, p2, None, 1.0, [0, 1, 2, 3])
    held = [i for i in range(4) if _margins_hold(ref["debug"][i])]
    for i in held:
        _compare_row(out, ref, i, i, COLLINEAR_F_TOL if i == 3 else None)
    print(f"degenerate LO-MSAC pairs compared with the oracle: {held} of [planar, rotation, identical, collinear]")


def test_msac_mixed_batch(cuda_dev):
    """B = 400 in one launch: every case above in the first rows, dead pairs (n < 7) between them, the rest ordinary
    pairs; clean pairs stop in the first chunk while 45 %-outlier and noise pairs run on (min 100 -> chunks of 101)."""
    B, N = 400, 512
    rng = np.random.default_rng(91)
    P1, P2 = [], []
    V = np.ones((B, N), bool)
    fr = rng.choice([0.0, 0.05, 0.45, 1.0], size=B, p=[0.3, 0.4, 0.2, 0.1])
    for b in range(B):
        _, _, p1, p2 = _geometry(rng, N)
        bad = rng.uniform(size=N) < fr[b]
        p2[bad] = rng.uniform(0, [W_IMG, H_IMG], size=(int(bad.sum()), 2))
        P1.append(p1)
        P2.append(p2)
    p1, p2 = np.stack(P1).astype(np.float32), np.stack(P2).astype(np.float32)
    d1, d2 = _degenerate_pairs(N, rng)
    p1[1:5], p2[1:5] = d1, d2
    for b in (5, 17, 200, 399):                                       # dead pairs
        V[b] = False
        V[b, rng.choice(N, size=b % 7, replace=False)] = True
    V[6] = False
    V[6, [31, 32, 255, 256, 257, 300, 511]] = True                    # exactly 7, across warp / tile boundaries
    V[7] = False
    V[7, [0, 63, 64, 127, 128, 255, 256, 511]] = True                 # exactly 8
    p1[8, ::3] = np.nan                                               # NaN among valid matches
    out = _msac_run(cuda_dev, p1, p2, V, 1.0, 700, 100)
    F, num, mask, iters = out[:4]
    assert not mask[~V].any() and np.array_equal(num, mask.sum(1))
    rows = sorted(set(np.linspace(0, B - 1, 12).astype(int).tolist()) | {0, 5, 8, 17, 200, 399})
    ref = _msac_oracle(p1, p2, V, 1.0, 700, 100, rows)
    _self_consistent(out, p1, p2, V, 1.0, range(B))
    for i, b in enumerate(rows):
        d = ref["debug"][i]
        if d["n"] < 7:
            assert iters[b] == 0 and num[b] == 0 and not F[b].any(), b
            continue
        assert _margins_hold(d), (b, d)
        _compare_row(out, ref, i, b)
    stops = set(int(x) for x in np.asarray(ref["iterations"]))
    assert 101 in stops and any(101 < s < 700 for s in stops), stops
    # the degenerate rows: self-consistent (above), and compared where the oracle's margins hold; the rows with exactly
    # 7 and 8 valid matches (scores tie to roundoff, as in test_msac_few_valid_scattered): the outcome
    ref2 = _msac_oracle(p1, p2, V, 1.0, 700, 100, [1, 2, 3, 4, 6, 7])
    for i, b in enumerate([1, 2, 3, 4, 6, 7]):
        if b < 6 and _margins_hold(ref2["debug"][i]):
            _compare_row(out, ref2, i, b, COLLINEAR_F_TOL if b == 4 else None)
        if b >= 6:
            assert iters[b] == ref2["iterations"][i] and np.array_equal(mask[b], ref2["inlier_mask"][i]), b
