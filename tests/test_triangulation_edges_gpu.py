"""GPU triangulation kernels against the float64 oracle at the benchmark's shape (400 frames x 4096 tracks) and at the
edges of their staging, sizing, gating and undistortion paths.

Bars: inlier counts and masks exact; points 1e-7 relative per point; filter `valid` / `detail` exact.  The oracle
reports how close each decision is to flipping (oracle/tri_oracle.py, return_debug): observations whose angular error
lies within GATE_TIE rad of the gate and hypotheses whose triangulation angle lies within TRI_TIE deg of the minimum
would make an exact comparison depend on rounding.  The scenes are built so that there are none, and every test
asserts that.  Score near-ties are not avoidable at 4096 tracks (two different hypotheses with the same inlier count
whose mean errors differ by ~1e-9): there the kernel may pick any hypothesis within SCORE_TIE of the best, and must
then agree with that hypothesis exactly."""
import ctypes
import os

import numpy as np
import pytest

from oracle import tri_oracle as to
from tests.helpers import to_dev

pytestmark = pytest.mark.gpu

GATE_TIE = 1e-10       # rad; the asin series and acos differ from the oracle's arccos by < 1e-14 rad here
TRI_TIE = 1e-9         # deg
SCORE_TIE = 1e-9       # score units (inlier count + normalised mean); kernel and oracle means differ by ~1e-15
GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "edges_undistort_gate8.npz")


def dead_track(S):
    """tn / vis / score of one track with no usable observation.  Each of its hypotheses has no inlier, so its mean
    is 2 pi on both sides (the kernel's `cnt > 0 ? sum / cnt : 2 pi`, the oracle's nan_to_num(0/0, 2 pi)), and no
    track can have a larger mean: every inlier's error is at most the gate < pi.  With it in the kernel's launch and
    in every oracle chunk, calculate_residual_indicator's grid-wide threshold is 2 pi + 1e-6 on both sides, so an
    oracle run on any subset of tracks scores them exactly as the kernel's run on all of them."""
    return np.full((S, 1, 2), 0.1), np.full((S, 1), 0.01, np.float32), np.ones((S, 1), np.float32)


def run_kernel(dev, E, tn, vis, score, pairs, **kw):
    from vggsfm_b200 import triangulation as tri
    p, n, m = tri.triangulate_tracks(to_dev(E, dev), to_dev(tn, dev), track_vis=to_dev(vis, dev),
                                     track_score=to_dev(score, dev) if score is not None else None,
                                     ransac_pairs=pairs, **kw)
    return p.cpu().numpy(), n.cpu().numpy(), m.cpu().numpy()


def run_oracle(E, tn, vis, score, pairs, idx, chunk=64, **kw):
    """oracle on tracks `idx` (whose last entry is the dead track), in chunks that each carry the dead track."""
    dead = idx[-1]
    outs = []
    for c0 in range(0, len(idx) - 1, chunk):
        sel = np.append(idx[c0:min(c0 + chunk, len(idx) - 1)], dead)
        outs.append(to.triangulate_tracks(E, tn[:, sel], pairs, vis[:, sel], None if score is None else score[:, sel],
                                          return_debug=True, **kw))
    keep = [slice(None, -1)] * (len(outs) - 1) + [slice(None)]
    p = np.concatenate([o[0][k] for o, k in zip(outs, keep)])
    n = np.concatenate([o[1][k] for o, k in zip(outs, keep)])
    m = np.concatenate([o[2][k] for o, k in zip(outs, keep)])
    dbg = {key: np.concatenate([o[3][key][k] for o, k in zip(outs, keep)])
           for key in ("allX", "score", "best", "cnt", "mask", "score_margin", "gate_dist_min", "tri_dist0", "tri_dist")}
    return p, n, m, dbg


def compare(kern, orac, idx, label):
    """exact counts / masks for every track, points 1e-7 relative per point for tracks with >= 2 inliers (with fewer
    the point is an unscored two-view DLT, possibly of two near-parallel rays); returns (near-tie tracks, max relative
    point error)."""
    pk, nk, mk = (a[idx] for a in kern)
    po, no, mo, d = orac
    near_gate = int((d["gate_dist_min"] < GATE_TIE).sum())
    near_tri = int((np.abs(d["tri_dist0"]) < TRI_TIE).sum() + (np.abs(d["tri_dist"]) < TRI_TIE).sum())
    assert near_gate == 0, f"{label}: {near_gate} tracks with an observation within {GATE_TIE} rad of the gate"
    assert near_tri == 0, f"{label}: {near_tri} hypotheses within {TRI_TIE} deg of min_tri_angle"
    rel = np.abs(pk - po).max(axis=1) / (1.0 + np.abs(po).max(axis=1))
    tie = d["score_margin"] < SCORE_TIE
    for i in np.nonzero(~tie)[0]:
        assert nk[i] == no[i] and np.array_equal(mk[i], mo[i]), f"{label}: track {idx[i]} counts/mask differ"
        assert no[i] < 2 or rel[i] <= 1e-7, f"{label}: track {idx[i]} point differs by {rel[i]:.2e}"
    for i in np.nonzero(tie)[0]:       # any hypothesis tied with the best: the kernel must agree with that one exactly
        cand = np.nonzero(d["score"][i] >= d["score"][i, d["best"][i]] - SCORE_TIE)[0]
        ok = [h for h in cand if nk[i] == d["cnt"][i, h] and np.array_equal(mk[i], d["mask"][i, h])
              and (nk[i] < 2 or np.abs(pk[i] - d["allX"][i, h]).max() <= 1e-7 * (1.0 + np.abs(d["allX"][i, h]).max()))]
        assert ok, f"{label}: near-tie track {idx[i]} matches none of its tied hypotheses {cand}"
    assert (nk == mk.sum(axis=1)).all()
    good = ~tie & (no >= 2)
    err = float(rel[good].max()) if good.any() else 0.0
    print(f"\n{label}: {len(idx)} tracks, near-tie tracks {int(tie.sum())}, gate/angle exclusions 0, "
          f"max rel point error {err:.2e}")
    return int(tie.sum()), err


# ------------------------------------------------------------------------------------------------------------------
# 1. the benchmark configuration: 400 x 4096, SIMPLE_RADIAL, one launch, oracle on a spread subset
# ------------------------------------------------------------------------------------------------------------------

@pytest.mark.parametrize("variant", ["bench", "outliers"])
def test_bench_configuration_against_oracle(cuda_dev, variant):
    import torch
    from vggsfm_b200 import triangulation as tri
    from vggsfm_b200.synthetic import make_scene
    S, N = 400, 4096
    if variant == "bench":
        sc = make_scene(S, N, "SIMPLE_RADIAL", seed=0)
    else:
        sc = make_scene(S, N, "SIMPLE_RADIAL", seed=0, invisible_frac=0.3, outlier_frac=0.1)
        sc.score = np.random.default_rng(1).uniform(0.3, 1.0, size=(S, N)).astype(np.float32)
    torch.manual_seed(0)
    pairs = tri.draw_ransac_pairs(S, 256)
    dev = cuda_dev
    tn = tri.cam_from_img(to_dev(sc.tracks, dev), to_dev(sc.intrinsics, dev), to_dev(sc.extra_params, dev)).cpu().numpy()
    dt, dv, ds = dead_track(S)
    tn = np.concatenate([tn, dt], axis=1)
    vis = np.concatenate([sc.vis, dv], axis=1)
    score = np.concatenate([sc.score, ds], axis=1)
    kern = run_kernel(dev, sc.extrinsics, tn, vis, score, pairs)           # all 4097 tracks in one launch
    idx = np.append(np.unique(np.linspace(0, N - 1, 320).astype(int)), N)  # first, last, spread; dead track last
    orac = run_oracle(sc.extrinsics, tn, vis, score, pairs, idx)
    assert orac[1][-1] == 0 and kern[1][N] == 0 and not kern[2][N].any()
    compare(kern, orac, idx, f"400x4096 {variant}")
    # the oracle's cam_from_img on the same subset
    sub = idx[:-1]
    ref = to.cam_from_img(sc.tracks[:, sub].astype(np.float64), sc.intrinsics, sc.extra_params)
    assert np.abs(tn[:, sub] - ref).max() < 1e-12


# ------------------------------------------------------------------------------------------------------------------
# 2. frame counts, hypothesis counts, the shared-memory limit
# ------------------------------------------------------------------------------------------------------------------

def scene_case(S, N, seed):
    from vggsfm_b200.synthetic import make_scene
    sc = make_scene(S, N, "SIMPLE_PINHOLE", seed=seed, invisible_frac=0.2, outlier_frac=0.1)
    tn = to.cam_from_img(sc.tracks.astype(np.float64), sc.intrinsics)
    dt, dv, ds = dead_track(S)
    return (sc, np.concatenate([tn, dt], axis=1), np.concatenate([sc.vis, dv], axis=1),
            np.concatenate([sc.score, ds], axis=1))


@pytest.mark.parametrize("S,N", [(2, 40), (3, 40), (31, 40), (32, 40), (33, 40), (63, 32), (65, 32), (129, 24),
                                 (1024, 5)])
def test_frame_counts_against_oracle(cuda_dev, S, N):
    """W = ceil(S/32) mask words, a word plus one frame, odd S (centres through plain loads), more than one 12 KB
    bulk-copy chunk of cameras (S > 128), and S = 1024 (~199 KB of shared memory)."""
    import torch
    sc, tn, vis, score = scene_case(S, N, seed=S)
    torch.manual_seed(S)
    pairs = to.draw_pairs(S, 256)
    kern = run_kernel(cuda_dev, sc.extrinsics, tn, vis, score, pairs)
    idx = np.arange(N + 1)
    compare(kern, run_oracle(sc.extrinsics, tn, vis, score, pairs, idx), idx, f"S={S}")


@pytest.mark.parametrize("H0", [1, 3, 20, 256, 512])
@pytest.mark.parametrize("lo_num", [5, 50, 600])
def test_hypothesis_counts_against_oracle(cuda_dev, H0, lo_num):
    """H0 > 256 puts more than one hypothesis on a thread in phase 1; H0 < lo_num shrinks lo and lo2."""
    S, N = 65, 24
    sc, tn, vis, score = scene_case(S, N, seed=100 + H0)
    rng = np.random.default_rng(H0)
    comb = to.generate_combinations(S)
    pairs = comb[rng.permutation(len(comb))[:H0]]
    kern = run_kernel(cuda_dev, sc.extrinsics, tn, vis, score, pairs, lo_num=lo_num)
    idx = np.arange(N + 1)
    compare(kern, run_oracle(sc.extrinsics, tn, vis, score, pairs, idx, lo_num=lo_num), idx, f"H0={H0} lo={lo_num}")


def test_shared_memory_limit_is_rejected_before_launch(cuda_dev):
    """S = 1200 needs ~231 KB of shared memory per CTA: VGG_EINVAL with the shared-memory message, outputs untouched."""
    import torch
    from vggsfm_b200 import _lib
    L = _lib.lib()
    S, N, H0 = 1200, 4, 256
    dev = cuda_dev
    E = torch.zeros(S, 12, dtype=torch.float64, device=dev)
    tn = torch.zeros(S, N, 2, dtype=torch.float64, device=dev)
    vis = torch.ones(S, N, dtype=torch.float32, device=dev)
    pairs = torch.from_numpy(to.generate_combinations(S)[:H0].astype(np.int32)).to(dev)
    nbytes = ctypes.c_size_t()
    assert L.vgg_tri_workspace_bytes(S, N, H0, 50, ctypes.byref(nbytes)) == 0
    ws = torch.empty(nbytes.value, dtype=torch.uint8, device=dev)
    pts = torch.full((N, 3), 7.0, dtype=torch.float64, device=dev)
    num = torch.full((N,), 7, dtype=torch.int64, device=dev)
    mask = torch.full((N, S), 7, dtype=torch.uint8, device=dev)
    torch.cuda.synchronize()
    rc = L.vgg_triangulate_tracks(S, N, E.data_ptr(), tn.data_ptr(), vis.data_ptr(), None, pairs.data_ptr(), H0, 50, 2.0,
                                  1.5, pts.data_ptr(), num.data_ptr(), mask.data_ptr(), ws.data_ptr(), ws.numel(),
                                  torch.cuda.current_stream(dev).cuda_stream)
    torch.cuda.synchronize()
    assert rc == -1                                          # VGG_EINVAL
    msg = L.vgg_last_error().decode()
    assert "shared memory" in msg and "S=1200" in msg, msg
    assert (pts == 7).all() and (num == 7).all() and (mask == 7).all()


# ------------------------------------------------------------------------------------------------------------------
# 3. gates: the asin series at its limit (5.7 deg), the acos branch above it, and a wide minimum angle
# ------------------------------------------------------------------------------------------------------------------

@pytest.mark.parametrize("gate", [2.0, 5.7, 5.8, 8.0])
@pytest.mark.parametrize("min_tri", [1.5, 10.0])
def test_gates_against_oracle(cuda_dev, gate, min_tri):
    import torch
    from vggsfm_b200.synthetic import make_scene
    S, N = 48, 64
    sc = make_scene(S, N, "SIMPLE_PINHOLE", seed=31, noise_px=3.0, invisible_frac=0.1, outlier_frac=0.2)
    tn = to.cam_from_img(sc.tracks.astype(np.float64), sc.intrinsics)
    dt, dv, ds = dead_track(S)
    tn, vis, score = (np.concatenate(a, axis=1) for a in ((tn, dt), (sc.vis, dv), (sc.score, ds)))
    torch.manual_seed(5)
    pairs = to.draw_pairs(S, 256)
    kw = dict(max_angular_error=gate, min_tri_angle=min_tri)
    kern = run_kernel(cuda_dev, sc.extrinsics, tn, vis, score, pairs, **kw)
    idx = np.arange(N + 1)
    orac = run_oracle(sc.extrinsics, tn, vis, score, pairs, idx, **kw)
    compare(kern, orac, idx, f"gate={gate} min_tri={min_tri}")
    # the scene exercises the gate: some inlier errors lie above 2 degrees at the wider gates
    if gate > 2.0:
        assert orac[1].sum() > run_oracle(sc.extrinsics, tn, vis, score, pairs, idx, min_tri_angle=min_tri)[1].sum()


def test_gate8_against_reference_golden(cuda_dev):
    """the reference's own triangulation at max_angular_error = 8 degrees (tools/make_golden.py edges)."""
    from vggsfm_b200 import triangulation as tri
    g = np.load(GOLDEN)
    dev = cuda_dev
    pts, num, mask = tri.triangulate_tracks(to_dev(g["extrinsics"], dev), to_dev(g["tn"], dev),
                                            track_vis=to_dev(g["vis"], dev), track_score=to_dev(g["score"], dev),
                                            ransac_pairs=g["pairs"], max_angular_error=float(g["max_angular_error"]))
    assert np.array_equal(num.cpu().numpy(), g["inlier_num"])
    assert np.array_equal(mask.cpu().numpy(), g["inlier_mask"])
    assert np.abs(pts.cpu().numpy() - g["points"]).max() <= 1e-7 * np.abs(g["points"]).max()


# ------------------------------------------------------------------------------------------------------------------
# 4. usable gating and degenerate tracks
# ------------------------------------------------------------------------------------------------------------------

def test_usable_gating_and_degenerate_tracks(cuda_dev):
    import torch
    from vggsfm_b200.synthetic import make_scene
    S, N = 40, 48
    sc = make_scene(S, N, "SIMPLE_PINHOLE", seed=41, invisible_frac=0.1, outlier_frac=0.05)
    E = sc.extrinsics.copy()
    E[1, :, 3] = 0.0                                              # frame 1 shares frame 0's centre (the origin)
    pc = np.einsum("sij,nj->sni", E[:, :, :3], sc.points3d) + E[:, None, :, 3]
    tn = pc[..., :2] / pc[..., 2:] + np.random.default_rng(0).normal(size=(S, N, 2)) * 3e-4
    vis, score = sc.vis.copy(), sc.score.copy()
    rng = np.random.default_rng(42)
    f05, f05up = np.float32(0.05), np.nextafter(np.float32(0.05), np.float32(1))
    s05, s05up = np.float32(0.5), np.nextafter(np.float32(0.5), np.float32(1))
    # tracks 0-7: vis / score exactly at the thresholds (unusable) and one float above (usable), on 15 frames each
    for n in range(8):
        fr = rng.choice(S, 15, replace=False)
        if n % 4 == 0:
            vis[fr, n] = f05
        elif n % 4 == 1:
            vis[fr, n] = f05up
        elif n % 4 == 2:
            score[fr, n] = s05
        else:
            score[fr, n] = s05up
    vis[:, 8] = 0.01                                              # seen in 0 frames
    vis[:, 9] = 0.01; vis[5, 9] = 0.9                             # 1 frame
    vis[:, 10] = 0.01; vis[[3, 30], 10] = 0.9                     # 2 frames
    tn[:, 11] = rng.uniform(-0.5, 0.5, size=(S, 2))               # every observation a gross outlier
    Xb = np.array([0.1, -0.2, -4.0])                              # behind every camera
    pb = np.einsum("sij,j->si", E[:, :, :3], Xb) + E[:, :, 3]
    tn[:, 12] = pb[:, :2] / pb[:, 2:]
    Xf = np.array([0.3, 0.1, 1e5])                                # every pair far below min_tri_angle
    pf = np.einsum("sij,j->si", E[:, :, :3], Xf) + E[:, :, 3]
    tn[:, 13] = pf[:, :2] / pf[:, 2:]
    assert np.array_equal(vis <= 0.05, (vis <= f05)) and (vis[vis == f05] <= 0.05).all()   # oracle compares in f32
    torch.manual_seed(7)
    pairs = to.draw_pairs(S, 256)
    dt, dv, ds = dead_track(S)
    # NaN observations: the oracle's eigh raises on NaN input ("Eigenvalues did not converge"), so these two tracks are
    # checked by the properties below only, and kept out of the oracle's subset
    nan_tn = tn[:, :2].copy()
    nan_tn[4, 0] = np.nan
    nan_tn[:, 1, 0] = np.nan
    tn_all = np.concatenate([tn, nan_tn, dt], axis=1)
    vis_all = np.concatenate([vis, vis[:, :2], dv], axis=1)
    score_all = np.concatenate([score, score[:, :2], ds], axis=1)
    idx = np.append(np.arange(N), N + 2)
    for sc_arg in (score_all, None):
        kern = run_kernel(cuda_dev, E, tn_all, vis_all, sc_arg, pairs)
        orac = run_oracle(E, tn_all, vis_all, sc_arg, pairs, idx)
        compare(kern, orac, idx, f"degenerate tracks, track_score={'set' if sc_arg is not None else 'None'}")
        pk, nk, mk = kern
        usable = (vis_all > 0.05) & ((sc_arg > 0.5) if sc_arg is not None else True)
        usable &= np.isfinite(tn_all).all(axis=-1)
        assert not (mk & ~usable.T).any()                         # no unusable or NaN observation is an inlier
        assert not mk[nk == 0].any() and (nk == mk.sum(axis=1)).all()
        assert nk[8] == 0 and nk[9] <= 1 and nk[10] <= 2 and nk[12] == 0 and nk[13] == 0
        assert not mk[N + 1].any()                                # all-NaN u: nothing usable
        # the exact-threshold tracks really differ: nothing on the unusable frames, something on the usable ones
        if sc_arg is not None:
            assert not mk[0][vis[:, 0] == f05].any() and not mk[2][score[:, 2] == s05].any()
            assert mk[1][vis[:, 1] == f05up].any() and mk[3][score[:, 3] == s05up].any()
        else:
            assert mk[2][score[:, 2] == s05].any()


# ------------------------------------------------------------------------------------------------------------------
# 5. undistortion through the ABI: iterations_run and the output
# ------------------------------------------------------------------------------------------------------------------

def undistort(dev, tn_d, k):
    import torch
    from vggsfm_b200 import _lib
    L = _lib.lib()
    S, N, _ = tn_d.shape
    t = to_dev(tn_d, dev)
    kk = to_dev(np.ascontiguousarray(k, dtype=np.float64), dev)
    out = torch.empty_like(t)
    ws = torch.empty(64, dtype=torch.uint8, device=dev)
    it = ctypes.c_int()
    _lib.check(L.vgg_undistort_simple_radial(S, N, t.data_ptr(), kk.data_ptr(), 100, 1e-10, 1e-6, out.data_ptr(),
                                             ctypes.byref(it), ws.data_ptr(), ws.numel(),
                                             torch.cuda.current_stream(dev).cuda_stream), "undistort")
    return out.cpu().numpy(), it.value


def test_undistortion_iterations_against_reference(cuda_dev):
    """corner tracks at k = 0.05 / -0.4 / -0.55 / -0.5: 11, 47, 80 (second mask word) and 100 (no convergence)
    iterations like the reference and the oracle; then one call mixing the converging k (the stop is global)."""
    g = np.load(GOLDEN)
    C = len(g["und_k"])
    for c in range(C):
        tn_d = (g["und_uv"][c:c + 1].astype(np.float64) - 512.0) / 1000.0
        out, it = undistort(cuda_dev, tn_d, g["und_k"][c])
        o_und, o_it = to.iterative_undistortion(g["und_k"][c], tn_d)
        assert it == g["und_iters"][c] == o_it
        assert np.abs(out - g["und_tn"][c]).max() < 1e-12 and np.abs(out - o_und).max() < 1e-12
    M = len(g["und_tn_mixed"])
    tn_d = (g["und_uv"][:M].astype(np.float64) - 512.0) / 1000.0
    out, it = undistort(cuda_dev, tn_d, g["und_k"][:M, 0])
    assert it == int(g["und_iters_mixed"]) and np.abs(out - g["und_tn_mixed"]).max() < 1e-12
    # the k = 0.05 frame alone stops at 11; inside the mixed call it runs all 80 iterations
    assert int(g["und_iters_mixed"]) > g["und_iters"][0]


@pytest.mark.parametrize("dtype", ["float32", "float64"])
def test_cam_from_img_corner_tracks(cuda_dev, dtype):
    """cam_from_img with float32 / float64 pixel tracks and float64 intrinsics on the same corner tracks."""
    import torch
    from vggsfm_b200 import triangulation as tri
    g = np.load(GOLDEN)
    dev = cuda_dev
    tdt = getattr(torch, dtype)
    for c in range(len(g["und_k"])):
        tn = tri.cam_from_img(to_dev(g["und_uv"][c:c + 1], dev, tdt), to_dev(g["und_intrinsics"][c:c + 1], dev),
                              to_dev(g["und_k"][c:c + 1], dev))
        assert tn.dtype == torch.float64
        assert np.abs(tn.cpu().numpy() - g["und_tn"][c]).max() < 1e-12


# ------------------------------------------------------------------------------------------------------------------
# 6. filter, projection and pair triangulation at S = 400
# ------------------------------------------------------------------------------------------------------------------

def planted_filter_case():
    from vggsfm_b200.synthetic import make_scene
    S, P = 400, 4099                                              # 4099 = 512 blocks of 8 warps + 3: a partial block
    sc = make_scene(S, P, "SIMPLE_RADIAL", seed=61, noise_px=0.6, invisible_frac=0.0, outlier_frac=0.05)
    X = sc.points3d + np.random.default_rng(62).normal(size=(P, 3)) * 2e-3
    uv = sc.tracks.astype(np.float64)
    E, K, ex = sc.extrinsics, sc.intrinsics, sc.extra_params
    assert np.array_equal(E[0], np.concatenate([np.eye(3), np.zeros((3, 1))], 1))    # frame 0: R = I, t = 0
    C = to.proj_centers(E)
    planted = {
        "behind frame 0": [0.2, 0.1, -0.5],
        "at frame 0's centre": [0.0, 0.0, 0.0],                   # camera coordinates exactly (0,0,0) in frame 0
        "depth 0, u = +inf": [1.0, 0.5, 0.0],
        "depth 0, v = NaN": [-1.0, 0.0, 0.0],
        "NaN": [np.nan, 0.0, 4.0],
        "|X| = hard_max": [0.5, 0.2, 300.0],
        "|X| > hard_max": [0.5, 0.2, np.nextafter(300.0, 400.0)],
        "depth 1e-306, x = +inf without distortion (v = 0 * inf = NaN with it)": [1.0, 0.0, 1e-306],
        "depth 1e-154, x = +inf with distortion": [1.0, 0.0, 1e-154],
    }
    # two-frame points: inliers only in frames 0 and b, with a triangulation angle just below / above 1.5 degrees
    Xt = np.array([0.1, 0.0, 4.0])
    ang = np.array([to.tri_angle_deg(C[0], C[b], Xt) for b in range(S)])
    planted["two frames, %.2f deg" % ang[np.argmin(np.abs(ang - 1.2))]] = ("two", Xt, int(np.argmin(np.abs(ang - 1.2))))
    planted["two frames, %.2f deg" % ang[np.argmin(np.abs(ang - 1.8))]] = ("two", Xt, int(np.argmin(np.abs(ang - 1.8))))
    names = list(planted)
    for i, name in enumerate(names):
        v = planted[name]
        j = 17 + 97 * i
        if isinstance(v, tuple):
            X[j] = v[1]
            p2, _ = to.project_3D_points(X[j:j + 1], E, K, ex)
            uv[:, j] = 1e4                                         # far from the projection ...
            uv[[0, v[2]], j] = p2[[0, v[2]], 0]                    # ... except in frames 0 and b
        else:
            X[j] = v
            p2, _ = to.project_3D_points(X[j:j + 1], E, K, ex)
            uv[:, j] = np.where(np.isfinite(p2[:, 0]) & (np.abs(p2[:, 0]) < 1e6), p2[:, 0], 0.0)
    uv[0, 17 + 97 * names.index("at frame 0's centre")] = 0.0      # NaN projection -> (0, 0): only depth <= 0 rejects it
    return S, P, X, uv, E, K, ex, [17 + 97 * i for i in range(len(names))]


def test_filter_points_at_400_frames(cuda_dev):
    import torch
    from vggsfm_b200 import triangulation as tri
    S, P, X, uv, E, K, ex, planted = planted_filter_case()
    dev = cuda_dev
    Xd, Ed, Kd, exd = to_dev(X, dev), to_dev(E, dev), to_dev(K, dev), to_dev(ex, dev)
    p2, _ = to.project_3D_points(X, E, K, ex)
    with np.errstate(invalid="ignore", over="ignore"):
        for u in (uv, uv.astype(np.float32).astype(np.float64)):
            assert not (np.abs(np.sum((p2 - u) ** 2, axis=-1) - 1.0) < 1e-9).any()   # nothing at the 1 px threshold
    seen = set()
    for dtype in (torch.float32, torch.float64):
        uvh = uv.astype(np.float32).astype(np.float64) if dtype == torch.float32 else uv
        for check in (True, False):
            for hard in (300.0, -1.0):
                v, d = tri.filter_all_points3D(Xd, to_dev(uv, dev, dtype), Ed, Kd, exd, max_reproj_error=1.0,
                                               check_triangle=check, return_detail=True, hard_max=hard)
                vo, do = to.filter_all_points3D(X, uvh, E, K, ex, max_reproj_error=1.0, check_triangle=check,
                                                return_detail=True, hard_max=hard)
                v, d = v.cpu().numpy(), d.cpu().numpy()
                assert np.array_equal(v, vo), (dtype, check, hard, np.nonzero(v != vo))
                assert np.array_equal(d, do), (dtype, check, hard)
                seen.add(tuple(vo[planted]))
    assert len(seen) >= 3                                          # the planted points change with the options
    # the two-frame points: below 1.5 degrees invalid, above valid; |X| = 300 passes hard_max = 300, the next float not
    vo, _ = to.filter_all_points3D(X, uv, E, K, ex, max_reproj_error=1.0)
    assert not vo[planted[-2]] and vo[planted[-1]]
    vo, _ = to.filter_all_points3D(X, uv, E, K, ex, max_reproj_error=1.0, check_triangle=False)
    assert vo[planted[5]] and not vo[planted[6]]


def test_project_points_at_400_frames(cuda_dev):
    from vggsfm_b200 import triangulation as tri
    S, P, X, uv, E, K, ex, planted = planted_filter_case()
    dev = cuda_dev
    for extra in (ex, None):
        p2d, pcam = tri.project_3D_points(to_dev(X, dev), to_dev(E, dev), to_dev(K, dev),
                                          to_dev(extra, dev) if extra is not None else None, return_points_cam=True)
        p2d, pcam = p2d.cpu().numpy(), pcam.cpu().numpy()
        r2d, rcam = to.project_3D_points(X, E, K, extra)
        assert np.isfinite(p2d).all()                              # +-inf clamped, NaN -> 0
        big = np.abs(r2d) == np.finfo(np.float64).max
        assert big.sum() == 1 and np.array_equal(big, np.abs(p2d) == np.finfo(np.float64).max)
        assert np.array_equal(np.sign(p2d[big]), np.sign(r2d[big]))
        assert np.allclose(p2d[~big], r2d[~big], rtol=1e-12, atol=1e-8)
        assert np.array_equal(np.isnan(pcam), np.isnan(rcam))
        fin = np.isfinite(rcam)
        assert np.allclose(pcam[fin], rcam[fin], rtol=1e-13, atol=1e-13)
        j = planted[1]                                             # at frame 0's centre: 0/0 -> NaN -> 0
        assert (p2d[0, j] == 0.0).all() and (pcam[0, :, j] == 0.0).all()


def test_triangulate_by_pair_at_bench_shape(cuda_dev):
    from vggsfm_b200 import triangulation as tri
    from vggsfm_b200.synthetic import make_scene
    S, N = 400, 4096
    sc = make_scene(S, N, "SIMPLE_RADIAL", seed=0)
    dev = cuda_dev
    tn = tri.cam_from_img(to_dev(sc.tracks, dev), to_dev(sc.intrinsics, dev), to_dev(sc.extra_params, dev))
    bp, bche, bang = tri.triangulate_by_pair(to_dev(sc.extrinsics, dev)[None], tn[None])
    bp, bche, bang, tn = bp.cpu().numpy(), bche.cpu().numpy(), bang.cpu().numpy(), tn.cpu().numpy()
    frames = np.unique(np.concatenate([np.arange(1, S, 21), [1, 2, S - 1]]))
    sel = np.concatenate([[0], frames])
    op, oche, oang = to.triangulate_by_pair(sc.extrinsics[sel], tn[sel])
    assert np.array_equal(bche[frames - 1], oche)
    rel = np.abs(bp[frames - 1] - op).max(axis=-1) / (1.0 + np.abs(op).max(axis=-1))
    print(f"\ntriangulate_by_pair 400x4096: {len(frames)} of 399 pairs checked, max rel point error {rel.max():.2e}, "
          f"max angle error {np.abs(bang[frames - 1] - oang).max():.2e} deg")
    assert rel.max() <= 1e-7
    assert np.abs(bang[frames - 1] - oang).max() <= 1e-7
