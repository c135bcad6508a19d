"""GPU parity of the bundle-adjustment kernels against the CPU oracle (oracle/ba_oracle.py).

Tolerances: the kernels compute in float64 with a different summation order than numpy, so block
sums are compared at 1e-10 relative; a whole LM solve (tens of Cholesky solves) at 1e-7 on the
trajectory and 1e-6 on the final parameters (rotation geodesic in degrees, translation/point L2)."""
import functools

import numpy as np
import pytest

from oracle import ba_oracle as bo
from tests.ba_harness import check_same_solve, check_trajectory, device_solve, options, oracle_solve, relerr
from tests.helpers import ba_case, to_dev, unpack_camrec, rotation_angle_deg

pytestmark = pytest.mark.gpu

CASES = [
    (8, 256, "SIMPLE_PINHOLE", bo.INTR_PER_FRAME),
    (8, 256, "SIMPLE_RADIAL", bo.INTR_SHARED),
    (5, 100, "SIMPLE_RADIAL", bo.INTR_PER_FRAME),     # N % 16 != 0 -> non-TMA path
    (13, 48, "SIMPLE_PINHOLE", bo.INTR_SHARED),
    (9, 64, "SIMPLE_RADIAL", bo.INTR_CONST),
    (20, 304, "SIMPLE_PINHOLE", bo.INTR_CONST),
]


BLOCK_CASES = CASES + [
    (45, 300, "SIMPLE_PINHOLE", bo.INTR_PER_FRAME),    # frame group 1: nf = 13 frames of dc = 7 -> plain-store W path
    (70, 1000, "SIMPLE_RADIAL", bo.INTR_SHARED),       # 3 frame groups
    (33, 130, "SIMPLE_RADIAL", bo.INTR_PER_FRAME),     # frame group 1 has nf = 1
    (70, 1001, "SIMPLE_PINHOLE", bo.INTR_SHARED),      # N % 4 != 0: scalar observation loads, several groups
]


@functools.lru_cache(maxsize=None)
def _blocks_oracle(S, N, cam, mode):
    c = ba_case(S, N, cam, mode, seed=S + N)
    pconst = np.zeros(N, dtype=bool)
    pconst[::7] = True
    ref = bo.build_blocks(c["poses"], c["intr"], c["points"], c["uv"], c["mask"], c["model"], mode, pconst)
    return c, pconst, ref


@pytest.mark.parametrize("S,N,cam,mode", BLOCK_CASES)
def test_blocks_match_oracle(cuda_dev, S, N, cam, mode):
    """the library's own warp sizing (tracks_per_warp = 0)"""
    _check_blocks(cuda_dev, S, N, cam, mode, 0)


# 36 and 100 put warp chunk boundaries inside a 32-track point tile; 64 is the sizing of banded problems
@pytest.mark.parametrize("tracks_per_warp", [4, 36, 64, 100])
@pytest.mark.parametrize("S,N,cam,mode", BLOCK_CASES)
def test_blocks_tracks_per_warp_match_oracle(cuda_dev, S, N, cam, mode, tracks_per_warp):
    _check_blocks(cuda_dev, S, N, cam, mode, tracks_per_warp)


def _check_blocks(cuda_dev, S, N, cam, mode, tracks_per_warp):
    import torch
    from vggsfm_b200 import bundle_adjustment as ba
    c, pconst, ref = _blocks_oracle(S, N, cam, mode)
    out = ba.build_blocks(to_dev(c["uv"], cuda_dev, torch.float32), to_dev(c["mask"].astype(np.uint8), cuda_dev),
                          to_dev(c["poses"], cuda_dev), to_dev(c["intr"], cuda_dev), to_dev(c["points"], cuda_dev),
                          c["model"], mode, point_const=to_dev(pconst.astype(np.uint8), cuda_dev),
                          tracks_per_warp=tracks_per_warp)
    torch.cuda.synchronize()
    dc, ns = bo.dims(c["model"], mode)
    g_c, H_cc, H_cs, g_s, H_ss = unpack_camrec(out["camrec"].cpu().numpy(), out["shared"].cpu().numpy(), S, dc, ns)
    tol = 1e-10
    assert abs(out["cost"].item() - ref["cost"]) <= tol * ref["cost"]
    assert relerr(g_c, ref["g_c"]) < tol
    assert relerr(H_cc, ref["H_cc"]) < tol
    assert relerr(out["g_p"].cpu().numpy(), ref["g_p"]) < tol
    Hpp = out["H_pp"].cpu().numpy()
    Hfull = np.stack([Hpp[:, [0, 1, 2]], Hpp[:, [1, 3, 4]], Hpp[:, [2, 4, 5]]], axis=1)
    assert relerr(Hfull, ref["H_pp"]) < tol
    W = out["W"].cpu().numpy()                       # track-major [N, pitch, 3]
    assert relerr(W[:, :S * dc].reshape(N, S, dc, 3).transpose(1, 2, 0, 3), ref["W"]) < tol
    if ns:
        assert relerr(W[:, S * dc:S * dc + ns].transpose(1, 0, 2), ref["W_s"]) < tol
        assert relerr(H_cs, ref["H_cs"]) < tol
        assert relerr(g_s, ref["g_s"]) < tol
        assert relerr(H_ss, ref["H_ss"]) < tol


@pytest.mark.parametrize("S,N,cam,mode", CASES[:4] + [
    (50, 2048, "SIMPLE_PINHOLE", bo.INTR_PER_FRAME),     # D = 350: three 128-column tiles
    (400, 4096, "SIMPLE_RADIAL", bo.INTR_SHARED),        # C3: D = 2402, 19 row blocks
])
def test_schur_matches_oracle(cuda_dev, S, N, cam, mode):
    """Sraw = H_cc - Z Z^T through z_build (which also produces the SYRK's column maxima) and the Ozaki SYRK, per entry
    within 1e-12 sqrt(S_ii S_jj) -- the accuracy the Cholesky of the reduced system needs (largest observed on an
    H100 80GB HBM3: 7.9e-14, at C3)."""
    import torch
    from vggsfm_b200 import bundle_adjustment as ba
    c = ba_case(S, N, cam, mode, seed=3 * S + N)
    dc, ns = bo.dims(c["model"], mode)
    D = S * dc + ns
    blocks = bo.build_blocks_c if bo._load_c() is not None else bo.build_blocks
    blk = blocks(c["poses"], c["intr"], c["points"], c["uv"], c["mask"], c["model"], mode)
    Hc, gc = bo._assemble_camera_system(blk, S, dc, ns)
    radius = 37.0
    sc_p = 1.0 / (1.0 + np.sqrt(np.einsum("nii->ni", blk["H_pp"])))
    Hs = blk["H_pp"] * sc_p[:, :, None] * sc_p[:, None, :]
    dpp = np.clip(np.einsum("nii->ni", Hs), 1e-6, 1e32)
    V = Hs + np.einsum("ni,ij->nij", dpp / radius, np.eye(3))
    Linv = np.linalg.inv(np.linalg.cholesky(V))
    M = sc_p[:, :, None] * np.transpose(Linv, (0, 2, 1))
    q = np.einsum("nji,nj->ni", M, blk["g_p"])
    Wf = bo._full_W(blk, S, dc, ns)
    Z = np.einsum("dnj,njk->dnk", Wf, M).reshape(D, N * 3)
    S_ref = Hc - Z @ Z.T
    rhs_ref = -(gc - Z @ q.reshape(-1))

    dev = cuda_dev
    args = (to_dev(c["uv"], dev, torch.float32), to_dev(c["mask"].astype(np.uint8), dev), to_dev(c["poses"], dev),
            to_dev(c["intr"], dev), to_dev(c["points"], dev), c["model"], mode)
    out = ba.build_blocks(*args)
    Sraw, rhs = ba.schur(*args, out, to_dev(sc_p, dev), radius)
    torch.cuda.synchronize()
    Sraw = Sraw.cpu().numpy()[:, :D]
    low = np.tril_indices(D)
    d = np.sqrt(np.diag(S_ref))
    assert (d > 0).all()
    ratio = (np.abs(Sraw - S_ref) / np.outer(d, d))[low].max()
    print(f"schur S={S} N={N}: max |dS_ij| / sqrt(S_ii S_jj) = {ratio:.3g}")
    assert ratio < 1e-12
    assert np.abs(rhs.cpu().numpy() - rhs_ref).max() < 1e-9 * np.abs(rhs_ref).max()


@pytest.mark.parametrize("S,N,cam,mode", [
    (8, 256, "SIMPLE_PINHOLE", bo.INTR_PER_FRAME),      # BASELINE config C1
    (8, 256, "SIMPLE_RADIAL", bo.INTR_SHARED),
    (12, 200, "SIMPLE_RADIAL", bo.INTR_PER_FRAME),
])
def test_lm_trajectory_matches_oracle(cuda_dev, S, N, cam, mode):
    ref, got = _solve_both(ba_case(S, N, cam, mode, seed=11), cuda_dev, 25)
    check_trajectory(got, ref)
    check_same_solve(got, ref)
    assert got["s"].kernel_launches > 0


def test_bundle_adjustment_wrapper_matches_oracle(cuda_dev):
    """global_BA-style call (triangulation.py:1033-1063): compaction, negative-depth filter, LM, normalize x2."""
    import torch
    from vggsfm_b200 import bundle_adjustment as ba
    c = ba_case(10, 300, "SIMPLE_RADIAL", bo.INTR_SHARED, seed=5, invisible_frac=0.4)
    sc = c["scene"]
    mask = sc.mask.copy()
    mask[:, :5] = False                      # tracks without inliers are dropped and ids compacted
    mask[1:, 5] = False                      # single-inlier track
    pts = c["points"].copy()
    pts[7] = [0.0, 0.0, -3.0]                # behind every camera -> negative depth filter deletes it
    ref = bo.bundle_adjustment(pts, c["poses"], c["K"], c["extra"], sc.tracks, mask, shared_camera=True,
                               camera_type="SIMPLE_RADIAL", options=bo.LMOptions.prepare_ba_options())
    dev = cuda_dev
    out = ba.bundle_adjustment(to_dev(pts, dev), to_dev(c["poses"], dev), to_dev(c["K"], dev), to_dev(c["extra"], dev),
                               to_dev(sc.tracks, dev), to_dev(mask, dev), shared_camera=True,
                               camera_type="SIMPLE_RADIAL", options=ba.prepare_ba_options())
    assert np.array_equal(out[4].cpu().numpy(), ref[4])
    assert out[5].iterations == ref[5]["iterations"]
    assert np.abs(out[0].cpu().numpy() - ref[0]).max() < 1e-6
    assert rotation_angle_deg(out[1].cpu().numpy()[:, :, :3], ref[1][:, :, :3]).max() < 1e-6
    assert np.abs(out[1].cpu().numpy()[:, :, 3] - ref[1][:, :, 3]).max() < 1e-6
    assert np.abs(out[2].cpu().numpy() - ref[2]).max() < 1e-5
    assert np.abs(out[3].cpu().numpy() - ref[3]).max() < 1e-7


def _solve_both(c, cuda_dev, max_it, use_c=False):
    """the oracle's and the GPU's solve of c with default options but max_num_iterations (tests/ba_harness.py)"""
    o, opt = options(max_num_iterations=max_it)
    return oracle_solve(c, opt=opt, use_c=use_c), device_solve(c, cuda_dev, options=o)


def test_c2_full_solve_matches_oracle(cuda_dev):
    """BASELINE config C2 (50 x 2048, SIMPLE_PINHOLE, per-frame focal) at FULL size, whole solve to convergence,
    against the oracle (C/OpenMP Jacobians + numpy Schur/Cholesky)."""
    c = ba_case(50, 2048, "SIMPLE_PINHOLE", bo.INTR_PER_FRAME, seed=2, invisible_frac=0.3)
    ref, got = _solve_both(c, cuda_dev, 100, use_c=bo._load_c() is not None)
    assert got["s"].termination == "CONVERGENCE_GRADIENT" and got["s"].iterations >= 5
    check_trajectory(got, ref)
    check_same_solve(got, ref)


def test_c3_bench_config_matches_oracle(cuda_dev):
    """The configuration bench.py publishes numbers on (C3: 400 x 4096, SIMPLE_RADIAL, shared camera, dense visibility;
    the same scene and perturbed start as bench.make_problem): first 3 LM iterations on the default product path
    (wgmma Ozaki SYRK + the in-repo Cholesky) against the oracle."""
    c = ba_case(400, 4096, "SIMPLE_RADIAL", bo.INTR_SHARED, seed=0, invisible_frac=0.0)
    ref, got = _solve_both(c, cuda_dev, 3, use_c=bo._load_c() is not None)
    assert got["s"].iterations == 3
    check_trajectory(got, ref)
    check_same_solve(got, ref)


def test_c2_full_size_properties(cuda_dev):
    """BASELINE config C2 (50 x 2048, SIMPLE_PINHOLE) at full size: size-independent properties --
    cost decreases monotonically over accepted steps, converges to the noise floor, recovers GT up to gauge."""
    import torch
    from vggsfm_b200 import bundle_adjustment as ba
    c = ba_case(50, 2048, "SIMPLE_PINHOLE", bo.INTR_PER_FRAME, seed=2, invisible_frac=0.3)
    dev = cuda_dev
    poses, intr, pts = to_dev(c["poses"], dev), to_dev(c["intr"], dev), to_dev(c["points"], dev)
    s = ba.lm_solve(to_dev(c["uv"], dev, torch.float32), to_dev(c["mask"].astype(np.uint8), dev), poses, intr, pts,
                    c["model"], c["mode"], want_trace=True)
    tr = s.trace.numpy()
    acc = tr[tr[:, 7] == 1]
    assert len(acc) >= 3
    assert np.all(acc[:, 2] < acc[:, 1])
    M = int(c["mask"].sum())
    rms = np.sqrt(2.0 * s.final_cost / M)
    assert 0.25 < rms < 0.5, rms            # 0.3 px noise per coordinate -> ~0.42 px per observation


@pytest.mark.parametrize("n", [64, 100, 343, 512, 2403])
def test_cholesky_matches_lapack(cuda_dev, n):
    """csrc/chol.cu -- the factorisation of the default LM path -- against numpy.linalg.cholesky (float64; 1e-10 of the
    factor's scale; L in the lower triangle, L^T mirrored into the upper one), plus failure reporting."""
    import ctypes
    import torch
    from vggsfm_b200 import _lib
    rng = np.random.default_rng(n)
    B = rng.normal(size=(n, n + 8))
    A = B @ B.T + n * 1e-3 * np.eye(n)
    lda = (n + 127) // 128 * 128
    buf = torch.zeros(n, lda, dtype=torch.float64, device=cuda_dev)
    buf[:, :n] = torch.from_numpy(np.tril(A)).to(cuda_dev)
    ws = torch.empty(((n + 127) // 128) * 131072 + 1024, dtype=torch.uint8, device=cuda_dev)
    info = ctypes.c_int(-1)
    L = _lib.lib()
    _lib.check(L.vgg_cholesky_lower(n, lda, buf.data_ptr(), ws.data_ptr(), ws.numel(), ctypes.byref(info),
                                    torch.cuda.current_stream().cuda_stream), "vgg_cholesky_lower")
    assert info.value == 0
    ref = np.linalg.cholesky(A)
    full = buf.cpu().numpy()[:, :n]
    got = np.tril(full)
    assert np.abs(got - ref).max() <= 1e-10 * np.abs(ref).max()
    assert np.array_equal(np.triu(full, 1), np.tril(full, -1).T)       # the mirror the backward substitution streams
    # not positive definite -> info reports the failing pivot (1-based)
    A2 = A.copy()
    A2[70 % n, 70 % n] = -1.0
    buf[:, :n] = torch.from_numpy(np.tril(A2)).to(cuda_dev)
    _lib.check(L.vgg_cholesky_lower(n, lda, buf.data_ptr(), ws.data_ptr(), ws.numel(), ctypes.byref(info),
                                    torch.cuda.current_stream().cuda_stream), "vgg_cholesky_lower")
    assert info.value == (70 % n) + 1


@pytest.mark.parametrize("nblk,bw,tail", [(12, 2, 0), (20, 3, 77), (9, 1, 5)])
def test_cholesky_band_plus_arrow_matches_lapack(cuda_dev, nblk, bw, tail):
    """The band-aware schedule of csrc/chol.cu (sequential / video problems: block band + dense arrow; panels and
    trailing tiles restricted to the structure, f64 REDs) against numpy on a random matrix WITH that structure."""
    import ctypes
    import torch
    from vggsfm_b200 import _lib
    n = nblk * 128 + tail                      # the arrow is the last full block (+ the partial tail)
    arrow = nblk - 1
    rng = np.random.default_rng(nblk * 10 + bw)
    G = rng.normal(size=(n, n)) * 0.05
    blk = np.arange(n) // 128
    keep = (np.abs(blk[:, None] - blk[None, :]) <= bw) | (blk[:, None] >= arrow) | (blk[None, :] >= arrow)
    A = (G + G.T) * keep
    A += np.diag(np.abs(A).sum(1) + 1.0)       # diagonally dominant: SPD with the same structure
    nb_all = (n + 127) // 128
    end = np.array([nb_all if b >= arrow else min(arrow, max(b + bw + 1, b + 2)) for b in range(nb_all)], dtype=np.int32)
    lda = nb_all * 128
    buf = torch.zeros(n, lda, dtype=torch.float64, device=cuda_dev)
    buf[:, :n] = torch.from_numpy(np.tril(A)).to(cuda_dev)
    ws = torch.empty(nb_all * 131072 + 1024, dtype=torch.uint8, device=cuda_dev)
    info = ctypes.c_int(-1)
    L = _lib.lib()
    _lib.check(L.vgg_dev_cholesky_band(n, lda, buf.data_ptr(), ws.data_ptr(), ws.numel(), ctypes.byref(info),
                                       torch.cuda.current_stream().cuda_stream, end.ctypes.data, end.size, arrow),
               "vgg_dev_cholesky_band")
    assert info.value == 0
    ref = np.linalg.cholesky(A)
    got = np.tril(buf.cpu().numpy()[:, :n])
    assert np.abs(got - ref).max() <= 1e-10 * np.abs(ref).max()
    # the factor keeps the structure (no fill outside band + arrow), which is what the schedule relies on
    assert not np.abs(ref * ~keep).max() > 1e-12
