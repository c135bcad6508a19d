"""The LM solve never stores the coupling blocks W = J_c^T J_p: z_build and backsub rebuild each block from its
observation.  These tests hold the rebuilt blocks against the W that vgg_ba_build_blocks stores, reduced in float64 on
the host:
  * the reduced system (Sraw, rhs) of vgg_ba_schur, whose Zt comes from the observations;
  * one LM iteration: the camera step the solver took has a normwise backward error <= 1e-12 in the damped reduced
    system built on the host from the stored W (so the Zt of the solve itself, banded or dense, is pinned), and the
    point step is d_p = -M M^T (g_p + W^T d_c) at that camera step;
  * structurally zero entries of the reduced system of vgg_ba_schur (which runs dense) stay exact zeros, which they
    only do if every Zt row that no observation reaches is zero: z_build skips those rows;
  * 1- and 2-frame solves follow the oracle's trajectory (CTAs of fewer warps than usual).
Masks put holes at the 32-frame groups' edges and blank whole (frame group, 8-track tile) regions; N % 32 != 0, S = 33
and 65 leave a one-frame last group; some points and (in the solve) the gauge poses are constant."""
import numpy as np
import pytest

from oracle import ba_oracle as bo
from tests.ba_harness import (band_record, check_one_step, check_same_solve, check_trajectory, device_args,
                              device_solve, options, oracle_solve)
from tests.helpers import ba_case, banded_ba_case, recovered_step, to_dev, unpack_camrec

pytestmark = pytest.mark.gpu

CASES = [
    (33, 130, "SIMPLE_PINHOLE", bo.INTR_CONST),
    (65, 203, "SIMPLE_PINHOLE", bo.INTR_PER_FRAME),
    (33, 97, "SIMPLE_PINHOLE", bo.INTR_SHARED),
    (65, 130, "SIMPLE_RADIAL", bo.INTR_CONST),
    (33, 250, "SIMPLE_RADIAL", bo.INTR_PER_FRAME),
    (65, 1001, "SIMPLE_RADIAL", bo.INTR_SHARED),
]


def _edge_case(S, N, cam, mode):
    c = ba_case(S, N, cam, mode, seed=5 * S + N)
    m = c["mask"].copy()
    rng = np.random.default_rng(S * N)
    for s in (31, 32, 63, 64):                       # holes at the frame-group edges
        if s < S:
            m[s, rng.uniform(size=N) < 0.5] = False
    m[32:64, 8:16] = False                           # a whole (frame group, track tile) region without observations
    m[:, N - 1] = False                              # a point nobody sees
    m[S - 1, N - 5:] = False                         # the one-frame last group, last partial tile
    c["mask"] = m
    pconst = np.zeros(N, dtype=bool)
    pconst[3::11] = True
    return c, pconst


def _blocks(c, pconst, dev):
    import torch
    from vggsfm_b200 import bundle_adjustment as ba
    args = device_args(c, dev)
    out = ba.build_blocks(*args, point_const=to_dev(pconst.astype(np.uint8), dev))
    torch.cuda.synchronize()
    return args, out, {k: v.cpu().numpy() for k, v in out.items()}


def _point_factor(H_pp, g_p, pconst, radius):
    """M = Dp L^-T (V = Dp H_pp Dp + diag/radius = L L^T), q = M^T g_p, in float64; zero for constant points"""
    N = H_pp.shape[0]
    H = np.stack([H_pp[:, [0, 1, 2]], H_pp[:, [1, 3, 4]], H_pp[:, [2, 4, 5]]], axis=1)
    sc_p = 1.0 / (1.0 + np.sqrt(np.einsum("nii->ni", H)))
    Hs = H * sc_p[:, :, None] * sc_p[:, None, :]
    dpp = np.clip(np.einsum("nii->ni", Hs), 1e-6, 1e32)
    V = Hs + np.einsum("ni,ij->nij", dpp / radius, np.eye(3))
    M = sc_p[:, :, None] * np.transpose(np.linalg.inv(np.linalg.cholesky(V)), (0, 2, 1))
    M[pconst] = 0.0
    q = np.einsum("nji,nj->ni", M, g_p)
    return sc_p, M, q.reshape(N, 3)


def _stored_W(h, S, N, dc, ns):
    """the stored blocks as [D, N, 3] (per-frame rows, then the shared-intrinsics rows)"""
    return np.ascontiguousarray(h["W"][:, :S * dc + ns].transpose(1, 0, 2))


def _camera_system(h, S, dc, ns):
    g_c, H_cc, H_cs, g_s, H_ss = unpack_camrec(h["camrec"], h["shared"], S, dc, ns)
    D = S * dc + ns
    Hc = np.zeros((D, D))
    for s in range(S):
        Hc[s * dc:(s + 1) * dc, s * dc:(s + 1) * dc] = H_cc[s]
        if ns:
            Hc[s * dc:s * dc + 6, S * dc:] = H_cs[s]
            Hc[S * dc:, s * dc:s * dc + 6] = H_cs[s].T
    gc = np.concatenate([g_c.reshape(-1), g_s.reshape(-1)]) if ns else g_c.reshape(-1)
    if ns:
        Hc[S * dc:, S * dc:] = H_ss
    return Hc, gc


def _host_schur(h, pconst, S, N, dc, ns, radius):
    """(Sraw [D,D], rhs [D], H_cc [D,D]) of the stored blocks at `radius`, in float64"""
    sc_p, M, q = _point_factor(h["H_pp"], h["g_p"], pconst, radius)
    Z = np.einsum("dnj,njk->dnk", _stored_W(h, S, N, dc, ns), M).reshape(S * dc + ns, 3 * N)
    Hc, gc = _camera_system(h, S, dc, ns)
    return Hc - Z @ Z.T, -(gc - Z @ q.reshape(-1)), Hc


def _schur(c, pconst, dev, radius=37.0):
    """(GPU Sraw [D,D] lower-valid, GPU rhs [D], host Sraw, host rhs) of the stored blocks at `radius`"""
    import torch
    from vggsfm_b200 import bundle_adjustment as ba
    S, N = c["mask"].shape
    dc, ns = bo.dims(c["model"], c["mode"])
    D = S * dc + ns
    args, out, h = _blocks(c, pconst, dev)
    sc_p, _, _ = _point_factor(h["H_pp"], h["g_p"], pconst, radius)
    Sraw, rhs = ba.schur(*args, out, to_dev(sc_p, dev), radius, point_const=to_dev(pconst.astype(np.uint8), dev))
    torch.cuda.synchronize()
    Sh, rh, _ = _host_schur(h, pconst, S, N, dc, ns, radius)
    return Sraw.cpu().numpy()[:, :D], rhs.cpu().numpy(), Sh, rh


def _frames_share_a_point(mask, dc, ns):
    """[D, D] True where two per-frame columns can couple (a common visible point) or a column is shared / the same frame"""
    S = mask.shape[0]
    common = (mask.astype(np.int64) @ mask.T.astype(np.int64)) > 0
    D = S * dc + ns
    out = np.ones((D, D), dtype=bool)
    out[:S * dc, :S * dc] = np.kron(common | np.eye(S, dtype=bool), np.ones((dc, dc), dtype=bool))
    return out


@pytest.mark.parametrize("S,N,cam,mode", CASES)
def test_schur_from_observations_matches_stored_W(cuda_dev, S, N, cam, mode):
    c, pconst = _edge_case(S, N, cam, mode)
    dc, ns = bo.dims(c["model"], mode)
    Sg, rg, Sh, rh = _schur(c, pconst, cuda_dev)
    D = S * dc + ns
    low = np.tril_indices(D)
    d = np.sqrt(np.abs(np.diag(Sh)))
    ratio = (np.abs(Sg - Sh) / np.maximum(np.outer(d, d), 1e-300))[low].max()
    print(f"matrix-free schur {S}x{N} {cam} mode {mode}: max |dS_ij| / sqrt(S_ii S_jj) = {ratio:.3g}")
    assert ratio < 1e-12
    assert np.abs(rg - rh).max() <= 1e-11 * np.abs(rh).max()
    zero = ~_frames_share_a_point(c["mask"], dc, ns)
    assert (Sg[low][zero[low]] == 0.0).all()


def _one_step_check(c, pconst, param_const, dev, label):
    """one accepted LM iteration (tests/ba_harness.py check_one_step), and against the stored W: the camera step's
    backward error in the damped reduced system (Jacobi-scaled, constant parameters pinned, as the solver forms it), and
    the point step at that camera step"""
    S, N = c["mask"].shape
    model, mode = c["model"], c["mode"]
    dc, ns = bo.dims(model, mode)
    _, _, h = _blocks(c, pconst, dev)
    o, _ = options(max_num_iterations=1, function_tolerance=0.0, gradient_tolerance=0.0, parameter_tolerance=0.0)
    got = device_solve(c, dev, param_const=param_const, point_const=pconst, options=o)
    check_one_step(c, got, param_const, pconst, label=label)
    radius = got["trace"][0, 5]
    new = (got["poses"], got["intr"], got["points"])
    d_c, u_c, d_p, u_p = recovered_step((c["poses"], c["intr"], c["points"]), new, S, dc, ns, model, mode)
    Sh, rh, Hc = _host_schur(h, pconst, S, N, dc, ns, radius)
    hd = np.diag(Hc)
    sc_c = 1.0 / (1.0 + np.sqrt(hd))
    fc = ~param_const.astype(bool)
    A = Sh * np.outer(sc_c, sc_c) + np.diag(np.clip(hd * sc_c * sc_c, 1e-6, 1e32) / radius)
    A[~fc, :] = 0.0
    A[:, ~fc] = 0.0
    A[~fc, ~fc] = 1.0
    b = np.where(fc, rh * sc_c, 0.0)
    x, ux = d_c / sc_c, u_c / sc_c
    assert not x[~fc].any()
    eta = np.abs(A @ x - b).max() / (np.abs(A).sum(1).max() * (np.abs(x).max() + ux.max()) + np.abs(b).max())
    _, M, _ = _point_factor(h["H_pp"], h["g_p"], pconst, radius)
    wacc = np.einsum("dnc,d->nc", _stored_W(h, S, N, dc, ns), d_c)
    ref = -np.einsum("nij,nkj,nk->ni", M, M, h["g_p"] + wacc)
    err = np.abs(d_p - ref)
    scale = np.abs(ref).max()
    print(f"matrix-free step {label}: camera step backward error {eta:.3g}, "
          f"max |d_p - ref| / max |ref| = {err.max() / scale:.3g}")
    assert eta <= 1e-12, (label, eta)
    assert not d_p[pconst].any()
    assert (err <= 1e-9 * scale + 4 * u_p).all(), label


@pytest.mark.parametrize("S,N,cam,mode", CASES)
def test_point_step_matches_stored_W(cuda_dev, S, N, cam, mode):
    c, pconst = _edge_case(S, N, cam, mode)
    param_const = bo.default_param_const(S, c["model"], mode)
    _one_step_check(c, pconst, param_const, cuda_dev, f"{S}x{N} {cam} mode {mode}")


def test_banded_skip_regions_stay_zero(cuda_dev):
    """a sequential problem with the band hint on: the solve's step against the reduced system of the stored W (a Zt
    region the band skip left wrong moves the camera step off it); then, through vgg_ba_schur (dense), exact zeros
    between frames without a common point"""
    c = banded_ba_case(160, 2050, "SIMPLE_RADIAL", bo.INTR_SHARED, life=24, seed=41)
    S, N = c["mask"].shape
    pconst = np.zeros(N, dtype=bool)
    pconst[7::13] = True
    _one_step_check(c, pconst, bo.default_param_const(S, c["model"], c["mode"]), cuda_dev, "banded 160x2050")
    assert band_record()["tables"], "the band tables were not used"
    dc, ns = bo.dims(c["model"], c["mode"])
    Sg, _, Sh, _ = _schur(c, pconst, cuda_dev)
    D = S * dc + ns
    low = np.tril_indices(D)
    zero = ~_frames_share_a_point(c["mask"], dc, ns)
    assert zero[low].sum() > D * D // 8
    assert (Sg[low][zero[low]] == 0.0).all()
    d = np.sqrt(np.abs(np.diag(Sh)))
    assert (np.abs(Sg - Sh) / np.maximum(np.outer(d, d), 1e-300))[low].max() < 1e-12


@pytest.mark.parametrize("S,N,cam,mode", [
    (1, 200, "SIMPLE_RADIAL", bo.INTR_PER_FRAME),
    (1, 64, "SIMPLE_PINHOLE", bo.INTR_CONST),
    (2, 150, "SIMPLE_PINHOLE", bo.INTR_SHARED),
    (2, 97, "SIMPLE_RADIAL", bo.INTR_CONST),
])
def test_few_frames_lm_matches_oracle(cuda_dev, S, N, cam, mode):
    """1 and 2 frames: backsub runs CTAs of one and two warps, z_build of one"""
    c = ba_case(S, N, cam, mode, seed=7)
    o, opt = options(max_num_iterations=10)
    ref = oracle_solve(c, opt=opt)
    got = device_solve(c, cuda_dev, options=o)
    check_trajectory(got, ref)
    seen = c["mask"].sum(0) >= 2                     # a point seen once has no depth; damping alone fixes it
    # a single frame fits its points exactly: final costs of 1e-18, held to 1e-9 absolute
    check_same_solve(got, ref, f"{S}x{N} {cam} mode {mode}", points=seen, min_cost=1.0)
