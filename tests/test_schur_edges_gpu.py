"""The reduced-system build of one LM iteration stage by stage, as the solve runs it, against the float64 references of
oracle/schur_oracle.py (each bar derived there):
  * ba_blocks_kernel without W (vgg_ba_build_blocks with W = NULL; vgg_dev_build_blocks_band for the band table and
    its sizing) per entry within (m + C0) u sum|terms|; the W-writing variant within the same bar;
  * point_prep (vgg_dev_schur_build): dpp bitwise, M exactly upper triangular, the backward check
    ||L^-1 V L^-T - I|| <= C_P u kappa(V), q within 3 u |M|^T|g|, failed factorisations counted with M = q = 0;
  * z_build: every Zt entry and rhs within its bar, the NaN sentinel left exactly on the complement of the written set
    (dense and banded), so invalid frames of a reached group are exact zeros and unreached rows are never written;
  * syrk_f64 (vgg_dev_syrk_f64_band): Kpad = 0 / 16 / 32 / 48 mod 64, 1 to 300 tiles, band hints with empty, one-block
    and partial-last-block ranges, a non-zero C0 whose skipped tiles stay bitwise, 2^+-300 columns, subnormal products,
    and one NaN whose NaN set equals the prediction from the work list (vgg_dev_syrk_work_list);
  * the whole Sraw per entry within c u (|H_cc| + |Z||Z|^T) at C3 and on a banded 160 x 4003 problem.
Every bar test prints its largest error-to-bar ratio."""
import ctypes

import numpy as np
import pytest

from oracle import ba_oracle as bo
from oracle import band_oracle as bd
from oracle import ozaki_oracle as oz
from oracle import schur_oracle as so
from tests.helpers import ba_case, banded_ba_case, to_dev

pytestmark = pytest.mark.gpu

U = 2.0 ** -53


def _prep_case(c, seed, edges=True):
    """float32 observations (what the kernels read); holes at frame-group edges, a whole (group, 8-track tile)
    region, an unobserved frame and point; constant points every 7th"""
    c["uv"] = c["uv"].astype(np.float32).astype(np.float64)
    S, N = c["mask"].shape
    m = c["mask"].copy()
    if edges:
        rng = np.random.default_rng(seed)
        for s in (31, 32, 63, 64, 127, 128):
            if s < S:
                m[s, rng.uniform(size=N) < 0.5] = False
        if S > 40 and N > 24:
            m[32:64, 16:24] = False
        if S > 3:
            m[S // 2] = False
        m[:, N // 3] = False
    c["mask"] = m
    pconst = np.zeros(N, dtype=bool)
    pconst[5::7] = True
    return c, pconst


def _problem(c, pconst, dev):
    import torch
    from vggsfm_b200 import _lib
    t = dict(uv=to_dev(c["uv"], dev, torch.float32), mask=to_dev(c["mask"].astype(np.uint8), dev),
             poses=to_dev(c["poses"], dev), intr=to_dev(c["intr"], dev), points=to_dev(c["points"], dev),
             pconst=to_dev(pconst.astype(np.uint8), dev))
    S, N = c["mask"].shape
    p = _lib.BAProblem()
    p.S, p.N, p.camera_model, p.intr_mode = S, N, c["model"], c["mode"]
    p.uv, p.mask, p.param_const, p.point_const = t["uv"].data_ptr(), t["mask"].data_ptr(), None, t["pconst"].data_ptr()
    p.poses, p.intr, p.points = t["poses"].data_ptr(), t["intr"].data_ptr(), t["points"].data_ptr()
    return p, t


def _blocks(c, pconst, dev, write_w=False, tpw=0, fg=None):
    """the block kernel's outputs (host arrays) through vgg_dev_build_blocks_band"""
    import torch
    from vggsfm_b200 import _lib
    L = _lib.lib()
    S, N = c["mask"].shape
    dc, ns = bo.dims(c["model"], c["mode"])
    KR = L.vgg_ba_camrec_len(c["model"], c["mode"])
    p, keep = _problem(c, pconst, dev)
    f64 = dict(dtype=torch.float64, device=dev)
    out = dict(cost=torch.zeros(1, **f64), camrec=torch.zeros(S, KR, **f64), g_p=torch.zeros(N, 3, **f64),
               H_pp=torch.zeros(N, 6, **f64), shared=torch.zeros(8, **f64))
    W = torch.zeros(N, (S * dc + ns + 1) // 2 * 2, 3, **f64) if write_w else None
    tab = None if fg is None else np.ascontiguousarray(fg, np.int32).reshape(-1)
    with torch.cuda.device(dev):
        st = torch.cuda.current_stream().cuda_stream
        _lib.check(L.vgg_dev_build_blocks_band(ctypes.byref(p), out["cost"].data_ptr(), out["camrec"].data_ptr(),
                                               out["g_p"].data_ptr(), out["H_pp"].data_ptr(),
                                               None if W is None else W.data_ptr(), out["shared"].data_ptr(), tpw,
                                               None if tab is None else tab.ctypes.data, 0 if tab is None else tab.size,
                                               st), "vgg_dev_build_blocks_band")
        torch.cuda.synchronize()
    return {k: v.cpu().numpy() for k, v in out.items()}, out


def _schur_build(c, pconst, dev, blk_dev, sc_p, radius, banded=0, zt_nan=1, min_diag=1e-6, max_diag=1e32, H_pp=None,
                 g_p=None):
    import torch
    from vggsfm_b200 import _lib
    from vggsfm_b200 import bundle_adjustment as ba
    L = _lib.lib()
    S, N = c["mask"].shape
    dc, ns = bo.dims(c["model"], c["mode"])
    D = S * dc + ns
    Dpad, Kpad = (D + 2 + 127) // 128 * 128, (3 * N + 15) // 16 * 16
    p, keep = _problem(c, pconst, dev)
    ws = ba.workspace(S, N, c["model"], c["mode"], dev)
    f64 = dict(dtype=torch.float64, device=dev)
    o = dict(M=torch.empty(N, 9, **f64), q=torch.empty(N, 3, **f64), dpp=torch.empty(N, 3, **f64),
             scal=torch.empty(16, **f64), Zt=torch.empty(Kpad, Dpad, **f64), Sraw=torch.empty(D, Dpad, **f64),
             rhs=torch.empty(Dpad, **f64))
    Hd = blk_dev["H_pp"] if H_pp is None else to_dev(H_pp, dev)
    gd = blk_dev["g_p"] if g_p is None else to_dev(g_p, dev)
    scd = to_dev(sc_p, dev)
    with torch.cuda.device(dev):
        st = torch.cuda.current_stream().cuda_stream
        _lib.check(L.vgg_dev_schur_build(ctypes.byref(p), blk_dev["camrec"].data_ptr(), gd.data_ptr(), Hd.data_ptr(),
                                         blk_dev["shared"].data_ptr(), scd.data_ptr(), radius, min_diag, max_diag,
                                         banded, zt_nan, ws.data_ptr(), ws.numel(), *[o[k].data_ptr() for k in
                                         ("M", "q", "dpp", "scal", "Zt", "Sraw", "rhs")], st), "vgg_dev_schur_build")
    return {k: v.cpu().numpy() for k, v in o.items()}, Kpad, Dpad


def _sc_p(H_pp):
    return 1.0 / (1.0 + np.sqrt(H_pp[:, [0, 3, 5]]))


def _gvec(h, S, dc, ns):
    return np.concatenate([h["camrec"][:, :dc].reshape(-1), h["shared"][:ns]])


def _ratio(err, bar):
    with np.errstate(invalid="ignore", divide="ignore"):
        q = np.where(err == 0, 0.0, err / bar)
    return float(np.max(np.where(np.isnan(q), np.inf, q), initial=0.0))


# (S, N, camera, mode): S = 1, 31, 32, 33, 128, 129 and 400 frames, N covering every residue mod 8, all six model /
# mode pairs; dc = 7 with an odd number of frames in the last group (S = 33, 129: one frame)
CASES = [
    (1, 203, "SIMPLE_PINHOLE", bo.INTR_CONST),
    (31, 130, "SIMPLE_PINHOLE", bo.INTR_SHARED),
    (32, 252, "SIMPLE_RADIAL", bo.INTR_CONST),
    (33, 97, "SIMPLE_PINHOLE", bo.INTR_PER_FRAME),
    (128, 1005, "SIMPLE_RADIAL", bo.INTR_SHARED),
    (129, 255, "SIMPLE_PINHOLE", bo.INTR_PER_FRAME),
    (65, 254, "SIMPLE_RADIAL", bo.INTR_PER_FRAME),
    (400, 200, "SIMPLE_PINHOLE", bo.INTR_CONST),
]


def _check_blocks(h, ref, label):
    r = so.check_blocks(h, ref)
    print(f"blocks {label}: max err/bar {max(r.values()):.3g} {r}")
    assert max(r.values()) <= 1.0, (label, r)


@pytest.mark.parametrize("S,N,cam,mode", CASES)
def test_blocks_solve_variant(cuda_dev, S, N, cam, mode):
    """the solve's variant (no W) with dense auto-sizing and tracks_per_warp 4 / 36 / 64 / 100, and the W-writing
    variant, per entry against the oracle"""
    c, pconst = _prep_case(ba_case(S, N, cam, mode, seed=S + N), S * N)
    ref = so.blocks_ref(c, pconst)
    for tpw in (0, 4, 36, 64, 100):
        h, _ = _blocks(c, pconst, cuda_dev, tpw=tpw)
        _check_blocks(h, ref, f"{S}x{N} {cam} {mode} no-W tpw={tpw}")
    h, _ = _blocks(c, pconst, cuda_dev, write_w=True)
    _check_blocks(h, ref, f"{S}x{N} {cam} {mode} W")


def _stage_checks(c, pconst, dev, radius, label, banded=0, fg=None):
    """point_prep, z_build and the NaN sentinel of one schur_build against the oracle; returns what the Sraw check needs"""
    S, N = c["mask"].shape
    dc, ns = bo.dims(c["model"], c["mode"])
    D = S * dc + ns
    h, blk_dev = _blocks(c, pconst, dev, fg=fg)
    sc = _sc_p(h["H_pp"])
    o, Kpad, Dpad = _schur_build(c, pconst, dev, blk_dev, sc, radius, banded=banded)
    # point_prep
    free = ~pconst
    dpp, V = so.point_prep_ref(h["H_pp"], sc, radius, 1e-6, 1e32)
    assert np.array_equal(o["dpp"][free].view(np.uint64), dpp[free].view(np.uint64)), label
    assert not o["M"][:, [3, 6, 7]].any() and not o["M"][pconst].any() and not o["q"][pconst].any()
    assert o["scal"][6] == 0.0, label
    err, bar = so.point_prep_backward(o["M"][free], V[free], sc[free])
    qref, qbar = so.q_bar(o["M"], h["g_p"])
    rp, rq = _ratio(err, bar), _ratio(np.abs(o["q"] - qref), qbar)
    # z_build
    wr = so.written_set(c["mask"], dc, ns, Kpad, Dpad, fg)
    Z, zbar, Zc, rhs, rbar = so.zt_ref(c, o["M"], o["q"], _gvec(h, S, dc, ns), Kpad, Dpad, pconst)
    nan_in, touched = so.check_sentinel(o["Zt"], wr)
    Zg = np.where(wr, o["Zt"], 0.0)
    rz = _ratio(np.abs(Zg - Z), zbar)
    rr = _ratio(np.abs(o["rhs"][:D] - rhs), rbar)
    print(f"stages {label}: point_prep backward {rp:.3g}, q {rq:.3g}, Zt {rz:.3g}, rhs {rr:.3g} (err/bar); "
          f"sentinel: {nan_in} written NaN, {touched} unwritten changed of {(~wr).sum()}")
    assert max(rp, rq, rz, rr) <= 1.0, label
    assert nan_in == 0 and touched == 0, label
    return h, blk_dev, sc, Z, zbar, Kpad, Dpad


@pytest.mark.parametrize("S,N,cam,mode", CASES)
def test_point_prep_and_z_build(cuda_dev, S, N, cam, mode):
    c, pconst = _prep_case(ba_case(S, N, cam, mode, seed=S + N), S * N)
    _stage_checks(c, pconst, cuda_dev, 37.0, f"{S}x{N} {cam} {mode}")


def _check_sraw(c, pconst, dev, h, blk_dev, sc, Z, zbar, radius, label, banded=0):
    """the whole Sraw of the solve's schur_build per entry against H_cc - Z Z^T of the oracle's Z (end to end: the
    kernel's Zt and the SYRK together).  With Zt within zbar of Z (test_point_prep_and_z_build's bar),
        |S_kernel - S| <= (2 K' + 8) u (|H_cc| + |Zt|^T |Zt|) + zbar^T |Zt| + |Z|^T zbar,
    K' = the non-zero products of the entry (one rounding each in the SYRK, plus its f64 REDs); H_cc is put exactly by
    assemble_hc from the block kernel's records (checked by test_blocks_solve_variant)"""
    import torch
    S, N = c["mask"].shape
    dc, ns = bo.dims(c["model"], c["mode"])
    D = S * dc + ns
    o, Kpad, Dpad = _schur_build(c, pconst, dev, blk_dev, sc, radius, banded=banded, zt_nan=0)
    from tests.test_ba_matrix_free_gpu import _camera_system
    Hc, _ = _camera_system(h, S, dc, ns)
    Zr = np.ascontiguousarray(Z[:3 * N, :D])
    ref = Hc - oz.exact_gram(Zr, device=dev)
    t = lambda a: torch.from_numpy(np.ascontiguousarray(a)).to(dev)
    Zg, Za, Zb = t(np.abs(o["Zt"][:3 * N, :D])), t(np.abs(Zr)), t(zbar[:3 * N, :D])
    nz = (Zg != 0).to(torch.float64)
    kprod = (nz.T @ nz).cpu().numpy()
    bar = ((2.0 * kprod + 8) * U * (np.abs(Hc) + (Zg.T @ Zg).cpu().numpy()) + (Zb.T @ Zg).cpu().numpy() +
           (Za.T @ Zb).cpu().numpy())
    low = np.tril(np.ones((D, D), bool))
    err = np.abs(o["Sraw"][:, :D] - ref)
    r = _ratio(err[low], bar[low])
    print(f"Sraw {label}: max err/bar {r:.3g}")
    assert r <= 1.0, label


def test_c3_stages_and_sraw(cuda_dev):
    """400 x 4096 SIMPLE_RADIAL with a shared camera (the bench configuration)"""
    c, pconst = _prep_case(ba_case(400, 4096, "SIMPLE_RADIAL", bo.INTR_SHARED, seed=3), 11)
    h, blk_dev, sc, Z, zbar, Kpad, Dpad = _stage_checks(c, pconst, cuda_dev, 1e4, "C3 400x4096")
    _check_blocks(h, so.blocks_ref(c, pconst), "C3 no-W")
    _check_sraw(c, pconst, cuda_dev, h, blk_dev, sc, Z, zbar, 1e4, "C3")


# frame group g of TILE_EDGE_RANGES sees tracks [lo, hi): every lo after the first is 7 mod 8 and every hi before the last
# 1 mod 8, so the first and last track of each range sit alone at an edge of z_build's 8-track CTA tile -- a band skip
# test off by one at either end drops a tile that holds an observation
TILE_EDGE_RANGES = [(0, 857), (807, 1665), (1615, 2473), (2423, 3281), (3231, 4003)]


def _tile_edge_case():
    c = ba_case(160, 4003, "SIMPLE_RADIAL", bo.INTR_SHARED, seed=13, invisible_frac=0.0)
    rng = np.random.default_rng(13)
    m = np.zeros((160, 4003), bool)
    for g, (lo, hi) in enumerate(TILE_EDGE_RANGES):
        m[32 * g:32 * g + 32, lo:hi] = rng.uniform(size=(32, hi - lo)) > 0.2
        m[32 * g + 5, [lo, hi - 1]] = True
    c["mask"] = m
    return c


@pytest.mark.parametrize("which", ["life24", "tile_edges"])
def test_banded_stages_and_sraw(cuda_dev, which):
    """160 x 4003 sequential problems: the solve's band plan (compute_band_hint) with fg_tracks active, the block kernel
    with the same table and its banded sizing; the sentinel is left exactly on the complement of the written set.
    life24: points seen for 24 to 36 frames; tile_edges: group ranges that start and end one track inside a tile"""
    if which == "life24":
        c = banded_ba_case(160, 4003, "SIMPLE_RADIAL", bo.INTR_SHARED, life=24, seed=9)
    else:
        c = _tile_edge_case()
    c, pconst = _prep_case(c, 4, edges=False)
    dc, ns = bo.dims(c["model"], c["mode"])
    fg = bd.band_tables(c["mask"], dc, ns)["fg_tracks"]
    if which == "tile_edges":
        assert fg.tolist() == [list(r) for r in TILE_EDGE_RANGES]
    label = f"banded 160x4003 {which}"
    h, blk_dev, sc, Z, zbar, Kpad, Dpad = _stage_checks(c, pconst, cuda_dev, 1e4, label, banded=1, fg=fg)
    from vggsfm_b200 import _lib
    meta, fgk = np.zeros(8, np.int32), np.zeros(2 * fg.shape[0], np.int32)
    _lib.check(_lib.lib().vgg_dev_last_band_hint(meta.ctypes.data, None, None, None, fgk.ctypes.data), "band hint")
    assert meta[0] == 1 and meta[2] == 1 and np.array_equal(fgk.reshape(-1, 2), fg)
    _check_blocks(h, so.blocks_ref(c, pconst), "banded no-W, band table")
    for tpw in (4, 100):
        hb, _ = _blocks(c, pconst, cuda_dev, tpw=tpw, fg=fg)
        _check_blocks(hb, so.blocks_ref(c, pconst), f"banded no-W tpw={tpw}")
    _check_sraw(c, pconst, cuda_dev, h, blk_dev, sc, Z, zbar, 1e4, label, banded=1)


# ----------------------------------------------------------------------------------------------
# point_prep at its edges
# ----------------------------------------------------------------------------------------------

def _point_block(J):
    """H_pp [6] of rows J [m, 3]"""
    H = J.T @ J
    return H[[0, 0, 0, 1, 1, 2], [0, 1, 2, 1, 2, 2]]


@pytest.mark.parametrize("radius", [1e-4, 1.0, 1e4, 1e16])
def test_point_prep_edges(cuda_dev, radius):
    """points seen by one frame (rank-2 H_pp), two nearly parallel rays (kappa up to 1e12), depth 1e5 (dpp at min_diag),
    a max_diag low enough to clip, planted NaN H_pp: exactly those points are counted bad and get M = q = 0.
    One-view points at radius >= 1e14: V = H + diag(dpp)/radius has a last Cholesky pivot at rounding level, and the
    kernel may count such a point bad (M = q = 0), which makes the LM step invalid.  This is a known divergence from
    Ceres (DESIGN 4.2): its Schur eliminator inverts the 3x3 block explicitly and rejects only a non-finite step.  The
    test pins the documented behaviour: such failures happen only to one-view points and only at radius >= 1e14"""
    c, pconst = _prep_case(ba_case(8, 64, "SIMPLE_PINHOLE", bo.INTR_CONST, seed=2), 1, edges=False)
    pconst[:] = False
    h, blk_dev = _blocks(c, pconst, cuda_dev)
    N = 64
    rng = np.random.default_rng(int(np.log10(radius)) + 20)
    H = h["H_pp"].copy()
    g = h["g_p"].copy()
    kinds = {}
    for n in range(N):
        kind = n % 5
        if kind == 0:                                  # one view: two rows
            J = rng.normal(size=(2, 3)) * 500.0
        elif kind == 1:                                # two nearly parallel rays
            a = rng.normal(size=3)
            b = a + rng.normal(size=3) * 10.0 ** -rng.uniform(3, 6)
            J = np.stack([np.cross(a, [0, 0, 1.0]), np.cross(a, [0, 1.0, 0]), np.cross(b, [0, 0, 1.0]),
                          np.cross(b, [0, 1.0, 0])]) * 300.0
        elif kind == 2:                                # depth 1e5: tiny point Jacobian
            J = rng.normal(size=(6, 3)) * 1e-4
        else:
            J = rng.normal(size=(6, 3)) * 300.0
        H[n] = _point_block(J)
        kinds[n] = kind
    bad_planted = [7, 33]
    H[7, 0] = np.nan
    H[33, 4] = np.nan
    sc = _sc_p(np.abs(H))
    sc[bad_planted] = 0.5
    for max_diag in (1e32, 0.3):
        o, _, _ = _schur_build(c, pconst, cuda_dev, blk_dev, sc, radius, H_pp=H, g_p=g, max_diag=max_diag)
        dpp, V = so.point_prep_ref(H, sc, radius, 1e-6, max_diag)
        assert np.array_equal(o["dpp"].view(np.uint64), dpp.view(np.uint64)), (radius, max_diag)
        if max_diag < 1:
            assert (o["dpp"] == max_diag).any()
        assert (dpp[[n for n in kinds if kinds[n] == 2]] == 1e-6).any()
        failed = np.nonzero(~o["M"].any(1))[0]
        assert set(bad_planted) <= set(failed.tolist())
        assert o["scal"][6] == len(failed), (o["scal"][6], failed)
        assert not o["q"][failed].any() and not o["M"][:, [3, 6, 7]].any()
        ok = np.setdiff1d(np.arange(N), failed)
        err, bar = so.point_prep_backward(o["M"][ok], V[ok], sc[ok])
        qref, qbar = so.q_bar(o["M"], g)
        unexpected = set(failed.tolist()) - set(bad_planted)
        print(f"point_prep radius {radius:g} max_diag {max_diag:g}: backward {_ratio(err, bar):.3g}, "
              f"q {_ratio(np.abs(o['q'] - qref), qbar):.3g} (err/bar); kappa max {np.linalg.cond(V[ok]).max():.3g}; "
              f"failed beyond the planted NaN: {sorted(unexpected)} (kinds {[kinds[n] for n in sorted(unexpected)]})")
        assert _ratio(err, bar) <= 1.0 and _ratio(np.abs(o["q"] - qref), qbar) <= 1.0
        if radius < 1e14:
            assert not unexpected, (radius, sorted(unexpected))
        else:
            assert all(kinds[n] == 0 for n in unexpected)


# ----------------------------------------------------------------------------------------------
# syrk_f64
# ----------------------------------------------------------------------------------------------

def _syrk(Z, C0, dev, ranges=None):
    from tests.test_syrk_f64_gpu import _syrk as run
    return run(Z, C0, dev, ranges)


def _syrk_bar(Z, C0, ref, dev):
    import torch
    Za = torch.from_numpy(np.abs(Z)).to(dev)
    nz = (Za != 0).to(torch.float64)
    scale = (Za.T @ Za).cpu().numpy()
    kprod = (nz.T @ nz).cpu().numpy()
    K = Z.shape[0]
    # one rounding per non-zero product, and one f64 RED per item (at most MAX_PARTS per tile) into C0
    return ((2.0 * kprod + 34) * U * scale + (so.MAX_PARTS + 1) * U * (np.abs(C0) + scale + np.abs(ref)) +
            2 * K * 2.0 ** -1074)


def _items(Kpad, Dpad, ranges, dev):
    import torch
    from tests.test_schur_oracle import _work_list
    sms = torch.cuda.get_device_properties(dev).multi_processor_count
    return _work_list(Kpad, Dpad, ranges, sms)


def _check_syrk(Z, C0, got, dev, label, ranges=None):
    ref = C0 - oz.exact_gram(Z, device=dev)
    Dpad = Z.shape[1]
    low = np.tril(np.ones((Dpad, Dpad), bool))
    bar = _syrk_bar(Z, C0, ref, dev)
    skipped = np.zeros((Dpad, Dpad), bool)
    if ranges is not None:
        want = so.tile_ranges(Z.shape[0], Dpad, ranges)
        nb = Dpad // 128
        for bj in range(nb):
            for bi in range(bj + 1):
                if (bi, bj) not in want:
                    skipped[bj * 128:bj * 128 + 128, bi * 128:bi * 128 + 128] = True
    r = _ratio(np.abs(got - ref)[low & ~skipped], bar[low & ~skipped])
    print(f"syrk {label}: max err/bar {r:.3g}")
    assert r <= 1.0, label
    assert np.array_equal(got[~low].view(np.uint64), C0[~low].view(np.uint64)), label
    assert np.array_equal(got[skipped].view(np.uint64), C0[skipped].view(np.uint64)), label


def _operand(Kpad, Dpad, seed, ranges=None):
    rng = np.random.default_rng(seed)
    Z = rng.normal(size=(Kpad, Dpad)) * np.exp(rng.uniform(-4, 4, size=(1, Dpad)))
    Z[rng.uniform(size=Z.shape) < 0.3] = 0.0
    if ranges is not None:
        for rb in range(Dpad // 128):
            Z[:ranges[2 * rb] * 64, rb * 128:rb * 128 + 128] = 0.0
            Z[ranges[2 * rb + 1] * 64:, rb * 128:rb * 128 + 128] = 0.0
    return Z


@pytest.mark.parametrize("Kpad,nb", [(1024, 1), (1040, 15), (1056, 16), (1072, 17), (1168, 23), (2112, 24),
                                     (16 * 37, 6), (48, 3)])
def test_syrk_shapes(cuda_dev, Kpad, nb):
    """Kpad = 0 / 16 / 32 / 48 mod 64 (items of 1 ... KB k blocks, not multiples of the 4-stage ring, so the ring's
    phase carries across items); nb = 1 ... 24 is 1 ... 300 upper tiles against the SM count"""
    Dpad = 128 * nb
    Z = _operand(Kpad, Dpad, Kpad + nb)
    C0 = np.random.default_rng(nb).normal(size=(Dpad, Dpad)) * 1e2
    items = _items(Kpad, Dpad, None, cuda_dev)
    assert not so.check_work_list(items, Kpad, Dpad)
    _check_syrk(Z, C0, _syrk(Z, C0, cuda_dev), cuda_dev, f"{Kpad}x{Dpad} ({len(items)} items)")


BAND_HINTS = [
    # (Kpad, ranges per row block): an empty row block, one-k-block ranges, ranges ending at the partial last block
    (1072, [0, 3, 0, 0, 5, 6, 6, 7, 16, 17, 2, 9, 9, 9, 0, 17, 15, 17, 0, 17]),
    # only the diagonal tiles survive
    (1072, sum(([b, b + 1] for b in range(10)), [])),
    # a one-block range in the partial last block (Kpad = 48 mod 64) next to dense ones
    (2096, [32, 33, 0, 33, 30, 33, 31, 32]),
]


@pytest.mark.parametrize("Kpad,ranges", BAND_HINTS)
def test_syrk_band_hints_with_c0(cuda_dev, Kpad, ranges):
    """band hints against a non-zero C0: computed tiles within the bar, skipped tiles and the upper triangle bitwise"""
    ranges = np.array(ranges, np.int32)
    Dpad = 64 * len(ranges)
    Z = _operand(Kpad, Dpad, Kpad, ranges)
    C0 = np.random.default_rng(3).normal(size=(Dpad, Dpad)) * 1e3
    assert not so.check_work_list(_items(Kpad, Dpad, ranges, cuda_dev), Kpad, Dpad, ranges)
    _check_syrk(Z, C0, _syrk(Z, C0, cuda_dev, ranges), cuda_dev, f"band {ranges.tolist()}", ranges)


def test_syrk_extreme_scales(cuda_dev):
    """columns scaled by 2^+300 and 2^-300, and columns whose products are subnormal (the bar adds K 2^-1074)"""
    Kpad, Dpad = 1040, 384
    Z = _operand(Kpad, Dpad, 5)
    Z[:, 0:128] *= 2.0 ** 300
    Z[:, 128:256] *= 2.0 ** -300
    Z[:, 256:320] *= 2.0 ** -530
    C0 = np.zeros((Dpad, Dpad))
    got = _syrk(Z, C0, cuda_dev)
    assert (np.abs(got[256:320, 256:320]) < 2.0 ** -1022).any() and (got[256:320, 256:320] != 0).any()
    _check_syrk(Z, C0, got, cuda_dev, "2^+-300, subnormal products")


@pytest.mark.parametrize("k,i,ranges", [(0, 0, None), (1039, 383, None), (700, 200, None),
                                        (330, 300, BAND_HINTS[0][1]), (1071, 1279, BAND_HINTS[0][1])])
def test_syrk_single_nan(cuda_dev, k, i, ranges):
    """one NaN in Zt: the NaN set of Cmat equals the prediction from the work list, nothing else is NaN"""
    Kpad, Dpad = (1040, 384) if ranges is None else (1072, 1280)
    r = None if ranges is None else np.array(ranges, np.int32)
    Z = _operand(Kpad, Dpad, k + i, r)
    if r is not None:
        assert r[2 * (i // 128)] <= k // 64 < r[2 * (i // 128) + 1]
    Z[k, i] = np.nan
    got = _syrk(Z, np.zeros((Dpad, Dpad)), cuda_dev, r)
    want = so.syrk_nan_set(_items(Kpad, Dpad, r, cuda_dev), Dpad, k, i)
    print(f"syrk NaN at ({k}, {i}): {int(np.isnan(got).sum())} NaN entries, predicted {int(want.sum())}")
    assert np.array_equal(np.isnan(got), want)
