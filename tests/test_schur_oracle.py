"""The bars of oracle/schur_oracle.py (cpu): each accepts an independent float64 / LAPACK / extended-precision
computation of its quantity and rejects a planted error; the written-set map equals a walk over z_build's loops; the
SYRK work lists the library builds (vgg_dev_syrk_work_list, host only) keep the cover contract for any CTA count and
their NaN prediction equals a float64 replay of the items."""
import ctypes

import numpy as np
import pytest

from oracle import ba_oracle as bo
from oracle import band_oracle as bd
from oracle import schur_oracle as so
from tests.helpers import ba_case, banded_mask


def _case(S, N, cam, mode, seed):
    c = ba_case(S, N, cam, mode, seed=seed)
    c["uv"] = c["uv"].astype(np.float32).astype(np.float64)
    m = c["mask"].copy()
    m[1, 3:] = False                              # frame 1 sees three points only
    c["mask"] = m
    return c


def _packed_H(blk, dc):
    iu = np.triu_indices(dc)
    return blk["H_cc"][:, iu[0], iu[1]]


@pytest.mark.parametrize("cam,mode", [("SIMPLE_PINHOLE", bo.INTR_CONST), ("SIMPLE_RADIAL", bo.INTR_PER_FRAME),
                                      ("SIMPLE_RADIAL", bo.INTR_SHARED)])
def test_blocks_bar_accepts_float64_and_rejects_lightly_observed_frame(cam, mode):
    c = _case(20, 150, cam, mode, seed=3)
    dc, ns = bo.dims(c["model"], mode)
    ref = so.blocks_ref(c)
    blk = bo.build_blocks(c["poses"], c["intr"], c["points"], c["uv"], c["mask"], c["model"], mode)
    parts = [blk["g_c"], _packed_H(blk, dc)] + ([blk["H_cs"].reshape(20, 6 * ns)] if ns else [])
    got = {"cost": [blk["cost"]], "camrec": np.concatenate(parts, 1), "g_p": blk["g_p"],
           "H_pp": blk["H_pp"][:, [0, 0, 0, 1, 1, 2], [0, 1, 2, 1, 2, 2]], "shared": np.zeros(5)}
    if ns:
        got["shared"][:ns] = blk["g_s"]
        got["shared"][2:2 + (3 if ns > 1 else 1)] = [blk["H_ss"][0, 0], blk["H_ss"][0, 1], blk["H_ss"][1, 1]][:3 if ns > 1 else 1]
    ratios = so.check_blocks(got, ref)
    print(cam, mode, ratios)
    assert max(ratios.values()) <= 1.0, ratios
    bad = dict(got, camrec=got["camrec"].copy())
    bad["camrec"][1, dc + 1] *= 1.0 + 1e-9           # H_cc[0, 1] of the frame that sees three points
    assert so.check_blocks(bad, ref)["camrec"] > 1.0


def _lapack_point_prep(H_pp, g_p, sc_p, radius, min_diag=1e-6, max_diag=1e32):
    dpp, V = so.point_prep_ref(H_pp, sc_p, radius, min_diag, max_diag)
    L = np.linalg.cholesky(V)
    M = sc_p[:, :, None] * np.transpose(np.linalg.inv(L), (0, 2, 1))
    q = np.einsum("nji,nj->ni", M, g_p)
    return dpp, V, M.reshape(-1, 9), q


def test_point_prep_bars():
    c = _case(12, 90, "SIMPLE_RADIAL", bo.INTR_CONST, seed=5)
    blk = bo.build_blocks(c["poses"], c["intr"], c["points"], c["uv"], c["mask"], c["model"], c["mode"])
    H = blk["H_pp"][:, [0, 0, 0, 1, 1, 2], [0, 1, 2, 1, 2, 2]]
    sc = 1.0 / (1.0 + np.sqrt(H[:, [0, 3, 5]]))
    for radius in (1e-4, 1.0, 1e4):
        dpp, V, M, q = _lapack_point_prep(H, blk["g_p"], sc, radius)
        dref, _ = so.point_prep_ref(H, sc, radius, 1e-6, 1e32)
        assert np.array_equal(dpp.view(np.uint64), dref.view(np.uint64))
        err, bar = so.point_prep_backward(M, V, sc)
        assert (err <= bar).all(), (radius, (err / bar).max())
        qref, qbar = so.q_bar(M, blk["g_p"])
        assert (np.abs(q - qref) <= qbar).all()
        # planted: one M entry off by 1e-10 relative, q off by 2^-40 relative
        n = int(np.argmin(bar))
        Mb = M.copy()
        Mb[n, 4] *= 1.0 + 1e-10
        err_b, _ = so.point_prep_backward(Mb, V, sc)
        assert err_b[n] > bar[n], (radius, err_b[n], bar[n])
        qb = qref.copy()
        qb[n, 2] *= 1.0 + 2.0 ** -40
        assert (np.abs(qb - qref) > qbar).any()
    # the clip of dpp is bitwise: the next float above max_diag is not max_diag
    d2, _ = so.point_prep_ref(H, sc, 1.0, 1e-6, 1e-3)
    assert (d2 == 1e-3).any() and not np.array_equal(d2, np.nextafter(d2, 1.0))


@pytest.mark.parametrize("cam,mode", [("SIMPLE_PINHOLE", bo.INTR_PER_FRAME), ("SIMPLE_RADIAL", bo.INTR_SHARED)])
def test_zt_bar_accepts_float64_and_rejects_planted_errors(cam, mode):
    S, N = 40, 61
    c = _case(S, N, cam, mode, seed=7)
    m = c["mask"].copy()
    m[32:, 8:16] = False                          # a whole (group, 8-track tile) region
    c["mask"] = m
    dc, ns = bo.dims(c["model"], mode)
    D = S * dc + ns
    Dpad, Kpad = (D + 2 + 127) // 128 * 128, (3 * N + 15) // 16 * 16
    blk = bo.build_blocks(c["poses"], c["intr"], c["points"], c["uv"], c["mask"], c["model"], mode)
    H = blk["H_pp"][:, [0, 0, 0, 1, 1, 2], [0, 1, 2, 1, 2, 2]]
    sc = 1.0 / (1.0 + np.sqrt(H[:, [0, 3, 5]]))
    _, _, M, q = _lapack_point_prep(H, blk["g_p"], sc, 37.0)
    g = np.concatenate([blk["g_c"].reshape(-1), blk["g_s"] if ns else []])
    Z, bar, _, rhs, rbar = so.zt_ref(c, M, q, g, Kpad, Dpad)
    # independent route: the float64 coupling blocks of ba_oracle times M
    W = blk["W"]                                              # [S,dc,N,3]
    Zi = np.zeros((Kpad, Dpad))
    Zi[:3 * N, :S * dc] = np.einsum("sinj,njc->ncsi", W, M.reshape(N, 3, 3)).reshape(3 * N, S * dc)
    if ns:
        Zi[:3 * N, S * dc:D] = np.einsum("inj,njc->nci", blk["W_s"], M.reshape(N, 3, 3)).reshape(3 * N, ns)
    assert (np.abs(Zi - Z) <= bar).all(), (np.abs(Zi - Z) / np.maximum(bar, 1e-300)).max()
    rhs_i = -g + Zi[:3 * N, :D].T @ q.reshape(-1)
    assert (np.abs(rhs_i - rhs) <= rbar).all()
    k, i = np.unravel_index(np.argmax(np.abs(Zi[:, :S * dc])), (Kpad, S * dc))
    Zb = Zi.copy()
    Zb[k, i] *= 1.0 + 2.0 ** -40
    assert not (np.abs(Zb - Z) <= bar).all()
    # the written set: a simulated kernel output over the NaN sentinel passes; writing zeros into a region no
    # observation reaches, or leaving a reached region unwritten, fails
    wr = so.written_set(c["mask"], dc, ns, Kpad, Dpad)
    sim = np.full((Kpad, Dpad), np.uint64(0xFFFFFFFFFFFFFFFF)).view(np.float64)
    sim[wr] = Zi[wr]
    assert so.check_sentinel(sim, wr) == (0, 0)
    assert not wr[3 * 8:3 * 16, 32 * dc:S * dc].any() and wr[3 * 8:3 * 16, :32 * dc].all()
    zeros = sim.copy()
    zeros[3 * 8:3 * 16, 32 * dc:S * dc] = 0.0
    assert so.check_sentinel(zeros, wr)[1] > 0
    skip = sim.copy()
    skip[3 * 20:3 * 21, 32 * dc:S * dc] = np.nan
    assert so.check_sentinel(skip, wr)[0] > 0


@pytest.mark.parametrize("S,N,banded", [(33, 97, False), (70, 203, False), (160, 1003, True), (129, 400, True)])
def test_written_set_equals_brute_force(S, N, banded):
    rng = np.random.default_rng(S + N)
    m = banded_mask(S, N, life=24, seed=S) if banded else rng.uniform(size=(S, N)) < 0.3
    m[:, N - 1] = False
    for dc, ns in ((6, 0), (7, 0), (6, 2)):
        D = S * dc + ns
        Dpad, Kpad = (D + 2 + 127) // 128 * 128, (3 * N + 15) // 16 * 16
        fg = bd.band_tables(m, dc, ns)["fg_tracks"] if banded else None
        a = so.written_set(m, dc, ns, Kpad, Dpad, fg)
        assert np.array_equal(a, so.written_set_brute(m, dc, ns, Kpad, Dpad, fg)), (dc, ns)
        assert not a[3 * N:].any() and not a[:, D:].any()
        if banded:
            # a correct band table changes nothing
            assert np.array_equal(a, so.written_set(m, dc, ns, Kpad, Dpad))


def _work_list(Kpad, Dpad, ranges, nworkers):
    from vggsfm_b200 import _lib
    L = _lib.lib()
    r = None if ranges is None else np.ascontiguousarray(ranges, np.int32)
    n = ctypes.c_int()
    args = (Kpad, Dpad, None if r is None else r.ctypes.data, 0 if r is None else r.size, nworkers)
    _lib.check(L.vgg_dev_syrk_work_list(*args, None, 0, ctypes.byref(n)), "vgg_dev_syrk_work_list")
    items = np.zeros((n.value, 4), np.int32)
    _lib.check(L.vgg_dev_syrk_work_list(*args, items.ctypes.data, n.value, ctypes.byref(n)), "vgg_dev_syrk_work_list")
    return items


def _shapes():
    """(label, Kpad, Dpad, ranges): Kpad = 0, 16, 32, 48 mod 64, nb = 1 ... 24, C3, C5 (banded) and band hints with an
    empty row block, one-k-block ranges, a range ending at the partial last block and only diagonal tiles left"""
    out = [(f"dense {k}x{d}", k, d, None) for k, d in ((64, 128), (16, 128), (1040, 1920), (2080, 2048), (3120, 2176),
                                                       (4144, 2944), (12288, 2432), (12304, 3072))]
    m = banded_mask(1000, 32768, life=40, seed=3)
    t = bd.band_tables(m, 6, 2)
    out.append(("C5 1000x32768 banded", (3 * 32768 + 15) // 16 * 16, t["Dpad"], t["rb_range"].reshape(-1)))
    Kpad, Dpad = 1072, 1280                                  # KB = 17, last block of 48 rows
    out.append(("empty row block, one-block ranges", Kpad, Dpad,
                np.array([0, 3, 0, 0, 5, 6, 6, 7, 16, 17, 2, 9, 9, 9, 0, 17, 15, 17, 0, 1], np.int32)))
    out.append(("diagonal tiles only", Kpad, Dpad, np.array(sum(([b, b + 1] for b in range(10)), []), np.int32)))
    return out


@pytest.mark.parametrize("label,Kpad,Dpad,ranges", _shapes(), ids=lambda v: v if isinstance(v, str) else "")
def test_syrk_work_list_cover_contract(label, Kpad, Dpad, ranges):
    for nw in (1, 7, 114, 132, 264):
        items = _work_list(Kpad, Dpad, ranges, nw)
        bad = so.check_work_list(items, Kpad, Dpad, ranges)
        assert not bad, (label, nw, bad[:5])
        if ranges is not None:
            # every band hint here leaves tiles out, so the list is checked against a clipped cover, not the dense one
            nb = Dpad // 128
            assert len(so.tile_ranges(Kpad, Dpad, ranges)) < nb * (nb + 1) // 2, label


def test_work_list_check_rejects_planted_errors():
    Kpad, Dpad = 2080, 1280
    items = _work_list(Kpad, Dpad, None, 132)
    assert not so.check_work_list(items, Kpad, Dpad)
    dropped = items.copy()
    dropped[:, 3] -= 1                                 # the last k block of every item
    assert so.check_work_list(dropped, Kpad, Dpad)
    dup = np.concatenate([items, items[-1:]])
    assert so.check_work_list(dup, Kpad, Dpad)
    assert not so.check_work_list([[0, 0, 1, 3], [0, 0, 0, 1]], 192, 128)
    assert any("longer" in b for b in so.check_work_list([[0, 0, 0, 1], [0, 0, 1, 3]], 192, 128))
    multi = np.array([[0, 0, k, k + 1] for k in range(33)], np.int32)
    assert not so.check_work_list(multi[:16], 1024, 128)
    assert any("items" in b for b in so.check_work_list(multi, 2112, 128))


@pytest.mark.parametrize("k,i", [(0, 0), (63, 130), (64, 255), (1000, 300), (1071, 1279)])
def test_syrk_nan_set_equals_replay(k, i):
    """a float64 replay of the work list (each item's partial product added into Cmat's lower triangle) puts NaN exactly
    where syrk_nan_set says"""
    Kpad, Dpad = 1072, 1280
    ranges = np.array([0, 3, 0, 0, 5, 6, 6, 7, 16, 17, 2, 9, 9, 9, 0, 17, 15, 17, 0, 17], np.int32)
    items = _work_list(Kpad, Dpad, ranges, 132)
    rng = np.random.default_rng(k + i)
    Z = rng.normal(size=(Kpad, Dpad))
    Z[k, i] = np.nan
    C = np.zeros((Dpad, Dpad))
    for bi, bj, k0, k1 in items.tolist():
        a = Z[k0 * 64:k1 * 64, bi * 128:bi * 128 + 128]
        b = Z[k0 * 64:k1 * 64, bj * 128:bj * 128 + 128]
        blk = -(a.T @ b).T                           # row index: column block bj, column index: row block bi
        if bi == bj:
            blk = np.tril(blk)
        C[bj * 128:bj * 128 + 128, bi * 128:bi * 128 + 128] += blk
    assert np.array_equal(np.isnan(C), so.syrk_nan_set(items, Dpad, k, i))
