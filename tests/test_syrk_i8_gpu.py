"""wgmma INT8 (Ozaki) SYRK (csrc/syrk_i8.cu, vgg_syrk_ozaki) checked two ways on every case:
  1. against the integer oracle (oracle/ozaki_oracle.py: the same digits, pair products and orders, exact), allowing
     only the float64 recombination: every work item's contribution is exact, so the kernel may differ by m roundings
     of at most 2^-53 of the entry's digit magnitude (m <= items per tile + orders).  Any wrong digit, slot, pair, order
     or k-block shows up here even where the normwise bound is loose;
  2. against Z^T Z computed exactly, under the normwise bound |err_ij| <= 2^-B (p_i ||Z_j||_1 / 2 + p_j ||Z_i||_1 / 2
     + c_s n_ij p_i p_j) (B = 8s-2, p = 2^e the column scale, n_ij rows where both columns are non-zero, c_s <= 6.02)
     plus the recombination term.  The error is NOT bounded relative to (|Z|^T |Z|)_ij (tests/test_ozaki_oracle.py).
Columns whose maximum is below 2^-900 are flushed to zero; a non-finite entry makes its row and column NaN.
Only entries whose true value is finite are compared.  Largest ratios observed on an H100 80GB HBM3 (700 W limit):
0.11 of the recombination term (check 1) and 0.14 of the normwise bound (check 2); each check prints its own.  The LM solve with VGG_SYRK=ozaki semantics is covered by
tests/test_ba_gpu.py."""
import ctypes

import numpy as np
import pytest

from oracle import ozaki_oracle as oz

pytestmark = pytest.mark.gpu


def _run(Z, s, dev):
    import torch
    from vggsfm_b200 import _lib
    L = _lib.lib()
    Kpad, Dpad = Z.shape
    Zt = torch.from_numpy(Z).to(dev)
    C = torch.zeros(Dpad, Dpad, dtype=torch.float64, device=dev)
    nb = ctypes.c_size_t()
    _lib.check(L.vgg_syrk_ozaki_workspace_bytes(Kpad, Dpad, s, ctypes.byref(nb)), "vgg_syrk_ozaki_workspace_bytes")
    ws = torch.empty(nb.value, dtype=torch.uint8, device=dev)
    with torch.cuda.device(dev):
        _lib.check(L.vgg_syrk_ozaki(Kpad, Dpad, Zt.data_ptr(), C.data_ptr(), s, ws.data_ptr(), ws.numel(),
                                    torch.cuda.current_stream().cuda_stream), "vgg_syrk_ozaki")
        torch.cuda.synchronize()
    full = C.cpu().numpy()
    del Zt, C, ws
    assert not np.triu(full, 1).any()                  # only the row-major LOWER triangle is written (csrc/chol.cu factors it)
    low = np.tril(full)
    return low + np.tril(low, -1).T


def _check(Z, got, s, dev, what):
    """got = -(Z^T Z) from the kernel; both checks of the module docstring on the entries with a finite true value."""
    got = -got
    ora = oz.syrk(Z, s, device=dev)
    rec = oz.recombination_bound(Z, s, device=dev)
    Zf = np.where(oz.flushed_columns(Z)[None, :], 0.0, Z)
    ref = oz.exact_gram(Zf, device=dev)
    fin = np.isfinite(ref) & np.isfinite(ora)
    e1 = np.abs(got - ora)[fin]
    r1 = (e1 / np.maximum(rec[fin], 1e-300)).max()
    bound = oz.normwise_bound(Z, s, device=dev) + rec + 2.0 ** -52 * np.abs(ref)
    e2 = np.abs(got - ref)[fin]
    r2 = (e2 / np.maximum(bound[fin], 1e-300)).max()
    print(f"syrk {what}: max err/recombination vs oracle = {r1:.3g}, max err/normwise bound = {r2:.3g}")
    assert np.all(e1 <= rec[fin]), (what, r1)
    assert np.all(e2 <= bound[fin]), (what, r2)
    fl = oz.flushed_columns(Z)
    assert not got[fl].any() and not got[:, fl].any()                 # flushed columns give exact zeros


def _case(Dpad, Kpad, seed):
    rng = np.random.default_rng(seed)
    Z = rng.normal(size=(Kpad, Dpad)) * np.exp(rng.uniform(-6, 6, size=(1, Dpad)))
    Z[rng.uniform(size=Z.shape) < 0.3] = 0.0
    Z[:, -5:] = 0.0
    return Z


def _varying(Dpad, Kpad, seed):
    """Rows scaled by 2^u, u in [-36, 36], and one large entry per column: the magnitudes vary along k."""
    rng = np.random.default_rng(seed)
    Z = rng.normal(size=(Kpad, Dpad)) * np.ldexp(1.0, rng.integers(-36, 37, size=(Kpad, 1)))
    Z[rng.integers(0, Kpad, size=Dpad), np.arange(Dpad)] = 2.0 ** 40
    return Z


@pytest.mark.parametrize("Dpad,Kpad,s,tol", [(128, 64, 7, 2.0 ** -44), (384, 1040, 7, 2.0 ** -44), (256, 640, 5, 2.0 ** -28),
                                             (256, 4096 + 16, 6, 2.0 ** -36), (640, 2000, 3, 2.0 ** -12), (256, 700, 4, 2.0 ** -20)])
def test_matches_float64(cuda_dev, Dpad, Kpad, s, tol):
    """Operands whose columns have a uniform magnitude along k.  For these the error also stays within
    tol (|Z|^T |Z|)_ij, tol = 2^-(8s-12), which is asserted as well; test_k_varying_magnitudes covers the
    operands where that componentwise form does not hold."""
    Z = _case(Dpad, Kpad, Dpad + s)
    got = _run(Z, s, cuda_dev)
    _check(Z, got, s, cuda_dev, f"uniform {Dpad}x{Kpad} s={s}")
    err = np.abs(-got - Z.T @ Z)
    bound = np.abs(Z).T @ np.abs(Z)
    assert np.all(err <= tol * bound + 1e-300), (err / (bound + 1e-300)).max()
    assert not got[:, -5:].any()


@pytest.mark.parametrize("Dpad,Kpad,s", [(384, 900, 7), (256, 1000, 3)])
def test_k_varying_magnitudes(cuda_dev, Dpad, Kpad, s):
    Z = _varying(Dpad, Kpad, Dpad + s)
    _check(Z, _run(Z, s, cuda_dev), s, cuda_dev, f"k-varying {Dpad}x{Kpad} s={s}")


def test_c3_reduced_order(cuda_dev):
    """C3: Dpad 2432 (19 row blocks, 190 tiles), K 12288."""
    Z = _case(2432, 12288, 3)
    _check(Z, _run(Z, 7, cuda_dev), 7, cuda_dev, "C3 2432x12288")


def test_int32_headroom_needs_the_forced_k_split(cuda_dev):
    """Dpad 2432, K = 3 x 16384, digits chosen so every pair product is positive and near 128^2
    (oz.worst_case_digits): load balancing alone leaves items of 384-768 k-blocks, and the top kept order wraps in
    int32 beyond about 340 k-blocks.  Only the forced split at 256 k-blocks (OZ_MAX_ITEM_KB) keeps it exact; with the
    limit at 512 this test fails."""
    Z = oz.worst_case_digits(3 * oz.ITEM_K_ROWS, 2432, 7, 1)
    _check(Z, _run(Z, 7, cuda_dev), 7, cuda_dev, "headroom 2432x49152")


def test_extreme_exponents(cuda_dev):
    """Columns at 2^+-500, one near 2^1000 paired with columns near 2^-800 (the ldexp branch of the epilogue), columns
    just above and below the 2^-900 flush, subnormal entries in a normal column."""
    rng = np.random.default_rng(5)
    Z = rng.normal(size=(600, 256))
    Z[rng.uniform(size=Z.shape) < 0.2] = 0.0
    Z[:, 0:10] *= 2.0 ** 500
    Z[:, 10:20] *= 2.0 ** -500
    Z[:, 20] *= 2.0 ** 1000 / np.abs(Z[:, 20]).max() * 0.9
    Z[:, 21:30] *= 2.0 ** -800
    Z[:, 30:34] *= 2.0 ** -905 / np.abs(Z[:, 30:34]).max(axis=0)
    Z[:, 34] *= 2.0 ** -899.5 / np.abs(Z[:, 34]).max()
    Z[::3, 35] = 5e-310
    Z[:, 200:] *= 2.0 ** 400
    assert oz.flushed_columns(Z)[30:34].all() and not oz.flushed_columns(Z)[34]
    got = _run(Z, 7, cuda_dev)
    _check(Z, got, 7, cuda_dev, "extreme exponents")
    assert np.isfinite(-got[20, 21:30]).all() and np.abs(got[20, 21:30]).max() > 0


def test_accumulates_and_flags_nonfinite(cuda_dev):
    Z = _case(256, 256, 1)
    got1 = _run(Z, 7, cuda_dev)
    assert np.abs(got1).max() > 0
    Z[17, 40] = np.nan
    Z[3, 41] = np.inf
    Z[200, 42] = -np.inf
    got = _run(Z, 7, cuda_dev)
    for c in (40, 41, 42):
        assert np.isnan(got[c, :250]).all() and np.isnan(got[:250, c]).all()
    ok = np.ones(256, bool)
    ok[40:43] = False
    assert np.isfinite(got[np.ix_(ok, ok)]).all()
    Zc = Z.copy()
    Zc[:, 40:43] = 0.0
    _check(Zc[:, ok], got[np.ix_(ok, ok)], 7, cuda_dev, "finite part")


def _banded(Dpad, KB, seed):
    """a sequential problem's operand: row block rb is non-zero in k blocks [2 rb, 2 rb + 7) only, the last (the shared
    camera's column) everywhere"""
    Z = _case(Dpad, KB * 64, seed)
    nb = Dpad // 128
    for rb in range(nb - 1):
        lo, hi = 2 * rb, min(KB, 2 * rb + 7)
        Z[:lo * 64, rb * 128:(rb + 1) * 128] = 0.0
        Z[hi * 64:, rb * 128:(rb + 1) * 128] = 0.0
    return Z


def test_plan_cache_alternating_shapes_and_slice_counts(cuda_dev):
    """The host plan is cached per (Kpad, Dpad, s): alternating them in one process must re-plan every time the key
    changes and reuse nothing stale."""
    cases = {"a": (_case(256, 640, 21), 7), "b": (_case(384, 1040, 22), 5), "c": (_case(256, 700, 23), 4),
             "band": (_banded(1024, 24, 12), 7)}
    for key in ["a", "b", "band", "a", "band", "c", "band", "b", "c"]:
        Z, s = cases[key]
        _check(Z, _run(Z, s, cuda_dev), s, cuda_dev, f"plan cache {key}")
