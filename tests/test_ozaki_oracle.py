"""CPU checks of the integer formulation behind the tensor-core SYRK (oracle/ozaki_oracle.py restates
csrc/syrk_i8.cu's arithmetic): digit identity, int32 exactness per work item, the flush of columns below 2^-900, and
the error bound against an exactly computed Z^T Z.

The bound is NORMWISE: with s slices, B = 8s-2, p_i = 2^e_i the column scale and n_ij the rows where both columns are
non-zero, |err_ij| <= 2^-B (p_i ||Z_j||_1 / 2 + p_j ||Z_i||_1 / 2 + c_s n_ij p_i p_j), c_s <= 6.02.  An entry's error is
NOT bounded relative to (|Z|^T |Z|)_ij: the two-spike operand below breaks any such bound."""
from fractions import Fraction

import numpy as np
import pytest

from oracle import ozaki_oracle as oz


def _Z(K, n, seed):
    rng = np.random.default_rng(seed)
    Z = rng.normal(size=(K, n)) * np.exp(rng.uniform(-8, 8, size=(1, n)))
    Z[rng.uniform(size=Z.shape) < 0.3] = 0.0
    Z[:, -2:] = 0.0
    return Z


def _rows_span(K, n, seed):
    """Rows scaled by 2^u, u uniform in [-36, 36]: inside one column the magnitudes vary along k."""
    rng = np.random.default_rng(seed)
    return rng.normal(size=(K, n)) * np.ldexp(1.0, rng.integers(-36, 37, size=(K, 1)))


OPERANDS = {
    "uniform": lambda s: _Z(1500, 40, 10 + s),
    "rows_span_2^36": lambda s: _rows_span(1200, 24, s),
    "two_spike": lambda s: oz.two_spike(2000, seed=s),
}


@pytest.mark.parametrize("s", [3, 5, 7])
def test_balanced_digits_reconstruct_the_rounded_value(s):
    Z = _Z(200, 17, s)
    Z[0, 0] = np.abs(Z[:, 0]).max() * (1 - 2.0 ** -52)        # an entry just below the column scale
    D, e, X = oz.slices(Z, s)
    assert D.dtype == np.int8 and np.abs(D[0].astype(int)).max() <= 65          # top digit has the headroom
    rec = sum(D[p].astype(np.int64) * (256 ** (s - 1 - p)) for p in range(s))
    assert np.array_equal(rec, X)                                                 # digits are exact
    B = 8 * s - 2
    back = np.ldexp(X.astype(np.float64), (e - B)[None, :])
    scale = np.ldexp(1.0, e)[None, :]
    assert np.all(np.abs(back - Z) <= 2.0 ** -(B + 1) * scale + 1e-300)           # rounding to B fractional bits


def test_exact_gram_is_exact():
    """The reference the bounds are checked against: Z^T Z of float64 entries over several binades, against rational
    arithmetic (it may differ only by the final rounding of each entry, and of the sum of its slice products)."""
    Z = _rows_span(60, 5, 1)
    ref = oz.exact_gram(Z)
    F = [[Fraction(float(v)) for v in row] for row in Z]
    for i in range(5):
        for j in range(5):
            exact = sum(F[k][i] * F[k][j] for k in range(60))
            assert abs(Fraction(float(ref[i, j])) - exact) <= 2 * 2.0 ** -52 * abs(exact) + Fraction(1, 2 ** 200)


def test_pair_products_are_exact_float64_gemms():
    """order_products computes the C_t as float64 GEMMs of int8 values; they equal the int64 products."""
    Z = _Z(300, 12, 4)
    s = 6
    D, _, _ = oz.slices(Z, s)
    C, _ = oz.order_products(Z, s)
    for t in range(2, s + 2):
        ref = sum(D[p - 1].astype(np.int64).T @ D[t - p - 1].astype(np.int64) for p in range(1, s + 1) if 1 <= t - p <= s)
        assert np.array_equal(C[t], ref.astype(np.float64))


@pytest.mark.parametrize("s,tol", [(7, 2.0 ** -44), (6, 2.0 ** -36), (5, 2.0 ** -28), (3, 2.0 ** -12)])
def test_syrk_error_bound(s, tol):
    """Columns of uniform magnitude along k: within the normwise bound, and for such operands also within
    tol (|Z|^T |Z|)_ij, tol = 2^-(8s-12) -- asserted too.  test_syrk_normwise_error_bound covers operands where
    that componentwise form fails."""
    Z = _Z(1500, 40, 10 + s)
    got = oz.syrk(Z, s)
    ref = oz.exact_gram(Z)
    err = np.abs(got - ref)
    assert np.all(err <= oz.normwise_bound(Z, s) + 2.0 ** -52 * np.abs(ref))
    bound = np.abs(Z).T @ np.abs(Z)
    assert np.all(np.abs(got - Z.T @ Z) <= tol * bound + 1e-300), (np.abs(got - Z.T @ Z) / (bound + 1e-300)).max()
    assert np.array_equal(got, got.T)


@pytest.mark.parametrize("kind", sorted(OPERANDS))
@pytest.mark.parametrize("s", [3, 5, 7])
def test_syrk_normwise_error_bound(s, kind):
    Z = OPERANDS[kind](s)
    got = oz.syrk(Z, s)
    ref = oz.exact_gram(Z)
    bound = oz.normwise_bound(Z, s)
    err = np.abs(got - ref)
    assert np.all(err <= bound + 2.0 ** -52 * np.abs(ref)), (err / (bound + 1e-300)).max()
    assert np.array_equal(got, got.T)


def test_two_spike_operand_breaks_the_componentwise_bound():
    """The two-spike operand is adversarial: at s = 7 the error of entry (3, 4) is orders of magnitude above
    2^-44 (|Z|^T |Z|)_34, while it stays tiny relative to sqrt(S_33 S_44) -- the accuracy a Cholesky needs."""
    Z = oz.two_spike(2000, seed=0)
    got = oz.syrk(Z, 7)
    ref = oz.exact_gram(Z)
    err = abs(got[3, 4] - ref[3, 4])
    comp = (np.abs(Z).T @ np.abs(Z))[3, 4]
    assert err > 1e6 * 2.0 ** -44 * comp
    assert err <= 2.0 ** -44 * np.sqrt(ref[3, 3] * ref[4, 4])
    assert err <= oz.normwise_bound(Z, 7)[3, 4]


def test_dropped_orders_are_below_the_rounding():
    """Keeping orders beyond s+1 changes the result by at most the dropped-order term c_s 2^-B n_ij p_i p_j, the same
    size as the slicing's own rounding term."""
    s = 6
    Z = _Z(800, 24, 3)
    a = oz.syrk(Z, s)
    b = oz.syrk(Z, s, max_order=2 * s)
    p = np.ldexp(1.0, oz.column_exponents(Z))
    nz = (Z != 0).astype(np.float64)
    term = oz.dropped_order_coefficient(s) * 2.0 ** -(8 * s - 2) * (nz.T @ nz) * p[:, None] * p[None, :]
    assert np.all(np.abs(a - b) <= term + 2.0 ** -52 * np.abs(b) + 1e-300)
    assert oz.dropped_order_coefficient(7) < 6.02


def test_int32_headroom_per_work_item():
    """|d| <= 128, at most 7 pairs per order: a work item of 256 k-blocks x 64 (csrc/syrk_i8.cu OZ_MAX_ITEM_KB) keeps
    every int32 accumulator exact even if all digits sit at -128; longer reductions are split into several items.
    The worst-case operand needs that split: over 2 x 16384 rows its top kept order leaves the int32 range."""
    assert 7 * 128 * 128 * oz.ITEM_K_ROWS < 2 ** 31
    s = 7
    Z = oz.worst_case_digits(2 * oz.ITEM_K_ROWS, 4, s, 0)
    D, _, X = oz.slices(Z, s)
    assert np.all(D[0] == -63) and np.all(D[1:] <= -127)                          # the digits are the chosen ones
    C, _ = oz.order_products(Z, s)                                                # per-item check passes
    assert np.abs(C[s + 1]).max() >= 2 ** 31                                      # one item over all of K would wrap
    assert np.abs(C[s + 1]).max() < 2 ** 32
    ref = oz.exact_gram(Z)
    assert np.all(np.abs(oz.syrk(Z, s) - ref) <= oz.normwise_bound(Z, s) + 2.0 ** -52 * np.abs(ref))


def test_columns_below_2_pow_minus_900_are_flushed():
    Z = _Z(100, 6, 2)
    Z[:, 0] *= 2.0 ** -905 / np.abs(Z[:, 0]).max()        # max exactly 2^-905: flushed
    Z[:, 1] *= 2.0 ** -899.5 / np.abs(Z[:, 1]).max()      # ilogb = -900 -> e = -899: kept
    assert list(oz.flushed_columns(Z)) == [True, False, False, False, False, False]
    D, e, _ = oz.slices(Z, 7)
    assert not D[:, :, 0].any() and e[0] == 0 and e[1] == -899
    got = oz.syrk(Z, 7)
    assert not got[0].any() and not got[:, 0].any()
    ref = oz.exact_gram(Z)
    keep = np.ix_(range(1, 6), range(1, 6))
    assert np.all(np.abs(got - ref)[keep] <= oz.normwise_bound(Z, 7)[keep] + 2.0 ** -52 * np.abs(ref)[keep])
