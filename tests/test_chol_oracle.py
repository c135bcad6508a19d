"""oracle/chol_oracle.py on the CPU: the generators plant what the Cholesky edge tests (test_chol_edges_gpu.py) claim
they plant, and the bars those tests apply pass a LAPACK factor and reject realistic ways a factor can be subtly
wrong."""
import numpy as np
import pytest

from oracle import chol_oracle as co


def _lapack_full(A):
    """LAPACK's factor laid out as the kernel leaves it: L below the diagonal, L^T above"""
    L = np.linalg.cholesky(A)
    return L + np.tril(L, -1).T


@pytest.mark.parametrize("n,p", [(300, 0), (300, 7), (300, 127), (2403, 1), (2403, 1033), (2403, 2402), (4500, 4097)])
def test_planted_negative_pivot_is_what_dpotrf_reports(n, p):
    A = co.spd(n, n)
    assert co.dpotrf_info(A) == 0
    A[p, p] = -1.0
    assert co.dpotrf_info(A) == p + 1


def test_two_planted_pivots_report_the_earlier():
    A = co.spd(700, 3)
    A[300, 300] = -1.0
    A[129, 129] = -5.0
    assert co.dpotrf_info(A) == 130


def test_graded_pairs_leave_the_two_pivot_range_on_both_sides():
    A = co.graded(384, 11)
    ac = co.pair_products(A)
    assert np.count_nonzero(ac < co.AC_LO) >= 10 and np.count_nonzero(ac > co.AC_HI) >= 10
    assert np.count_nonzero((ac >= co.AC_LO) & (ac <= co.AC_HI)) >= 10      # and the two-pivot path runs too
    assert np.isfinite(A).all() and np.abs(A).max() < 1e250
    ratio, bad = co.backward_error(A, np.linalg.cholesky(A))
    assert bad == 0 and ratio <= 1.0


def test_bordered_corner_takes_the_sequential_fallback():
    for D in (296, 297):
        A = co.bordered(D, D, pinned=(0, 5, 6, 128))
        ac = co.pair_products(A)
        assert ac[D // 2] > co.AC_HI
        assert np.all(A[5, :5] == 0) and A[5, 5] == 1.0 and A[D, 5] == 0.0


def test_ill_conditioned_generators():
    A = co.jacobi_ill(300, 1e12, 5)
    assert np.allclose(np.diag(A), 1.0) and 1e11 < np.linalg.cond(A) < 1e13
    B = co.dependent_pairs(300, 1e-6, 5)
    assert np.allclose(np.diag(B), 1.0) and np.linalg.cond(B) > 1e10
    S = np.linalg.cholesky(B)
    piv = np.diag(S)[1::2] ** 2                         # second pivot of each pair against its C
    C = piv + np.diag(S, -1)[0::2] ** 2
    assert np.median(C / piv) > 1e10


def test_block_diagonal_first_rows_have_known_pivots():
    A, firsts = co.block_diagonal(257, 2)
    assert firsts[0] == 0 and {0, 1} <= set(firsts % 2)
    L = np.linalg.cholesky(A)
    assert np.all(co.ulps(np.diag(L)[firsts], np.sqrt(np.diag(A)[firsts])) <= 1)


@pytest.mark.parametrize("n", [1, 2, 9, 64, 300, 2403])
def test_lapack_factor_passes_the_bars(n):
    for A in (co.spd(n, n), co.graded(n, n), co.diagonal(n, n)):
        full = _lapack_full(A)
        ratio, bad = co.backward_error(A, full)
        print(f"LAPACK n={n}: backward-error ratio {ratio:.3e}")
        assert bad == 0 and ratio <= 1.0
        assert co.mirror_ok(full)


@pytest.mark.parametrize("n", [1, 64, 300, 512])
def test_bar_rejects_a_diagonal_off_by_2_pow_minus_44(n):
    """what one Newton step fewer in the kernel's rsqrt would leave on every pivot"""
    for A in (co.spd(n, n), co.diagonal(n, n)):
        L = np.linalg.cholesky(A)
        L[np.diag_indices(n)] *= 1.0 + 2.0 ** -44
        ratio, bad = co.backward_error(A, L)
        print(f"n={n}: diagonal * (1 + 2^-44) -> ratio {ratio:.2f}")
        assert ratio > 1.0
    # ... and the known-diagonal bar sees it at any order
    d = np.sqrt(np.diag(co.diagonal(n, n)))
    assert np.all(co.ulps(d * (1.0 + 2.0 ** -44), d) > co.ULPS_SECOND)


@pytest.mark.parametrize("n", [300, 2403])
def test_bar_rejects_one_perturbed_tile(n):
    A = co.spd(n, 1)
    L = np.linalg.cholesky(A)
    L[64:128, 0:64] *= 1.0 + 1e-12
    ratio, bad = co.backward_error(A, L)
    print(f"n={n}: one 64 x 64 tile * (1 + 1e-12) -> ratio {ratio:.2f}")
    assert ratio > 1.0


def test_bar_rejects_a_swapped_mirror_entry():
    A = co.spd(200, 4)
    full = _lapack_full(A)
    full[3, 150] = full[150, 4]                     # the wrong mirror entry in the upper triangle
    assert not co.mirror_ok(full)
    assert co.backward_error(A, full)[1] == 0       # (bar 1 reads the lower triangle only)


def test_bar_rejects_a_non_zero_pinned_entry():
    D = 200
    A = co.bordered(D, 1, pinned=(40, 41))
    L = np.linalg.cholesky(np.tril(A) + np.tril(A, -1).T)
    ratio, bad = co.backward_error(A, L)
    assert ratio <= 1.0 and bad == 0
    assert np.all(L[40, :40] == 0) and np.all(L[41:, 40][1:] == 0)
    L[41, 40] = 1e-300                              # the smallest thing that is not zero, in a pinned column
    ratio, bad = co.backward_error(A, L)
    assert ratio > 1.0 or bad > 0


def test_bar_rejects_a_non_zero_outside_the_band():
    A, keep, end, arrow = co.band_arrow(6, 1, 5, 3)
    L = np.linalg.cholesky(A)
    assert np.all(L[~keep & np.tri(len(A), dtype=bool)] == 0)
    assert co.backward_error(A, L)[1] == 0
    L[400, 10] = 1e-300                             # outside the band, below the arrow
    ratio, bad = co.backward_error(A, L)
    assert ratio > 1.0 or bad > 0


def test_expected_nan_index():
    assert co.nan_info(9, 9) == 10 and co.nan_info(33, 2) == 34 and co.nan_info(127, 126) == 128
