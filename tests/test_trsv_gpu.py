"""The backward substitution of the LM loop (csrc/trsv.cu, U x = y through the launcher the solver calls) on its own.

U is L^T of a random SPD matrix whose rows and columns are scaled by 10^U(-3,3), the way Jacobi-scaled BA systems are.
It sits in the upper triangle of a row-major buffer with lda = the solver's padded order; the strictly lower triangle and
the padding columns hold NaN (the kernel may read only j >= i, j < n), and the right-hand sides are columns of the same
buffer read with stride lda, as in the LM loop, where y is the bordered column D of the factor.  Two right-hand sides go
through the same x buffer one after the other (the sentinel fill of the second call must not see the first result).

The residual is computed in extended precision and bounded by

    |y - U x|_inf <= 8 (n + max_b kappa_inf(U_bb)) 2^-53 (|U|_inf |x|_inf + |y|_inf),

U_bb being the 64 x 64 diagonal blocks the kernel inverts explicitly (the explicit inverse costs a factor of their
condition number over a substitution).  Orders: one partial block, exact multiples of 64, C3 (2402) and its bordered
order, and the largest order the one-wave kernel takes (7000, 110 blocks)."""
import numpy as np
import pytest

pytestmark = pytest.mark.gpu

ORDERS = [1, 5, 63, 64, 65, 128, 448, 2402, 2403, 4096, 6999, 7000]
U53 = 2.0 ** -53


def _scaled_upper(n, rng):
    G = rng.normal(size=(n, n)) * (0.25 / np.sqrt(n))
    A = G + G.T + np.eye(n)                          # eigenvalues within about [0.3, 1.7]
    s = 10.0 ** rng.uniform(-3.0, 3.0, size=n)
    return np.linalg.cholesky(A * s[:, None] * s[None, :]).T


def _residual(U, x, y):
    """y - U x in extended precision, a block of rows at a time"""
    r = np.empty(len(y), dtype=np.longdouble)
    xl = x.astype(np.longdouble)
    for i in range(0, len(y), 512):
        r[i:i + 512] = y[i:i + 512].astype(np.longdouble) - U[i:i + 512].astype(np.longdouble) @ xl
    return np.abs(r).max()


def _max_block_kappa(U):
    from scipy.linalg import solve_triangular
    n = U.shape[0]
    k = 0.0
    for r0 in range(0, n, 64):
        B = U[r0:r0 + 64, r0:r0 + 64]
        Bi = solve_triangular(B, np.eye(B.shape[0]))
        k = max(k, np.abs(B).sum(1).max() * np.abs(Bi).sum(1).max())
    return k


@pytest.mark.parametrize("n", ORDERS)
def test_trsv_matches_extended_precision_residual(cuda_dev, n):
    import torch
    from vggsfm_b200 import _lib
    rng = np.random.default_rng(1000 + n)
    U = _scaled_upper(n, rng)
    lda = (n + 2 + 127) // 128 * 128                 # the solver's Dpad: >= n + 2, so two right-hand-side columns fit
    buf = np.full((n, lda), np.nan)
    iu = np.triu_indices(n)
    buf[iu] = U[iu]
    ys = [rng.normal(size=n) * 10.0 ** rng.uniform(-2.0, 2.0, size=n) for _ in range(2)]
    buf[:, n] = ys[0]
    buf[:, n + 1] = ys[1]
    A = torch.from_numpy(buf).to(cuda_dev)
    x = torch.empty(n, dtype=torch.float64, device=cuda_dev)
    L = _lib.lib()
    kmax = _max_block_kappa(U)
    normU = np.abs(U).sum(1).max()
    for col, y in zip((n, n + 1), ys):
        torch.cuda.synchronize()
        _lib.check(L.vgg_dev_trsv_probe(n, lda, A.data_ptr(), A.data_ptr() + 8 * col, lda, x.data_ptr(), None),
                   "vgg_dev_trsv_probe")
        xh = x.cpu().numpy()
        assert np.isfinite(xh).all(), (n, col)
        res = _residual(U, xh, y)
        bound = 8.0 * (n + kmax) * U53 * (normU * np.abs(xh).max() + np.abs(y).max())
        print(f"trsv n={n} rhs column {col}: |y - Ux| = {float(res):.3e}  bound {bound:.3e}  ratio {float(res / bound):.3e}  "
              f"max kappa(U_bb) {kmax:.2e}")
        assert res <= bound, (n, col, float(res), bound)
