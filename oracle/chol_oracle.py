"""TEST INFRASTRUCTURE ONLY (never imported by the product path).

What the reduced-system Cholesky (vggsfm_b200/csrc/chol.cu) is checked against: matrix generators that plant what a
case needs (failing pivots, graded scales, nearly dependent pivot pairs, the bordered BA matrix, band + arrow
structure), the componentwise backward-error bar, the expected `info` of a failing matrix, a float64 replay of the
kernel's two-pivot sequence, and a runner that calls the exported factorisation on a device buffer.

Backward-error bar.  For the computed factor L of A (order n), every entry of the lower triangle must satisfy

    |A - L L^T|_ij <= c_n u (|L| |L^T|)_ij,    u = 2^-53,    c_n = n + ceil(n / 8) + 32,

i.e. c (n + 1) u with c = c_n / (n + 1) <= 4 for n >= 9 (-> 1.13 for large n).  c_n counts the kernel's roundings:
  * the update of entry (i, j) before its pivot, a_ij - sum_{k<j} L_ik L_jk, runs in chunks: 8-column FMA chains in the
    8 x 8 leaves, rank-32 DMMA accumulators inside the diagonal block, 128-column DMMA accumulators (fused update, tile
    update) between panels.  A term passes at most its chunk's length (<= j) plus one rounding per chunk subtracted
    after it (chunks have >= 8 columns): <= j + ceil(j/8) + 1; the pre-scaled leaf rows (x *= dinv first, then FMAs
    with Lh = L dinv, each Lh rounded once) add 2.  Together <= n + ceil(n/8) + 2 (gamma_d to first order).
  * the pivot: 1/sqrt(p) is the hardware seed + two Newton steps, each step leaving 2.5 u (t = hp r, the FMA, r f);
    L_jj = p r adds u, so L_jj dinv_j = 1 + 6 u (first pivot of a pair).  The second pivot of the two-pivot step uses
    ib = (A ia) rsqrt(det) and L_11 = (det rsqrt(det)) ia, so L_11 ib = 1 + 14 u; its square carries det's rounding,
    eps C / (C - B^2/A) relative to the pivot, which is eps C absolutely, C <= (|L||L^T|)_jj -- the same bound as the
    sequential C - l10^2.  Off the diagonal L_ij = s dinv_j adds u: <= 15 u of |L_ij L_jj|; on the diagonal <= 23 u.
  * 25 u -> 32 u of slack.
Where the bound is 0 (structural zeros of band and arrow, pinned rows) the residual must be exactly 0.  The residual is
evaluated in np.longdouble up to n = 512 and in float64 above, and its own evaluation error gamma_{n+1}(|A| + |L||L^T|)
in that precision is added to the bound.

Known diagonals.  For a pivot with nothing above it in its row (diagonal matrices, the first row of a diagonal block)
L_jj = p r with r = 1/sqrt(p) (1 + 2.5 u): < 3.5 u from sqrt(p), plus half an ulp for rounding np.sqrt -> <= 4 ulps
for the first pivot of a pair; the second is L_11 = (det rsqrt(det)) ia with det = A C (1 + u): < 8.5 u -> <= 9 ulps.
A one-Newton-step rsqrt leaves 2^-44 relative, 2^9 ulps, and fails both.
"""
from __future__ import annotations

import math

import numpy as np

U = 2.0 ** -53
LONG_MAX_N = 512                     # residuals in np.longdouble up to this order, float64 above
PMIN = 2.2250738585072014e-308       # the kernel's smallest acceptable pivot (smallest normal double)
AC_LO, AC_HI = 1e-280, 1e280         # outside this range the two-pivot step falls back to the sequential formula
ULPS_FIRST, ULPS_SECOND = 4, 9


def c_bar(n):
    return n + -(-n // 8) + 32


def _gamma(k, u):
    return k * u / (1.0 - k * u)


def backward_error(A, L, matmul=None):
    """Componentwise backward error of L (lower triangle used) as a factor of A (lower triangle used).

    Returns (ratio, bad): ratio = max over the lower triangle of |A - L L^T| / bound (0 where both are 0), bad = number of
    entries with a zero bound and a non-zero residual (NaN counts as bad).  `matmul(X, Y)` computes X @ Y^T in float64
    for n > 512 (any summation order: its error is inside gamma_{n+1}); default numpy."""
    n = A.shape[0]
    L = np.tril(L)
    Al = np.tril(A)
    if n <= LONG_MAX_N:
        T = np.longdouble
        Lx = L.astype(T)
        R = Al.astype(T) - np.tril(Lx @ Lx.T)
        absLL = np.tril(np.abs(Lx) @ np.abs(Lx).T)
    else:
        T = np.float64
        mm = matmul or (lambda X, Y: X @ Y.T)
        R = Al - np.tril(mm(L, L))
        absL = np.abs(L)
        absLL = np.tril(mm(absL, absL))
    uT = float(np.finfo(T).eps) / 2
    g = _gamma(n + 1, uT)
    bound = c_bar(n) * U * (1.0 - g) * absLL + g * (np.abs(Al).astype(T) + absLL)
    R = np.abs(R)
    zero = bound == 0
    bad = int(np.count_nonzero(zero & ~(R == 0))) + int(np.count_nonzero(np.isnan(R)))
    ratio = float(np.max(np.where(zero, 0.0, R / np.where(zero, 1.0, bound)), initial=0.0))
    return ratio, bad


def mirror_ok(full):
    """the strict upper triangle equals tril(L, -1)^T bitwise"""
    n = full.shape[0]
    iu = np.triu_indices(n, 1)
    return np.array_equal(full[iu].view(np.uint64), full.T[iu].view(np.uint64))


def ulps(x, ref):
    """|x - ref| in units of the last place of ref (elementwise)"""
    return np.abs(np.asarray(x, dtype=np.float64) - ref) / np.spacing(np.abs(ref))


def pair_ulp_limits(idx):
    """ULPS_FIRST for the first pivot of a leaf pair (even index), ULPS_SECOND for the second"""
    return np.where(np.asarray(idx) % 2 == 0, ULPS_FIRST, ULPS_SECOND)


# ---------------------------------------------------------------------------------------------------- generators
def spd(n, seed):
    """well-conditioned dense SPD matrix, entries O(1)"""
    rng = np.random.default_rng(seed)
    G = rng.normal(size=(n, n + 8))
    return G @ G.T / (n + 8) + 0.5 * np.eye(n)


def unit_diagonal(A):
    d = 1.0 / np.sqrt(np.diag(A))
    M = A * d[:, None] * d[None, :]
    np.fill_diagonal(M, 1.0)
    return M


def graded(n, seed, lo=-120.0, hi=120.0):
    """S M S, M a unit-diagonal well-conditioned SPD matrix, s_i = 10^U(lo, hi): the pivot pairs' A C spans 1e-480 .. 1e480"""
    rng = np.random.default_rng(seed)
    s = 10.0 ** rng.uniform(lo, hi, size=n)
    return unit_diagonal(spd(n, seed + 1)) * s[:, None] * s[None, :]


def jacobi_ill(n, kappa, seed):
    """unit-diagonal (Jacobi-scaled) SPD matrix with a random eigenbasis and condition number about kappa"""
    rng = np.random.default_rng(seed)
    Q, _ = np.linalg.qr(rng.normal(size=(n, n)))
    lam = np.logspace(0.0, -np.log10(kappa), n)
    A = (Q * lam) @ Q.T
    return unit_diagonal((A + A.T) / 2)


def dependent_pairs(n, eps, seed):
    """unit-diagonal SPD matrix whose rows 2k and 2k+1 are nearly dependent (A = G G^T with g_{2k+1} = g_{2k} + eps h):
    every leaf pair of the kernel has C / (C - B^2/A) ~ 1/eps^2, and the rows below couple to both members"""
    rng = np.random.default_rng(seed)
    G = rng.normal(size=(n, n + 8))
    m = (n // 2) * 2
    G[1:m:2] = G[0:m:2] + eps * rng.normal(size=(m // 2, n + 8))
    return unit_diagonal(G @ G.T)


def diagonal(n, seed, lo=-30.0, hi=30.0):
    rng = np.random.default_rng(seed)
    return np.diag(10.0 ** rng.uniform(lo, hi, size=n))


def block_diagonal(n, seed):
    """SPD blocks of sizes 1..9 at random offsets (both parities); returns (A, first row of every block)"""
    rng = np.random.default_rng(seed)
    A = np.zeros((n, n))
    firsts = []
    r = 0
    while r < n:
        b = min(int(rng.integers(1, 10)), n - r)
        A[r:r + b, r:r + b] = spd(b, seed + r) * 10.0 ** rng.uniform(-20, 20)
        firsts.append(r)
        r += b
    return A, np.array(firsts)


def band_arrow(nblk, bw, tail, seed, arrow=None):
    """random diagonally dominant matrix with a block band of half-width bw and a dense arrow from block `arrow`
    (default: the last full block); returns (A, structure mask, end_blk table, arrow_blk) in the layout
    vgg_dev_cholesky_band takes"""
    n = nblk * 128 + tail
    arrow = nblk - 1 if arrow is None else arrow
    rng = np.random.default_rng(seed)
    G = rng.normal(size=(n, n)) * 0.05
    blk = np.arange(n) // 128
    keep = (np.abs(blk[:, None] - blk[None, :]) <= bw) | (blk[:, None] >= arrow) | (blk[None, :] >= arrow)
    A = (G + G.T) * keep
    A += np.diag(np.abs(A).sum(1) + 1.0)
    nb_all = (n + 127) // 128
    end = np.array([nb_all if b >= arrow else min(arrow, max(b + bw + 1, b + 2)) for b in range(nb_all)], dtype=np.int32)
    return A, keep, end, arrow


def bordered(D, seed, pinned=()):
    """the bordered matrix scale_damp_kernel (csrc/ba_schur.cu) hands to the factorisation, order D + 1: a unit-scale
    damped SPD block, pinned parameters as identity rows and columns, row D = b (0 at pinned rows), corner 1e300"""
    rng = np.random.default_rng(seed)
    S = unit_diagonal(spd(D, seed)) + 1e-2 * np.eye(D)
    pin = np.zeros(D, dtype=bool)
    pin[list(pinned)] = True
    S[pin, :] = 0.0
    S[:, pin] = 0.0
    S[pin, pin] = 1.0
    b = rng.normal(size=D)
    b[pin] = 0.0
    A = np.zeros((D + 1, D + 1))
    A[:D, :D] = S
    A[D, :D] = b
    A[:D, D] = b
    A[D, D] = 1e300
    return A


# ---------------------------------------------------------------------------------------------------- expectations
def dpotrf_info(A):
    from scipy.linalg import lapack
    return int(lapack.dpotrf(A, lower=1, clean=0, overwrite_a=0)[1])


def nan_info(i, j):
    """a NaN planted at (i, j) of the lower triangle (i >= j) makes pivot max(i, j) the first NaN one: the row's
    entries right of column j all depend on it, and nothing before row i does"""
    return max(i, j) + 1


def pair_products(A):
    """float64 replay of the kernel's pivot sequence (right-looking, two pivots at a time, as the 8 x 8 leaves take
    them): A C of every pair (2k, 2k+1); an odd last pivot pairs with the identity padding (C = 1)"""
    S = np.array(np.tril(A) + np.tril(A, -1).T, dtype=np.float64)
    n = S.shape[0]
    out = []
    for k in range(0, n, 2):
        a = S[k, k]
        if k + 1 < n:
            c = S[k + 1, k + 1]
            with np.errstate(over="ignore", under="ignore"):
                out.append(a * c)
            P = np.linalg.cholesky(S[k:k + 2, k:k + 2])
            X = np.linalg.solve(P, S[k:k + 2, k + 2:]).T
            S[k + 2:, k + 2:] -= X @ X.T
        else:
            out.append(a * 1.0)
    return np.array(out)


# ---------------------------------------------------------------------------------------------------- runner
def workspace_bytes(n):
    return ((n + 127) // 128) * 131072 + 1024


def cholesky_device(A_ptr, n, lda, ws, band=None):
    """vgg_cholesky_lower (band=None) or vgg_dev_cholesky_band (band = (end_blk int32 array, arrow_blk)) in place on the
    device matrix at A_ptr on the current torch stream; ws a device uint8 tensor of >= workspace_bytes(n).  Returns
    info (0, the 1-based failing pivot, or INT_MAX for a stalled hand-off, which callers assert never happens)."""
    import ctypes
    import torch
    from vggsfm_b200 import _lib
    L = _lib.lib()
    info = ctypes.c_int(-1)
    args = (n, lda, A_ptr, ws.data_ptr(), ws.numel(), ctypes.byref(info), torch.cuda.current_stream().cuda_stream)
    if band is None:
        _lib.check(L.vgg_cholesky_lower(*args), "vgg_cholesky_lower")
    else:
        end = np.ascontiguousarray(band[0], dtype=np.int32)
        _lib.check(L.vgg_dev_cholesky_band(*args, end.ctypes.data, end.size, int(band[1])), "vgg_dev_cholesky_band")
    return info.value


INFO_STALLED = 2 ** 31 - 1
