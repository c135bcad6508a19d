"""The reduced-system Cholesky (csrc/chol.cu) against its own contract, at its edges.

Bars, applied to every successful call (derivations in oracle/chol_oracle.py):
  1. componentwise backward error |A - L L^T| <= c_n u (|L||L^T|), c_n = n + ceil(n/8) + 32 (<= 4 (n + 1) for n >= 9),
     exact zeros where the bound is zero (structure of band and arrow, pinned rows); residual in extended precision up
     to n = 512, in float64 (on the device) above with its own evaluation error added;
  2. the strict upper triangle equals tril(L, -1)^T bitwise;
  3. where the pivot is known (diagonal matrices, the first row of a diagonal block) L_jj is within 4 ulps of
     sqrt(a_jj) for the first pivot of a leaf pair and 9 for the second;
  4. info is never INT_MAX (a stalled hand-off between CTAs) -- asserted on every call.
Cases: orders across the one-block / two-block / captured-graph boundaries and every leaf, sub-panel and panel boundary;
failing pivots (negative, NaN, subnormal, +inf, two of them, both of a pair, in band and arrow) at every leaf position
class of the first, a middle and the last block, each followed by a good matrix on the same buffer; graded scales whose
pivot pairs leave the two-pivot range; ill-conditioned and nearly dependent pairs; the bordered matrix of the LM loop;
NaN sentinels around the matrix and lda = n; the graph cache; band shapes.  Each case prints its backward-error ratio
and worst ulp count."""
import functools

import numpy as np
import pytest

from oracle import chol_oracle as co

pytestmark = pytest.mark.gpu

ORDERS = [1, 2, 7, 8, 9, 31, 32, 33, 127, 128, 129, 255, 256, 257, 383, 384, 385, 2402, 2403]
POSITIONS = [0, 1, 6, 7, 8, 9, 30, 31, 32, 33, 126, 127]


def _r128(n):
    return (n + 127) // 128 * 128


def _dev():
    import torch
    return torch.device("cuda:0")


def _matmul(X, Y):
    """X @ Y^T in float64 on the device (cuBLAS; any summation order is inside the bar's evaluation term)"""
    import torch
    tX = torch.from_numpy(np.ascontiguousarray(X)).to(_dev())
    tY = tX if Y is X else torch.from_numpy(np.ascontiguousarray(Y)).to(_dev())
    return (tX @ tY.T).cpu().numpy()


class Slot:
    """a device matrix buffer [rows, lda] and a workspace, reused across calls like the LM loop reuses its own"""

    def __init__(self, n, lda=None, rows=None):
        import torch
        self.n, self.lda, self.rows = n, lda or _r128(n), rows or n
        self.buf = torch.zeros(self.rows, self.lda, dtype=torch.float64, device=_dev())
        self.ws = torch.empty(co.workspace_bytes(n), dtype=torch.uint8, device=_dev())

    def factor(self, A, band=None, n=None, fill=0.0):
        import torch
        n = n or self.n
        h = np.full((self.rows, self.lda), fill)
        h[:n, :n] = np.tril(A) + (np.triu(np.full((n, n), fill), 1) if fill != 0.0 else 0.0)
        self.h = h
        self.buf.copy_(torch.from_numpy(h))
        info = co.cholesky_device(self.buf.data_ptr(), n, self.lda, self.ws, band)
        assert info != co.INFO_STALLED
        return info, self.buf.cpu().numpy()


def check(tag, A, full, known=None):
    """bars 1 and 2 (+ 3 on the indices in `known`); prints the ratio and the ulp count"""
    n = A.shape[0]
    F = full[:n, :n]
    ratio, bad = co.backward_error(A, F, matmul=_matmul)
    msg = f"chol {tag}: n={n} backward-error ratio {ratio:.3e}"
    if known is not None and len(known):
        d = np.diag(F)[known]
        u = co.ulps(d, np.sqrt(np.diag(A)[known]))
        lim = co.pair_ulp_limits(known)
        msg += f"  worst ulps first/second {u[known % 2 == 0].max(initial=0):.1f}/{u[known % 2 == 1].max(initial=0):.1f}"
        assert np.all(u <= lim), (tag, known[u > lim][:8], u[u > lim][:8])
    print(msg)
    assert bad == 0, (tag, "non-zero residual where the bound is zero", bad)
    assert ratio <= 1.0, (tag, ratio)
    assert co.mirror_ok(F), tag


@functools.lru_cache(maxsize=4)
def _spd(n):
    A = co.spd(n, n)
    A.setflags(write=False)
    return A


# ---------------------------------------------------------------------------------------------------- orders
@pytest.mark.parametrize("n", ORDERS)
def test_orders(cuda_dev, n):
    s = Slot(n)
    A = _spd(n)
    info, full = s.factor(A)
    assert info == 0
    check(f"orders spd", A, full)
    for lo, hi in ((-30.0, 30.0), (-120.0, 120.0)):          # pairs inside and outside the two-pivot range
        D = co.diagonal(n, n + 1, lo, hi)
        info, full = s.factor(D)
        assert info == 0
        check(f"orders diagonal 1e{int(hi)}", D, full, known=np.arange(n))
    B, firsts = co.block_diagonal(n, n + 2)
    info, full = s.factor(B)
    assert info == 0
    check("orders block-diagonal", B, full, known=firsts)


# ---------------------------------------------------------------------------------------------------- failures
def _pivot_cases():
    out = []
    for n in (2403, 200, 4500):
        nblk = (n + 127) // 128
        blocks = {"first": 0, "last": nblk - 1}
        if nblk > 2:
            blocks["middle"] = nblk // 2
        for where, b in blocks.items():
            for p in POSITIONS:
                if b * 128 + p < n:
                    out.append((n, where, b * 128 + p))
    return out


def _fail_then_good(s, A, bad, want, tag, band=None):
    info, _ = s.factor(bad, band=band)
    assert info == want, (tag, info, want)
    info, full = s.factor(A, band=band)                      # the same buffer, workspace and cached graph
    assert info == 0, tag
    check(tag, A, full)


@pytest.mark.parametrize("n,where,p", _pivot_cases())
def test_negative_pivot(cuda_dev, n, where, p):
    A = _spd(n)
    bad = A.copy()
    bad[p, p] = -1.0
    want = co.dpotrf_info(bad)
    assert want == p + 1
    _fail_then_good(Slot(n), A, bad, want, f"after negative pivot {p}")


@pytest.mark.parametrize("n,i,j", [(2403, 0, 0), (2403, 1, 1), (2403, 7, 7), (2403, 1030, 1030), (2403, 2402, 2402),
                                   (2403, 9, 3), (2403, 128, 127), (2403, 33, 32), (2403, 1033, 5), (2403, 2402, 2401),
                                   (200, 1, 0), (200, 150, 140), (9, 8, 0)])
def test_nan_entry(cuda_dev, n, i, j):
    """OpenBLAS dpotrf returns 0 for a NaN pivot, so the expected index is analytic: max(i, j) + 1"""
    A = _spd(n)
    bad = A.copy()
    bad[i, j] = np.nan
    _fail_then_good(Slot(n), A, bad, co.nan_info(i, j), f"after NaN at ({i},{j})")


@pytest.mark.parametrize("n,ps", [(2403, (1500, 300)), (2403, (640, 641)), (2403, (9, 7)), (200, (150, 131)),
                                  (4500, (4400, 700))])
def test_two_failing_pivots_report_the_earlier(cuda_dev, n, ps):
    A = _spd(n)
    bad = A.copy()
    for p in ps:
        bad[p, p] = -2.0
    want = co.dpotrf_info(bad)
    assert want == min(ps) + 1
    _fail_then_good(Slot(n), A, bad, want, f"after pivots {ps}")


@pytest.mark.parametrize("n,p", [(300, 0), (300, 1), (300, 131), (2403, 2402), (2403, 1001)])
def test_subnormal_pivot_fails(cuda_dev, n, p):
    """1e-310 on an uncoupled row: LAPACK accepts it, the kernel's rule (pivot < smallest normal) reports p + 1"""
    A = _spd(n).copy()
    A[p, :] = 0.0
    A[:, p] = 0.0
    A[p, p] = 1e-310
    assert co.dpotrf_info(A) == 0
    good = _spd(n).copy()
    good[p, :] = 0.0
    good[:, p] = 0.0
    good[p, p] = 1.0
    _fail_then_good(Slot(n), good, A, p + 1, f"after subnormal pivot {p}")


@pytest.mark.parametrize("n,p", [(300, 0), (300, 1), (2403, 1200), (2403, 2402)])
def test_inf_pivot_is_flagged(cuda_dev, n, p):
    """+inf on the diagonal: LAPACK says info 0 with a non-finite factor; the LM loop needs info != 0 or a non-finite L"""
    A = _spd(n).copy()
    A[p, p] = np.inf
    s = Slot(n)
    info, full = s.factor(A)
    assert info != 0 or not np.isfinite(np.tril(full[:n, :n])).all()
    info, full = s.factor(_spd(n))
    assert info == 0
    check(f"after +inf pivot {p}", _spd(n), full)


def test_failures_in_band_and_arrow(cuda_dev):
    A, keep, end, arrow = co.band_arrow(20, 3, 77, 21)
    n = len(A)
    s = Slot(n)
    for p in (700, 701, arrow * 128 + 9, n - 2):
        bad = A.copy()
        bad[p, p] = -1.0
        want = co.dpotrf_info(bad)
        assert want == p + 1
        _fail_then_good(s, A, bad, want, f"band+arrow after pivot {p}", band=(end, arrow))


# ---------------------------------------------------------------------------------------------------- scales
@pytest.mark.parametrize("n", [129, 257, 384, 2403])
def test_graded_scales(cuda_dev, n):
    A = co.graded(n, n)
    ac = co.pair_products(A) if n <= 512 else None
    if ac is not None:
        assert (ac < co.AC_LO).any() and (ac > co.AC_HI).any()
    info, full = Slot(n).factor(A)
    assert info == 0
    check("graded 1e+-120", A, full)


def test_smallest_normal_diagonal(cuda_dev):
    n = 300
    d = 10.0 ** np.random.default_rng(3).uniform(-5, 5, n)
    d[[0, 1, 6, 9, 130, 131, 299]] = 2.0 ** -1022            # first / second of a pair, a whole pair, the last
    A = np.diag(d)
    info, full = Slot(n).factor(A)
    assert info == 0
    check("2^-1022 diagonal", A, full, known=np.arange(n))


@pytest.mark.parametrize("n,kind,k", [(300, "eig", 1e6), (300, "eig", 1e12), (2403, "eig", 1e12),
                                      (300, "pairs", 1e-3), (300, "pairs", 1e-4), (2403, "pairs", 1e-3)])
def test_ill_conditioned(cuda_dev, n, kind, k):
    """Jacobi-scaled systems, kappa up to 1e12: a random eigenbasis, and nearly dependent pivot pairs (rows 2k, 2k+1),
    where a second pivot taken from C - l10^2 while its column is scaled by a reciprocal root of det leaves
    ~eps C / (C - B^2/A) of backward error below it"""
    A = co.jacobi_ill(n, k, n) if kind == "eig" else co.dependent_pairs(n, k, n)
    info, full = Slot(n).factor(A)
    assert info == 0
    check(f"ill-conditioned {kind} {k:g}", A, full)


# ---------------------------------------------------------------------------------------------------- bordered
@pytest.mark.parametrize("D", [296, 297, 302, 2407, 384, 2431, 2402])
def test_bordered_ba_matrix(cuda_dev, D):
    """the matrix scale_damp_kernel builds: the corner 1e300 at D = 0, 1, 6, 7 mod 8 (first / second of a pair) and
    0 / 127 mod 128 (a lone last panel / the last row of a full one)"""
    pinned = [0, 1, 40, 128, 129, 200, D - 1]
    A = co.bordered(D, D, pinned)
    n = D + 1
    info, full = Slot(n).factor(A)
    assert info == 0
    F = full[:n, :n]
    check("bordered leading D x D", A[:D, :D], full[:D, :D])
    L = np.tril(F)
    y = L[D, :D]
    b = A[D, :D]
    # L y = b componentwise (this is row D of bar 1)
    LD = L[:D, :D].astype(np.longdouble) if D <= co.LONG_MAX_N else L[:D, :D]
    r = np.abs(b - LD @ y)
    bound = co.c_bar(n) * co.U * (np.abs(LD) @ np.abs(y)) + co._gamma(n + 1, float(np.finfo(LD.dtype).eps) / 2) * (
        np.abs(b) + np.abs(LD) @ np.abs(y))
    assert np.all((r <= bound) | ((r == 0) & (bound == 0))), float(np.max(r / np.where(bound > 0, bound, 1)))
    want = float(np.sqrt(np.longdouble(1e300) - np.dot(y.astype(np.longdouble), y)))
    uc = float(co.ulps(F[D, D], want))
    print(f"chol bordered D={D}: corner {uc:.1f} ulps, L y = b ratio {float(np.max(r / np.where(bound > 0, bound, 1))):.3e}")
    assert uc <= (co.ULPS_FIRST if D % 2 == 0 else co.ULPS_SECOND)
    for p in pinned:
        assert F[p, p] == 1.0 or co.ulps(F[p, p], 1.0) <= co.ULPS_SECOND
        assert np.all(L[p, :p] == 0) and np.all(L[p + 1:, p] == 0), p


# ---------------------------------------------------------------------------------------------------- sentinels
@pytest.mark.parametrize("n", [33, 100, 257, 2403])
def test_nan_sentinels_around_the_matrix(cuda_dev, n):
    """NaN in the strict upper triangle, the padding columns n .. lda-1 and 5 extra rows: padding and extra rows come
    back bitwise unchanged, and the bars hold"""
    s = Slot(n, rows=n + 5)
    A = _spd(n)
    info, full = s.factor(A, fill=np.nan)
    assert info == 0
    same = full.view(np.uint64) == s.h.view(np.uint64)
    assert same[:, n:].all() and same[n:].all()
    check("NaN sentinels", A, full)


@pytest.mark.parametrize("n", [2, 100, 258, 2402])
def test_lda_equals_n_at_the_end_of_the_allocation(cuda_dev, n):
    import torch
    A = _spd(n)
    pre, tail = 6, 4096
    h = np.full(pre + n * n + tail, np.nan)
    h[pre:pre + n * n] = np.tril(A).ravel()
    buf = torch.from_numpy(h).to(cuda_dev)
    ws = torch.empty(co.workspace_bytes(n), dtype=torch.uint8, device=cuda_dev)
    info = co.cholesky_device(buf.data_ptr() + 8 * pre, n, n, ws)
    assert info == 0
    out = buf.cpu().numpy()
    same = out.view(np.uint64) == h.view(np.uint64)
    assert same[:pre].all() and same[pre + n * n:].all()
    check("lda = n", A, out[pre:pre + n * n].reshape(n, n))


# ---------------------------------------------------------------------------------------------------- schedules
def _band_case():
    return co.band_arrow(12, 2, 77, 5)


def test_representative_set_graph(cuda_dev):
    """257 (the smallest captured order), 2403, 4500 (second wave) and a band + arrow matrix under bars 1 and 2, with a failure and
    a recovery on each buffer"""
    for n in (257, 2403, 4500):
        s = Slot(n)
        A = _spd(n)
        bad = A.copy()
        bad[n - 3, n - 3] = -1.0
        assert s.factor(bad)[0] == n - 2
        info, full = s.factor(A)
        assert info == 0
        check("schedule", A, full)
    A, keep, end, arrow = _band_case()
    info, full = Slot(len(A)).factor(A, band=(end, arrow))
    assert info == 0
    check("schedule band+arrow", A, full)


def test_graph_cache_eviction_and_reuse(cuda_dev):
    """ten (buffer, order) keys so the cache of eight clears, then an evicted key again; the same buffer with new
    contents; the same buffer dense -> banded -> dense"""
    s = Slot(420, lda=512)
    orders = [384 + 4 * k for k in range(10)]
    for n in orders + [orders[0], orders[1]]:
        A = co.spd(n, 1000 + n)
        info, full = s.factor(A, n=n)
        assert info == 0
        check("graph cache", A, full[:n, :n])
    A2 = co.graded(orders[0], 77)
    info, full = s.factor(A2, n=orders[0])
    assert info == 0
    check("graph cache new contents", A2, full[:orders[0], :orders[0]])
    A, keep, end, arrow = co.band_arrow(9, 1, 5, 8)
    t = Slot(len(A))
    D = co.spd(len(A), 9)
    for M, band in ((D, None), (A, (end, arrow)), (D, None), (A, (end, arrow))):
        info, full = t.factor(M, band=band)
        assert info == 0
        check("dense/banded alternation", M, full)


# ---------------------------------------------------------------------------------------------------- band shapes
def test_band_shapes(cuda_dev):
    A, keep, end, arrow = co.band_arrow(10, 2, 40, 13)
    n = len(A)
    nb = len(end)
    s = Slot(n)
    cases = {
        "structure": (end, arrow),
        "arrow_blk = 1": (np.full(nb, nb, dtype=np.int32), 1),
        "band reaching the arrow": (np.array([max(b + 2, min(nb, arrow + 1)) if b < arrow else nb for b in range(nb)],
                                             dtype=np.int32), arrow),
        "wider tables": (np.array([nb if b >= arrow - 2 else min(end[b] + 2, arrow - 2) for b in range(nb)],
                                  dtype=np.int32), arrow - 2),
        "end_blk = nblk": (np.full(nb, nb, dtype=np.int32), arrow),
    }
    for tag, band in cases.items():
        info, full = s.factor(A, band=band)
        assert info == 0
        check(f"band shape {tag}", A, full)
    info, full = s.factor(A)
    assert info == 0
    check("band shape dense path", A, full)
    # arrow_blk = 1 on a matrix that is dense below the first block
    D = _spd(n)
    info, full = s.factor(D, band=(np.full(nb, nb, dtype=np.int32), 1))
    assert info == 0
    check("band shape arrow_blk = 1 dense", D, full)
