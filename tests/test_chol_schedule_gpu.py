"""The device-sized panel schedule of csrc/chol.cu: panels whose rows below the diagonal block need more than 16
ride-along rows per CTA to fit the SMs in one wave (20 .. 32 rows, and a second wave beyond 32), dense and banded,
against numpy.linalg.cholesky at 1e-10 of the factor's scale."""
import ctypes

import numpy as np
import pytest

pytestmark = pytest.mark.gpu


def _factor(cuda_dev, A, band=None):
    import torch
    from vggsfm_b200 import _lib
    n = A.shape[0]
    lda = (n + 127) // 128 * 128
    buf = torch.zeros(n, lda, dtype=torch.float64, device=cuda_dev)
    buf[:, :n] = torch.from_numpy(np.tril(A)).to(cuda_dev)
    ws = torch.empty(((n + 127) // 128) * 131072 + 1024, dtype=torch.uint8, device=cuda_dev)
    info = ctypes.c_int(-1)
    L = _lib.lib()
    args = (n, lda, buf.data_ptr(), ws.data_ptr(), ws.numel(), ctypes.byref(info), torch.cuda.current_stream().cuda_stream)
    if band is None:
        _lib.check(L.vgg_cholesky_lower(*args), "vgg_cholesky_lower")
    else:
        _lib.check(L.vgg_dev_cholesky_band(*args, band[0].ctypes.data, band[0].size, band[1]), "vgg_dev_cholesky_band")
    return info.value, buf.cpu().numpy()[:, :n]


# on 132 SMs: n = 2700 -> 20 rows in the first panel, 3300 -> 28, 4500 -> 32 and a second wave
@pytest.mark.parametrize("n", [2700, 3300, 4500])
def test_cholesky_wide_panels_match_lapack(cuda_dev, n):
    rng = np.random.default_rng(n)
    B = rng.normal(size=(n, n + 8))
    A = B @ B.T + n * 1e-3 * np.eye(n)
    info, full = _factor(cuda_dev, A)
    assert info == 0
    ref = np.linalg.cholesky(A)
    got = np.tril(full)
    assert np.abs(got - ref).max() <= 1e-10 * np.abs(ref).max()
    assert np.array_equal(np.triu(full, 1), np.tril(full, -1).T)
    # a failing pivot in a later panel (the first panels run with the widest row chunks)
    A2 = A.copy()
    bad = n - 700
    A2[bad, bad] = -1.0
    info, _ = _factor(cuda_dev, A2)
    assert info == bad + 1


def test_cholesky_wide_band_plus_arrow_matches_lapack(cuda_dev):
    """A band of 16 blocks plus the arrow: more than 16 rows per panel CTA, so row chunks end early at the band's end."""
    nblk, bw, tail = 24, 16, 77
    n = nblk * 128 + tail
    arrow = nblk - 1
    rng = np.random.default_rng(7)
    G = rng.normal(size=(n, n)) * 0.05
    blk = np.arange(n) // 128
    keep = (np.abs(blk[:, None] - blk[None, :]) <= bw) | (blk[:, None] >= arrow) | (blk[None, :] >= arrow)
    A = (G + G.T) * keep
    A += np.diag(np.abs(A).sum(1) + 1.0)
    nb_all = (n + 127) // 128
    end = np.array([nb_all if b >= arrow else min(arrow, max(b + bw + 1, b + 2)) for b in range(nb_all)], dtype=np.int32)
    info, full = _factor(cuda_dev, A, band=(end, arrow))
    assert info == 0
    ref = np.linalg.cholesky(A)
    got = np.tril(full)
    assert np.abs(got - ref).max() <= 1e-10 * np.abs(ref).max()
