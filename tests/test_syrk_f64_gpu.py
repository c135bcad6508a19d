"""FP64 tensor-core Schur SYRK of the LM loop (csrc/ba_schur.cu syrk_f64_kernel, through the vgg_dev_syrk_f64 probe):
Cmat -= Zt^T Zt into the row-major LOWER triangle, checked against Z^T Z computed to a few units in the last place
(oracle/ozaki_oracle.py exact_gram).  Every entry is a float64 dot product over at most K rows, accumulated in FP64 MMA
registers per work item and added into Cmat with one f64 RED per item (at most 16 items per tile), so
|err_ij| <= c K 2^-53 (|Z|^T |Z|)_ij + 2^-48 |C0_ij|, c = 2."""
import ctypes

import numpy as np
import pytest

from oracle import ozaki_oracle as oz

pytestmark = pytest.mark.gpu


def _syrk(Z, C0, dev, ranges=None):
    import torch
    from vggsfm_b200 import _lib
    L = _lib.lib()
    Kpad, Dpad = Z.shape
    Zt = torch.from_numpy(np.ascontiguousarray(Z)).to(dev)
    C = torch.from_numpy(np.ascontiguousarray(C0)).to(dev)
    with torch.cuda.device(dev):
        args = (Kpad, Dpad, Zt.data_ptr(), C.data_ptr(), torch.cuda.current_stream().cuda_stream)
        if ranges is None:
            _lib.check(L.vgg_dev_syrk_f64(*args), "vgg_dev_syrk_f64")
        else:
            r = np.ascontiguousarray(ranges, dtype=np.int32)
            _lib.check(L.vgg_dev_syrk_f64_band(*args, r.ctypes.data, r.size), "vgg_dev_syrk_f64_band")
        torch.cuda.synchronize()
    return C.cpu().numpy()


def _check(Z, C0, got, dev, what):
    """Lower triangle: C0 - Z^T Z within the bound of the module docstring; strict upper triangle: C0 untouched."""
    import torch
    K = Z.shape[0]
    ref = C0 - oz.exact_gram(Z, device=dev)
    Za = torch.from_numpy(np.abs(Z)).to(dev)
    scale = (Za.T @ Za).cpu().numpy()
    bound = 2.0 * K * 2.0 ** -53 * scale * (1 + 1e-6) + 2.0 ** -48 * np.abs(C0) + 2.0 ** -50 * np.abs(ref)
    low = np.tril(np.ones(C0.shape, dtype=bool))
    err = np.abs(got - ref)[low]
    ratio = (err / np.maximum(bound[low], 1e-300)).max()
    print(f"syrk_f64 {what}: max err/bound = {ratio:.3g}")
    assert np.all(err <= bound[low]), (what, ratio)
    assert np.array_equal(got[~low], C0[~low]), what


def _operand(Kpad, Dpad, seed):
    rng = np.random.default_rng(seed)
    Z = rng.normal(size=(Kpad, Dpad)) * np.exp(rng.uniform(-6, 6, size=(1, Dpad)))
    Z[rng.uniform(size=Z.shape) < 0.3] = 0.0
    Z[:, -5:] = 0.0
    return Z


@pytest.mark.parametrize("Kpad,Dpad", [(64, 128), (16, 128), (1040, 384), (12288, 2432)])
def test_matches_float64(cuda_dev, Kpad, Dpad):
    """One tile (a full and a partial k block), three row blocks with a k tail, and the C3 shape (400 x 4096,
    SIMPLE_RADIAL, shared camera: D = 2402)."""
    Z = _operand(Kpad, Dpad, Kpad + Dpad)
    C0 = np.zeros((Dpad, Dpad))
    _check(Z, C0, _syrk(Z, C0, cuda_dev), cuda_dev, f"{Kpad}x{Dpad}")


def test_accumulates_into_lower_triangle(cuda_dev):
    """Cmat already holds the camera block (assemble_hc) when the SYRK runs: it subtracts from the lower triangle and
    leaves the strict upper triangle alone."""
    Kpad, Dpad = 2000, 640
    Z = _operand(Kpad, Dpad, 7)
    rng = np.random.default_rng(8)
    C0 = rng.normal(size=(Dpad, Dpad)) * 1e3
    _check(Z, C0, _syrk(Z, C0, cuda_dev), cuda_dev, "accumulate")


def _banded(Kpad, Dpad, seed):
    """Row block rb of Zt is non-zero only inside its k-block range (a sliding window, like a video), except the last
    row block, which is dense (the shared-intrinsics arrow)."""
    nb, KB = Dpad // 128, (Kpad + 63) // 64
    Z = _operand(Kpad, Dpad, seed)
    ranges = np.zeros(2 * nb, dtype=np.int32)
    for rb in range(nb):
        lo, hi = (max(0, 2 * rb - 3), min(KB, 2 * rb + 4)) if rb < nb - 1 else (0, KB)
        ranges[2 * rb], ranges[2 * rb + 1] = lo, hi
        Z[:lo * 64, rb * 128:(rb + 1) * 128] = 0.0
        Z[hi * 64:, rb * 128:(rb + 1) * 128] = 0.0
    return Z, ranges


def test_band_hint(cuda_dev):
    """With the band hint the kernel skips the tiles whose ranges do not meet and clips the others to the intersection;
    the result is the dense one up to rounding order, and the skipped tiles stay exactly as they were."""
    Kpad, Dpad = 1600, 1280
    Z, ranges = _banded(Kpad, Dpad, 11)
    C0 = np.zeros((Dpad, Dpad))
    dense = _syrk(Z, C0, cuda_dev)
    band = _syrk(Z, C0, cuda_dev, ranges)
    _check(Z, C0, dense, cuda_dev, "banded operand, no hint")
    _check(Z, C0, band, cuda_dev, "banded operand, hint")
    nb = Dpad // 128
    for bi in range(nb):
        for bj in range(bi + 1):
            if min(ranges[2 * bi + 1], ranges[2 * bj + 1]) <= max(ranges[2 * bi], ranges[2 * bj]):
                assert not band[bi * 128:(bi + 1) * 128, bj * 128:(bj + 1) * 128].any(), (bi, bj)
    ref = -oz.exact_gram(Z, device=cuda_dev)
    low = np.tril(np.ones(C0.shape, dtype=bool))
    assert np.abs(band - dense)[low].max() <= 2.0 ** -40 * np.abs(ref).max()


def test_work_list_cache(cuda_dev):
    """The work list is cached per shape and band hint: alternating shapes (and a hint in between) must each get theirs."""
    shapes = [(640, 384), (1040, 1280), (640, 384), (1600, 1280), (1040, 1280)]
    for i, (Kpad, Dpad) in enumerate(shapes):
        if i == 3:
            Z, ranges = _banded(Kpad, Dpad, 20 + i)
        else:
            Z, ranges = _operand(Kpad, Dpad, 20 + i), None
        C0 = np.zeros((Dpad, Dpad))
        _check(Z, C0, _syrk(Z, C0, cuda_dev, ranges), cuda_dev, f"cache step {i}: {Kpad}x{Dpad}")
