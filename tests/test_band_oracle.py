"""The band tables of oracle/band_oracle.py (= the formulas of csrc/ba_solve.cu compute_band_hint) against the brute-force
sparsity of random banded visibility masks: nothing non-zero may fall outside what the banded kernels visit."""
import numpy as np
import pytest

from oracle import band_oracle as bo
from tests.helpers import banded_mask as _banded_mask


@pytest.mark.parametrize("S,N,life,dc,ns,seed", [(160, 1400, 24, 6, 1, 0), (220, 2000, 40, 6, 2, 1), (130, 1100, 16, 7, 0, 2),
                                                  (96, 1200, 96, 6, 1, 3)])
def test_tables_cover_the_true_sparsity(S, N, life, dc, ns, seed):
    mask = _banded_mask(S, N, life, seed)
    t = bo.band_tables(mask, dc, ns)
    Z, Sp, ZtZ = bo.brute_force_pattern(mask, dc, ns)
    D, nb, KB = t["D"], t["nb"], t["KB"]
    # 1. Zt is zero outside every row block's k range (what the slicing kernel, z_build and the SYRK work list skip)
    for rb in range(nb):
        cols = slice(rb * 128, min(D, rb * 128 + 128))
        lo, hi = t["rb_range"][rb]
        assert not Z[:lo * 64, cols].any() and not Z[hi * 64:, cols].any(), rb
    # 2. SYRK tiles whose ranges do not meet are structurally zero in Zt^T Zt
    for bi in range(nb):
        for bj in range(bi + 1):
            a, b = t["rb_range"][bi], t["rb_range"][bj]
            if min(a[1], b[1]) <= max(a[0], b[0]):
                assert not ZtZ[bi * 128:min(D, bi * 128 + 128), bj * 128:min(D, bj * 128 + 128)].any(), (bi, bj)
    # 3. the factorisation's structure contains the envelope of the reduced system (and is monotone)
    end, arrow = t["end_blk"], t["arrow_blk"]
    assert np.all(np.diff(end) >= 0)
    nblk = (D + 1 + 127) // 128
    for b in range(min(arrow, nblk)):
        assert end[b] >= min(b + 2, arrow)
        rows_beyond = slice(end[b] * 128, arrow * 128)
        assert not Sp[rows_beyond, b * 128:min(D, b * 128 + 128)].any(), b
    # 4. backsub: W[n][row] != 0 only inside the point's k-block row range or the arrow
    for n in range(0, N, 7):
        ka, kb = (3 * n) >> 6, (3 * n + 2) >> 6
        lo = min(t["kb_rows"][ka][0], t["kb_rows"][kb][0])
        hi = max(t["kb_rows"][ka][1], t["kb_rows"][kb][1])
        rows = np.nonzero(Z[3 * n, :S * dc])[0]
        if rows.size:
            ok = ((rows >= lo) & (rows < hi)) | (rows >= arrow * 128)
            assert ok.all(), n
    # 5. ba_blocks: every visible (frame, track) lies inside its frame group's track range
    for g, (lo, hi) in enumerate(t["fg_tracks"]):
        sub = mask[32 * g:32 * g + 32]
        cols = np.nonzero(sub.any(0))[0]
        if cols.size:
            assert cols[0] >= lo and cols[-1] < hi


def test_unordered_points_give_wide_but_valid_ranges():
    mask = _banded_mask(128, 1500, 20, 5)
    perm = np.random.default_rng(0).permutation(mask.shape[1])
    t = bo.band_tables(mask[:, perm], 6, 1)
    Z, _, _ = bo.brute_force_pattern(mask[:, perm], 6, 1)
    for rb in range(t["nb"]):
        lo, hi = t["rb_range"][rb]
        cols = slice(rb * 128, min(t["D"], rb * 128 + 128))
        assert not Z[:lo * 64, cols].any() and not Z[hi * 64:, cols].any()
    # nothing to gain: almost every row block spans almost all of K
    assert np.mean(t["rb_range"][:t["arrow_blk"], 1] - t["rb_range"][:t["arrow_blk"], 0]) > 0.8 * t["KB"]
