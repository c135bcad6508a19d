"""CPU restatement of the integer arithmetic of csrc/syrk_i8.cu -- TEST INFRASTRUCTURE ONLY.

This is not a reference-side algorithm (the reference's SYRK lives inside Ceres' Schur eliminator, in plain FP64);
it restates OUR tensor-core formulation so that its arithmetic can be checked without a GPU:
  * column scales p = 2^e >= max|z|, x = z 2^-e rounded to B = 8s-2 fractional bits; columns whose maximum is below
    2^-900 are flushed to zero (the kernel does the same so that 2^(B-e) stays finite);
  * balanced base-256 digits from one add: bytes of (X + 0x80..80) xor 0x80;
  * exact integer pair products C_t = sum_{p+q=t} D_p^T D_q for t <= s+1, recombined in float64.

The pair products are float64 GEMMs of int8-valued arrays: every partial sum is an integer below 7 2^14 K < 2^53, so
they are exact in any summation order, on the CPU (numpy) or on a GPU (torch, `device=`).

Error bounds (tests/test_ozaki_oracle.py, tests/test_syrk_i8_gpu.py):
  * normwise_bound -- |syrk - Z^T Z|_ij <= 2^-B (p_i ||Z_j||_1 / 2 + p_j ||Z_i||_1 / 2 + c_s n_ij p_i p_j), n_ij the rows
    where both columns are non-zero.  The first two terms are the rounding of the slices, the last one the dropped
    orders t > s+1 (c_s = sum_j (s-1-j) 256^-j + 2^-B / 4 <= 6.02).  It is NOT a componentwise bound relative to
    (|Z|^T |Z|)_ij: one large entry in column j sets p_j for the whole column.
  * recombination_bound -- what the kernel may differ from `syrk` by: every work item's contribution is exact (int32
    accumulators, power-of-two scaling), the only roundings are the float64 additions of at most m items into one
    entry and the oracle's own sum over orders.
"""
from __future__ import annotations

import numpy as np

FLUSH_EXP = -900          # columns with max|z| < 2^-900 are treated as exact zeros
ITEM_K_ROWS = 256 * 64    # OZ_MAX_ITEM_KB k-blocks of 64 rows: the longest reduction one int32 accumulator sees


def column_exponents(Z):
    """e_d with |Z[:, d]| 2^-e_d < 1 (ilogb(max) + 1); 0 for all-zero and flushed columns."""
    m = np.abs(Z).max(axis=0)
    e = np.zeros(Z.shape[1], dtype=np.int64)
    nz = m > 0
    e[nz] = np.frexp(m[nz])[1]            # m = f 2^e, f in [0.5, 1)  ->  m 2^-e < 1
    e[e < FLUSH_EXP] = 0
    return e


def flushed_columns(Z):
    """Columns the kernel treats as zero: non-zero, but every entry below 2^-900."""
    m = np.abs(Z).max(axis=0)
    return (m > 0) & (np.frexp(m)[1] < FLUSH_EXP)


def slices(Z, s):
    """int8 digit matrices D[p] (p = 0 most significant) and exponents e: Z ~ 2^(e - B) sum_p D[p] 256^(s-1-p)."""
    B = 8 * s - 2
    e = column_exponents(Z)
    X = np.rint(np.ldexp(Z, (B - e)[None, :])).astype(np.int64)
    X[:, flushed_columns(Z)] = 0
    bias = int.from_bytes(b"\x80" * s, "little")
    Y = (X + bias) ^ bias
    D = np.empty((s,) + Z.shape, dtype=np.int8)
    for p in range(s):
        j = s - 1 - p
        D[p] = ((Y >> (8 * j)) & 255).astype(np.uint8).view(np.int8)
    return D, e, X


def _dev(a, device):
    """float64 copy of a numpy array on `device` (torch), or the numpy array itself for device None."""
    a = np.ascontiguousarray(a, dtype=np.float64)
    if device is None:
        return a
    import torch
    return torch.from_numpy(a).to(device)


def _host(x):
    return x if isinstance(x, np.ndarray) else x.cpu().numpy()


def _gram(cols, K, device):
    """sum over k-chunks of A^T A, A = cols(k0, k1) (float64 [k1-k0, n]), on `device`."""
    out = None
    for k0 in range(0, K, ITEM_K_ROWS):
        a = _dev(cols(k0, min(K, k0 + ITEM_K_ROWS)), device)
        g = _host(a.T @ a)
        out = g if out is None else out + g
    return out


def order_products(Z, s, max_order=None, device=None):
    """{t: C_t} for t = 2 .. max_order (default s+1) as exact float64 integers, and the exponents e.

    The int32 headroom of the kernel is checked per ITEM_K_ROWS block of k, the longest reduction a work item runs."""
    D, e, _ = slices(Z, s)
    tmax = s + 1 if max_order is None else max_order
    n = Z.shape[1]
    C = {t: np.zeros((n, n)) for t in range(2, tmax + 1)}
    for k0 in range(0, Z.shape[0], ITEM_K_ROWS):
        Dk = [_dev(D[p, k0:k0 + ITEM_K_ROWS], device) for p in range(s)]
        for t in range(2, tmax + 1):
            Ck = 0
            for p in range(1, s + 1):
                q = t - p
                if 1 <= q <= s:
                    Ck = Ck + Dk[p - 1].T @ Dk[q - 1]
            Ck = _host(Ck)
            assert np.abs(Ck).max() < 2 ** 31, "int32 accumulator would overflow"
            C[t] += Ck
        del Dk
    return C, e


def syrk(Z, s, max_order=None, device=None):
    """Z^T Z through the sliced integer products, recombined like the kernel's epilogue (float64)."""
    B = 8 * s - 2
    C, e = order_products(Z, s, max_order, device)
    out = np.zeros_like(C[2])
    for t in sorted(C, reverse=True):                  # least significant order first
        out += np.ldexp(C[t], 8 * (2 * s - t) - 2 * B)
    return np.ldexp(np.ldexp(out, e[:, None]), e[None, :])     # two steps: no intermediate overflow to inf


def dropped_order_coefficient(s):
    """c_s: |sum over the dropped orders t > s+1| <= c_s 2^-B p_i p_j per row k (|d_p| <= 128 for p >= 2), plus the
    product of the two roundings (<= 2^-2B p_i p_j / 4)."""
    B = 8 * s - 2
    return sum((s - 1 - j) * 256.0 ** -j for j in range(s - 1)) + 2.0 ** -B / 4


def normwise_bound(Z, s, device=None):
    """Bound on |syrk(Z, s) - Z^T Z| per entry (see the module docstring); flushed columns count as zero."""
    Zf = np.where(flushed_columns(Z)[None, :], 0.0, Z)
    B = 8 * s - 2
    e = column_exponents(Zf)
    p = np.where(np.abs(Zf).max(axis=0) > 0, np.ldexp(1.0, e), 0.0)
    l1 = np.abs(Zf).sum(axis=0)
    n = _gram(lambda k0, k1: Zf[k0:k1] != 0, Zf.shape[0], device)
    return 2.0 ** -B * (0.5 * p[:, None] * l1[None, :] + 0.5 * l1[:, None] * p[None, :]
                        + dropped_order_coefficient(s) * n * p[:, None] * p[None, :])


def max_items_per_tile(Kpad, s):
    """Upper bound on the work items that add into one 128 x 128 tile: ceil(s/2) order groups (two orders per group)
    times at most max(16, ceil(KB / 256)) k-parts each (csrc/syrk_i8.cu build_work_list, oz_max_parts)."""
    KB = -(-Kpad // 64)
    return -(-s // 2) * max(16, -(-KB // 256))


def digit_magnitude(Z, s, device=None):
    """T_ij = p_i p_j sum_k A_ki A_kj with A = 2^-B sum_p |d_p| 256^(s-1-p): bounds the sum of |contribution| of all
    work items to entry (i, j), whatever the order groups and k-splits."""
    D, e, _ = slices(Z, s)
    B = 8 * s - 2
    A = lambda k0, k1: sum(np.abs(D[p, k0:k1].astype(np.float64)) * 256.0 ** (s - 1 - p) for p in range(s)) * 2.0 ** -B
    return np.ldexp(np.ldexp(_gram(A, Z.shape[0], device), e[:, None]), e[None, :])


def recombination_bound(Z, s, device=None):
    """Allowed |kernel - syrk(Z, s)| per entry: m float64 additions into the entry (m <= max_items_per_tile) and the
    oracle's sum of s orders, each rounding by at most 2^-53 of a partial sum bounded by digit_magnitude; plus one
    2^-1074 per addition for results in the subnormal range."""
    m = max_items_per_tile(Z.shape[0], s) + s
    return m * (2.0 ** -53 * digit_magnitude(Z, s, device) + 2.0 ** -1074)


def exact_gram(Z, device=None, pieces=4, bits=18):
    """Z^T Z to a few units in the last place, for K < 2^17 rows: every column is split on its own 2^e grid into
    `pieces` integer slices of `bits` bits (their products, summed over k, are exact float64 integers), and the slice
    products are added least significant first.  The split drops nothing above 2^-(pieces * bits) p."""
    e = column_exponents(Z)
    K, n = Z.shape
    assert K * 2.0 ** (2 * bits) < 2.0 ** 53
    G = {(a, b): np.zeros((n, n)) for a in range(pieces) for b in range(a, pieces)}
    for k0 in range(0, K, ITEM_K_ROWS):
        rest = np.ldexp(Z[k0:k0 + ITEM_K_ROWS], -e[None, :])
        parts = []
        for a in range(pieces):
            hi = np.trunc(np.ldexp(rest, bits))
            parts.append(_dev(hi, device))
            rest = np.ldexp(rest, bits) - hi
        for a, b in G:
            G[a, b] += _host(parts[a].T @ parts[b])
        del parts
    out = np.zeros((n, n))
    for a, b in sorted(G, key=lambda ab: -(ab[0] + ab[1])):
        g = np.ldexp(G[a, b], -bits * (a + b + 2))
        out += g if a == b else g + g.T
    return np.ldexp(np.ldexp(out, e[:, None]), e[None, :])


def two_spike(K=2000, seed=0):
    """An operand that defeats a bound relative to (|Z|^T |Z|)_ij: rows of N(0,1), except that row 0 is 2^30 in
    columns 0-3 (zero elsewhere) and row 1 is 2^30 in columns 4-7 (zero in 0-3).  Entry (3, 4) then sees both column
    scales 2^31 but none of the spikes, so its slicing error is large against (|Z|^T |Z|)_34 ~ 1e3 and small against
    sqrt(S_33 S_44)."""
    rng = np.random.default_rng(seed)
    Z = rng.normal(size=(K, 8))
    Z[0, :] = 0.0
    Z[1, :] = 0.0
    Z[0, :4] = 2.0 ** 30
    Z[1, 4:] = 2.0 ** 30
    return Z


def worst_case_digits(K, n, s, seed):
    """Z whose non-leading balanced digits are all -128 or -127 and leading digit -63, so every pair product is
    positive and near 128^2: the int32 accumulators of a work item sit close to their worst case."""
    rng = np.random.default_rng(seed)
    B = 8 * s - 2
    X = np.full((K, n), -63 * 256 ** (s - 1), dtype=np.int64)
    for p in range(1, s):
        X += np.where(rng.uniform(size=(K, n)) < 0.9, -128, -127).astype(np.int64) * 256 ** (s - 1 - p)
    e = rng.integers(-4, 5, size=n)
    return np.ldexp(X.astype(np.float64), (e - B)[None, :])
