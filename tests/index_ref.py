# coding=utf-8
"""Plain references for the graph preprocessing kernels (csrc/index_ops.cu, csrc/scan.cuh, the flag and compaction
entries of csrc/sample_ops.cu, colsum and l2_normalize in csrc/gemm.cu).  numpy and integer arithmetic only, no CUDA:
tests/test_index_ref_host.py checks these references on the CPU, tests/test_gpu_index_contract.py checks the kernels
against them.

Exact references restate the kernel's own operation order (`select_ref`, `unique_ref`, `rowsum_seq`, `deg_inv_exact`,
`scale_edges_ref`), so the kernels must match them bit for bit.  The two reductions whose order is a blocking choice
(colsum, l2_normalize) get forward error bounds instead (`colsum_bound`, `l2_bound`), derived below with the usual
gamma_k = k u / (1 - k u), u = 2^-24 (fp32 round to nearest)."""
import math
from fractions import Fraction

import numpy as np

F32 = np.float32
U32 = 2.0 ** -24                 # unit roundoff of fp32
FLT_MAX = float(np.finfo(F32).max)
TFGK_POW_INV_SQRT, TFGK_POW_INV = 0, 1


def gamma(k):
    k = float(k)
    return k * U32 / (1.0 - k * U32)


# ---- compaction and unique -------------------------------------------------------------------------------------------

def select_ref(flag):
    """tfgk_select_flagged_i32: ascending positions of the non-zero flags (any non-zero value counts once)."""
    return np.flatnonzero(np.asarray(flag)).astype(np.int32)


def unique_ref(row, col):
    """tfgk_edge_unique / tf.unique over the hash row * N + col (N = max id + 1, as merge_duplicated_edge hashes):
    the unique pairs in first-occurrence order (int32 [2, U]) and, per edge, the index of its pair (int32 [E])."""
    row = np.asarray(row).astype(np.int64)
    col = np.asarray(col).astype(np.int64)
    if row.size == 0:
        return np.zeros((2, 0), np.int32), np.zeros(0, np.int32)
    n = int(max(row.max(), col.max())) + 1
    h = row * n + col
    _, first, inverse = np.unique(h, return_index=True, return_inverse=True)
    order = np.argsort(first, kind="stable")            # sorted slot -> first-occurrence rank
    rank = np.empty_like(order)
    rank[order] = np.arange(order.size)
    uniq = np.stack([row[first[order]], col[first[order]]]).astype(np.int32)
    return uniq, rank[inverse.reshape(-1)].astype(np.int32)


# ---- GCN normalisation helpers ---------------------------------------------------------------------------------------

def rowsum_seq(rowptr, w):
    """csr_rowsum_kernel: out[r] = (((+0 + w[p]) + w[p+1]) + ...) in fp32, strictly left to right over the row.
    Vectorised over "the j-th entry of every row with degree > j": rows sorted by degree (descending) make those rows a
    prefix, so the cost is max degree numpy steps of shrinking size, E element operations in all."""
    rowptr = np.asarray(rowptr, dtype=np.int64)
    w = np.asarray(w, dtype=F32)
    n = rowptr.size - 1
    deg = np.diff(rowptr)
    order = np.argsort(-deg, kind="stable")
    deg_sorted = deg[order]
    start = rowptr[:-1][order]
    acc = np.zeros(n, F32)                                   # +0.0, as the kernel starts
    max_deg = int(deg.max()) if n else 0
    # live[j] = how many rows have degree > j (a prefix of `order`)
    live = np.searchsorted(-deg_sorted, -np.arange(max_deg), side="left") if max_deg else []
    for j in range(max_deg):
        k = int(live[j])
        acc[:k] = acc[:k] + w[start[:k] + j]                 # fp32 + fp32 -> fp32, round to nearest
    out = np.empty(n, F32)
    out[order] = acc
    return out


def _round_positive_to_f32(y, exact_cmp):
    """Correct rounding to fp32 of positive values known in float64 as `y` (relative error << 2^-28).
    exact_cmp(i, m) returns the sign of (true value - m) for element i and a float64 midpoint m, exactly."""
    y = np.asarray(y, dtype=np.float64)
    with np.errstate(over="ignore"):
        r = y.astype(F32)                                    # nearest fp32 of the float64 value (may be inf)
        lo = np.where(r.astype(np.float64) > y, np.nextafter(r, F32(0)), r)  # largest fp32 <= y (FLT_MAX if r == inf)
        hi32 = np.nextafter(lo, F32(np.inf))
    hi = np.where(np.isinf(hi32), 2.0 ** 128, hi32.astype(np.float64))        # round-to-nearest treats 2^128 as next
    mid = (lo.astype(np.float64) + hi) * 0.5                 # 25 significant bits: exact in float64
    out = np.where(y < mid, lo, hi32).astype(F32)
    near = np.flatnonzero(np.abs(y - mid) <= 2.0 ** -28 * y)
    for i in near:                                           # settle midpoint-adjacent cases with integers
        s = exact_cmp(int(i), float(mid[i]))
        if s < 0:
            out[i] = lo[i]
        elif s > 0:
            out[i] = hi32[i]
        else:                                                # an exact tie: to even
            out[i] = lo[i] if (lo[i].view(np.uint32) & 1) == 0 else hi32[i]
    return out


def deg_inv_exact(d, power):
    """deg_inv_kernel: the correctly rounded fp32 of d^-1/2 (power TFGK_POW_INV_SQRT) or 1/d (TFGK_POW_INV), then
    inf and NaN -> +0 (gcn.py's _remove_inf_and_nan).  1/(-inf) stays -0.0, as __frcp_rn gives.

    The float64 value is within 2^-52 relative of the true one, so it rounds to the right fp32 unless it lies within
    2^-28 relative of an fp32 midpoint m; those cases are settled exactly: m^2 d against 1 (or m d against 1) with the
    dyadic rationals of m and d as Python integers."""
    d = np.asarray(d, dtype=F32).reshape(-1)
    out = np.zeros(d.shape, F32)
    a = np.abs(d.astype(np.float64))
    if power == TFGK_POW_INV_SQRT:
        ok = np.isfinite(d) & (d > 0)                         # 0, -0 -> inf; negative, -inf, NaN -> NaN; +inf -> +0
        idx = np.flatnonzero(ok)
        with np.errstate(divide="ignore"):
            y = 1.0 / np.sqrt(a[idx])

        def cmp(i, m):                                       # sign(d^-1/2 - m) = sign(1 - m^2 d)
            mn, md = Fraction(m).numerator, Fraction(m).denominator
            dn, dd = Fraction(float(a[idx[i]])).numerator, Fraction(float(a[idx[i]])).denominator
            lhs, rhs = md * md * dd, mn * mn * dn
            return (lhs > rhs) - (lhs < rhs)
        out[idx] = _round_positive_to_f32(y, cmp)
    elif power == TFGK_POW_INV:
        ok = np.isfinite(d) & (d != 0)                        # +-0 -> +-inf -> 0; NaN -> 0; +-inf -> +-0 below
        idx = np.flatnonzero(ok)
        y = 1.0 / a[idx]

        def cmp(i, m):                                       # sign(1/|d| - m) = sign(1 - m |d|)
            mn, md = Fraction(m).numerator, Fraction(m).denominator
            dn, dd = Fraction(float(a[idx[i]])).numerator, Fraction(float(a[idx[i]])).denominator
            lhs, rhs = md * dd, mn * dn
            return (lhs > rhs) - (lhs < rhs)
        mag = _round_positive_to_f32(y, cmp)
        out[idx] = np.where(d[idx] < 0, -mag, mag)
        out[np.isinf(d)] = np.where(d[np.isinf(d)] < 0, F32(-0.0), F32(0.0))
    else:
        raise ValueError("unknown power {}".format(power))
    out[np.isinf(out)] = 0                                   # an overflowed 1/d (d subnormal) -> 0 as well
    return out


def scale_edges_ref(row, col, w, dl=None, dr=None):
    """scale_edges_kernel: v = w (or 1), v = dl[row] * v, v = v * dr[col], each product rounded to fp32."""
    v = np.ones(np.asarray(row if row is not None else col).shape, F32) if w is None else np.asarray(w, F32).copy()
    with np.errstate(over="ignore"):                        # an overflow to inf is the fp32 product's value
        if dl is not None:
            v = (np.asarray(dl, F32)[row] * v).astype(F32)
        if dr is not None:
            v = (v * np.asarray(dr, F32)[col]).astype(F32)
    return v


# ---- colsum and l2_normalize bounds ----------------------------------------------------------------------------------

def _sm_count(sm_count):
    if sm_count is None:
        from tf_geometric_b200 import ops
        sm_count = ops.device_info()["sm_count"]
    return int(sm_count)


def colsum_blocks(n_rows, sm_count=None):
    """The block count of tfgk_colsum_f32, restated from colsum_blocks() in csrc/gemm.cu:
    min(ceil(n_rows / 512), 8 * SMs), at least 1.  SMs defaults to the current device's (ops.device_info())."""
    sm_count = _sm_count(sm_count)
    b = -(-int(n_rows) // 512)
    return max(1, min(b, 8 * int(sm_count)))


def colsum_terms(n_rows, sm_count=None):
    """k of colsum_bound: the most roundings any one entry of x meets on its way to out[c].
    A block owns rpb = ceil(n / nb) rows and sums them into four accumulators (rows r, r+1, r+2, r+3), the < 4 left-over
    rows into the first: at most ceil(rpb / 4) + 2 additions per accumulator; then (a0 + a1) + (a2 + a3) is 2 more, and
    the final kernel adds the nb partials in block order from +0: at most nb more."""
    nb = colsum_blocks(n_rows, sm_count)
    rpb = -(-max(int(n_rows), 1) // nb)
    return -(-rpb // 4) + 2 + nb


def colsum_bound(x, n_rows, sm_count=None):
    """|colsum(x)[c] - sum_r x[r, c]| <= gamma_k * sum_r |x[r, c]| (float64), k = colsum_terms.  x: float64 [n, D]
    or the float64 column sums of |x| directly (a 1-D array)."""
    a = np.asarray(x, dtype=np.float64)
    abs_sum = a if a.ndim == 1 else np.abs(a).sum(axis=0)
    return gamma(colsum_terms(n_rows, sm_count)) * abs_sum


def l2_bound(D):
    """Per-entry relative bound of l2_normalize_kernel against float64 x / sqrt(max(sum x^2, 1e-12)), for rows whose
    sum of squares S is a normal fp32 number above the 1e-12 clamp.

    Lane l squares and adds its ceil(D/32) entries (x[l], x[l+32], ...; a product and an add each, fused or not), then
    5 butterfly shuffle adds combine the lanes: every term meets at most k = ceil(D/32) + 6 roundings, so the computed
    s = S (1 + t) with |t| <= gamma_k (all terms are >= 0, so the bound is relative to S itself).  Through the square
    root the relative error of s^-1/2 is (1 + t)^-1/2 - 1, at most e1 = (1 - gamma_k)^-1/2 - 1 ~ gamma_k / 2.
    rsqrtf has at most 2 ulp of error (CUDA Programming Guide, mathematical functions): e2 = 2 * 2^-23 relative.
    The final product x * inv is rounded once: e3 = 2^-24.  So |out - y| <= ((1 + e1)(1 + e2)(1 + e3) - 1) |y|."""
    k = -(-int(D) // 32) + 6
    e1 = 1.0 / math.sqrt(1.0 - gamma(k)) - 1.0
    e2 = 2.0 ** -22
    e3 = 2.0 ** -24
    return (1.0 + e1) * (1.0 + e2) * (1.0 + e3) - 1.0
