# coding=utf-8
"""CPU checks of tests/index_ref.py, the references the preprocessing-kernel contract (test_gpu_index_contract.py)
compares against: unique_ref against the oracle's tf.unique restatement, rowsum_seq against an explicit loop,
deg_inv_exact against exact rational arithmetic, and the colsum / l2_normalize bounds against float64 over numpy
restatements of the two kernels' summation orders."""
import math
from fractions import Fraction

import numpy as np
import pytest

from oracle import tfg_oracle as o
import index_ref as R

F32 = np.float32


# ---- unique_ref ------------------------------------------------------------------------------------------------------

@pytest.mark.parametrize("n,e,seed", [(1, 1, 0), (1, 50, 1), (7, 200, 2), (300, 5000, 3), (70000, 20000, 4)])
def test_unique_ref_matches_oracle(n, e, seed):
    rs = np.random.RandomState(seed)
    ei = rs.randint(0, n, (2, e)).astype(np.int32)
    ei[:, rs.randint(0, e, e // 5)] = ei[:, :1]                # a long run of one pair
    uniq, of_edge = R.unique_ref(ei[0], ei[1])
    want_index, _ = o.merge_duplicated_edge(ei)
    np.testing.assert_array_equal(uniq, want_index)
    h, _ = o.convert_edge_index_to_edge_hash(ei)
    _, want_of_edge = o.tf_unique(h)
    np.testing.assert_array_equal(of_edge, want_of_edge)
    np.testing.assert_array_equal(uniq[:, of_edge], ei)          # every edge points at its own pair


# ---- rowsum_seq ------------------------------------------------------------------------------------------------------

@pytest.mark.parametrize("seed", range(4))
def test_rowsum_seq_matches_a_loop(seed):
    rs = np.random.RandomState(seed)
    n = 60
    deg = rs.randint(0, 9, n)
    deg[rs.randint(0, n, 10)] = 0                                # empty rows
    deg[3] = 300                                                 # a hub
    rowptr = np.concatenate([[0], np.cumsum(deg)]).astype(np.int64)
    w = (rs.randn(rowptr[-1]) * 10.0 ** rs.randint(-3, 4, rowptr[-1])).astype(F32)
    got = R.rowsum_seq(rowptr, w)
    for r in range(n):
        acc = F32(0.0)
        for p in range(rowptr[r], rowptr[r + 1]):
            acc = F32(acc + w[p])
        assert got[r].view(np.uint32) == acc.view(np.uint32), r


# ---- deg_inv_exact ---------------------------------------------------------------------------------------------------

def _round_fraction_f32(q):
    """q (a positive Fraction) rounded to nearest-even fp32, as a float (inf above the overflow threshold)."""
    e = q.numerator.bit_length() - q.denominator.bit_length()
    if Fraction(2) ** e > q:
        e -= 1
    ulp = Fraction(2) ** (max(e, -126) - 23)
    n, rem = divmod(q, ulp)
    n = int(n)
    if rem * 2 > ulp or (rem * 2 == ulp and n % 2 == 1):
        n += 1
    v = n * ulp
    return math.inf if v >= Fraction(2) ** 128 else float(v)


def _f32_neighbours(r):
    r = F32(r)
    lo = np.nextafter(r, F32(0))
    hi = np.nextafter(r, F32(np.inf))
    hi = Fraction(2) ** 128 if np.isinf(hi) else Fraction(float(hi))
    return Fraction(float(lo)), hi


def _deg_inv_sample():
    rs = np.random.RandomState(7)
    special = np.array([0.0, -0.0, -1.0, -3.5, np.inf, -np.inf, np.nan, 1.0, 2.0, 4.0, 3.0, 0.25,
                        1e-45, 2e-45, 1e-40, 1.17549435e-38, 2.9e-39, 5.9e-39, 3.4028235e38, 1e38, 65536.0,
                        16777216.0, 16777217.0], np.float32)
    bits = rs.randint(0, 0x7F800000, 3000).astype(np.uint32)      # positive finite, subnormals included
    rand = bits.view(np.float32)
    sub = (rs.randint(1, 1 << 23, 300).astype(np.uint32)).view(np.float32)
    # midpoint-adjacent values: d with 1/d (or d^-1/2) within a few fp32 ulps of d of an fp32 midpoint m
    m = rs.uniform(1.0, 2.0, 600).astype(F32).astype(np.float64)
    m = m + np.spacing(m.astype(F32)).astype(np.float64) / 2
    near_rcp = (1.0 / m * rs.choice([0.25, 1.0, 1024.0, 2.0 ** -100], 600)).astype(F32)
    near_rsqrt = (1.0 / (m * m) * rs.choice([0.25, 1.0, 4.0 ** 30, 4.0 ** -40], 600)).astype(F32)
    return np.concatenate([special, rand, sub, near_rcp, near_rsqrt, -rand[:50]])


@pytest.mark.parametrize("power", [R.TFGK_POW_INV_SQRT, R.TFGK_POW_INV])
def test_deg_inv_exact_is_correctly_rounded(power):
    d = _deg_inv_sample()
    got = R.deg_inv_exact(d, power)
    assert got.dtype == np.float32 and got.shape == d.shape
    n_near = 0
    for x, g in zip(d, got):
        xf = float(x)
        if power == R.TFGK_POW_INV_SQRT:
            if not (math.isfinite(xf) and xf > 0):                   # 0, -0, negatives, -inf, NaN, +inf -> +0
                assert g.view(np.uint32) == 0, (x, g)
                continue
            # g is d^-1/2 correctly rounded iff the midpoints around g bracket d^-1/2: lo^2 d <= 1 <= hi^2 d
            lo, hi = _f32_neighbours(g)
            gq = Fraction(float(g))
            mlo, mhi = (lo + gq) / 2, (gq + hi) / 2
            dq = Fraction(xf)
            assert mlo * mlo * dq <= 1 <= mhi * mhi * dq, (x, g)
            n_near += min(abs(1 - mlo * mlo * dq), abs(mhi * mhi * dq - 1)) < Fraction(1, 1 << 26)
        else:
            if math.isnan(xf) or xf == 0:
                assert g.view(np.uint32) == 0, (x, g)
                continue
            if math.isinf(xf):
                assert g == 0 and math.copysign(1.0, g) == math.copysign(1.0, xf), (x, g)
                continue
            want = _round_fraction_f32(1 / Fraction(abs(xf)))
            want = 0.0 if math.isinf(want) else math.copysign(want, xf)
            assert F32(want).view(np.uint32) == g.view(np.uint32), (x, g, want)
    if power == R.TFGK_POW_INV_SQRT:
        assert n_near > 100                                         # the sample does reach the exact settling path


# ---- colsum_bound and l2_bound ---------------------------------------------------------------------------------------

def _colsum_kernel_order(x, sm_count):
    """colsum_partial_kernel + colsum_final_kernel restated in fp32 (four accumulators per block, blocks in order)."""
    n, d = x.shape
    nb = R.colsum_blocks(n, sm_count)
    rpb = -(-max(n, 1) // nb)
    partial = np.zeros((nb, d), F32)
    for b in range(nb):
        r0, r1 = b * rpb, min(b * rpb + rpb, n)
        a = np.zeros((4, d), F32)
        r = r0
        while r + 4 <= r1:
            for j in range(4):
                a[j] = a[j] + x[r + j]
            r += 4
        while r < r1:
            a[0] = a[0] + x[r]
            r += 1
        partial[b] = (a[0] + a[1]) + (a[2] + a[3])
    out = np.zeros(d, F32)
    for b in range(nb):
        out = out + partial[b]
    return out


def test_colsum_blocks_restates_the_kernel_rule():
    assert R.colsum_blocks(0, 132) == 1 and R.colsum_blocks(1, 132) == 1 and R.colsum_blocks(512, 132) == 1
    assert R.colsum_blocks(513, 132) == 2 and R.colsum_blocks(10 ** 9, 132) == 8 * 132
    # 1 row: 1 block, 1 row per block -> ceil(1/4) + 2 + 1
    assert R.colsum_terms(1, 132) == 4


@pytest.mark.parametrize("n,d,sm", [(1, 3, 2), (7, 5, 2), (3001, 33, 2), (9000, 17, 1), (2048, 8, 4)])
def test_colsum_bound_holds_in_float64(n, d, sm):
    rs = np.random.RandomState(n + d)
    x = (rs.randn(n, d) * 10.0 ** rs.randint(-2, 3, (n, d))).astype(F32)
    x[:, 0] = np.abs(x[:, 0])                                   # a column without cancellation
    x[:, 1 % d] += F32(1e4)                                     # a column with a large common offset
    got = _colsum_kernel_order(x, sm).astype(np.float64)
    exact = x.astype(np.float64).sum(axis=0)
    bound = R.colsum_bound(x.astype(np.float64), n, sm)
    assert np.all(np.abs(got - exact) <= bound)
    assert np.all(bound <= 1e-4 * np.abs(x).astype(np.float64).sum(axis=0) + 1e-30)


def _l2_kernel_order(x):
    """l2_normalize_kernel restated in fp32: lane l sums x[c]^2 for c = l, l+32, ... (product and add rounded
    separately: the unfused case, one rounding more than an FMA), 5 butterfly adds, a 2-ulp-accurate rsqrt (here the
    correctly rounded one) and one product."""
    n, d = x.shape
    lanes = np.zeros((n, 32), F32)
    for c in range(d):
        lanes[:, c % 32] = lanes[:, c % 32] + (x[:, c] * x[:, c]).astype(F32)
    for off in (16, 8, 4, 2, 1):
        lanes = (lanes + lanes[:, np.arange(32) ^ off]).astype(F32)
    ss = np.maximum(lanes[:, 0], F32(1e-12))
    inv = (1.0 / np.sqrt(ss.astype(np.float64))).astype(F32)
    return (x * inv[:, None]).astype(F32)


@pytest.mark.parametrize("d", [1, 31, 32, 33, 100, 602])
def test_l2_bound_holds_in_float64(d):
    rs = np.random.RandomState(d)
    x = (rs.randn(301, d) * 10.0 ** rs.randint(-3, 4, (301, 1))).astype(F32)
    got = _l2_kernel_order(x).astype(np.float64)
    x64 = x.astype(np.float64)
    y = x64 / np.sqrt(np.maximum((x64 * x64).sum(axis=1, keepdims=True), 1e-12))
    b = R.l2_bound(d)
    assert np.all(np.abs(got - y) <= b * np.abs(y))
    assert b < 1.1e-6                                          # gamma_25 / 2 + 2.5 ulp at D = 602
    # the bound is not vacuous: it is within a small factor of the error fp32 arithmetic can reach
    assert b >= 2.0 ** -22
