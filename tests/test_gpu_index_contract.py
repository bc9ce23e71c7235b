# coding=utf-8
"""Contract of the graph preprocessing kernels: the integer and normalisation work that builds every graph before the
message-passing kernels run (csrc/index_ops.cu, csrc/scan.cuh, the flag and compaction entries of csrc/sample_ops.cu,
colsum and l2_normalize in csrc/gemm.cu).  References are in tests/index_ref.py (checked on the CPU by
test_index_ref_host.py) and the oracle.

Exact, bit for bit:
- select_flagged against np.flatnonzero, across the 4 096-entry scan tile and the 1 024-tile chunk of scan_sums_kernel
  (n > 2^22 carries between chunks), for every non-zero flag value (2, -1, INT32_MAX count once, like 1);
- edge_flags in its three structural modes and three Bernoulli rules against the oracle's Philox restatement, and
  drop_edge / remove_self_loop_edge on the device against the oracle;
- edge_unique (index and per-edge group) against unique_ref with 1 to 4 radix passes per key, several thousand-key tiles,
  duplicate runs longer than a tile, and n_unique below 4 096, above 4 096 and above 2^22 (the first-occurrence ranking
  sort on one and on many blocks); merge_duplicated_edge's props in its four modes (a zero max or min takes K1's
  order of signed zeros, -0.0 < +0.0, where numpy keeps the first zero; DESIGN §5), convert_edge_to_upper and
  convert_edge_to_directed against the oracle and against the numpy-input route.  Sums of duplicate runs longer than a
  K1 hub slice (2 048 edges) are taken over dyadic props, which every summation order adds exactly: such a row is summed
  in slices (DESIGN §4, work plan), the one place the merge does not add strictly left to right;
  NaN props are outside the exact contract: test_merge_with_nan_props_device_and_host_routes pins what each route does;
- csr_rowsum (left to right from +0 per row), deg_inv (correctly rounded, inf / NaN -> 0) and scale_edges (two
  products in a fixed order) against their restatements.

Bounded:
- colsum within gamma_k * sum |x| of float64 (index_ref.colsum_bound; the blocking depends only on n_rows), and bit
  identical run to run and between a contiguous matrix and a column slice of a wider one;
- l2_normalize within index_ref.l2_bound(D) of float64, and the fp32 oracle within that bound plus the oracle's own
  (numpy sums the squares pairwise, the kernel by lanes, so the last bits may differ).  Its edge cases are exact:
  zero rows, a sum of squares that overflows fp32 (zeros, as the oracle's fp32 gives; pinned to fp32 semantics, float64
  would give finite values), an inf entry (NaN there) and rows below the 1e-12 clamp (x * rsqrtf(1e-12))."""
import numpy as np
import pytest
import torch

import tf_geometric_b200 as tfg
from tf_geometric_b200 import ops, _ffi
from oracle import tfg_oracle as o
from conftest import random_graph
import index_ref as R

pytestmark = pytest.mark.gpu

F32 = np.float32
I32_MAX = np.iinfo(np.int32).max


def dev(a, dtype=None):
    return ops.as_device(a, dtype)


def host(t):
    return t.detach().cpu().numpy()


def assert_bits(got, want, what=""):
    got, want = np.asarray(got), np.asarray(want)
    assert got.shape == want.shape, "{}: shape {} != {}".format(what, got.shape, want.shape)
    assert got.dtype == want.dtype, "{}: dtype {} != {}".format(what, got.dtype, want.dtype)
    g = got.view(np.uint32) if got.dtype == np.float32 else got
    w = want.view(np.uint32) if want.dtype == np.float32 else want
    bad = np.flatnonzero(g.reshape(-1) != w.reshape(-1))
    assert bad.size == 0, "{}: {} mismatches, first at {}: got {!r}, want {!r}".format(
        what, bad.size, bad[0], got.reshape(-1)[bad[0]], want.reshape(-1)[bad[0]])


# ---- select_flagged --------------------------------------------------------------------------------------------------

SELECT_SIZES = [1, 4095, 4096, 4097, (1 << 22) - 1, 1 << 22, (1 << 22) + 1, 3 * (1 << 22) + 17]


def _flag_patterns(n, rs):
    yield "zero", np.zeros(n, np.int32)
    yield "one", np.ones(n, np.int32)
    yield "alternating", (np.arange(n) % 2).astype(np.int32)
    yield "random", (rs.rand(n) < 0.5).astype(np.int32)
    last = np.zeros(n, np.int32)
    last[-1] = 1
    yield "last", last


@pytest.mark.parametrize("n", SELECT_SIZES)
def test_select_flagged_zero_one(n):
    rs = np.random.RandomState(n % 1000)
    for name, flag in _flag_patterns(n, rs):
        got = ops.select_flagged(dev(flag))
        assert got.dtype == torch.int32
        assert_bits(host(got), R.select_ref(flag), "n={} {}".format(n, name))


@pytest.mark.parametrize("value", [2, 5, I32_MAX])
def test_select_flagged_count_of_one_large_flag(value):
    """One non-zero flag, at the end: the count is 1 and the only position written is out[0].  (Adding the flag values
    in the scan instead of counting them gave a count of `value` here, with every write still in bounds.)"""
    for n in (2, 4097, (1 << 22) + 1):
        flag = np.zeros(n, np.int32)
        flag[-1] = value
        got = host(ops.select_flagged(dev(flag)))
        assert got.tolist() == [n - 1], "n={}: {} entries".format(n, got.shape[0])


@pytest.mark.parametrize("n", SELECT_SIZES)
def test_select_flagged_counts_non_zero_values_once(n):
    """Any non-zero flag selects its position once: the offsets count non-zero flags, not add their values (a flag of
    2 used to double the count and write past the output, a flag of -1 to give negative offsets)."""
    rs = np.random.RandomState(n % 997 + 1)
    for value in (2, -1, I32_MAX):
        for name, flag in _flag_patterns(n, rs):
            flag = flag * np.int32(value)
            got = host(ops.select_flagged(dev(flag)))
            assert got.shape[0] == np.count_nonzero(flag), "n={} {}x{}".format(n, name, value)
            assert_bits(got, R.select_ref(flag), "n={} {}x{}".format(n, name, value))
    mixed = rs.choice(np.array([0, 1, 2, -1, I32_MAX, -I32_MAX - 1, 7], np.int32), n)
    got = host(ops.select_flagged(dev(mixed)))
    assert got.shape[0] == np.count_nonzero(mixed)
    assert_bits(got, R.select_ref(mixed), "n={} mixed".format(n))


# ---- edge_flags, drop_edge, remove_self_loop_edge --------------------------------------------------------------------

@pytest.mark.parametrize("mode", [ops.FLAG_ALL, ops.FLAG_UPPER, ops.FLAG_MAPPED])
@pytest.mark.parametrize("bern", [ops.BERNOULLI_NONE, ops.BERNOULLI_DROPOUT, ops.BERNOULLI_KEEP])
def test_edge_flags_against_the_philox_restatement(mode, bern):
    n, e, prob, seed, stream = 5000, 100003, 0.3, 12345678901, ops.RNG_STREAM_SAMPLER   # e spans 25 scan tiles
    ei = random_graph(n, e, seed=3)
    rs = np.random.RandomState(4)
    row_map = np.where(rs.rand(n) < 0.3, -1, rs.randint(0, n, n)).astype(np.int32)
    col_map = np.where(rs.rand(n) < 0.2, -1, rs.randint(0, n, n)).astype(np.int32)
    if mode == ops.FLAG_ALL:
        keep = np.ones(e, bool)
    elif mode == ops.FLAG_UPPER:
        keep = ei[0] < ei[1]
    else:
        keep = (row_map[ei[0]] >= 0) & (col_map[ei[1]] >= 0)
    if bern != ops.BERNOULLI_NONE:
        u = o.random_uniform(seed, stream, np.arange(e, dtype=np.uint64))
        keep &= (u >= F32(prob)) if bern == ops.BERNOULLI_DROPOUT else (u <= F32(prob))
    want = keep.astype(np.int32)
    maps = (dev(row_map), dev(col_map)) if mode == ops.FLAG_MAPPED else (None, None)
    flag = ops.edge_flags(dev(ei[0]), dev(ei[1]), e, mode=mode, row_map=maps[0], col_map=maps[1], bernoulli=bern,
                          prob=prob, seed=seed, rng_stream=stream)
    assert_bits(host(flag), want, "flags")
    assert_bits(host(ops.select_flagged(flag)), R.select_ref(want), "selected")


def test_drop_edge_and_remove_self_loops_at_5m_edges():
    n, e = 400000, 5000000
    ei = random_graph(n, e, seed=9)
    ei[1, ::7] = ei[0, ::7]                                      # self loops
    w = np.random.RandomState(10).randn(e).astype(F32)
    for force_undirected in (False, True):
        want = o.drop_edge([ei, w], 0.4, force_undirected, True, seed=77)
        got = tfg.nn.drop_edge([dev(ei, torch.int32), dev(w)], 0.4, force_undirected, True, seed=77)
        assert_bits(host(got[0]), want[0].astype(np.int32), "drop_edge index")
        assert_bits(host(got[1]), want[1], "drop_edge weight")
    want_i, want_w = o.remove_self_loop_edge(ei, w)
    got_i, got_w = tfg.utils.remove_self_loop_edge(dev(ei, torch.int32), dev(w))
    assert_bits(host(got_i), want_i.astype(np.int32), "remove_self_loop index")
    assert_bits(host(got_w), want_w, "remove_self_loop weight")


# ---- edge_unique, merge_duplicated_edge, convert_edge_to_upper / _directed --------------------------------------------

def _edges(n, e, dup, seed, run=0, loops=0.0):
    """int32 [2, e] over ids [0, n) with max id n - 1: about a fraction `dup` of duplicate edges, a fraction `loops`
    of self loops and one contiguous run of `run` copies of a single pair."""
    rs = np.random.RandomState(seed)
    if dup == 0.0:
        h = np.unique(rs.randint(0, n * n, int(e * 1.2) + 16, dtype=np.int64))
        h = rs.permutation(h)[:e]
        ei = np.stack([h // n, h % n])
    else:
        pool = rs.randint(0, n, (2, max(1, int(e * (1.0 - dup)))))
        ei = pool[:, rs.randint(0, pool.shape[1], e)]
    if loops:
        at = rs.rand(e) < loops
        ei[1, at] = ei[0, at]
    if run:
        s = rs.randint(0, e - run + 1)
        ei[:, s:s + run] = ei[:, s:s + 1]
    ei[1, rs.randint(0, e)] = n - 1
    return ei.astype(np.int32)


def _k1_zero_signs(want, prop, of_edge, mode):
    """The device merge takes max and min with K1's MAX (fmaxf), which orders -0.0 below +0.0 whatever the edge order:
    a group whose max is zero gives +0.0 if it holds a +0.0, a group whose min is zero gives -0.0 if it holds a -0.0.
    numpy keeps the first of equal values in edge order.  `want` (numpy's result) with the device's zero signs."""
    zero = prop == 0
    has = np.zeros(want.shape, bool)
    np.logical_or.at(has, of_edge, zero & (np.signbit(prop) == (mode == "min")))
    out = want.copy()
    z = want == 0
    signed, other = (F32(0.0), F32(-0.0)) if mode == "max" else (F32(-0.0), F32(0.0))
    out[z] = np.where(has[z], signed, other)
    return out


def _props(e, seed, dyadic):
    """Random fp32 props with some -0.0, or dyadic ones (multiples of 2^-8 below 8) that sum exactly in any order."""
    rs = np.random.RandomState(seed)
    if dyadic:
        p = (rs.randint(-2048, 2048, e) / 256.0).astype(F32)
    else:
        p = (rs.randn(e) * 10.0 ** rs.randint(-3, 4, e)).astype(F32)
    p[rs.rand(e) < 0.02] = F32(-0.0)
    return p


UNIQUE_CASES = [
    # n (max id + 1: 1, 2, 3, 4 radix passes per key), e, duplicates, long run, self loops
    (1, 1, 0.0, 0, 0.0),
    (1, 9000, 0.5, 0, 0.0),                    # one pair 9 000 times: only self loops
    (256, 200000, 0.5, 5000, 0.05),
    (257, 300000, 0.95, 0, 0.05),
    (65536, 1000000, 0.0, 0, 0.0),             # n_unique ~ 1 M: the ranking sort on many blocks
    (65537, 1000000, 0.5, 10000, 0.01),
    (65537, 100000, 0.98, 0, 0.0),             # n_unique < 4 096: the ranking sort on one block
    ((1 << 24) + 1, 4095, 0.5, 0, 0.0),
    ((1 << 24) + 1, 4097, 0.0, 0, 0.0),
    ((1 << 24) + 1, 4300000, 0.0, 0, 0.001),   # n_unique > 2^22
    ((1 << 24) + 1, 4300000, 0.95, 6000, 0.0),
]


@pytest.mark.parametrize("n,e,dup,run,loops", UNIQUE_CASES)
def test_edge_unique_and_merge(n, e, dup, run, loops):
    ei = _edges(n, e, dup, seed=n % 1009 + e % 1013, run=run, loops=loops)
    assert int(ei.max()) == n - 1
    want_index, want_of_edge = R.unique_ref(ei[0], ei[1])
    got_index, got_of_edge = ops.edge_unique(dev(ei[0]), dev(ei[1]), n)
    assert_bits(host(got_index), want_index, "unique index")
    assert_bits(host(got_of_edge), want_of_edge, "unique_of_edge")
    n_unique = want_index.shape[1]
    if dup == 0.0 and e > 5000:
        assert n_unique > 4096
    # props: a hub row of K1 (> 2 048 duplicates of one pair) is summed in slices, so those sums take dyadic props
    dyadic = np.bincount(want_of_edge).max() > ops.HUB_THRESHOLD
    props = [_props(e, s, dyadic) for s in range(4)]
    modes = ["sum", "min", "max", "mean"]
    want_i, want_p = o.merge_duplicated_edge(ei, props, modes)
    got_i, got_p = tfg.utils.merge_duplicated_edge(dev(ei, torch.int32), [dev(p) for p in props], modes)
    assert_bits(host(got_i), want_i, "merged index")
    for m, p, g, w in zip(modes, props, got_p, want_p):
        if m in ("max", "min"):
            w = _k1_zero_signs(w, p, want_of_edge, m)
        assert_bits(host(g), w, "merged props ({})".format(m))


@pytest.mark.parametrize("n,e,dup,run,loops", UNIQUE_CASES + [(500, 20000, 0.5, 0, 1.0)])
def test_convert_edge_to_upper_and_directed(n, e, dup, run, loops):
    ei = _edges(n, e, dup, seed=n % 1013 + e % 1019 + 1, run=run, loops=loops)
    if loops == 1.0:
        ei[1] = ei[0]                                            # nothing but self loops
    rs = np.random.RandomState(e % 101)
    flip = rs.rand(e) < 0.5
    ei[:, flip] = ei[::-1, flip]                                 # both orientations of an undirected edge
    upper = np.stack([ei.min(axis=0), ei.max(axis=0)])
    dyadic = np.bincount(R.unique_ref(upper[0], upper[1])[1]).max() > ops.HUB_THRESHOLD
    props = [_props(e, 11, dyadic), _props(e, 12, dyadic)]
    modes = ["sum", "max"]
    for fn in ("convert_edge_to_upper", "convert_edge_to_directed"):
        want_i, want_p = getattr(o, fn)(ei, props, modes)
        got_i, got_p = getattr(tfg.utils, fn)(dev(ei, torch.int32), [dev(p) for p in props], modes)
        np_i, np_p = getattr(tfg.utils, fn)(ei, props, modes)
        assert_bits(host(got_i), np.asarray(want_i, np.int32), fn + " index")
        assert_bits(np.asarray(np_i, np.int32), np.asarray(want_i, np.int32), fn + " numpy-route index")
        for m, g, h, w in zip(modes, got_p, np_p, want_p):
            # max: the sign of a zero maximum follows K1's rule on the device (test_edge_unique_and_merge), so +0 == -0
            fold = (lambda a: np.asarray(a, F32) + F32(0.0)) if m == "max" else (lambda a: np.asarray(a, F32))
            assert_bits(fold(host(g)), fold(w), "{} props ({})".format(fn, m))
            assert_bits(np.asarray(h, F32), np.asarray(w), "{} numpy-route props ({})".format(fn, m))
        if loops == 1.0 and fn == "convert_edge_to_directed":
            assert_bits(host(got_i), ei, "self loops only: the input comes back")


@pytest.mark.filterwarnings("ignore::RuntimeWarning")
def test_merge_with_nan_props_device_and_host_routes():
    """NaN props are outside the bit-exact contract; what each route does is pinned here (DESIGN §5).
    sum and mean propagate a NaN into its group on both routes.  max and min: the host route (numpy) propagates it;
    the device route merges with K1's MAX (fmaxf), which ignores a NaN, so a group whose props are all NaN gives the
    empty-segment value (-FLT_MAX for max, FLT_MAX for min)."""
    ei = np.array([[0, 1, 0, 2, 2, 3, 1], [1, 2, 1, 3, 3, 0, 2]], np.int32)
    p = np.array([np.nan, 1.0, 2.0, np.nan, np.nan, 5.0, -3.0], F32)
    modes = ["sum", "mean", "max", "min"]
    got_i, got_p = tfg.utils.merge_duplicated_edge(dev(ei, torch.int32), [dev(p)] * 4, modes)
    host_i, host_p = tfg.utils.merge_duplicated_edge(ei, [p] * 4, modes)
    assert host(got_i).tolist() == [[0, 1, 2, 3], [1, 2, 3, 0]] == np.asarray(host_i).tolist()
    fmax = float(np.finfo(F32).max)
    want_dev = {"sum": [np.nan, -2.0, np.nan, 5.0], "mean": [np.nan, -1.0, np.nan, 5.0],
                "max": [2.0, 1.0, -fmax, 5.0], "min": [2.0, -3.0, fmax, 5.0]}
    want_host = {"sum": [np.nan, -2.0, np.nan, 5.0], "mean": [np.nan, -1.0, np.nan, 5.0],
                 "max": [np.nan, 1.0, np.nan, 5.0], "min": [np.nan, -3.0, np.nan, 5.0]}
    for m, g, h in zip(modes, got_p, host_p):
        np.testing.assert_array_equal(host(g), np.array(want_dev[m], F32), err_msg="device " + m)
        np.testing.assert_array_equal(np.asarray(h), np.array(want_host[m], F32), err_msg="host " + m)


# ---- GCN normalisation helpers ---------------------------------------------------------------------------------------

def test_csr_rowsum_is_left_to_right():
    n = 100000
    ei = random_graph(n, 400000, seed=5, isolated=20000, hub=(777, 60000))   # empty rows and a 60 000-edge hub
    rs = np.random.RandomState(6)
    w = (rs.randn(ei.shape[1]) * 10.0 ** rs.randint(-4, 5, ei.shape[1])).astype(F32)
    w[1::2] = -w[0::2][:w[1::2].size] * F32(1.0000001)           # near-cancelling pairs
    w[rs.rand(w.size) < 0.01] = F32(-0.0)
    csr = ops.csr_build(dev(ei[0]), dev(ei[1]), n)
    perm = host(csr.perm)
    w_csr = np.ascontiguousarray(w[perm])
    got = ops.csr_rowsum(csr, dev(w_csr))
    assert_bits(host(got), R.rowsum_seq(host(csr.rowptr), w_csr), "rowsum")


def test_deg_inv_is_correctly_rounded():
    rs = np.random.RandomState(8)
    special = np.array([0.0, -0.0, -1.0, -2.5e-40, np.inf, -np.inf, np.nan, -np.nan, 1.0, 4.0, 1e-45, 1e-40,
                        1.17549435e-38, 2.9e-39, 3.4028235e38, 16777217.0], F32)
    bits = rs.randint(1, 0x7F800000, 1000000).astype(np.uint32)          # positive finite fp32, subnormals included
    bits[:20000] = rs.randint(1, 0x00800000, 20000)                    # plenty of subnormals
    d = np.concatenate([special, bits.view(F32), -bits[:1000].view(F32)])
    for power in (R.TFGK_POW_INV_SQRT, R.TFGK_POW_INV):
        got = ops.deg_inv(dev(d), power)
        assert_bits(host(got), R.deg_inv_exact(d, power), "deg_inv power {}".format(power))


def test_scale_edges_four_forms():
    n, e = 50000, 700000
    ei = random_graph(n, e, seed=13)
    rs = np.random.RandomState(14)
    w = (rs.randn(e) * 10.0 ** rs.randint(-20, 20, e)).astype(F32)
    dl = (rs.rand(n) * 10.0 ** rs.randint(-20, 20, n)).astype(F32)
    dr = (rs.rand(n) * 10.0 ** rs.randint(-20, 20, n)).astype(F32)
    row, col = dev(ei[0]), dev(ei[1])
    for wl, l, r in ((w, dl, dr), (w, dl, None), (w, None, dr), (None, dl, dr)):
        what = "scale_edges w={} dl={} dr={}".format(wl is not None, l is not None, r is not None)
        dl_d, dr_d = (None if l is None else dev(l)), (None if r is None else dev(r))
        if wl is not None:
            got = ops.scale_edges(row, col, dev(wl), dl_d, dr_d)
        else:                                                     # w = NULL: the kernel starts from 1.0 per edge
            got = torch.empty(e, dtype=torch.float32, device=row.device)
            _ffi.call("tfgk_scale_edges_f32", ops._p(row), ops._p(col), None, e, ops._p(dl_d), ops._p(dr_d),
                      ops._p(got), ops._stream(got))
        assert_bits(host(got), R.scale_edges_ref(ei[0], ei[1], wl, l, r), what)


def test_gcn_norm_adj_at_300k_nodes_with_a_hub():
    n = 300000
    ei = random_graph(n, 1500000, seed=23, symmetric=True, isolated=11, hub=(12345, 60000))
    w = (np.random.RandomState(24).rand(ei.shape[1]) + 0.05).astype(F32)
    want = o.gcn_norm_adj(o.SparseMatrix(ei, w, [n, n]), "both", True, True, True, False)
    got = tfg.nn.gcn_norm_adj(tfg.SparseMatrix(ei, w, [n, n]), "both", True, True, True, False)
    assert_bits(host(got.index), want.index.astype(np.int32), "index")
    np.testing.assert_allclose(host(got.value), want.value, rtol=6e-7, atol=0)


# ---- colsum ----------------------------------------------------------------------------------------------------------

def _sm():
    return ops.device_info()["sm_count"]


def _colsum_cases():
    for n in (0, 1, 511, 512, 513, "4096sm+1", 2500000):
        for d in (1, 3, 100, 255, 256, 257, 1000):
            if n == 2500000 and d == 1000:
                continue                                          # 10 GB of x: the 2.5 M-row cases stop at D = 257
            yield n, d


@pytest.mark.parametrize("n,d", list(_colsum_cases()))
def test_colsum_within_bound_and_bit_stable(n, d):
    if n == "4096sm+1":
        n = 4096 * _sm() + 1
    g = torch.Generator(device="cuda").manual_seed(n * 7 + d)
    wide = torch.empty((n, d + 5), dtype=torch.float32, device="cuda")
    x = wide[:, 2:2 + d]
    x.copy_(torch.randn((n, d), generator=g, device="cuda") * 3.0 + torch.linspace(-50, 50, d, device="cuda"))
    xc = x.contiguous()
    got = ops.colsum(xc)
    if n == 0:
        assert_bits(host(got), np.zeros(d, F32), "empty")
        return
    # float64 reference and sum |x|, in row chunks
    exact = torch.zeros(d, dtype=torch.float64, device="cuda")
    mag = torch.zeros(d, dtype=torch.float64, device="cuda")
    for r0 in range(0, n, 1 << 18):
        c = xc[r0:r0 + (1 << 18)].double()
        exact += c.sum(0)
        mag += c.abs().sum(0)
    err = (got.double() - exact).abs().cpu().numpy()
    bound = R.colsum_bound(mag.cpu().numpy(), n)
    assert np.all(err <= bound), "max err/bound {}".format((err / bound).max())
    assert_bits(host(ops.colsum(xc)), host(got), "run to run")
    assert_bits(host(ops.colsum(x)), host(got), "column slice (ldx = {}) vs contiguous".format(d + 5))


# ---- l2_normalize ----------------------------------------------------------------------------------------------------

@pytest.mark.parametrize("d", [1, 31, 32, 33, 100, 128, 602])
def test_l2_normalize_within_bound(d):
    n = 1001
    rs = np.random.RandomState(d)
    xv = (rs.randn(n, d) * 10.0 ** rs.randint(-3, 4, (n, 1))).astype(F32)
    x_wide = torch.full((n, d + 3), 7.0, dtype=torch.float32, device="cuda")
    x_wide[:, 1:1 + d] = dev(xv)
    out_wide = torch.full((n, d + 5), 3.0, dtype=torch.float32, device="cuda")
    ops.l2_normalize(x_wide[:, 1:1 + d], out=out_wide[:, 2:2 + d])
    ow = host(out_wide)
    assert np.all(ow[:, :2] == 3.0) and np.all(ow[:, 2 + d:] == 3.0), "writes outside the output columns"
    got = ow[:, 2:2 + d].astype(np.float64)
    x64 = xv.astype(np.float64)
    y = x64 / np.sqrt(np.maximum((x64 * x64).sum(axis=1, keepdims=True), 1e-12))
    b = R.l2_bound(d)
    assert np.all(np.abs(got - y) <= b * np.abs(y)), "max rel err {}".format((np.abs(got - y) / np.abs(y)).max())
    # the fp32 oracle: its own sum of squares (pairwise) is within gamma_{log2 D + 2} / 2 + 1.5 ulp of float64
    want = o.l2_normalize(xv).astype(np.float64)
    b_oracle = R.gamma(int(np.ceil(np.log2(d))) + 2) / 2 + 1.5 * 2.0 ** -23
    assert np.all(np.abs(got - want) <= (b + b_oracle) * np.abs(y))


@pytest.mark.filterwarnings("ignore::RuntimeWarning")
def test_l2_normalize_edge_cases():
    d = 40
    xv = np.random.RandomState(1).randn(6, d).astype(F32)
    xv[0] = 0.0                                                   # zero row -> exact zeros
    xv[1] = 1e20                                                  # sum of squares overflows fp32 -> zeros
    xv[2, 5] = np.inf                                             # inf entry -> NaN there, zeros elsewhere
    xv[3] = F32(2.0 ** -21)                                       # sum 40 * 2^-42 = 9.1e-12: above the clamp
    xv[4] = 0.0
    xv[4, :4] = F32(2.0 ** -21)                                   # sum 4 * 2^-42 = 9.1e-13 < 1e-12: clamped
    xv[5] = 0.0
    xv[5, 7] = F32(-2.0 ** -30)                                   # far below the clamp
    got = host(ops.l2_normalize(dev(xv)))
    want = o.l2_normalize(xv)
    assert_bits(got[0], np.zeros(d, F32), "zero row")
    assert_bits(got[1], np.zeros(d, F32), "overflowing row (fp32 semantics)")
    assert_bits(want[1], np.zeros(d, F32), "the fp32 oracle gives zeros too")
    assert np.isnan(got[2, 5]) and np.isnan(want[2, 5])
    assert_bits(np.delete(got[2], 5), (np.delete(xv[2], 5) * F32(0)).astype(F32), "finite entries of the inf row")
    assert_bits(np.delete(got[2], 5), np.delete(want[2], 5), "inf row against the oracle")
    # below the clamp: out = x * rsqrtf(1e-12); with power-of-two x the product is exact, so out / x is that constant
    c = F32(got[4, 0] / xv[4, 0])
    assert_bits(got[4, :4], (xv[4, :4] * c).astype(F32), "clamped row")
    assert_bits(got[4, 4:], np.zeros(d - 4, F32), "clamped row zeros")
    assert got[5, 7] == F32(xv[5, 7] * c), "every clamped row uses the same factor"
    exact_c = 1.0 / np.sqrt(np.float64(F32(1e-12)))
    assert abs(float(c) - exact_c) <= 2 * np.spacing(F32(exact_c)), "rsqrtf(1e-12) within 2 ulp"
    # the row just above the clamp is normalised by its own sum
    y3 = xv[3].astype(np.float64) / np.sqrt((xv[3].astype(np.float64) ** 2).sum())
    assert np.all(np.abs(got[3] - y3) <= R.l2_bound(d) * np.abs(y3))
