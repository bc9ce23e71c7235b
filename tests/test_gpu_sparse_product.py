# coding=utf-8
"""SparseMatrix @ SparseMatrix on the H100: the product is K10's (bit-identical to ops.spgemm and to the numpy Gustavson
restatement, whatever requires grad and whatever the chunking); K12, its gradient in both operands' values, is
bit-identical to the numpy restatement of tests/spgemm_grad_ref.py (duplicates, exact zeros, NaN and inf in dC, a B row
and an A column of 60 000 entries, a C pattern with missing entries), identical across runs, and within a stated bound
of float64; gradients flow through (A @ B) @ h and through the reference's normalisation diags(d) @ A @ diags(d)."""
import numpy as np
import pytest
import scipy.sparse as sp
import torch

import asap_fake_backend as fake_k10
import spgemm_grad_ref as ref
from conftest import assert_close

pytestmark = pytest.mark.gpu

DEV = "cuda"


def _dev(a, dtype=None):
    t = torch.as_tensor(np.ascontiguousarray(a), device=DEV)
    return t if dtype is None else t.to(dtype)


def _coo(rs, n_rows, n_cols, nnz, dup=0, zeros=0):
    r, c = rs.randint(0, n_rows, nnz), rs.randint(0, n_cols, nnz)
    if dup:
        r, c = np.concatenate([r, r[:dup]]), np.concatenate([c, c[:dup]])
    order = rs.permutation(len(r))
    v = rs.uniform(-1, 1, len(r)).astype(np.float32)
    v[:zeros] = 0.0
    return np.stack([r[order], c[order]]).astype(np.int32), v


def _csr_arrays(M):
    """(rowptr, col, values in CSR order) of a SparseMatrix, as numpy."""
    return M.csr.rowptr.cpu().numpy(), M.csr.col.cpu().numpy(), M.value_csr.cpu().numpy()


def _dense64(index, value, shape):
    out = torch.zeros(shape, dtype=torch.float64)
    return out.index_put((torch.as_tensor(index[0]).long(), torch.as_tensor(index[1]).long()), value, accumulate=True)


# ---- the forward: K10 ----------------------------------------------------------------------------------------------

def test_product_is_k10_bit_for_bit():
    import tf_geometric_b200 as tfg
    from tf_geometric_b200 import ops
    rs = np.random.RandomState(0)
    ai, av = _coo(rs, 300, 200, 2000, dup=50, zeros=20)
    bi, bv = _coo(rs, 200, 250, 1500, dup=40, zeros=20)
    A, B = tfg.SparseMatrix(_dev(ai), _dev(av), [300, 200]), tfg.SparseMatrix(_dev(bi), _dev(bv), [200, 250])
    C = A @ B
    assert C.shape == [300, 250] and C.index.dtype == torch.int32
    a, b = _csr_arrays(A), _csr_arrays(B)
    want = fake_k10.spgemm_reference(*a, *b, 250)
    ci = C.index.cpu().numpy()
    np.testing.assert_array_equal(ci[0], np.repeat(np.arange(300), np.diff(want[0])))
    np.testing.assert_array_equal(ci[1], want[1])
    np.testing.assert_array_equal(C.value.cpu().numpy(), want[2])
    for budget in (None, 0, 97):
        kw = {} if budget is None else {"budget": budget}
        got = ops.spgemm(A.csr.rowptr, A.csr.col, A.value_csr, B.csr.rowptr, B.csr.col, B.value_csr, 250, **kw)
        assert torch.equal(got[0], C.csr.rowptr) and torch.equal(got[1], C.csr.col) and torch.equal(got[2], C.value)
    # requires_grad changes no bit; the prebuilt CSR has the identity permutation
    Ag = tfg.SparseMatrix(_dev(ai), _dev(av).requires_grad_(), [300, 200])
    Bg = tfg.SparseMatrix(_dev(bi), _dev(bv).requires_grad_(), [200, 250])
    Cg = Ag @ Bg
    assert Cg.value.requires_grad and torch.equal(Cg.value.detach(), C.value) and torch.equal(Cg.index, C.index)
    assert torch.equal(C.csr.perm.cpu(), torch.arange(C.nnz, dtype=torch.int32))
    # a following C @ h uses the prebuilt CSR
    h = _dev(rs.randn(250, 16).astype(np.float32))
    assert torch.equal(C @ h, ops.spmm(C.csr, C.value, h))


# ---- K12 against its restatement -----------------------------------------------------------------------------------

def _grad_both(mode, x, y, c_rowptr, c_col, g, m, k, n, perm=None):
    from tf_geometric_b200 import ops
    args = [_dev(v) for v in (x[0], x[1], y[0], y[1], y[2], c_rowptr, c_col, g)]
    got = ops.spgemm_grad(mode, *args, m, k, n, perm=None if perm is None else _dev(perm))
    again = ops.spgemm_grad(mode, *args, m, k, n, perm=None if perm is None else _dev(perm))
    assert torch.equal(got.view(torch.int32), again.view(torch.int32))            # the same bits, NaN included
    want = ref.spgemm_grad_reference(mode, x[0], x[1], y[0], y[1], y[2], c_rowptr, c_col, g, perm)
    np.testing.assert_array_equal(got.cpu().numpy(), want, err_msg=mode)
    return got.cpu().numpy()


def _csr(index, value, shape):
    """(rowptr, col, values, perm) of a COO matrix, stable by row as the CSR build is; perm[p] = COO position of slot p."""
    order = np.argsort(index[0], kind="stable")
    rowptr = np.zeros(shape[0] + 1, np.int64)
    rowptr[1:] = np.cumsum(np.bincount(index[0], minlength=shape[0]))
    return rowptr, index[1][order].astype(np.int32), value[order].astype(np.float32), order.astype(np.int32)


def _k12_case(ai, av, bi, bv, m, k, n, g_fn):
    a = _csr(ai, av, (m, k))
    b = _csr(bi, bv, (k, n))
    at = _csr(ai[::-1].copy(), av, (k, m))
    c_rowptr, c_col, _ = fake_k10.spgemm_reference(a[0], a[1], a[2], b[0], b[1], b[2], n)
    g = g_fn(len(c_col))
    dA = _grad_both("left", a, b, c_rowptr, c_col, g, m, k, n, perm=a[3])
    dB = _grad_both("right", b, at, c_rowptr, c_col, g, m, k, n, perm=b[3])
    return dA, dB, c_rowptr, c_col, g


def test_k12_duplicates_zeros_and_non_finite_gradients():
    rs = np.random.RandomState(1)
    ai, av = _coo(rs, 400, 300, 3000, dup=100, zeros=30)
    bi, bv = _coo(rs, 300, 350, 2500, dup=80, zeros=30)

    def g_fn(nnz):
        g = rs.randn(nnz).astype(np.float32)
        g[rs.choice(nnz, 30, replace=False)] = np.array([np.nan, np.inf, -np.inf] * 10, np.float32)
        return g

    dA, dB, *_ = _k12_case(ai, av, bi, bv, 400, 300, 350, g_fn)
    assert np.isnan(dA).any() and np.isnan(dB).any() and np.isfinite(dA).any()
    # finite dC: against float64 dense autograd
    dA, dB, c_rowptr, c_col, g = _k12_case(ai, av, bi, bv, 400, 300, 350, lambda nnz: rs.randn(nnz).astype(np.float32))
    a64, b64 = torch.tensor(av, dtype=torch.float64, requires_grad=True), torch.tensor(bv, dtype=torch.float64,
                                                                                        requires_grad=True)
    c64 = _dense64(ai, a64, (400, 300)) @ _dense64(bi, b64, (300, 350))
    rows = np.repeat(np.arange(400), np.diff(c_rowptr))
    (c64[rows, c_col] * torch.tensor(g, dtype=torch.float64)).sum().backward()
    assert_close(dA, a64.grad.numpy(), rtol=1e-5, what="dA")
    assert_close(dB, b64.grad.numpy(), rtol=1e-5, what="dB")


def test_k12_hub_rows_of_60000_entries():
    """B's row 5 and A's column 7 hold 60 000 entries each: every A entry of column 5 (left) and every B entry of row 7
    (right) walks 60 000 entries, in 938 slices.  Against scipy float64 (dC B^T) and (A^T dC) sampled on the patterns,
    within 1e-4 of the sum of the terms' magnitudes: sequential fp32 sums over slices of 64 and then over at most 938
    slice sums have a relative error below (64 + 938) * 2^-24 < 1e-4 of that sum."""
    rs = np.random.RandomState(2)
    m, k, n, hub = 70000, 1000, 70000, 60000
    ai, av = _coo(rs, m, k, 20000, dup=200)
    ai = np.concatenate([ai, np.stack([rs.permutation(m)[:hub], np.full(hub, 7)]).astype(np.int32)], 1)
    av = np.concatenate([av, rs.uniform(-1, 1, hub).astype(np.float32)])
    ai[1, :40] = 5                                             # column 5 of A: about 40 entries walking B's hub row
    bi, bv = _coo(rs, k, n, 20000, dup=200)
    bi = np.concatenate([bi, np.stack([np.full(hub, 5), rs.permutation(n)[:hub]]).astype(np.int32)], 1)
    bv = np.concatenate([bv, rs.uniform(-1, 1, hub).astype(np.float32)])
    bi[0, :40] = 7                                             # row 7 of B: about 40 entries walking A's hub column
    dA, dB, c_rowptr, c_col, g = _k12_case(ai, av, bi, bv, m, k, n, lambda nnz: rs.randn(nnz).astype(np.float32))
    G = sp.csr_matrix((g.astype(np.float64), c_col, c_rowptr), shape=(m, n))
    A = sp.csr_matrix((av.astype(np.float64), (ai[0], ai[1])), shape=(m, k))
    B = sp.csr_matrix((bv.astype(np.float64), (bi[0], bi[1])), shape=(k, n))
    for got, full, mag, idx in ((dA, G @ B.T, abs(G) @ abs(B).T, ai), (dB, A.T @ G, abs(A).T @ abs(G), bi)):
        want = np.asarray(full.tocsr()[idx[0], idx[1]]).ravel()
        bound = np.asarray(mag.tocsr()[idx[0], idx[1]]).ravel()
        assert np.all(np.abs(got - want) <= 1e-4 * bound + 1e-30), np.abs(got - want).max()


def test_k12_missing_entries_of_c_contribute_zero():
    """A hand-made C: half the product's entries dropped and columns the product does not have added."""
    rs = np.random.RandomState(3)
    ai, av = _coo(rs, 200, 150, 1500, dup=20)
    bi, bv = _coo(rs, 150, 180, 1200, dup=20)
    a, b = _csr(ai, av, (200, 150)), _csr(bi, bv, (150, 180))
    at = _csr(ai[::-1].copy(), av, (150, 200))
    rp, col, _ = fake_k10.spgemm_reference(a[0], a[1], a[2], b[0], b[1], b[2], 180)
    rows, cols = [], []
    for i in range(200):
        keep = col[rp[i]:rp[i + 1]][rs.rand(rp[i + 1] - rp[i]) < 0.5]
        extra = np.setdiff1d(rs.choice(180, 5), col[rp[i]:rp[i + 1]])
        c = np.union1d(keep, extra)
        rows.append(np.full(len(c), i))
        cols.append(c)
    rows, cols = np.concatenate(rows), np.concatenate(cols).astype(np.int32)
    c_rowptr = np.zeros(201, np.int64)
    c_rowptr[1:] = np.cumsum(np.bincount(rows, minlength=200))
    g = rs.randn(len(cols)).astype(np.float32)
    dA = _grad_both("left", a, b, c_rowptr, cols, g, 200, 150, 180, perm=a[3])
    dB = _grad_both("right", b, at, c_rowptr, cols, g, 200, 150, 180, perm=b[3])
    G = sp.csr_matrix((g.astype(np.float64), cols, c_rowptr), shape=(200, 180))
    A = sp.csr_matrix((av.astype(np.float64), (ai[0], ai[1])), shape=(200, 150))
    B = sp.csr_matrix((bv.astype(np.float64), (bi[0], bi[1])), shape=(150, 180))
    assert_close(dA, np.asarray((G @ B.T).tocsr()[ai[0], ai[1]]).ravel(), rtol=1e-5, what="dA")
    assert_close(dB, np.asarray((A.T @ G).tocsr()[bi[0], bi[1]]).ravel(), rtol=1e-5, what="dB")


def test_k12_rejects_out_of_range_columns():
    from tf_geometric_b200 import ops, _ffi
    x = (np.array([0, 1], np.int64), np.array([3], np.int32))               # A [1, 2]: column 3 is outside [0, 2)
    y = (np.array([0, 1, 1], np.int64), np.array([0], np.int32), np.ones(1, np.float32))
    c = (np.array([0, 1], np.int64), np.array([0], np.int32), np.ones(1, np.float32))
    with pytest.raises(_ffi.TfgkError) as err:
        ops.spgemm_grad("left", *[_dev(v) for v in x + y + c], 1, 2, 1)
    assert err.value.code == _ffi.ERR_INDEX_OUT_OF_RANGE
    x = (np.array([0, 1], np.int64), np.array([0], np.int32))               # A [1, 1]
    y = (np.array([0, 1], np.int64), np.array([4], np.int32), np.ones(1, np.float32))   # B [1, 1]: column 4
    with pytest.raises(_ffi.TfgkError) as err:
        ops.spgemm_grad("left", *[_dev(v) for v in x + y + c], 1, 1, 1)
    assert err.value.code == _ffi.ERR_INDEX_OUT_OF_RANGE
    with pytest.raises(ValueError, match="rowptr"):
        ops.spgemm_grad("right", *[_dev(v) for v in x + y + c], 3, 1, 1)


# ---- the public product --------------------------------------------------------------------------------------------

def test_gradient_through_a_composition():
    """(A @ B) @ h with trainable A, B and h: K7 gives C's value gradient, K12 takes it to A's and B's values."""
    import tf_geometric_b200 as tfg
    rs = np.random.RandomState(4)
    ai, av = _coo(rs, 120, 90, 800, dup=30)
    bi, bv = _coo(rs, 90, 110, 700, dup=30)
    hv = rs.randn(110, 24).astype(np.float32)
    at, bt, ht = _dev(av).requires_grad_(), _dev(bv).requires_grad_(), _dev(hv).requires_grad_()
    y = (tfg.SparseMatrix(_dev(ai), at, [120, 90]) @ tfg.SparseMatrix(_dev(bi), bt, [90, 110])) @ ht
    gy = rs.randn(120, 24)
    (y * _dev(gy, torch.float32)).sum().backward()
    a64, b64, h64 = (torch.tensor(v, dtype=torch.float64, requires_grad=True) for v in (av, bv, hv))
    y64 = _dense64(ai, a64, (120, 90)) @ _dense64(bi, b64, (90, 110)) @ h64
    (y64 * torch.tensor(gy)).sum().backward()
    assert_close(y.detach().cpu().numpy(), y64.detach().numpy(), rtol=1e-5, what="y")
    for name, got, want in (("A", at, a64), ("B", bt, b64), ("h", ht, h64)):
        assert_close(got.grad.cpu().numpy(), want.grad.numpy(), rtol=1e-4, what="d " + name)


def test_reference_normalisation_with_diags_matches_gcn_norm_adj():
    """diags(d) @ A.add_diag(1.0) @ diags(d), d = deg^-1/2 of A + I (gcn.py:83-94), gives gcn_norm_adj(A)'s entries:
    the same (row, col) set and values within 2 ulp."""
    import tf_geometric_b200 as tfg
    rs = np.random.RandomState(5)
    n = 3000
    r, c = rs.randint(0, n, 20000), rs.randint(0, n, 20000)
    keep = r != c
    pairs = np.unique(np.stack([np.concatenate([r[keep], c[keep]]), np.concatenate([c[keep], r[keep]])]), axis=1)
    ei = pairs[:, rs.permutation(pairs.shape[1])].astype(np.int32)
    w = rs.uniform(0.5, 1.5, ei.shape[1]).astype(np.float32)
    A = tfg.SparseMatrix(_dev(ei), _dev(w), [n, n])
    norm = tfg.nn.gcn_norm_adj(A)
    from tf_geometric_b200 import ops
    loops = A.add_diag(1.0)
    d = ops.deg_inv(loops.segment_sum(axis=-1), ops.POW_INV_SQRT)
    P = tfg.sparse.diags(d) @ loops @ tfg.sparse.diags(d)
    ni, nv = norm.index.cpu().numpy(), norm.value.cpu().numpy()
    order = np.lexsort((ni[1], ni[0]))
    np.testing.assert_array_equal(P.index.cpu().numpy(), ni[:, order])
    want, got = nv[order], P.value.cpu().numpy()
    assert np.all(np.abs(got - want) <= 2 * np.spacing(np.abs(want))), np.abs(got - want).max()
    # and it is differentiable in d and in A's values
    wt = _dev(w).requires_grad_()
    dt = d.clone().requires_grad_()
    P = tfg.sparse.diags(dt) @ tfg.SparseMatrix(_dev(ei), wt, [n, n]).add_diag(1.0) @ tfg.sparse.diags(dt)
    assert P.value.requires_grad


def test_errors():
    import tf_geometric_b200 as tfg
    rs = np.random.RandomState(6)
    ai, av = _coo(rs, 10, 8, 30)
    bi, bv = _coo(rs, 9, 7, 30)
    A, B = tfg.SparseMatrix(_dev(ai), _dev(av), [10, 8]), tfg.SparseMatrix(_dev(bi), _dev(bv), [9, 7])
    with pytest.raises(ValueError, match="inner dimensions"):
        A @ B
    B = tfg.SparseMatrix(_dev(bi[:, bi[0] < 8]), _dev(bv[bi[0] < 8]), [8, 7])
    with pytest.raises(TypeError):
        A.matmul(B, num_or_size_splits=7)
    with pytest.raises(TypeError):
        A.matmul(B, act=1)
    Bc = tfg.SparseMatrix(torch.tensor(bi[:, bi[0] < 8]), torch.tensor(bv[bi[0] < 8]), [8, 7])
    Bc.index, Bc.value = Bc.index.cpu(), Bc.value.cpu()
    with pytest.raises(ValueError, match="operands on"):
        A @ Bc
