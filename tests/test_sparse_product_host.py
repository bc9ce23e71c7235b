# coding=utf-8
"""SparseMatrix @ SparseMatrix and its gradient in both operands' values without a GPU: the host logic over the CPU fake
of the kernel layer, with the numpy K10 of tests/asap_fake_backend.py and the numpy K12 of tests/spgemm_grad_ref.py,
against float64 dense autograd over to_dense(A) @ to_dense(B)."""
import ctypes

import numpy as np
import pytest
import torch

import spgemm_grad_ref
from conftest import assert_close


@pytest.fixture
def fake(monkeypatch):
    spgemm_grad_ref.install(monkeypatch)
    import tf_geometric_b200 as tfg
    return tfg


def _coo(rs, n_rows, n_cols, nnz, dup=0, empty_rows=(), empty_cols=()):
    """COO (index int32 [2, nnz], values float32) in shuffled order, `dup` repeated (row, col) pairs, the given rows and
    columns empty."""
    rows = np.setdiff1d(np.arange(n_rows), empty_rows)
    cols = np.setdiff1d(np.arange(n_cols), empty_cols)
    r, c = rs.choice(rows, nnz), rs.choice(cols, nnz)
    if dup:
        r, c = np.concatenate([r, r[:dup]]), np.concatenate([c, c[:dup]])
    order = rs.permutation(len(r))
    return np.stack([r[order], c[order]]).astype(np.int32), rs.uniform(-1, 1, len(r)).astype(np.float32)


def _dense64(index, value, shape):
    out = torch.zeros(shape, dtype=torch.float64)
    return out.index_put((torch.as_tensor(index[0]).long(), torch.as_tensor(index[1]).long()), value, accumulate=True)


def _check_product(tfg, a, b, rs, same=False):
    """a, b: (index, values, shape).  C = A @ B against float64 dense: pattern, values, and dA / dB for a random dC."""
    (ai, av, ash), (bi, bv, bsh) = a, b
    if same:                                                  # B = A.transpose(), sharing A's value tensor
        bi, bv = ai[::-1].copy(), av
    at = torch.tensor(av, requires_grad=True)
    bt = at if same else torch.tensor(bv, requires_grad=True)
    A = tfg.SparseMatrix(torch.tensor(ai), at, ash)
    B = tfg.SparseMatrix(torch.tensor(bi), bt, bsh) if not same else A.transpose()
    C = A @ B
    assert isinstance(C, tfg.SparseMatrix) and C.shape == [ash[0], bsh[1]]
    assert C.index.dtype == torch.int32
    ci = C.index.numpy()
    # row-major, ascending unique columns per row: the structural pattern of the product
    key = ci[0].astype(np.int64) * bsh[1] + ci[1]
    assert np.all(np.diff(key) > 0)
    pat = (_dense64(ai, torch.ones(ai.shape[1], dtype=torch.float64), ash) != 0).double() @ \
        (_dense64(bi, torch.ones(bi.shape[1], dtype=torch.float64), bsh) != 0).double()
    np.testing.assert_array_equal(np.stack(np.nonzero(pat.numpy())), ci)
    # the prebuilt CSR: identity permutation
    np.testing.assert_array_equal(C.csr.perm.numpy(), np.arange(C.nnz))
    np.testing.assert_array_equal(C.csr.col.numpy(), ci[1])

    a64 = torch.tensor(av, dtype=torch.float64, requires_grad=True)
    b64 = a64 if same else torch.tensor(bv, dtype=torch.float64, requires_grad=True)
    c64 = _dense64(ai, a64, ash) @ _dense64(bi, b64, bsh)
    want = c64[ci[0], ci[1]]
    assert_close(C.value.detach().numpy(), want.detach().numpy(), rtol=1e-5, what="C")
    g = rs.randn(C.nnz)
    (C.value * torch.tensor(g, dtype=torch.float32)).sum().backward()
    (want * torch.tensor(g)).sum().backward()
    assert_close(at.grad.numpy(), a64.grad.numpy(), rtol=1e-4, what="dA")
    if not same:
        assert_close(bt.grad.numpy(), b64.grad.numpy(), rtol=1e-4, what="dB")
    return C


# ---- the ABI and the argument checks, before any device work -----------------------------------------------------

def test_k12_is_exported_with_the_declared_arity():
    from tf_geometric_b200 import _ffi
    lib = _ffi.lib()
    for name, n_args in (("tfgk_spgemm_grad_workspace_bytes", 2), ("tfgk_spgemm_grad_plan", 14),
                         ("tfgk_spgemm_grad_f32", 19)):
        assert hasattr(lib, name)
        assert len(_ffi.SIGNATURES[name]) == n_args
    assert _ffi.ABI_VERSION == 7


def test_k12_validates_without_gpu():
    from tf_geometric_b200 import _ffi
    need = ctypes.c_size_t()
    _ffi.call("tfgk_spgemm_grad_workspace_bytes", 1000, ctypes.byref(need))
    assert need.value >= 1000 * 8
    with pytest.raises(_ffi.TfgkError) as err:
        _ffi.call("tfgk_spgemm_grad_workspace_bytes", -1, ctypes.byref(need))
    assert err.value.code == _ffi.ERR_INVALID_ARGUMENT
    n = ctypes.c_int64()
    with pytest.raises(_ffi.TfgkError) as err:
        _ffi.call("tfgk_spgemm_grad_plan", 2, None, None, 0, None, None, 1, 1, 1, None, ctypes.byref(n), None, 0, None)
    assert err.value.code == _ffi.ERR_INVALID_ARGUMENT and "mode" in str(err.value)
    with pytest.raises(_ffi.TfgkError) as err:
        _ffi.call("tfgk_spgemm_grad_plan", 0, None, None, 0, None, None, -1, 1, 1, None, ctypes.byref(n), None, 0, None)
    assert err.value.code == _ffi.ERR_INVALID_ARGUMENT
    with pytest.raises(_ffi.TfgkError) as err:
        _ffi.call("tfgk_spgemm_grad_f32", 1, None, None, None, 5, None, None, None, 1, 1, 1, None, None, None, None, 0,
                  None, None, None)
    assert err.value.code == _ffi.ERR_INVALID_ARGUMENT and "null" in str(err.value)
    # no entries of X: nothing to compute
    _ffi.call("tfgk_spgemm_grad_f32", 1, None, None, None, 0, None, None, None, 1, 1, 1, None, None, None, None, 0, None,
              None, None)


def test_ops_spgemm_grad_argument_errors():
    from tf_geometric_b200 import ops
    i64, i32, f32 = torch.zeros(2, dtype=torch.int64), torch.zeros(1, dtype=torch.int32), torch.zeros(1)
    with pytest.raises(ValueError, match="mode"):
        ops.spgemm_grad("middle", i64, i32, i64, i32, f32, i64, i32, f32, 1, 1, 1)
    with pytest.raises(TypeError, match="CUDA"):
        ops.spgemm_grad("left", i64, i32, i64, i32, f32, i64, i32, f32, 1, 1, 1)


def test_sparse_operand_errors(fake):
    rs = np.random.RandomState(0)
    ai, av = _coo(rs, 4, 5, 8)
    bi, bv = _coo(rs, 6, 3, 8)
    A, B = fake.SparseMatrix(ai, av, [4, 5]), fake.SparseMatrix(bi, bv, [6, 3])
    with pytest.raises(ValueError, match="inner dimensions"):
        A @ B
    B = fake.SparseMatrix(bi[:, bi[0] < 5], bv[bi[0] < 5], [5, 3])
    with pytest.raises(TypeError, match="num_or_size_splits"):
        A.matmul(B, num_or_size_splits=2)
    with pytest.raises(TypeError, match="epilogue"):
        A.matmul(B, bias=torch.zeros(3))
    meta = fake.SparseMatrix(torch.zeros((2, 1), dtype=torch.int32, device="meta"), torch.zeros(1, device="meta"), [5, 3])
    with pytest.raises(ValueError, match="operands on"):
        A @ meta


def test_products_past_the_int32_index_are_refused(fake, monkeypatch):
    from tf_geometric_b200 import ops
    huge = 2 ** 31

    def spgemm(*args, **kw):
        return (torch.tensor([0, huge], dtype=torch.int64), torch.zeros(1, dtype=torch.int32).expand(huge),
                torch.zeros(1).expand(huge))

    monkeypatch.setattr(ops, "spgemm", spgemm)
    A = fake.SparseMatrix(np.array([[0], [0]], np.int32), np.ones(1, np.float32), [1, 1])
    with pytest.raises(ValueError, match="int32 index"):
        A @ A


# ---- the restatement of K12 --------------------------------------------------------------------------------------

def test_reference_summation_order_and_misses():
    """Slices of the Y row summed from +0 in order, and a C entry that is missing contributes 0."""
    f = np.float32
    y_val = f([1e8, 1.0, -1e8, 1.0, 3.0])
    # left mode, one A entry (0, 0); B's row 0 has five entries in columns 0..4; dC = 1 everywhere
    c_rowptr, c_col = [0, 5], np.arange(5)
    got = spgemm_grad_ref.spgemm_grad_reference("left", [0, 1], [0], [0, 5], np.arange(5), y_val, c_rowptr, c_col,
                                                np.ones(5, f), slice_size=2)
    want = f(0) + (f(1e8) + f(1.0)) + (f(-1e8) + f(1.0)) + f(3.0)       # slices (0, 1), (2, 3), (4)
    assert got[0] == f(f(f(f(1e8) + f(1.0)) + f(f(-1e8) + f(1.0))) + f(3.0)) == want
    whole = spgemm_grad_ref.spgemm_grad_reference("left", [0, 1], [0], [0, 5], np.arange(5), y_val, c_rowptr, c_col,
                                                  np.ones(5, f))
    assert whole[0] == f(f(f(f(f(1e8) + f(1.0)) + f(-1e8)) + f(1.0)) + f(3.0))
    # C without columns 1 and 3: their products are left out, even with an infinite Y value
    y_inf = f([2.0, np.inf, 5.0, -np.inf, 7.0])
    got = spgemm_grad_ref.spgemm_grad_reference("left", [0, 1], [0], [0, 5], np.arange(5), y_inf, [0, 3], [0, 2, 4],
                                                f([1.0, 10.0, 100.0]))
    assert got[0] == f(2 + 50 + 700)


def test_reference_against_float64():
    rs = np.random.RandomState(3)
    import scipy.sparse as sp
    a = sp.random(30, 40, density=0.1, random_state=1, format="csr", dtype=np.float32)
    b = sp.random(40, 25, density=0.2, random_state=2, format="csr", dtype=np.float32)
    import asap_fake_backend
    c_rowptr, c_col, _ = asap_fake_backend.spgemm_reference(a.indptr, a.indices, a.data, b.indptr, b.indices, b.data, 25)
    g = rs.randn(len(c_col)).astype(np.float32)
    G = sp.csr_matrix((g.astype(np.float64), c_col, c_rowptr), shape=(30, 25))
    dA = (G @ b.astype(np.float64).T).toarray()
    got = spgemm_grad_ref.spgemm_grad_reference("left", a.indptr, a.indices, b.indptr, b.indices, b.data, c_rowptr, c_col, g)
    rows = np.repeat(np.arange(30), np.diff(a.indptr))
    assert_close(got, dA[rows, a.indices], rtol=1e-5, what="dA")
    at = a.T.tocsr()
    dB = (a.astype(np.float64).T @ G).toarray()
    got = spgemm_grad_ref.spgemm_grad_reference("right", b.indptr, b.indices, at.indptr, at.indices, at.data, c_rowptr,
                                                c_col, g)
    rows = np.repeat(np.arange(40), np.diff(b.indptr))
    assert_close(got, dB[rows, b.indices], rtol=1e-5, what="dB")


# ---- SparseMatrix @ SparseMatrix against float64 dense autograd ----------------------------------------------------

def test_product_duplicates_empty_rows_and_columns(fake):
    rs = np.random.RandomState(1)
    ai, av = _coo(rs, 30, 20, 120, dup=15, empty_rows=(0, 7), empty_cols=(3, 19))
    bi, bv = _coo(rs, 20, 25, 90, dup=10, empty_rows=(4, 5), empty_cols=(0, 24))
    _check_product(fake, (ai, av, [30, 20]), (bi, bv, [20, 25]), rs)


def test_product_rectangular_and_long_rows(fake):
    """Rows of B and columns of A longer than a slice, so that both gradients sum several slices."""
    rs = np.random.RandomState(2)
    ai, av = _coo(rs, 7, 300, 400)
    ai[1, :150] = 11                                          # column 11 of A: at least 150 entries
    bi, bv = _coo(rs, 300, 5, 500)
    bi[0, :140] = 11                                          # row 11 of B: at least 140 entries
    _check_product(fake, (ai, av, [7, 300]), (bi, bv, [300, 5]), rs)


def test_product_with_its_own_transpose(fake):
    rs = np.random.RandomState(3)
    ai, av = _coo(rs, 25, 18, 100, dup=8)
    _check_product(fake, (ai, av, [25, 18]), (None, None, [18, 25]), rs, same=True)


def test_diags_on_either_side(fake):
    rs = np.random.RandomState(4)
    ai, av = _coo(rs, 12, 12, 50, dup=5)
    d = rs.uniform(0.5, 2.0, 12).astype(np.float32)
    eye = np.stack([np.arange(12), np.arange(12)]).astype(np.int32)
    _check_product(fake, (eye, d, [12, 12]), (ai, av, [12, 12]), rs)
    _check_product(fake, (ai, av, [12, 12]), (eye, d, [12, 12]), rs)
    D = fake.sparse.diags(torch.tensor(d))
    assert D.shape == [12, 12] and D.nnz == 12
    np.testing.assert_array_equal(D.to_dense().numpy(), np.diag(d))
    with pytest.raises(ValueError, match="1-D"):
        fake.sparse.diags(torch.zeros(2, 2))


def test_gcn_normalisation_written_with_diags_is_differentiable(fake):
    """diags(d) @ A @ diags(d) with trainable d and A's values, against float64 dense autograd."""
    rs = np.random.RandomState(5)
    ai, av = _coo(rs, 15, 15, 60)
    d = rs.uniform(0.5, 2.0, 15).astype(np.float32)
    dt, at = torch.tensor(d, requires_grad=True), torch.tensor(av, requires_grad=True)
    C = fake.sparse.diags(dt) @ fake.SparseMatrix(ai, at, [15, 15]) @ fake.sparse.diags(dt)
    d64, a64 = torch.tensor(d, dtype=torch.float64, requires_grad=True), torch.tensor(av, dtype=torch.float64,
                                                                                      requires_grad=True)
    c64 = torch.diag(d64) @ _dense64(ai, a64, [15, 15]) @ torch.diag(d64)
    ci = C.index.numpy()
    want = c64[ci[0], ci[1]]
    assert_close(C.value.detach().numpy(), want.detach().numpy(), rtol=1e-5, what="C")
    g = rs.randn(C.nnz)
    (C.value * torch.tensor(g, dtype=torch.float32)).sum().backward()
    (want * torch.tensor(g)).sum().backward()
    assert_close(dt.grad.numpy(), d64.grad.numpy(), rtol=1e-4, what="d d")
    assert_close(at.grad.numpy(), a64.grad.numpy(), rtol=1e-4, what="d A")


def test_only_the_requested_gradients_are_computed(fake, monkeypatch):
    from tf_geometric_b200 import ops
    rs = np.random.RandomState(6)
    ai, av = _coo(rs, 10, 8, 30)
    bi, bv = _coo(rs, 8, 9, 30)
    modes = []
    inner = ops.spgemm_grad
    monkeypatch.setattr(ops, "spgemm_grad", lambda mode, *a, **k: modes.append(mode) or inner(mode, *a, **k))
    plain = (fake.SparseMatrix(ai, av, [10, 8]) @ fake.SparseMatrix(bi, bv, [8, 9])).value
    assert not plain.requires_grad
    bt = torch.tensor(bv, requires_grad=True)
    C = fake.SparseMatrix(ai, av, [10, 8]) @ fake.SparseMatrix(bi, bt, [8, 9])
    assert torch.equal(C.value.detach(), plain)
    C.value.sum().backward()
    assert modes == ["right"] and bt.grad.shape == (bt.shape[0],)
