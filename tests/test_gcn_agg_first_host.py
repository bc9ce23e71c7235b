# coding=utf-8
"""Aggregate-then-project GCN without a GPU: tfgk_spmm_proj_f32 is exported with the header's arity and validates its
arguments, and the GCN inference route is taken exactly for the shapes the entry supports (checked on the CPU test double
with a numpy stand-in for the kernel)."""
import ctypes
import os
import re

import numpy as np
import pytest
import torch

import fake_backend
from tf_geometric_b200 import _ffi, ops
import tf_geometric_b200 as tfg

NAME = "tfgk_spmm_proj_f32"


def _header_arity(name):
    header = open(os.path.join(os.path.dirname(__file__), "..", "include", "tfgk.h")).read()
    m = re.search(r"int {}\(([^;]*)\);".format(name), header)
    assert m, name
    return len(m.group(1).split(","))


def test_symbol_is_exported_with_the_header_arity():
    assert hasattr(_ffi.lib(), NAME)
    assert len(_ffi.SIGNATURES[NAME]) == _header_arity(NAME) == 15


def _status(*args):
    with pytest.raises(_ffi.TfgkError) as err:
        _ffi.call(NAME, *args)
    return err.value


def test_validates_arguments_before_any_device_work():
    fake = ctypes.c_void_p(256)
    #       rowptr col   w     x     ldx  n  F    W     U    bias  act out   ldo  plan  stream
    base = [fake, fake, None, fake, 100, 8, 100, fake, 128, None, 0, fake, 128, None, None]
    bad = list(base)
    bad[5] = -1
    assert "negative size" in str(_status(*bad))
    bad = list(base)
    bad[10] = 5
    assert "activation" in str(_status(*bad))
    bad = list(base)
    bad[12] = 100
    assert "leading dimension" in str(_status(*bad))
    bad = list(base)
    bad[0] = None
    assert "null pointer" in str(_status(*bad))
    # shapes outside 4 <= F < U <= 128, F % 4 == 0, ldx % 4 == 0, 16-byte aligned x: TFGK_ERR_UNSUPPORTED
    for i, v in ((6, 128), (6, 102), (6, 2), (8, 200), (8, 100), (4, 102), (3, ctypes.c_void_p(260))):
        bad = list(base)
        bad[i] = v
        if i == 6:
            bad[4] = max(v, 100)
        assert _status(*bad).code == _ffi.ERR_UNSUPPORTED, (i, v)
    bad = list(base)
    bad[5] = 0
    assert _ffi.call(NAME, *bad) == _ffi.OK                          # nothing to do


class _CudaLike(object):
    """What spmm_proj_supported reads of a tensor, for a 'CUDA' tensor on a machine without one."""

    def __init__(self, shape, ld=None, ptr=0, dtype=torch.float32):
        self.shape, self.dtype, self.is_cuda = tuple(shape), dtype, True
        self._ld, self._ptr = shape[-1] if ld is None else ld, ptr

    def dim(self):
        return len(self.shape)

    def stride(self, i=None):
        s = (self._ld, 1)
        return s if i is None else s[i]

    def data_ptr(self):
        return self._ptr


@pytest.mark.parametrize("F,U,ld,ptr,routed", [
    (100, 128, None, 0, True), (4, 8, None, 0, True), (124, 128, None, 0, True), (100, 128, 108, 0, True),
    (128, 128, None, 0, False), (100, 100, None, 0, False), (130, 256, None, 0, False), (102, 128, None, 0, False),
    (2, 8, None, 0, False), (64, 200, None, 0, False), (100, 128, 102, 0, False), (100, 128, None, 4, False)])
def test_route_predicate(F, U, ld, ptr, routed):
    assert ops.spmm_proj_supported(_CudaLike((10, F), ld, ptr), _CudaLike((F, U))) == routed
    assert not ops.spmm_proj_supported(_CudaLike((10, F), ld, ptr, dtype=torch.float64), _CudaLike((F, U)))
    assert not ops.spmm_proj_supported(torch.zeros((10, F)), torch.zeros((F, U)))     # host tensors never take it


@pytest.fixture
def fake_proj(monkeypatch):
    """The CPU test double, with the aggregate-first entry replaced by a numpy stand-in that records its calls."""
    fake_backend.install(monkeypatch)
    calls = []

    def supported(x, W):
        return x.dim() == 2 and W.dim() == 2 and W.shape[0] == x.shape[1] and 4 <= x.shape[1] < W.shape[1] <= 128 and \
            x.shape[1] % 4 == 0

    def spmm_proj(csr, w_csr, x, W, bias=None, act=ops.ACT_NONE, out=None):
        calls.append((tuple(x.shape), tuple(W.shape)))
        rowptr, col = csr.rowptr.numpy(), csr.col.numpy()
        w = np.ones(len(col)) if w_csr is None else w_csr.numpy().astype(np.float64)
        xh = x.numpy().astype(np.float64)
        agg = np.stack([(w[rowptr[r]:rowptr[r + 1], None] * xh[col[rowptr[r]:rowptr[r + 1]]]).sum(0)
                        for r in range(len(rowptr) - 1)])
        h = agg @ W.numpy().astype(np.float64) + (0.0 if bias is None else bias.numpy())
        if act == ops.ACT_RELU:
            h = np.maximum(h, 0.0)
        return torch.from_numpy(h.astype(np.float32))

    monkeypatch.setattr(ops, "spmm_proj_supported", supported)
    monkeypatch.setattr(ops, "spmm_proj", spmm_proj)
    yield calls
    from tf_geometric_b200 import _structure
    _structure.clear()


def _graph(n=60, e=400, f=12, seed=0):
    rs = np.random.RandomState(seed)
    ei = rs.randint(0, n, (2, e)).astype(np.int32)
    return rs.randn(n, f).astype(np.float32), ei


@pytest.mark.parametrize("units,splits,routed", [(16, None, True), (12, None, False), (8, None, False),
                                                 (200, None, False), (16, 2, False)])
def test_gcn_inference_takes_the_route_for_supported_shapes(fake_proj, units, splits, routed):
    x, ei = _graph()
    n = x.shape[0]
    rs = np.random.RandomState(1)
    W = rs.randn(x.shape[1], units).astype(np.float32)
    b = rs.randn(units).astype(np.float32)
    adj = tfg.SparseMatrix(ei, None, [n, n])
    got = tfg.nn.gcn(x, adj, W, b, activation=tfg.nn.relu, num_or_size_splits=splits, cache={})
    assert len(fake_proj) == (1 if routed else 0)
    # both routes compute act(norm(A) x W + b): compare with float64
    normed = tfg.nn.conv.gcn.gcn_norm_adj(adj, cache=None)
    A = np.zeros((n, n))
    np.add.at(A, (normed.index[0].numpy(), normed.index[1].numpy()), normed.value.numpy().astype(np.float64))
    want = np.maximum(A @ x.astype(np.float64) @ W.astype(np.float64) + b, 0.0)
    np.testing.assert_allclose(got.numpy(), want, rtol=1e-5, atol=1e-5)


def test_training_and_other_message_dtypes_keep_their_routes(fake_proj):
    x, ei = _graph()
    n = x.shape[0]
    W = torch.randn(12, 16, requires_grad=True)
    adj = tfg.SparseMatrix(ei, None, [n, n])
    tfg.nn.gcn(torch.from_numpy(x), adj, W, None, cache={})
    assert fake_proj == []
