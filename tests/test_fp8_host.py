# coding=utf-8
"""fp8 message rows without a GPU: the new entry points are exported with the header's arity and validate their
arguments; GCN and GAT refuse what the fp8 mode does not support before any device work; the exponent rule of the
format holds on hand-picked edge cases; and the GCN / GAT fp8 plumbing runs end to end on the CPU test double."""
import ctypes
import re

import numpy as np
import pytest
import torch

import fp8_fake_backend
import fp8_ref
from tf_geometric_b200 import _ffi, ops
import tf_geometric_b200 as tfg

FP8 = torch.float8_e4m3fn


def _call_err(name, *args):
    with pytest.raises(_ffi.TfgkError) as err:
        _ffi.call(name, *args)
    return err.value


def _header_arity(name):
    import os
    header = open(os.path.join(os.path.dirname(__file__), "..", "include", "tfgk.h")).read()
    m = re.search(r"int {}\(([^;]*)\);".format(name), header)
    assert m, name
    return len(m.group(1).split(","))


def test_symbols_are_exported_with_the_header_arity():
    for name in ("tfgk_spmm_fp8", "tfgk_gat_fused_fp8", "tfgk_gemm_proj_fp8", "tfgk_quantize_fp8"):
        assert hasattr(_ffi.lib(), name)
        assert len(_ffi.SIGNATURES[name]) == _header_arity(name)
    assert ctypes.sizeof(_ffi.ProjBlockFp8) == ctypes.sizeof(_ffi.ProjBlockOut) + 16
    assert _ffi.DTYPE_FP8_E4M3 == 2


def test_spmm_fp8_validates_arguments():
    fake = ctypes.c_void_p(256)
    base = [fake, fake, None, fake, 16, fake, 4, 8, 0, 1.0, None, 0, 0.0, None, 0, fake, 8, None, None]
    bad = list(base)
    bad[6] = -1
    assert "negative size" in str(_call_err("tfgk_spmm_fp8", *bad))
    bad = list(base)
    bad[8] = 7
    assert "reduce" in str(_call_err("tfgk_spmm_fp8", *bad))
    bad = list(base)
    bad[5] = None
    assert "exponent" in str(_call_err("tfgk_spmm_fp8", *bad))
    bad = list(base)
    bad[4] = 7
    assert "leading dimension" in str(_call_err("tfgk_spmm_fp8", *bad))
    bad = list(base)
    bad[5], bad[7] = ctypes.c_void_p(257), 200                      # two groups: 2-byte aligned exponents
    bad[4], bad[16] = 208, 200
    assert "aligned" in str(_call_err("tfgk_spmm_fp8", *bad))
    empty = list(base)
    empty[6] = 0
    assert _ffi.call("tfgk_spmm_fp8", *empty) == _ffi.OK


def test_gat_fused_fp8_validates_arguments():
    fake = ctypes.c_void_p(256)
    base = [fake, fake, fake, 128, fake, 256, fake, 10, 8, 16, 4.0, None, 0, fake, 128, None, None]
    bad = list(base)
    bad[8] = 0
    assert _call_err("tfgk_gat_fused_fp8", *bad).code == _ffi.ERR_INVALID_ARGUMENT
    bad = list(base)
    bad[10] = 0.0
    assert _call_err("tfgk_gat_fused_fp8", *bad).code == _ffi.ERR_INVALID_ARGUMENT
    for H, dqk in ((3, 16), (8, 32), (4, 12), (1, 2)):               # not a power of two, A > 128, dqk / 4 not a power of 2
        bad = list(base)
        bad[8], bad[9] = H, dqk
        assert _call_err("tfgk_gat_fused_fp8", *bad).code == _ffi.ERR_UNSUPPORTED
    bad = list(base)
    bad[5] = 264                                                     # ldkv % 16 != 0
    assert _call_err("tfgk_gat_fused_fp8", *bad).code == _ffi.ERR_UNSUPPORTED
    bad = list(base)
    bad[4] = None
    assert _call_err("tfgk_gat_fused_fp8", *bad).code == _ffi.ERR_INVALID_ARGUMENT


def test_gemm_proj_fp8_and_quantize_validate_arguments():
    fake = ctypes.c_void_p(256)
    parts = (ctypes.c_void_p * 1)(256)
    blk = (_ffi.ProjBlockFp8 * 1)(_ffi.ProjBlockFp8(256, 64, 64, 0, None, 0, 256, 64, 9, None, 0))
    assert "unknown dtype" in str(_call_err("tfgk_gemm_proj_fp8", parts, 1, 0, 64, 8, 64, blk, 1, 0, 0, None))
    blk = (_ffi.ProjBlockFp8 * 1)(_ffi.ProjBlockFp8(256, 64, 64, 0, None, 0, 256, 64, _ffi.DTYPE_FP8_E4M3, None, 0))
    assert "exponents" in str(_call_err("tfgk_gemm_proj_fp8", parts, 1, 0, 64, 8, 64, blk, 1, 0, 0, None))
    assert "negative" in str(_call_err("tfgk_quantize_fp8", fake, 8, -1, 8, fake, 16, fake, 1, None))
    assert "leading dimension" in str(_call_err("tfgk_quantize_fp8", fake, 8, 4, 200, fake, 208, fake, 1, None))
    assert "null" in str(_call_err("tfgk_quantize_fp8", fake, 8, 4, 8, fake, 16, None, 1, None))
    assert _ffi.call("tfgk_quantize_fp8", None, 0, 0, 8, None, 16, None, 1, None) == _ffi.OK


@pytest.mark.parametrize("m, k", [(0.0, 0), (448.0, 0), (449.0, 1), (1.0, -8), (1.75, -8), (1.7500001, -7), (896.0, 1),
                                  (np.float32(3.4028235e38), 120), (1e-45, -126), (448.0 * 2.0 ** -126, -126),
                                  (448.0 * 2.0 ** -118, -118), (2.0 ** -110, -118)])
def test_exponent_rule(m, k):
    assert fp8_ref.exponent(float(m)) == k
    if m:
        assert float(m) * 2.0 ** -k <= 448.0 and (k == -126 or float(m) * 2.0 ** -(k - 1) > 448.0)


def test_quantize_edge_cases_against_float64():
    x = np.array([[0.0] * 4, [-0.0, 1.0, -2.0, 0.5], [np.inf, 3.0, np.nan, -np.inf], [1e-40, -3e-39, 0.0, 2e-39],
                  [3.4e38, -3.0e38, 1.0, 1e30]], np.float32)
    q, k = fp8_ref.quantize(x)
    assert list(k[:, 0]) == [0, -7, -7, -126, 120]
    assert q[0].tolist() == [0, 0, 0, 0] and q[1, 0] == 0x80
    assert q[2, 0] == 0x7F and q[2, 3] == 0xFF and (q[2, 2] & 0x7F) == 0x7F
    xh = fp8_ref.dequantize(q, k)
    assert xh[4, 0] == np.inf          # 3.4e38 rounds to 256 * 2^120 = 2^128: past FLT_MAX, x^ is inf
    fin = np.isfinite(x) & np.isfinite(xh)
    assert np.all(np.abs(xh[fin].astype(np.float64) - x[fin]) <= fp8_ref.error_bound(x, k)[fin])


def test_message_dtype_values():
    assert ops.conv_message_dtype(FP8) is FP8 and ops.conv_message_dtype("float8_e4m3fn") is FP8
    assert ops.conv_message_dtype(torch.bfloat16) is torch.bfloat16 and ops.conv_message_dtype(None) is None
    for bad in (torch.float8_e5m2, torch.float16, "fp8"):
        with pytest.raises(ValueError):
            ops.conv_message_dtype(bad)
    with pytest.raises(ValueError):
        ops.message_dtype(FP8)                      # the other convolutions keep refusing fp8
    with pytest.raises(ValueError):
        tfg.layers.GCN(4, message_dtype=torch.float8_e5m2)
    with pytest.raises(ValueError):
        tfg.layers.GAT(4, message_dtype=torch.float8_e5m2)
    tfg.layers.GCN(4, message_dtype=FP8)
    tfg.layers.GAT(4, message_dtype=FP8)


def _graph(n=12, f=6, seed=0):
    rng = np.random.default_rng(seed)
    ei = np.stack([rng.integers(0, n, 40), rng.integers(0, n, 40)]).astype(np.int32)
    return rng.standard_normal((n, f)).astype(np.float32), ei


def test_refusals_come_before_device_work(monkeypatch):
    calls = fp8_fake_backend.install(monkeypatch)
    x, ei = _graph()
    xt, eit = torch.from_numpy(x), torch.from_numpy(ei)
    adj = tfg.SparseMatrix(eit, shape=[12, 12])
    w = torch.ones(6, 8, requires_grad=True)
    with pytest.raises(NotImplementedError):
        tfg.nn.gcn(xt, adj, w, message_dtype=FP8)
    with pytest.raises(NotImplementedError):
        tfg.nn.gcn(xt, adj, w.detach(), edge_drop_rate=0.5, training=True, message_dtype=FP8)
    wq, wk, wv = torch.ones(6, 8), torch.ones(6, 8), torch.ones(6, 8)
    args = (xt, eit, wq, None, None, wk, None, None, wv)
    with pytest.raises(NotImplementedError):
        tfg.nn.gat(*args, num_heads=2, return_attention=True, message_dtype=FP8)
    with pytest.raises(NotImplementedError):
        tfg.nn.gat(*args, num_heads=2, edge_drop_rate=0.3, training=True, message_dtype=FP8)
    with pytest.raises(NotImplementedError):
        tfg.nn.gat(xt, eit, wq, None, None, wk, None, None, w, num_heads=2, message_dtype=FP8)
    with pytest.raises(NotImplementedError, match="bfloat16 or float32"):
        tfg.nn.gat(*args, num_heads=3, message_dtype=FP8)             # 8 units, 3 heads
    with pytest.raises(NotImplementedError, match="bfloat16 or float32"):
        tfg.nn.gat(*args, num_heads=2, split_value_heads=False, message_dtype=FP8)
    with pytest.raises(NotImplementedError, match="bfloat16 or float32"):
        tfg.nn.gat(xt, eit, torch.ones(6, 256), None, None, torch.ones(6, 256), None, None, torch.ones(6, 256),
                   num_heads=8, message_dtype=FP8)
    with pytest.raises(NotImplementedError):
        tfg.nn.gat(xt, eit, torch.ones(6, 12), None, None, torch.ones(6, 12), None, None, torch.ones(6, 12), num_heads=1,
                   message_dtype=FP8)                                  # dqk / 4 = 3
    with pytest.raises(ValueError):
        tfg.nn.gat(*args, num_heads=2, message_dtype=torch.float8_e5m2)
    with pytest.raises(ValueError):
        tfg.nn.gcn(xt, adj, w.detach(), message_dtype=torch.float8_e5m2)
    assert calls == []


def test_gcn_and_gat_plumbing_on_the_test_double(monkeypatch):
    calls = fp8_fake_backend.install(monkeypatch)
    x, ei = _graph(seed=3)
    xt, eit = torch.from_numpy(x), torch.from_numpy(ei)
    rng = np.random.default_rng(4)
    w = torch.from_numpy(rng.standard_normal((6, 8)).astype(np.float32))
    b = torch.from_numpy(rng.standard_normal(8).astype(np.float32))
    adj = tfg.SparseMatrix(eit, shape=[12, 12])
    got = tfg.nn.gcn(xt, adj, w, b, activation=ops.relu, message_dtype=FP8)
    assert calls == ["gemm_proj", "spmm_fp8"]
    # the fp32 composition over the dequantised projection
    xw = fp8_fake_backend.dequantized((xt @ w).numpy())
    ref = tfg.nn.gcn(torch.from_numpy(xw), tfg.SparseMatrix(eit, shape=[12, 12]), None, b, activation=ops.relu)
    assert torch.equal(got, ref)
    calls.clear()
    got = tfg.nn.gcn(xt, adj, None, message_dtype=FP8)
    assert calls == ["quantize_fp8", "spmm_fp8"] and tuple(got.shape) == (12, 6)

    calls.clear()
    wq, wk, wv = (torch.from_numpy(rng.standard_normal((6, 8)).astype(np.float32)) for _ in range(3))
    got = tfg.nn.gat(xt, eit, wq, None, ops.relu, wk, None, ops.relu, wv, b, num_heads=2, message_dtype=FP8)
    assert calls == ["gemm_proj", "gat_fused_fp8"]
    K = fp8_fake_backend.dequantized(np.maximum((xt @ wk).numpy(), 0))
    V = fp8_fake_backend.dequantized((xt @ wv).numpy())
    Q = np.maximum((xt @ wq).numpy(), 0)
    from tf_geometric_b200 import _structure
    csr, _ = _structure.csr_for_edge_index(eit, 12, add_self_loop=True)
    ref = ops.gat_fused(csr, torch.from_numpy(Q), torch.from_numpy(K), torch.from_numpy(V), 2, bias=b)
    np.testing.assert_allclose(got.numpy(), ref.numpy(), rtol=1e-5, atol=1e-5)
    layer = tfg.layers.GAT(8, num_heads=2, message_dtype=FP8)
    assert tuple(layer([xt, eit]).shape) == (12, 8)
    layer = tfg.layers.GCN(8, message_dtype=FP8)
    assert tuple(layer([xt, eit]).shape) == (12, 8)


def _cpu_csr(n=12):
    rowptr = torch.arange(n + 1, dtype=torch.int64)
    col = torch.arange(n, dtype=torch.int32)
    return ops.CSR(rowptr, col, col.clone(), n, n)


def test_gathers_refuse_strided_exponents_and_host_tables():
    """The K1 / K3 kernels index exponents as row * groups + group: a column block of a wider table (its exponents are a
    strided column), a table with too few exponent columns and a table in host memory are refused before any launch."""
    csr = _cpu_csr()
    wide = ops.fp8_table(12, 200, "cpu")                               # two groups
    with pytest.raises(ValueError, match="dense"):
        ops.spmm(csr, None, wide.block(0, 128))                        # exponents [12, 1] with row stride 2
    thin = ops.Fp8Table(wide.data, wide.exps[:, :1].contiguous(), 200)
    with pytest.raises(ValueError, match="dense"):
        ops.spmm(csr, None, thin)                                      # 200 columns need two exponent columns
    with pytest.raises(TypeError, match="CUDA"):
        ops.spmm(csr, None, wide)                                      # a host table
    with pytest.raises(ValueError, match="rows"):
        ops.spmm(ops.CSR(csr.rowptr, csr.col, csr.perm, 12, 40), None, wide)
    kv = ops.fp8_table(12, 16, "cpu", groups=2)
    q = torch.zeros((12, 8))
    with pytest.raises(TypeError, match="CUDA"):
        ops.gat_fused(csr, q, kv, None, 2)                             # host K | V
    with pytest.raises(ValueError, match="rows"):
        ops.gat_fused(csr, torch.zeros((11, 8)), kv, None, 2)          # Q does not cover the graph's rows
    with pytest.raises(ValueError, match="dense"):
        ops.gat_fused(csr, q, ops.Fp8Table(kv.data, kv.exps[:, :1], 16), None, 2)
