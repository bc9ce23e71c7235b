# coding=utf-8
"""K4 tensor-core path (wgmma, 3xTF32 split): fp32-level accuracy against float64, far inside the 1e-4 gate that a
single TF32 pass would miss.  Shapes cover the projections of the hot path and the ragged edges (M, N, K tails)."""
import os

import numpy as np
import pytest
import torch

from tf_geometric_b200 import ops
from conftest import assert_close

pytestmark = [pytest.mark.gpu,
              pytest.mark.skipif(os.environ.get("TFGK_GEMM_TC") == "0", reason="tensor-core GEMM disabled by TFGK_GEMM_TC=0")]


def dev(a):
    return ops.as_device(a)


@pytest.mark.parametrize("m,n,k", [
    (128, 128, 32), (128, 16, 8), (4096, 128, 100), (5000, 128, 128), (2708, 16, 184), (3000, 7, 16),
    (1000, 64, 20), (777, 200, 160), (130000, 128, 100), (300, 256, 64), (129, 48, 5)])
def test_gemm_tc_matches_float64(m, n, k):
    rs = np.random.RandomState(m + n + k)
    a = rs.randn(m, k).astype(np.float32)
    b = (rs.randn(k, n) / np.sqrt(k)).astype(np.float32)
    bias = rs.randn(n).astype(np.float32)
    want = a.astype(np.float64) @ b.astype(np.float64)
    got = ops.gemm(dev(a), dev(b)).cpu().numpy()
    err = np.abs(got - want).max() / np.abs(want).max()
    assert err < 5e-6, "3xTF32 relative error {:.2e} (single-pass TF32 would be ~1e-3)".format(err)
    got = ops.gemm(dev(a), dev(b), bias=dev(bias), act=ops.ACT_RELU).cpu().numpy()
    assert_close(got, np.maximum(want + bias, 0), rtol=1e-5, atol_scale=5e-6, what="tc gemm + bias + relu")


@pytest.mark.parametrize("m,n,k", [(2708, 16, 512), (777, 200, 333)])
def test_gemm_wide_k_runs_simt_and_matches_float64(monkeypatch, m, n, k):
    """K above ops.GEMM_PROJ_MAX_K: W (hi | lo) does not fit in shared memory next to the A ring, so the exact-fp32 SIMT
    kernel runs (the same bits as with the tensor-core route switched off)."""
    assert k > ops.GEMM_PROJ_MAX_K
    rs = np.random.RandomState(m + n + k)
    a = rs.randn(m, k).astype(np.float32)
    b = (rs.randn(k, n) / np.sqrt(k)).astype(np.float32)
    bias = rs.randn(n).astype(np.float32)
    want = a.astype(np.float64) @ b.astype(np.float64)
    got = ops.gemm(dev(a), dev(b))
    with monkeypatch.context() as mp:
        mp.setenv("TFGK_GEMM_TC", "0")
        assert torch.equal(got, ops.gemm(dev(a), dev(b)))
    got = got.cpu().numpy()
    err = np.abs(got - want).max() / np.abs(want).max()
    assert err < 5e-6, "SIMT relative error {:.2e}".format(err)
    got = ops.gemm(dev(a), dev(b), bias=dev(bias), act=ops.ACT_RELU).cpu().numpy()
    assert_close(got, np.maximum(want + bias, 0), rtol=1e-5, atol_scale=5e-6, what="SIMT gemm + bias + relu")


def test_gemm_tc_strided_operands_and_output_slices():
    rs = np.random.RandomState(0)
    m, k, n = 3000, 100, 128
    big_a = rs.randn(m, 3 * k + 4).astype(np.float32)          # lda = 304
    a = dev(big_a)[:, 4:4 + k]                                  # 16-byte aligned column offset
    b = dev((rs.randn(k, n) / 10).astype(np.float32))
    out = torch.zeros((m, 2 * n), dtype=torch.float32, device="cuda")
    ops.gemm(a, b, out=out[:, n:])
    want = big_a[:, 4:4 + k].astype(np.float64) @ b.cpu().numpy().astype(np.float64)
    assert_close(out[:, n:].cpu().numpy(), want, rtol=1e-5, atol_scale=5e-6, what="strided tc gemm")
    assert float(out[:, :n].abs().max()) == 0.0
    a2 = dev(big_a)[:, 1:1 + k]                                  # unaligned column offset -> scalar-load variant
    ops.gemm(a2, b, out=out[:, :n])
    want2 = big_a[:, 1:1 + k].astype(np.float64) @ b.cpu().numpy().astype(np.float64)
    assert_close(out[:, :n].cpu().numpy(), want2, rtol=1e-5, atol_scale=5e-6, what="unaligned tc gemm")


def test_gemm_tc_is_deterministic():
    rs = np.random.RandomState(1)
    a, b = dev(rs.randn(20000, 100).astype(np.float32)), dev(rs.randn(100, 128).astype(np.float32))
    first = ops.gemm(a, b)
    for _ in range(3):
        assert torch.equal(first, ops.gemm(a, b))
