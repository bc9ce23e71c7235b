# coding=utf-8
"""bf16 message rows without a GPU: the new entry points are exported, bound and validate their arguments before they
touch the device; the Python layer rejects what the bf16 mode does not support."""
import ctypes

import pytest
import torch

from tf_geometric_b200 import _ffi, ops


def _call_err(name, *args):
    with pytest.raises(_ffi.TfgkError) as err:
        _ffi.call(name, *args)
    return err.value


def test_symbols_are_bound():
    for name in ("tfgk_spmm_bf16", "tfgk_gat_fused_bf16", "tfgk_gemm_proj_mixed", "tfgk_round_bf16"):
        assert name in _ffi.SIGNATURES and hasattr(_ffi.lib(), name)
    assert len(_ffi.SIGNATURES["tfgk_spmm_bf16"]) == len(_ffi.SIGNATURES["tfgk_spmm_f32"])
    assert len(_ffi.SIGNATURES["tfgk_gat_fused_bf16"]) == len(_ffi.SIGNATURES["tfgk_gat_fused_f32"])
    assert ctypes.sizeof(_ffi.ProjBlockOut) == ctypes.sizeof(_ffi.ProjBlock) + 8


def test_spmm_bf16_validates_arguments():
    fake = ctypes.c_void_p(256)
    e = _call_err("tfgk_spmm_bf16", fake, fake, None, fake, 8, -1, 8, 0, 1.0, None, 0, 0.0, None, 0, fake, 8, None, None)
    assert e.code == _ffi.ERR_INVALID_ARGUMENT and "negative size" in str(e)
    e = _call_err("tfgk_spmm_bf16", fake, fake, None, fake, 8, 4, 8, 7, 1.0, None, 0, 0.0, None, 0, fake, 8, None, None)
    assert e.code == _ffi.ERR_INVALID_ARGUMENT and "reduce" in str(e)
    e = _call_err("tfgk_spmm_bf16", fake, fake, None, None, 8, 4, 8, 0, 1.0, None, 0, 0.0, None, 0, fake, 8, None, None)
    assert e.code == _ffi.ERR_INVALID_ARGUMENT and "null" in str(e)
    e = _call_err("tfgk_spmm_bf16", fake, fake, None, fake, 7, 4, 8, 0, 1.0, None, 0, 0.0, None, 0, fake, 8, None, None)
    assert e.code == _ffi.ERR_INVALID_ARGUMENT and "leading dimension" in str(e)
    assert _ffi.call("tfgk_spmm_bf16", None, None, None, None, 0, 0, 8, 0, 1.0, None, 0, 0.0, None, 0, None, 0, None,
                     None) == _ffi.OK


def test_gat_fused_bf16_validates_arguments():
    fake = ctypes.c_void_p(256)
    args = [fake, fake, fake, 128, fake, 256, fake, 256, 10, 8, 16, 16, 4.0, 1, None, 0, None, 0, fake, 128, None, None]
    bad = list(args)
    bad[9] = 0                                            # H
    assert _call_err("tfgk_gat_fused_bf16", *bad).code == _ffi.ERR_INVALID_ARGUMENT
    bad = list(args)
    bad[12] = 0.0                                         # scale
    assert _call_err("tfgk_gat_fused_bf16", *bad).code == _ffi.ERR_INVALID_ARGUMENT
    bad = list(args)
    bad[4] = None                                         # K
    assert _call_err("tfgk_gat_fused_bf16", *bad).code == _ffi.ERR_INVALID_ARGUMENT
    bad = list(args)
    bad[5] = 64                                           # ldk < A
    assert _call_err("tfgk_gat_fused_bf16", *bad).code == _ffi.ERR_INVALID_ARGUMENT
    bad = list(args)
    bad[17] = 1                                           # write_att
    assert _call_err("tfgk_gat_fused_bf16", *bad).code == _ffi.ERR_UNSUPPORTED


def test_gemm_proj_mixed_and_round_validate_arguments():
    fake = ctypes.c_void_p(256)
    blk = _ffi.ProjBlockOut(256, 32, 32, 0, None, 0, 512, 32, 5)         # unknown dtype
    parts = (ctypes.c_void_p * 1)(256)
    e = _call_err("tfgk_gemm_proj_mixed", parts, 1, 0, 16, 64, 16, ctypes.byref(blk), 1, 0, 0, None)
    assert e.code == _ffi.ERR_INVALID_ARGUMENT and "dtype" in str(e)
    blk = _ffi.ProjBlockOut(256, 32, 32, 0, None, 0, 513, 32, _ffi.DTYPE_BF16)   # odd bf16 address
    e = _call_err("tfgk_gemm_proj_mixed", parts, 1, 0, 16, 64, 16, ctypes.byref(blk), 1, 0, 0, None)
    assert e.code == _ffi.ERR_INVALID_ARGUMENT
    blk = _ffi.ProjBlockOut(256, 32, 32, 0, None, 0, 512, 32, _ffi.DTYPE_BF16)
    e = _call_err("tfgk_gemm_proj_mixed", parts, 1, 0, 16, 64, 16, ctypes.byref(blk), 5, 0, 0, None)
    assert e.code == _ffi.ERR_INVALID_ARGUMENT and "n_blocks" in str(e)
    e = _call_err("tfgk_gemm_proj_mixed", None, 1, 0, 16, 64, 16, ctypes.byref(blk), 1, 0, 0, None)
    assert e.code == _ffi.ERR_INVALID_ARGUMENT
    e = _call_err("tfgk_gemm_proj_mixed", (ctypes.c_void_p * 2)(256, 256), 2, 128, 16, 64, 16, ctypes.byref(blk), 1, 0, 0,
                  None)
    assert e.code == _ffi.ERR_UNSUPPORTED
    e = _call_err("tfgk_round_bf16", fake, 4, 2, 8, fake, 8, None)
    assert e.code == _ffi.ERR_INVALID_ARGUMENT and "leading dimension" in str(e)
    e = _call_err("tfgk_round_bf16", None, 8, 2, 8, fake, 8, None)
    assert e.code == _ffi.ERR_INVALID_ARGUMENT


def test_message_dtype_values():
    assert ops.message_dtype(None) is None and ops.message_dtype(torch.float32) is None
    assert ops.message_dtype(torch.bfloat16) is torch.bfloat16 and ops.message_dtype("bfloat16") is torch.bfloat16
    for bad in (torch.float16, torch.float64, "fp8", 16):
        with pytest.raises(ValueError):
            ops.message_dtype(bad)
    import tf_geometric_b200 as tfg
    with pytest.raises(ValueError):
        tfg.layers.GCN(8, message_dtype=torch.float16)
    with pytest.raises(ValueError):
        tfg.layers.GAT(8, message_dtype="half")
    with pytest.raises(TypeError):
        ops.spmm(None, None, torch.zeros(3, 2, dtype=torch.bfloat16))      # CPU tensor
