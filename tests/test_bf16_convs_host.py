# coding=utf-8
"""bf16 message rows for the remaining convolutions, without a GPU: the dual-store aggregation entry is exported, bound
with the header's arity and validates its arguments before it touches the device; every function and layer takes
`message_dtype` and refuses on the host what the mode does not support."""
import ctypes
import inspect
import os
import re

import numpy as np
import pytest
import torch

import tf_geometric_b200 as tfg
from tf_geometric_b200 import _ffi

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))

FUNCTIONS = ["mean_graph_sage", "sum_graph_sage", "gcn_graph_sage", "mean_pool_graph_sage", "max_pool_graph_sage", "gin",
             "le_conv", "appnp", "sgc", "ssgc", "tagcn", "chebynet"]
LAYERS = ["MeanGraphSage", "SumGraphSage", "GCNGraphSage", "MeanPoolGraphSage", "MaxPoolGraphSage", "GIN", "LEConv",
          "APPNP", "SGC", "SSGC", "TAGCN", "ChebyNet"]


def _call_err(*args):
    with pytest.raises(_ffi.TfgkError) as err:
        _ffi.call("tfgk_spmm_bf16_dual", *args)
    return err.value


def test_dual_entry_is_exported_with_the_header_arity():
    assert hasattr(_ffi.lib(), "tfgk_spmm_bf16_dual")
    header = open(os.path.join(ROOT, "include", "tfgk.h")).read()
    decl = re.search(r"int tfgk_spmm_bf16_dual\(([^)]*)\)", header).group(1)
    assert len(_ffi.SIGNATURES["tfgk_spmm_bf16_dual"]) == len(decl.split(","))
    assert len(_ffi.SIGNATURES["tfgk_spmm_bf16_dual"]) == len(_ffi.SIGNATURES["tfgk_spmm_bf16"]) + 2


def _args(**over):
    fake = ctypes.c_void_p(256)
    a = dict(rowptr=fake, col=fake, w=None, h=fake, ldh=48, n=4, D=47, reduce=0, alpha=1.0, addend=None, lda=0,
             beta=0.0, bias=None, act=0, out=fake, ldo=47, outb=ctypes.c_void_p(512), ldob=47, plan=None, stream=None)
    a.update(over)
    return list(a.values())


def test_dual_entry_validates_arguments():
    e = _call_err(*_args(out=None, outb=None))
    assert e.code == _ffi.ERR_INVALID_ARGUMENT and "both outputs" in str(e)
    e = _call_err(*_args(out=None, outb=None, n=0))                    # even for an empty launch
    assert e.code == _ffi.ERR_INVALID_ARGUMENT
    e = _call_err(*_args(n=-1))
    assert e.code == _ffi.ERR_INVALID_ARGUMENT and "negative size" in str(e)
    e = _call_err(*_args(D=-3))
    assert e.code == _ffi.ERR_INVALID_ARGUMENT and "negative size" in str(e)
    e = _call_err(*_args(ldh=40))
    assert e.code == _ffi.ERR_INVALID_ARGUMENT and "leading dimension" in str(e)
    e = _call_err(*_args(ldob=46))
    assert e.code == _ffi.ERR_INVALID_ARGUMENT and "leading dimension" in str(e)
    e = _call_err(*_args(out=None, ldob=46))
    assert e.code == _ffi.ERR_INVALID_ARGUMENT and "leading dimension" in str(e)
    e = _call_err(*_args(h=ctypes.c_void_p(257)))                      # padded ldh, rows at an odd address
    assert e.code == _ffi.ERR_INVALID_ARGUMENT and "misaligned" in str(e)
    e = _call_err(*_args(outb=ctypes.c_void_p(513)))
    assert e.code == _ffi.ERR_INVALID_ARGUMENT and "misaligned" in str(e)
    e = _call_err(*_args(reduce=9))
    assert e.code == _ffi.ERR_INVALID_ARGUMENT and "reduce" in str(e)
    e = _call_err(*_args(h=None))
    assert e.code == _ffi.ERR_INVALID_ARGUMENT and "null" in str(e)
    assert _ffi.call("tfgk_spmm_bf16_dual", *_args(n=0, out=None)) == _ffi.OK


def test_every_function_and_layer_takes_message_dtype():
    for name in FUNCTIONS:
        fn = getattr(tfg.nn, name)
        p = inspect.signature(fn).parameters
        assert "message_dtype" in p and p["message_dtype"].default is None, name
    for name in LAYERS:
        cls = getattr(tfg.layers, name)
        args = (lambda h: h,) if name == "GIN" else ((8,) if name not in ("APPNP", "SSGC", "ChebyNet") else
                                                    ([8],) if name != "ChebyNet" else (8, 2))
        assert cls(*args).message_dtype is None
        assert cls(*args, message_dtype=torch.bfloat16).message_dtype is torch.bfloat16
        assert cls(*args, message_dtype="bfloat16").message_dtype == "bfloat16"
        with pytest.raises(ValueError):
            cls(*args, message_dtype=torch.float16)


def test_host_refusals():
    n, f = 40, 6
    rs = np.random.RandomState(0)
    ei = rs.randint(0, n, (2, 200)).astype(np.int32)
    x = torch.randn((n, f))
    w = torch.randn((f, 4))
    b16 = torch.bfloat16
    for bad in (torch.float16, torch.float64, "half", 8):
        with pytest.raises(ValueError):
            tfg.nn.sgc(x, ei, None, 2, w, message_dtype=bad)
        with pytest.raises(ValueError):
            tfg.nn.mean_graph_sage(x, ei, None, w, w, message_dtype=bad)
    # training and active dropout are refused before any device work (a sparse x is refused on the GPU)
    with pytest.raises(NotImplementedError):
        tfg.nn.le_conv(x, ei, None, w.clone().requires_grad_(True), None, w, None, w, None, message_dtype=b16)
    with pytest.raises(NotImplementedError):
        tfg.nn.max_pool_graph_sage(x.clone().requires_grad_(True), ei, torch.ones(200), w, w, w, message_dtype=b16)
    with pytest.raises(NotImplementedError):
        tfg.nn.gcn_graph_sage(x, ei, None, w.clone().requires_grad_(True), message_dtype=b16)
    with pytest.raises(NotImplementedError):
        tfg.nn.tagcn(x, ei, None, 2, torch.randn((3 * f, 4), requires_grad=True), message_dtype=b16)
    with pytest.raises(NotImplementedError):
        tfg.nn.chebynet(x, ei, None, 2, [w, w.clone().requires_grad_(True)], message_dtype=b16)
    with pytest.raises(NotImplementedError):
        tfg.nn.appnp(x, ei, None, [w], [None], dense_drop_rate=0.5, last_dense_drop_rate=0.5, training=True,
                     message_dtype=b16)
    with pytest.raises(NotImplementedError):
        tfg.nn.appnp(x, ei, None, [w], [None], edge_drop_rate=0.5, training=True, message_dtype=b16)
    with pytest.raises(NotImplementedError):
        tfg.nn.ssgc(x, ei, None, [w], [None], dense_drop_rate=0.1, last_dense_drop_rate=0.1, training=True,
                    message_dtype=b16)
    mlp = torch.nn.Linear(f, 4)
    with pytest.raises(NotImplementedError):
        tfg.nn.gin(x, ei, mlp, message_dtype=b16)                      # the MLP's weights require grad
