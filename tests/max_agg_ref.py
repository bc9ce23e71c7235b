# coding=utf-8
"""Numpy restatement of K11 (tfgk_spmm_max_f32 and tfgk_spmm_max_bwd_f32) and a TEST DOUBLE that installs it as
ops.spmm_max / ops.spmm_max_bwd over the CPU fake of the kernel layer (tests/fake_backend.py), so that the host logic of
the max aggregation routes runs without a GPU.  Injected with monkeypatch; the product has no such path."""
import numpy as np
import torch

import fake_backend
from fake_backend import _np, _t

F32 = np.float32
LOWEST = np.finfo(np.float32).min


def k11a(rowptr, col, w, h):
    """(out, cnt) of K11a in CSR order: out = fmax chain from -FLT_MAX over w_e * h[col_e] (fp32 products), cnt = the
    running tie count (restarts at 1 above the maximum, +1 on IEEE equality), which ends as #{e : m_e == out}."""
    h = np.asarray(h, F32)
    n, D = len(rowptr) - 1, h.shape[1]
    out = np.full((n, D), LOWEST, F32)
    cnt = np.zeros((n, D), np.int32)
    with np.errstate(invalid="ignore"):
        for r in range(n):
            a, k = out[r].copy(), cnt[r].copy()
            for e in range(int(rowptr[r]), int(rowptr[r + 1])):
                m = (h[col[e]] * (F32(1) if w is None else F32(w[e]))).astype(F32)
                k = np.where(m > a, 1, np.where(m == a, k + 1, k)).astype(np.int32)
                a = np.fmax(a, m)
            out[r], cnt[r] = a, k
    return out, cnt


def k11b(rowptr_t, dst_t, w_t, h, out, cnt, g):
    """dh of K11b over the transposed CSR: sum from 0, in edge order, of ((Gn[r] * sel) * w_e) with Gn = g / max(cnt, 1)
    in fp32 and sel = (w_e * h[c] == out[r]); every edge adds its term."""
    h, out, g = np.asarray(h, F32), np.asarray(out, F32), np.asarray(g, F32)
    gn = (g / np.maximum(cnt, 1).astype(F32)).astype(F32)
    n, D = len(rowptr_t) - 1, h.shape[1]
    dh = np.zeros((n, D), F32)
    with np.errstate(invalid="ignore", over="ignore"):
        for c in range(n):
            acc = np.zeros(D, F32)
            for p in range(int(rowptr_t[c]), int(rowptr_t[c + 1])):
                r = int(dst_t[p])
                we = F32(1) if w_t is None else F32(w_t[p])
                sel = ((h[c] * we).astype(F32) == out[r]).astype(F32)
                acc = (acc + ((gn[r] * sel).astype(F32) * we).astype(F32)).astype(F32)
            dh[c] = acc
    return dh


def install(monkeypatch):
    """The CPU fake of the kernel layer plus K11; host tensors take the device routes (NeighborMax)."""
    fake_backend.install(monkeypatch)
    from tf_geometric_b200 import ops, autograd
    calls = {"spmm_max": 0, "spmm_max_bwd": 0}

    def spmm_max(csr, w_csr, h):
        calls["spmm_max"] += 1
        out, cnt = k11a(_np(csr.rowptr), _np(csr.col), _np(w_csr), _np(h))
        return _t(out), _t(cnt)

    def spmm_max_bwd(csr_t, w_t, h, out, cnt, g):
        calls["spmm_max_bwd"] += 1
        return _t(k11b(_np(csr_t.rowptr), _np(csr_t.col), _np(w_t), _np(h), _np(out), _np(cnt), _np(g)))

    monkeypatch.setattr(ops, "spmm_max", spmm_max)
    monkeypatch.setattr(ops, "spmm_max_bwd", spmm_max_bwd)
    monkeypatch.setattr(autograd, "_is_device", lambda t: torch.is_tensor(t))
    return calls
