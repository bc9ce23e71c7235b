# coding=utf-8
"""TEST DOUBLE for the fp8 message rows: the CPU fake kernel layer of tests/fake_backend.py plus numpy restatements of
the fp8 entry points (K4's fp8 blocks, tfgk_quantize_fp8, tfgk_spmm_fp8, tfgk_gat_fused_fp8) built on tests/fp8_ref.py,
so that the GCN and GAT fp8 plumbing runs without a GPU.  It lives under tests/ and is injected with monkeypatch; the
product has no such path."""
import fake_backend
import fp8_ref
from fake_backend import _np, _t


def install(monkeypatch):
    fake_backend.install(monkeypatch)
    from tf_geometric_b200 import ops
    calls = []
    fake_spmm, fake_gat, fake_proj = ops.spmm, ops.gat_fused, ops.gemm_proj

    def quantize_into(src, table):
        q, k = fp8_ref.quantize(_np(src))
        table.data.copy_(_t(q))
        table.exps[:, :k.shape[1]].copy_(_t(k))
        return table

    def dequant(table, exps=None):
        return _t(fp8_ref.dequantize(_np(table.data), _np(table.exps if exps is None else exps)))

    def quantize_fp8(src, out=None):
        calls.append("quantize_fp8")
        if out is None:
            out = ops.fp8_table(src.shape[0], src.shape[1], src.device)
        return quantize_into(src, out)

    def gemm_proj(a, blocks, a_parts=None, part_rows=0, first_part=0, max_ctas=0, num_rows=None):
        calls.append("gemm_proj")
        plain = [tuple(b[:3]) + (None,) + tuple(b[4:]) if isinstance(b[3], ops.Fp8Table) else b for b in blocks]
        res = fake_proj(a, plain, a_parts, part_rows, first_part, max_ctas, num_rows)
        return [quantize_into(r, b[3]) if isinstance(b[3], ops.Fp8Table) else r for r, b in zip(res, blocks)]

    def spmm(csr, w_csr, h, *args, **kwargs):
        if isinstance(h, ops.Fp8Table):
            calls.append("spmm_fp8")
            h = dequant(h)
        return fake_spmm(csr, w_csr, h, *args, **kwargs)

    def gat_fused(csr, Q, K, V, num_heads, *args, **kwargs):
        if isinstance(K, ops.Fp8Table):
            calls.append("gat_fused_fp8")
            A = K.cols // 2
            K, V = dequant(K.block(0, A, group=0)), dequant(K.block(A, 2 * A, group=1))
        return fake_gat(csr, Q, K, V, num_heads, *args, **kwargs)

    for name, fn in (("quantize_fp8", quantize_fp8), ("gemm_proj", gemm_proj), ("spmm", spmm), ("gat_fused", gat_fused)):
        monkeypatch.setattr(ops, name, fn)
    return calls


def dequantized(x):
    """x^ of a float32 numpy array under the format."""
    q, k = fp8_ref.quantize(x)
    return fp8_ref.dequantize(q, k)

