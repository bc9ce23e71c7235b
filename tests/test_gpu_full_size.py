# coding=utf-8
"""Parity at BASELINE.json's full size (synthetic ogbn-products shape: 2,449,029 nodes, 123,718,280 edges, D=128)
through size-independent properties plus bit-exact spot checks of sampled destination rows against the oracle's
arithmetic (sequential fp32 in edge order), so the whole thing runs in seconds on the GPU."""
import numpy as np
import pytest
import torch

import tf_geometric_b200 as tfg
from tf_geometric_b200 import ops
from oracle import c_oracle

pytestmark = pytest.mark.gpu

N, PAIRS, D, H = 2449029, 61859140, 128, 8


@pytest.fixture(scope="module")
def big():
    dev = torch.device("cuda")
    gen = torch.Generator(device=dev)
    gen.manual_seed(0)
    u = torch.randint(0, N, (PAIRS,), generator=gen, device=dev, dtype=torch.int32)
    v = torch.randint(0, N - 1, (PAIRS,), generator=gen, device=dev, dtype=torch.int32)
    v = v + (v >= u).to(torch.int32)
    ei = torch.stack([torch.cat([u, v]), torch.cat([v, u])])
    del u, v
    w = torch.rand((ei.shape[1],), generator=gen, device=dev, dtype=torch.float32) + 0.5
    adj = tfg.SparseMatrix(ei, w, [N, N])
    h = torch.randn((N, D), generator=gen, device=dev, dtype=torch.float32)
    return {"ei": ei, "w": w, "adj": adj, "h": h, "gen": gen}


def test_csr_is_a_stable_sort_at_full_size(big):
    csr = big["adj"].csr
    row = big["ei"][0]
    rowptr = csr.rowptr
    assert int(rowptr[0]) == 0 and int(rowptr[-1]) == row.numel()
    sorted_rows = row[csr.perm.long()]
    assert bool((sorted_rows[1:] >= sorted_rows[:-1]).all())                       # sortedness
    same = sorted_rows[1:] == sorted_rows[:-1]
    assert bool((csr.perm[1:][same] > csr.perm[:-1][same]).all())                  # stability: ties keep input order
    assert bool((torch.bincount(row.long(), minlength=N) == (rowptr[1:] - rowptr[:-1])).all())
    assert int(csr.perm.long().sum()) == row.numel() * (row.numel() - 1) // 2      # a permutation (checksum)
    assert bool((csr.col == big["ei"][1][csr.perm.long()]).all())


def _expected_rows(csr, w_csr, h, rows):
    """Oracle arithmetic for a handful of destination rows: sequential fp32 sum of w_e * h[col_e] in CSR order."""
    rp = csr.rowptr[torch.as_tensor(np.stack([rows, rows + 1]), device=h.device)].cpu().numpy()
    out = []
    for (s, e) in zip(rp[0], rp[1]):
        cols = csr.col[s:e].long()
        hw = h[cols].cpu().numpy()
        ww = np.ones(e - s, np.float32) if w_csr is None else w_csr[s:e].cpu().numpy()
        ids = np.zeros(e - s, np.int32)
        out.append(c_oracle.aggregate(ids, np.arange(e - s, dtype=np.int32), ww, hw, 1, "sum")[0])
    return np.stack(out)


def test_spmm_sampled_rows_bit_exact_and_properties(big):
    adj, h = big["adj"], big["h"]
    out = adj @ h
    rows = np.random.RandomState(1).randint(0, N, 512)
    want = _expected_rows(adj.csr, adj.value_csr, h, rows)
    np.testing.assert_array_equal(out[torch.as_tensor(rows, device=h.device)].cpu().numpy(), want)
    # A @ ones == row sums of the values (checksum of every edge weight, sequential order on both sides)
    ones = torch.ones((N, 4), dtype=torch.float32, device=h.device)
    np.testing.assert_array_equal((adj @ ones)[:, 0].cpu().numpy(), adj.segment_sum(axis=-1).cpu().numpy())
    # linearity within fp32 tolerance
    g = torch.randn((N, D), generator=big["gen"], device=h.device, dtype=torch.float32)
    lhs = adj @ (2.0 * h + 0.5 * g)
    rhs = 2.0 * out + 0.5 * (adj @ g)
    err = (lhs - rhs).abs().max().item()
    assert err <= 1e-4 * rhs.abs().max().item(), err
    # idempotent / deterministic
    assert torch.equal(out, adj @ h)


def test_mean_and_max_sampled_rows(big):
    adj, h = big["adj"], big["h"]
    csr = adj.csr
    rows = np.random.RandomState(2).randint(0, N, 256)
    idx = torch.as_tensor(rows, device=h.device)
    mean = ops.spmm(csr, None, h, reduce="mean")[idx].cpu().numpy()
    mx = ops.spmm(csr, None, h, reduce="max")[idx].cpu().numpy()
    rp = csr.rowptr[torch.as_tensor(np.stack([rows, rows + 1]), device=h.device)].cpu().numpy()
    for i, (s, e) in enumerate(zip(rp[0], rp[1])):
        hw = h[csr.col[s:e].long()].cpu().numpy()
        ids = np.zeros(e - s, np.int32)
        loc = np.arange(e - s, dtype=np.int32)
        np.testing.assert_array_equal(mean[i], c_oracle.aggregate(ids, loc, None, hw, 1, "mean")[0])
        np.testing.assert_array_equal(mx[i], c_oracle.aggregate(ids, loc, None, hw, 1, "max")[0])


def test_gat_full_size_attention_is_a_distribution_and_rows_match(big):
    h = big["h"]
    gen = big["gen"]
    ei = big["ei"]
    q = torch.randn((N, D), generator=gen, device=h.device, dtype=torch.float32)
    k = torch.randn((N, D), generator=gen, device=h.device, dtype=torch.float32)
    from tf_geometric_b200 import _structure
    csr, full = _structure.csr_for_edge_index(ei, N, add_self_loop=True)
    out, att = ops.gat_fused(csr, q, k, h, H, return_attention=True)
    seg = torch.repeat_interleave(torch.arange(N, device=h.device), (csr.rowptr[1:] - csr.rowptr[:-1]))
    sums = torch.zeros((N, H), dtype=torch.float64, device=h.device).index_add_(0, seg, att.double())
    assert float((sums - 1.0).abs().max()) < 1e-5                                 # softmax over each (dst, head)
    rows = np.random.RandomState(3).randint(0, N, 128)
    rp = csr.rowptr[torch.as_tensor(np.stack([rows, rows + 1]), device=h.device)].cpu().numpy()
    for r, s, e in zip(rows, rp[0], rp[1]):
        cols = csr.col[s:e].long()
        kk, vv = k[cols].cpu().numpy(), h[cols].cpu().numpy()
        qq = np.concatenate([q[r:r + 1].cpu().numpy(), kk[:0]])                   # local graph: node 0 = dst, 1.. = sources
        loc_q = np.concatenate([qq, np.zeros_like(kk)])
        loc_k = np.concatenate([np.zeros_like(qq), kk])
        loc_v = np.concatenate([np.zeros_like(qq), vv])
        m = e - s
        want = c_oracle.gat_core(np.zeros(m, np.int32), np.arange(1, m + 1, dtype=np.int32), loc_q, loc_k, loc_v, H)[0]
        got = out[r].cpu().numpy()
        assert np.all(np.abs(got - want) <= 2e-5 * np.abs(want) + 2e-6 * np.abs(want).max()), (r, np.abs(got - want).max())
    out2 = ops.gat_fused(csr, q, k, h, H)           # no attention output: the cp.async kernel
    assert float((out - out2).abs().max()) <= 2e-6 * float(out.abs().max())
    assert torch.equal(out2, ops.gat_fused(csr, q, k, h, H))       # deterministic


def test_graph_sage_mean_forward_backward_full_size(big):
    """BASELINE config 4 (GraphSAGE mean-aggregate fwd+bwd at ogbn-products shape, D = F = 100): the backward aggregation
    is the adjoint of the forward one, <mean_agg(x), g> == <x, d/dx>, checked in float64 over all 2.4M x 100 entries; the
    end-to-end layer gradient is checked on sampled rows against the explicit formula."""
    import time
    ei, gen = big["ei"], big["gen"]
    dev = ei.device
    F, U = 100, 128
    x = torch.randn((N, F), generator=gen, device=dev, dtype=torch.float32).requires_grad_(True)
    ws = (torch.randn((F, U), generator=gen, device=dev) * 0.1).requires_grad_(True)
    wn = (torch.randn((F, U), generator=gen, device=dev) * 0.1).requires_grad_(True)
    b = torch.zeros((2 * U,), device=dev).requires_grad_(True)
    g = torch.randn((N, 2 * U), generator=gen, device=dev, dtype=torch.float32)

    from tf_geometric_b200 import autograd
    agg = autograd.NeighborAggregate.apply(x, ei, None, "mean", N)
    gg = torch.randn((N, F), generator=gen, device=dev, dtype=torch.float32)
    (grad_x,) = torch.autograd.grad((agg * gg).sum(), x)
    lhs = float((agg.double() * gg.double()).sum())
    rhs = float((x.detach().double() * grad_x.double()).sum())
    assert abs(lhs - rhs) <= 1e-6 * max(abs(lhs), abs(rhs), 1.0), (lhs, rhs)

    torch.cuda.synchronize()
    t0 = time.perf_counter()
    out = tfg.nn.mean_graph_sage(x, ei, None, ws, wn, b, tfg.nn.relu, concat=True)
    (out * g).sum().backward()
    torch.cuda.synchronize()
    print("GraphSAGE mean fwd+bwd at products shape (first call, incl. CSC build): %.1f ms" % ((time.perf_counter() - t0) * 1e3))
    x.grad = ws.grad = wn.grad = b.grad = None
    t0 = time.perf_counter()
    out = tfg.nn.mean_graph_sage(x, ei, None, ws, wn, b, tfg.nn.relu, concat=True)
    (out * g).sum().backward()
    torch.cuda.synchronize()
    ms = (time.perf_counter() - t0) * 1e3
    print("GraphSAGE mean fwd+bwd at products shape (warm): %.1f ms -> %.2f G edges/s" % (ms, ei.shape[1] / ms / 1e6))
    # db = column sums of the masked upstream gradient; dWs = x^T (mask * g)[:, :U]
    mask_g = g * (out.detach() > 0)
    want_db = mask_g.double().sum(0)
    assert float((b.grad.double() - want_db).abs().max()) <= 1e-4 * float(want_db.abs().max())
    want_dws = (x.detach().double().t() @ mask_g[:, :U].double())
    assert float((ws.grad.double() - want_dws).abs().max()) <= 1e-4 * float(want_dws.abs().max())
    assert torch.isfinite(x.grad).all()
