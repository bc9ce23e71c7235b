# coding=utf-8
"""Whole-layer training contract at shapes that reach the fast kernels: forward and every gradient (x, each weight, the
bias, the edge weights where they are differentiable) of each convolution against float64 torch autograd, entry by
entry, within the bound of tests/train_bound.py; three SGD steps with in-place updates, each checked against a float64
reference built from the parameters the GPU holds at that step.

Graph (one family, `_graph`): n = 20 000 nodes, about 8 random in-edges each, plus
  * destination hub 101 (in-degree HUB_THRESHOLD + 500): a hub row of the forward CSR;
  * source hub 202 (out-degree HUB_THRESHOLD + 500): a hub row of the transposed CSR only, which every backward
    gather (dX = A^T G) cuts into slices and merges with the fix-up kernel;
  * nodes 0-9 without in-edges, nodes n-10 .. n-1 without out-edges, 500 duplicated edges and 50 explicit self loops
    (the layers that add self loops append theirs as well).
Widths F = 100 and U = 128: every projection has M·K >= 16384 and K <= GEMM_PROJ_MAX_K = 184, so x W and dX = G W^T run
on K4 (tfgk_gemm_proj_f32, transB for dX); the weight gradients reduce over K = n >= 4096 rows with split-K; K1 runs its
TMA ring at D = 100 and D = 128.  U = 30 (D % 4 != 0) takes K1's scalar kernel.

Bounds.  Linear chains (every case but GAT): |got - ref| <= e · S per entry, S the magnitude replay and e the sum of the
stages' roundings plus K4's term (tests/train_bound.py); each case lists its stages.  For the node-indexed outputs (the
forward and dx) e is per row, from that row's own chain (G.fwd_hops / bwd_hops); the weight gradients and column sums,
which sum over every node, take the largest degrees and n.
GAT: the tolerance test_gpu_gat_backward.py derives for the attention kernels, |got - ref| <= 1e-4 |ref| + 1e-5 max|ref|,
applied to the whole layer (the projections add K4's 2^-19-relative term and the weight gradients about sqrt(n)·2^-24
relative, both far below it).  The worst err / bound ratio of every output is printed (run with -s).

Max aggregation (K11a / K11b) runs through aggregate_neighbors(max_reducer) with ties from the duplicated edges;
max-pool GraphSAGE is not a case here: this graph has nodes without in-edges, whose float32-lowest maximum overflows
in the projection that follows (test_gpu_train.py trains it on a graph where every node has an in-edge).

Route pins (`test_routes_reached`): the kernels named in ROUTE_PINS are recorded with torch.profiler (and the ABI entry
names with _ffi.CallTrace) in a fresh interpreter while the backward of the cases that should reach them runs, so a change
of the dispatch that routes around a kernel fails here instead of leaving this suite green."""
import json
import os
import subprocess
import sys

import numpy as np
import pytest
import torch

import tf_geometric_b200 as tfg
from tf_geometric_b200 import ops, _ffi, _structure
from oracle import tfg_oracle as o
from oracle import torch_cpu_port as port
import train_bound as tb
from conftest import glorot

pytestmark = pytest.mark.gpu

N, F, UNITS = 20000, 100, 128
GAT_RTOL, GAT_ATOL_SCALE = 1e-4, 1e-5
DST_HUB, SRC_HUB = 101, 202


def _graph(seed=0, dst_hub=True):
    rs = np.random.RandomState(seed)
    n = N
    e = 8 * n
    row, col = rs.randint(10, n, e), rs.randint(0, n - 10, e)
    parts_r, parts_c = [row], [col]
    if dst_hub:
        parts_r.append(np.full(ops.HUB_THRESHOLD + 500, DST_HUB))
        parts_c.append(rs.randint(0, n - 10, ops.HUB_THRESHOLD + 500))
    parts_r.append(rs.randint(10, n, ops.HUB_THRESHOLD + 500))
    parts_c.append(np.full(ops.HUB_THRESHOLD + 500, SRC_HUB))
    row, col = np.concatenate(parts_r), np.concatenate(parts_c)
    w = (rs.rand(len(row)) + 0.2).astype(np.float32)
    dup = rs.randint(0, len(row), 500)
    loops = rs.randint(10, n - 10, 50)
    # a duplicate keeps its original's weight, so that its messages tie with the original's in a max aggregation
    row, col = np.concatenate([row, row[dup], loops]), np.concatenate([col, col[dup], loops])
    w = np.concatenate([w, w[dup], (rs.rand(50) + 0.2).astype(np.float32)])
    p = rs.permutation(len(row))
    return np.stack([row[p], col[p]]).astype(np.int32), w[p]


class G(object):
    """The graph of a case with its degrees and the float64 index tensors of the references.
    din_v / dout_v: in- and out-degree per node, plus the self loop some layers append (slack for the others); din /
    dout their maxima, which bound the chains of the outputs that sum over every node (weight gradients, column sums).
    The chains of node-indexed outputs are per row (train_bound's per-row chains): fwd_hops / bwd_hops give them for
    k hops over the forward / transposed CSR, each hop adding its row's reduction and the longest chain of the rows it
    gathers from, and, for normalised values, the degree sums behind them (those of the row and of each neighbour)."""

    def __init__(self, ei, w):
        self.ei, self.w, self.n = ei, w, N
        self.row, self.col = torch.from_numpy(ei[0].astype(np.int64)), torch.from_numpy(ei[1].astype(np.int64))
        self.din_v, self.dout_v = tb.degrees(ei[0], ei[1], N, loops=1)
        self.din, self.dout = int(self.din_v.max()), int(self.dout_v.max())
        self.fwd_norm = tb.neighbour_max(ei[0], ei[1], self.din_v)       # degree sums behind row r's values
        self.bwd_norm = tb.neighbour_max(ei[1], ei[0], self.din_v)       # ... behind the values source c is gathered by
        self.eid, self.wd = ops.as_device(ei, torch.int32), ops.as_device(w)

    def fwd_hops(self, k, start=0, norm=True):
        c = np.full(N, start, np.int64)
        for _ in range(k):
            c = self.din_v + 6 + np.maximum(tb.neighbour_max(self.ei[0], self.ei[1], c), self.fwd_norm if norm else 0)
        return c

    def bwd_hops(self, k, start=0, norm=True):
        c = np.full(N, start, np.int64)
        for _ in range(k):
            c = self.dout_v + 6 + np.maximum(tb.neighbour_max(self.ei[1], self.ei[0], c), self.bwd_norm if norm else 0)
        return c


_GRAPHS = {}


def graph(dst_hub=True):
    if dst_hub not in _GRAPHS:
        _GRAPHS[dst_hub] = G(*_graph(dst_hub=dst_hub))
    return _GRAPHS[dst_hub]


def host(t):
    return t.detach().cpu().numpy()


def _mask(t):
    return torch.from_numpy((host(t) > 0).astype(np.float64))


def _relu_out(d, y):
    return {"out": _mask(y)}


# ---- cases ----------------------------------------------------------------------------------------------------------
# A case is a dict:
#   params : {name: float32 array}, the differentiable inputs (x included when its gradient is checked)
#   mine   : (device params, g) -> y, the layer on the GPU
#   ref    : (Replay, float64 params, masks, g) -> y, the same layer in float64
#   masks  : (device params, y) -> {name: float64 0/1 tensor}, the ReLU masks the float32 path applied
#   eps    : {output name ("y" or a parameter): relative bound}, from the stages of that output's chain

def _x(rs, f=F):
    return rs.randn(N, f).astype(np.float32)


def _hidden_mask(x, k, b):
    """The mask of relu(x W + b) as the layer's own projection computes it (same kernel, same bits)."""
    return _mask(ops.gemm(x.detach(), k.detach(), bias=b.detach(), act=ops.ACT_RELU))


def case_gcn(g, units=UNITS, edge_grad=False):
    rs = np.random.RandomState(1 + units + edge_grad)
    P = dict(x=_x(rs), k=glorot(rs, F, units), b=rs.randn(units).astype(np.float32) * 0.1)
    if edge_grad:
        P["w"] = g.w

    def mine(d, g):
        adj = tfg.SparseMatrix(g.eid, d["w"] if edge_grad else g.wd, [N, N])
        return tfg.nn.gcn(d["x"], adj, d["k"], d["b"], tfg.nn.relu, cache=None)

    def ref(R, p, m, g):
        w = p["w"] if edge_grad else R.const(g.w)
        r2, c2, v = R.gcn_norm(g.row, g.col, w if edge_grad else w.detach(), N)
        return R.relu(R.spmm(r2, c2, v, p["x"] @ p["k"], N) + p["b"], m["out"])

    norm = g.din + 6                                  # degree sums, rsqrt, two scalings
    e = dict(y=tb.eps(g.fwd_hops(1) + 6, F), x=tb.gcn_dx_eps(g.ei[0], g.ei[1], N, units),
             k=tb.eps(int(g.bwd_hops(1).max()) + N + 6), b=tb.eps(N + 6))
    if edge_grad:                                     # K7's dot over U, then the normalisation's two segment sums
        e["w"] = tb.eps(2 * norm + units + 2 * g.din + g.dout + 20, F)
    return dict(params=P, mine=mine, ref=ref, masks=_relu_out, eps=e)


def case_sparse_matmul(g, units=UNITS):
    rs = np.random.RandomState(3 + units)
    P = dict(h=rs.randn(N, units).astype(np.float32), b=rs.randn(units).astype(np.float32) * 0.1,
             w=(g.w - 0.6).astype(np.float32))                                # signed values
    A = {}

    def mine(d, g):
        if "A" not in A or A["A"].value is not d["w"]:
            A["A"] = tfg.SparseMatrix(g.eid, d["w"], [N, N])
        return A["A"].matmul(d["h"], bias=d["b"], act=ops.ACT_RELU)

    def ref(R, p, m, g):
        return R.relu(R.spmm(g.row, g.col, p["w"], p["h"], N) + p["b"], m["out"])

    e = dict(y=tb.eps(g.din_v + 3), h=tb.transposed_gather_eps(g.ei[0], g.ei[1], N), w=tb.eps(units + 3),
             b=tb.eps(N + 3))
    return dict(params=P, mine=mine, ref=ref, masks=_relu_out, eps=e, holder=A)


def case_sage(g, reduce="mean", concat=True):
    rs = np.random.RandomState(5 + concat + len(reduce))
    P = dict(x=_x(rs), ws=glorot(rs, F, UNITS), wn=glorot(rs, F, UNITS),
             b=rs.randn(2 * UNITS if concat else UNITS).astype(np.float32) * 0.1)
    fn = {"mean": tfg.nn.mean_graph_sage, "sum": tfg.nn.sum_graph_sage}[reduce]
    cnt = torch.from_numpy(np.maximum(np.bincount(g.ei[0], minlength=N), 1).astype(np.float64)).unsqueeze(1)

    def mine(d, g):
        return fn(d["x"], g.eid, g.wd, d["ws"], d["wn"], d["b"], tfg.nn.relu, concat=concat)

    def ref(R, p, m, g):
        agg = R.spmm(g.row, g.col, R.const(g.w), p["x"], N)
        if reduce == "mean":
            agg = agg / cnt
        z = torch.cat([p["x"] @ p["ws"], agg @ p["wn"]], 1) if concat else p["x"] @ p["ws"] + agg @ p["wn"]
        return R.relu(z + p["b"], m["out"])

    # y: agg W_n may run on the SIMT kernel (it accumulates onto x W_s when not concatenated): F more roundings
    e = dict(y=tb.eps(g.din_v + F + 8, F), x=tb.eps(g.dout_v + 8, UNITS, UNITS), ws=tb.eps(N + 4),
             wn=tb.eps(g.din + N + 8), b=tb.eps(N + 4))
    return dict(params=P, mine=mine, ref=ref, masks=_relu_out, eps=e)


def case_gcn_graph_sage(g):
    rs = np.random.RandomState(7)
    P = dict(x=_x(rs), k=glorot(rs, F, UNITS), b=rs.randn(UNITS).astype(np.float32) * 0.1)
    normed = o.gcn_norm_adj(o.SparseMatrix(g.ei, np.ones_like(g.w), [N, N]), renorm=False)   # weights -> ones
    ni, nv = torch.from_numpy(normed.index.astype(np.int64)), normed.value

    def mine(d, g):
        return tfg.nn.gcn_graph_sage(d["x"], g.eid, g.wd, d["k"], d["b"], tfg.nn.relu)

    def ref(R, p, m, g):
        return R.relu(R.spmm(ni[0], ni[1], R.const(nv), p["x"], N) @ p["k"] + p["b"], m["out"])

    e = dict(y=tb.eps(g.fwd_hops(1) + 6, F), x=tb.eps(g.bwd_hops(1) + 6, UNITS), k=tb.eps(g.din + N + 6),
             b=tb.eps(N + 4))
    return dict(params=P, mine=mine, ref=ref, masks=_relu_out, eps=e)


def case_mean_pool_sage(g):
    rs = np.random.RandomState(8)
    H = 64
    P = dict(x=_x(rs), ws=glorot(rs, F, UNITS), wm=glorot(rs, F, H), wn=glorot(rs, H, UNITS),
             bm=rs.randn(H).astype(np.float32) * 0.1, b=rs.randn(2 * UNITS).astype(np.float32) * 0.1)
    cnt = torch.from_numpy(np.maximum(np.bincount(g.ei[0], minlength=N), 1).astype(np.float64)).unsqueeze(1)

    def mine(d, g):
        return tfg.nn.mean_pool_graph_sage(d["x"], g.eid, g.wd, d["ws"], d["wm"], d["wn"], d["bm"], d["b"], tfg.nn.relu)

    def masks(d, y):
        return dict(out=_mask(y), hid=_hidden_mask(d["x"], d["wm"], d["bm"]))

    def ref(R, p, m, g):
        h = R.relu(p["x"] @ p["wm"] + p["bm"], m["hid"])
        red = R.spmm(g.row, g.col, torch.ones(g.row.shape[0], dtype=torch.float64), h, N) / cnt
        return R.relu(torch.cat([p["x"] @ p["ws"], red @ p["wn"]], 1) + p["b"], m["out"])

    e = {k: tb.eps(2 * g.din + g.dout + N + 12, F, H, UNITS, UNITS) for k in ("ws", "wm", "wn", "bm", "b")}
    e.update(y=tb.eps(g.din_v + 12, F, H, UNITS, UNITS), x=tb.eps(g.dout_v + 12, F, H, UNITS, UNITS))
    return dict(params=P, mine=mine, ref=ref, masks=masks, eps=e)


def case_max_aggregate(g):
    """aggregate_neighbors(gcn_mapper, max_reducer, sum_updater): x + max_e w_e x[col_e] (K11a / K11b).  The maximum is
    chosen among the float32 products w_e x[col_e] (one IEEE multiply on the device as in numpy), so the reference routes
    the gradient to exactly the messages the kernel found, shared among ties (a duplicated edge carries its original's
    weight, so their messages tie); rows without in-edges hold float32 lowest."""
    rs = np.random.RandomState(9)
    D = F
    P = dict(x=_x(rs, D))
    msg32 = P["x"][g.ei[1]] * g.w[:, None]                                     # float32 products
    best = np.full((N, D), np.finfo(np.float32).min, np.float32)
    np.maximum.at(best, g.ei[0], msg32)
    sel = (msg32 == best[g.ei[0]]).astype(np.float64)
    ties = np.zeros((N, D))
    np.add.at(ties, g.ei[0], sel)
    assert (ties > 1).sum() >= 100, int((ties > 1).sum())              # the tie-sharing backward is exercised
    share = torch.from_numpy(sel / np.maximum(ties, 1)[g.ei[0]])
    empty = torch.from_numpy((np.bincount(g.ei[0], minlength=N) == 0).astype(np.float64)).unsqueeze(1)
    lowest = float(np.finfo(np.float32).min)

    def mine(d, g):
        return tfg.nn.aggregate_neighbors(d["x"], g.eid, g.wd, tfg.nn.gcn_mapper, tfg.nn.max_reducer,
                                          tfg.nn.sum_updater)

    def ref(R, p, m, g):
        msg = p["x"][g.col] * R.const(g.w).unsqueeze(1) * share
        agg = torch.zeros((N, D), dtype=torch.float64).index_add(0, g.row, msg)
        if R.magnitude:
            return p["x"] + agg
        return p["x"] + agg + empty * (lowest - p["x"].detach())        # lowest there, and dx = g as x + agg gives

    return dict(params=P, mine=mine, ref=ref, masks=lambda d, y: {}, eps=dict(y=tb.eps(3), x=tb.eps(g.dout_v + 6)))


def _normed(g, renorm=True):
    m = o.gcn_norm_adj(o.SparseMatrix(g.ei, g.w, [N, N]), renorm=renorm)
    return torch.from_numpy(m.index.astype(np.int64)), m.value


def case_appnp(g, k=3, alpha=0.15):
    rs = np.random.RandomState(10)
    P = dict(x=_x(rs), k0=glorot(rs, F, UNITS), b0=rs.randn(UNITS).astype(np.float32) * 0.1,
             k1=glorot(rs, UNITS, UNITS), b1=rs.randn(UNITS).astype(np.float32) * 0.1)
    ni, nv = _normed(g)

    def mine(d, g):
        return tfg.nn.appnp(d["x"], g.eid, g.wd, [d["k0"], d["k1"]], [d["b0"], d["b1"]], k=k, alpha=alpha,
                            training=True)

    def masks(d, y):
        return dict(hid=_hidden_mask(d["x"], d["k0"], d["b0"]))

    def ref(R, p, m, g):
        h = R.relu(p["x"] @ p["k0"] + p["b0"], m["hid"]) @ p["k1"] + p["b1"]
        out = h
        for _ in range(k):
            out = R.spmm(ni[0], ni[1], R.const(nv), out, N) * (1.0 - alpha) + h * alpha
        return out

    c = k * (max(g.din, g.dout) + 8) + g.din + N + 16
    e = {name: tb.eps(c, F, UNITS, UNITS, UNITS) for name in P}
    e.update(y=tb.eps(g.fwd_hops(k, start=8) + 8, F, UNITS), x=tb.eps(g.bwd_hops(k) + 16, F, UNITS, UNITS, UNITS))
    return dict(params=P, mine=mine, ref=ref, masks=masks, eps=e)


def case_sgc(g, k=2):
    rs = np.random.RandomState(11)
    P = dict(x=_x(rs), k=glorot(rs, F, UNITS), b=rs.randn(UNITS).astype(np.float32) * 0.1)
    ni, nv = _normed(g)

    def mine(d, g):
        return tfg.nn.sgc(d["x"], g.eid, g.wd, k, d["k"], d["b"], tfg.nn.relu)

    def ref(R, p, m, g):
        h = p["x"] @ p["k"]
        for _ in range(k):
            h = R.spmm(ni[0], ni[1], R.const(nv), h, N)
        return R.relu(h + p["b"], m["out"])

    e = dict(y=tb.eps(g.fwd_hops(k) + 4, F), x=tb.eps(g.bwd_hops(k) + 4, UNITS),
             k=tb.eps(int(g.bwd_hops(k).max()) + N + 4), b=tb.eps(N + 4))
    return dict(params=P, mine=mine, ref=ref, masks=_relu_out, eps=e)


def case_ssgc(g, k=3, alpha=0.2):
    rs = np.random.RandomState(12)
    P = dict(x=_x(rs), k0=glorot(rs, F, UNITS), b0=rs.randn(UNITS).astype(np.float32) * 0.1,
             k1=glorot(rs, UNITS, UNITS), b1=rs.randn(UNITS).astype(np.float32) * 0.1)
    ni, nv = _normed(g)

    def mine(d, g):
        return tfg.nn.ssgc(d["x"], g.eid, g.wd, [d["k0"], d["k1"]], [d["b0"], d["b1"]], k=k, alpha=alpha)

    def masks(d, y):
        return dict(hid=_hidden_mask(d["x"], d["k0"], d["b0"]))

    def ref(R, p, m, g):
        h = R.relu(p["x"] @ p["k0"] + p["b0"], m["hid"]) @ p["k1"] + p["b1"]
        out = h * alpha
        for _ in range(k):
            h = R.spmm(ni[0], ni[1], R.const(nv), h, N)
            out = out + (1 - alpha) * h / k
        return out

    c = k * (max(g.din, g.dout) + 8) + g.din + N + 16
    e = {name: tb.eps(c, F, UNITS, UNITS, UNITS) for name in P}
    e.update(y=tb.eps(g.fwd_hops(k, start=8) + 16, F, UNITS), x=tb.eps(g.bwd_hops(k) + 16, F, UNITS, UNITS, UNITS))
    return dict(params=P, mine=mine, ref=ref, masks=masks, eps=e)


def case_tagcn(g, k=2):
    rs = np.random.RandomState(13)
    P = dict(x=_x(rs), k=glorot(rs, (k + 1) * F, UNITS), b=rs.randn(UNITS).astype(np.float32) * 0.1)
    ni, nv = _normed(g, renorm=False)

    def mine(d, g):
        return tfg.nn.tagcn(d["x"], g.eid, g.wd, k, d["k"], d["b"], tfg.nn.relu)

    def ref(R, p, m, g):
        hops = [p["x"]]
        for _ in range(k):
            hops.append(R.spmm(ni[0], ni[1], R.const(nv), hops[-1], N))
        return R.relu(torch.cat(hops, 1) @ p["k"] + p["b"], m["out"])

    norm = g.din + 6
    c = norm + k * (max(g.din, g.dout) + 4) + (k + 1) * F + N + 8        # K = 300 > 184: the SIMT product
    e = {name: tb.eps(c) for name in ("k", "b")}
    e.update(y=tb.eps(g.fwd_hops(k) + (k + 1) * F + 8), x=tb.eps(g.bwd_hops(k, start=UNITS + 8) + 8))
    return dict(params=P, mine=mine, ref=ref, masks=_relu_out, eps=e)


def case_gin(g, eps_=0.3):
    rs = np.random.RandomState(14)
    P = dict(x=_x(rs), m=glorot(rs, F, UNITS), eps=np.array([eps_], np.float32))
    from tf_geometric_b200 import autograd

    def mine(d, g):
        return tfg.nn.gin(d["x"], g.eid, lambda h, training=None: autograd.dense(h, d["m"], None, tfg.nn.relu),
                          eps=d["eps"])

    def ref(R, p, m, g):
        ones = torch.ones(g.row.shape[0], dtype=torch.float64)
        return R.relu((p["x"] * (1.0 + p["eps"]) + R.spmm(g.row, g.col, ones, p["x"], N)) @ p["m"], m["out"])

    c = max(g.din, g.dout) + 8
    e = dict(y=tb.eps(g.din_v + 8, F), x=tb.eps(g.dout_v + 8, UNITS), m=tb.eps(c + N),
             eps=tb.eps(c + N * F + UNITS, UNITS))
    return dict(params=P, mine=mine, ref=ref, masks=_relu_out, eps=e)


def case_le_conv(g):
    rs = np.random.RandomState(15)
    P = dict(x=_x(rs))
    for k_ in ("ws", "wa", "wn"):
        P[k_] = glorot(rs, F, UNITS)
    for k_ in ("bs", "ba", "bn"):
        P[k_] = rs.randn(UNITS).astype(np.float32) * 0.1

    def mine(d, g):
        return tfg.nn.le_conv(d["x"], g.eid, g.wd, d["ws"], d["bs"], d["wa"], d["ba"], d["wn"], d["bn"], tfg.nn.relu)

    def ref(R, p, m, g):
        diff = R.sub(p["x"] @ p["wa"] + p["ba"], p["x"] @ p["wn"] + p["bn"])
        return R.relu(R.spmm(g.row, g.col, R.const(g.w), diff, N) + p["x"] @ p["ws"] + p["bs"], m["out"])

    c = max(g.din, g.dout) + N + 12
    e = {name: tb.eps(c, F, UNITS, UNITS) for name in P}
    e.update(y=tb.eps(g.din_v + 3 * F + 12, F, UNITS, UNITS), x=tb.eps(g.dout_v + 12, F, UNITS, UNITS))
    return dict(params=P, mine=mine, ref=ref, masks=_relu_out, eps=e)


def case_chebynet(g, k=3):
    rs = np.random.RandomState(16)
    P = dict(x=_x(rs), k0=glorot(rs, F, UNITS), k1=glorot(rs, F, UNITS), k2=glorot(rs, F, UNITS),
             b=rs.randn(UNITS).astype(np.float32) * 0.1)
    li, lv = o.chebynet_norm_edge(g.ei, N, g.w, "sym")
    li = torch.from_numpy(np.asarray(li).astype(np.int64))

    def mine(d, g):
        return tfg.nn.chebynet(d["x"], g.eid, g.wd, k, [d["k0"], d["k1"], d["k2"]], d["b"], tfg.nn.relu)

    def ref(R, p, m, g):
        t0 = p["x"]
        t1 = R.spmm(li[0], li[1], R.const(lv), t0, N)
        t2 = R.sub(R.spmm(li[0], li[1], R.const(lv), t1, N) * 2.0, t0)
        return R.relu(t0 @ p["k0"] + t1 @ p["k1"] + t2 @ p["k2"] + p["b"], m["out"])

    c = 2 * (max(g.din, g.dout) + 8) + g.din + N + 16
    e = {name: tb.eps(c, F, F, F, UNITS, UNITS, UNITS) for name in P}
    # y: the three projections accumulate through the GEMM's beta, which the SIMT kernel takes: 3F more roundings
    e.update(y=tb.eps(g.fwd_hops(2) + 3 * F + 16, F, F, F), x=tb.eps(g.bwd_hops(2) + 16, UNITS, UNITS, UNITS))
    return dict(params=P, mine=mine, ref=ref, masks=_relu_out, eps=e)


CASES = {
    "gcn": lambda: case_gcn(graph()),
    "gcn_edge_weight": lambda: case_gcn(graph(), edge_grad=True),
    "gcn_u30": lambda: case_gcn(graph(), units=30),
    "sparse_matmul": lambda: case_sparse_matmul(graph()),
    "sparse_matmul_u30": lambda: case_sparse_matmul(graph(), units=30),
    "sage_mean_concat": lambda: case_sage(graph(), "mean", True),
    "sage_mean": lambda: case_sage(graph(), "mean", False),
    "sage_sum_concat": lambda: case_sage(graph(), "sum", True),
    "sage_sum": lambda: case_sage(graph(), "sum", False),
    "sage_gcn": lambda: case_gcn_graph_sage(graph()),
    "mean_pool_sage": lambda: case_mean_pool_sage(graph()),
    "max_aggregate": lambda: case_max_aggregate(graph()),
    "appnp": lambda: case_appnp(graph()),
    "sgc": lambda: case_sgc(graph()),
    "ssgc": lambda: case_ssgc(graph()),
    "tagcn": lambda: case_tagcn(graph()),
    "gin": lambda: case_gin(graph()),
    "le_conv": lambda: case_le_conv(graph()),
    "chebynet": lambda: case_chebynet(graph()),
}


def _gout(rs, y):
    return rs.randn(*y.shape).astype(np.float32)


def run_linear_case(case, g, tag, gout_seed=0):
    """Forward + backward on the GPU and both float64 replays; returns {output: worst err / bound}.  case["params"]
    holds float32 arrays, or device tensors that already exist (the optimiser's parameters of the step tests)."""
    d = case["params"]
    if not torch.is_tensor(next(iter(d.values()))):
        d = {k: ops.as_device(v).requires_grad_(True) for k, v in d.items()}
    for v in d.values():
        v.grad = None
    y = case["mine"](d, g)
    gout = _gout(np.random.RandomState(gout_seed), y)
    (y * ops.as_device(gout)).sum().backward()
    masks = case["masks"](d, y)
    res = {}
    for magnitude in (False, True):
        R = tb.Replay(magnitude)
        p = {k: R.leaf(host(v)) for k, v in d.items()}
        yr = case["ref"](R, p, masks, g)
        (yr * R.upstream(gout)).sum().backward()
        res[magnitude] = dict(y=yr.detach().numpy(), **{k: p[k].grad.numpy() for k in p})
    got = dict(y=host(y), **{k: host(v.grad) for k, v in d.items()})
    ratios = {}
    for name, e in case["eps"].items():
        r = tb.ratio(got[name], res[False][name], res[True][name], e)
        ratios[name] = r
        if not r <= 1.0:
            i, a, b, bd = tb.worst_entry(got[name], res[False][name], res[True][name], e)
            raise AssertionError("{} {}: entry {} = {!r}, float64 {!r}, bound {:.3e} (ratio {:.3g})".format(
                tag, name, i, a, b, bd, r))
    print("{:<24s} worst err/bound {:.3g}  ({})".format(tag, max(ratios.values()),
                                                         ", ".join("{} {:.2g}".format(k, v) for k, v in ratios.items())))
    return ratios


@pytest.mark.parametrize("name", sorted(CASES))
def test_layer_matches_float64(name):
    run_linear_case(CASES[name](), graph(), name)


# ---- GAT -------------------------------------------------------------------------------------------------------------

def _gat_params(rs, H=8, dh=16):
    A = H * dh
    return dict(x=_x(rs), wq=glorot(rs, F, A), bq=rs.randn(A).astype(np.float32) * .1, wk=glorot(rs, F, A),
                bk=rs.randn(A).astype(np.float32) * .1, wv=glorot(rs, F, A), b=rs.randn(A).astype(np.float32) * .1)


GAT_NAMES = ("wq", "bq", "wk", "bk", "wv", "b", "x")


def _gat_ref(t, masks, row, col, H, att_scale):
    """port.gat_forward (split heads, no output activation) with the query / key ReLU masks of the float32 projections:
    a key of the source hub whose pre-activation lies within rounding of 0 would otherwise route its whole gradient
    (thousands of edges) differently in float64."""
    n = t["x"].shape[0]
    Q = ((t["x"] @ t["wq"] + t["bq"]) * masks[0]).index_select(0, row)
    K = ((t["x"] @ t["wk"] + t["bk"]) * masks[1]).index_select(0, col)
    V = t["x"] @ t["wv"]
    Q_ = torch.cat(torch.split(Q, Q.shape[1] // H, dim=-1), dim=0)
    K_ = torch.cat(torch.split(K, K.shape[1] // H, dim=-1), dim=0)
    rows_ = torch.cat([row + i * n for i in range(H)])
    cols_ = torch.cat([col + i * n for i in range(H)])
    att = port.segment_softmax((Q_ * K_).sum(-1) / (Q_.shape[-1] ** 0.5), rows_, n * H)
    if att_scale is not None:
        att = att * att_scale
    V_ = torch.cat(torch.split(V, V.shape[1] // H, dim=-1), dim=0)
    h_ = port.spmm(rows_, cols_, att, V_, n * H)
    return torch.cat(torch.split(h_, n, dim=0), dim=-1) + t["b"]


def _gat_ratio(got, ref):
    got, ref = np.asarray(got, np.float64), np.asarray(ref, np.float64)
    bound = GAT_RTOL * np.abs(ref) + GAT_ATOL_SCALE * float(np.abs(ref).max())
    return float((np.abs(got - ref) / np.maximum(bound, 1e-300)).max())


def run_gat(g, P, rate, seed, tag, H=8, gout_seed=0):
    """GAT(128, 8 heads of 16), relu query / key projections, no output activation; returns {output: ratio} and the
    device params (so that a caller can step them)."""
    d = P if torch.is_tensor(P["x"]) else {k: ops.as_device(v).requires_grad_(True) for k, v in P.items()}
    trace = _ffi.CallTrace()
    prev = _ffi.set_trace(trace)
    try:
        y = tfg.nn.gat(d["x"], g.eid, d["wq"], d["bq"], tfg.nn.relu, d["wk"], d["bk"], tfg.nn.relu, d["wv"], d["b"],
                       None, num_heads=H, edge_drop_rate=rate, training=True, seed=seed)
        gout = _gout(np.random.RandomState(gout_seed), y)
        (y * ops.as_device(gout)).sum().backward()
    finally:
        _ffi.set_trace(prev)
    recompute = trace.counts.get("tfgk_gat_bwd_dst_f32", 0)
    table = trace.counts.get("tfgk_gat_softmax_bwd_f32", 0)
    assert (recompute, table) == ((0, 1) if rate > 0 or g is graph(True) else (1, 0)), trace.counts

    ei_loops = o.add_self_loop_edge(g.ei, N)[0]
    att_scale = None
    if rate > 0.0:
        csr, _ = _structure.csr_for_edge_index(g.eid, N, add_self_loop=True)
        perm = host(csr.perm).astype(np.int64)
        mult_csr = o.dropout_scale(ei_loops.shape[1] * H, rate, seed).reshape(-1, H)
        mult = np.empty_like(mult_csr)
        mult[perm] = mult_csr
        att_scale = torch.tensor(mult.T.reshape(-1).astype(np.float64))
    t = {k: torch.tensor(host(v).astype(np.float64), requires_grad=True) for k, v in d.items()}
    masks = (_hidden_mask(d["x"], d["wq"], d["bq"]), _hidden_mask(d["x"], d["wk"], d["bk"]))
    yr = _gat_ref(t, masks, torch.from_numpy(ei_loops[0].astype(np.int64)),
                  torch.from_numpy(ei_loops[1].astype(np.int64)), H, att_scale)
    (yr * torch.tensor(gout.astype(np.float64))).sum().backward()
    ratios = dict(y=_gat_ratio(host(y), yr.detach().numpy()))
    for name in GAT_NAMES:
        ratios[name] = _gat_ratio(host(d[name].grad), t[name].grad.numpy())
    print("{:<24s} worst err/bound {:.3g}  ({})".format(tag, max(ratios.values()),
                                                         ", ".join("{} {:.2g}".format(k, v) for k, v in ratios.items())))
    bad = {k: v for k, v in ratios.items() if not v <= 1.0}
    assert not bad, "{}: outside the GAT bound: {}".format(tag, bad)
    return ratios, d


@pytest.mark.parametrize("path", ["recompute", "table_dropout"])
def test_gat_matches_float64(path):
    """recompute: no dropout and no destination hub (the stats forward takes no hub plan); table_dropout: the full graph
    (destination hub) with edge_drop_rate 0.3, so the DROP instantiations of spmm_heads128 / gat_softmax_bwd128 run."""
    g = graph(dst_hub=path != "recompute")
    run_gat(g, _gat_params(np.random.RandomState(17)), 0.3 if path == "table_dropout" else 0.0, 4242, "gat_" + path)


# ---- steps ---------------------------------------------------------------------------------------------------------

STEPS = 3


@pytest.mark.parametrize("name", ["gcn_edge_weight", "sparse_matmul"])
def test_sgd_steps_match_float64(name):
    """Three SGD steps (in-place updates of every parameter, edge weights included), each checked against the bound of
    step 0.  Each step's reference starts from the float32 parameters the GPU holds at that step; the SparseMatrix of
    `sparse_matmul` is built once and kept, so its cached CSR-ordered values must follow the updates, and GCN's
    SparseMatrix over the learnable weights is rebuilt and normalised again at every step."""
    case = CASES[name]()
    g = graph()
    d = {k: ops.as_device(v).requires_grad_(True) for k, v in case["params"].items()}
    opt = torch.optim.SGD(list(d.values()), lr=1e-3)          # small enough that the edge weights stay positive
    before = {k: host(v) for k, v in d.items()}
    for step in range(STEPS):
        if name == "gcn_edge_weight":
            assert float(d["w"].detach().min()) > 0          # the premise of Replay.inv_sqrt's magnitude mode
        opt.zero_grad(set_to_none=True)
        run_linear_case(dict(case, params=d), g, "{} step {}".format(name, step), gout_seed=step)
        opt.step()
    for k, v in d.items():                                          # the steps did move every parameter
        assert not np.array_equal(host(v), before[k]), k
    if name == "sparse_matmul":
        assert case["holder"]["A"].value is d["w"]                  # one matrix across the steps


def test_gat_dropout_sgd_steps():
    """Three SGD steps of GAT with attention dropout (a new mask each step).  The weight gradients sum over 20 000 nodes
    and reach hundreds, so the step is kept small enough (lr 1e-4) that the attention logits stay at the scale the GAT
    bound is stated for: a step of 0.05 multiplies them by about a hundred, and the rounding of exp grows with them."""
    g = graph()
    d = {k: ops.as_device(v).requires_grad_(True) for k, v in _gat_params(np.random.RandomState(18)).items()}
    opt = torch.optim.SGD(list(d.values()), lr=1e-4)
    for step in range(STEPS):
        opt.zero_grad(set_to_none=True)
        run_gat(g, d, 0.3, 1000 + step, "gat_dropout step {}".format(step), gout_seed=step)
        opt.step()


# ---- route pins ------------------------------------------------------------------------------------------------------
# (scenario, kernel-name fragments the profiler must record in its backward, ABI entries CallTrace must count)

ROUTE_PINS = [
    ("sage_mean", ["spmm_tma4_kernel", "spmm_hub_fixup_kernel", "gemm_proj_kernel", "splitk_reduce_kernel"], []),
    ("gat_table_dropout", ["spmm_heads128_kernel<4, true", "gat_softmax_bwd128_kernel<4, 4, true"], []),
    ("max_aggregate", ["max_bwd_kernel", "max_bwd_fixup_kernel"], []),
    ("gcn_edge_weight", [], ["tfgk_sddmm_csr_f32"]),
]


def _record_backward(name):
    """(kernel names, ABI counts) of the backward of one scenario; the forward runs before the profiler starts."""
    from torch.profiler import ProfilerActivity, profile
    if name == "gat_table_dropout":
        g = graph()
        d = {k: ops.as_device(v).requires_grad_(True) for k, v in _gat_params(np.random.RandomState(17)).items()}
        y = tfg.nn.gat(d["x"], g.eid, d["wq"], d["bq"], tfg.nn.relu, d["wk"], d["bk"], tfg.nn.relu, d["wv"], d["b"],
                       None, num_heads=8, edge_drop_rate=0.3, training=True, seed=7)
    else:
        case = CASES[name]()
        d = {k: ops.as_device(v).requires_grad_(True) for k, v in case["params"].items()}
        y = case["mine"](d, graph())
    loss = (y * torch.randn_like(y)).sum()
    trace = _ffi.CallTrace()
    torch.cuda.synchronize()
    prev = _ffi.set_trace(trace)
    try:
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            loss.backward()
            torch.cuda.synchronize()
    finally:
        _ffi.set_trace(prev)
    names = sorted({e.name for e in prof.events() if "tfgk::" in e.name})
    return names, dict(trace.counts)


def _record_routes():
    return {name: _record_backward(name) for name, _, _ in ROUTE_PINS}


@pytest.fixture(scope="module")
def route_record():
    """Recorded in a fresh interpreter, as test_gpu_k1k3_contract's dispatch table is: an earlier torch.profiler
    session in the same process can leave later ones without kernel records."""
    here = os.path.dirname(os.path.abspath(__file__))
    code = ("import json, sys; sys.path[:0] = [{!r}, {!r}]; import test_gpu_train_contract as t; "
            "print('@@' + json.dumps(t._record_routes()))").format(here, os.path.dirname(here))
    flags = ["-I"] if sys.flags.isolated else ["-s"] if sys.flags.no_user_site else []
    res = subprocess.run([sys.executable] + flags + ["-c", code], capture_output=True, text=True, timeout=900)
    assert res.returncode == 0, res.stdout[-2000:] + res.stderr[-4000:]
    return json.loads([line for line in res.stdout.splitlines() if line.startswith("@@")][-1][2:])


@pytest.mark.parametrize("name,kernels,entries", ROUTE_PINS, ids=[p[0] for p in ROUTE_PINS])
def test_routes_reached(name, kernels, entries, route_record):
    names, counts = route_record[name]
    assert names, "{}: the profiler recorded no tfgk kernel".format(name)
    for k in kernels:
        hit = [n for n in names if k in n]
        assert hit, "{}: no {} in the backward ({})".format(name, k, names)
        print("{:<20s} {:<40s} {}".format(name, k, hit[0]))
    for entry in entries:
        assert counts.get(entry, 0) >= 1, "{}: {} not called ({})".format(name, entry, counts)
        print("{:<20s} {:<40s} called {}x".format(name, entry, counts[entry]))
