# coding=utf-8
"""Multi-GPU execution of the hot path: 1-D partition by DESTINATION row block + halo all-gather of source rows.

The reference has no graph partitioning (its two "distributed" demos replicate the whole graph under
tf.distribute.MirroredStrategy, demo/demo_distributed_gcn.py:37-57); this is the new design of SURVEY.md section 8e.

  * rank r owns destination rows [r*B, min((r+1)*B, N)), B = ceil(N / R), all their in-edges and the same rows of x;
  * dense projections are row-local (weights replicated);
  * each aggregation needs the projected rows of every SOURCE: one all-gather (torch.distributed, NCCL over
    NVLink/NVSwitch between GPUs, gloo in the CPU tests) into a [R*B, D] buffer indexed by global node id;
  * softmax / mean / max are per destination, so nothing is reduced across ranks; the GCN normalisation exchanges only
    the [N] vector of deg^-1/2.
Per-row edge order is the caller's order, so every output row is bit-identical to the single-GPU result.

Round 2 - how the source rows reach a rank (the exchange step):
  * "p2p" (default on GPUs of one node): NO collective on the data path.  Every rank publishes rows in a peer-mapped
    buffer (peer.RowExchange: CUDA IPC mappings set up once; per publication one device-to-device copy and a device-side
    flag barrier over NVLink) and the other ranks pull them with tfgk_peer_pull (copy engine by default) on a side stream.
      - input narrower than what is aggregated (the bench: F = 100 against 128 + 256 projected columns): x itself is
        published and pulled into a local [N, F] table, and tfgk_gemm_proj_f32 projects every block as soon as it has
        landed - the pull of block j+1 travels while the tensor core works on block j.  3.8x fewer NVLink bytes than
        shipping projected rows; the projections replicated on every rank are tensor-core work.  Rows are identical to the
        ones the owner would compute (row-local arithmetic, same kernel).
      - input at least as wide (config 5): the local rows are projected straight into the published slot and the peers'
        projected rows are pulled (no replicated GEMM).
  * "p2p_fused": measured alternative - the projection GEMM's producers cp.async the owners' rows in place (a_parts of
    tfgk_gemm_proj_f32).  Correct, slower (peer reads bypass the local L2).
  * "collective": the round-1 path - project the local rows, all-gather the projected rows (NCCL on GPUs, gloo in the
    CPU tests); also the fallback when peer mappings cannot be set up.
tfg.layers.GCN / GAT accept [x_local, partitioned_graph] (or the result of partitioned_graph.share(...)).
"""
import os

import torch
import torch.distributed as dist

from . import ops
from .ops import CSR  # noqa: F401

ROW_ALIGN = 128       # partition blocks are multiples of the GEMM row tile, so a tile never straddles two owners


class RowPartition(object):
    """Block partition of node ids: rank r owns [lo(r), hi(r))."""

    def __init__(self, num_nodes, world_size, rank, align=1):
        self.num_nodes = int(num_nodes)
        self.world_size = int(world_size)
        self.rank = int(rank)
        self.block = (self.num_nodes + self.world_size - 1) // self.world_size
        if align > 1 and self.world_size > 1:
            self.block = (self.block + align - 1) // align * align
        self.lo = min(self.rank * self.block, self.num_nodes)
        self.hi = min(self.lo + self.block, self.num_nodes)
        self.n_local = self.hi - self.lo
        self.padded_nodes = self.block * self.world_size

    def owner_of(self, node_ids):
        return node_ids // self.block


class PartitionedGraph(object):
    """The slice of a graph one rank works on: edges whose destination it owns, destinations renumbered locally,
    sources kept as GLOBAL ids (they index the all-gathered buffer)."""

    def __init__(self, partition, local_edge_index, local_edge_weight=None, group=None, exchange=None):
        self.part = partition
        self.edge_index = local_edge_index          # int32 [2, E_local]: row in [0, n_local), col in [0, N)
        self.edge_weight = local_edge_weight
        self.group = group
        self.cache = {}
        # "p2p" | "collective"; default: p2p on CUDA with more than one rank (TFGK_DIST_EXCHANGE overrides)
        self.exchange = exchange or os.environ.get("TFGK_DIST_EXCHANGE") or (
            "p2p" if local_edge_index.is_cuda and partition.world_size > 1 else "collective")
        self._row_exchanges = {}
        self._pull_stream = None
        self._work = {}                             # persistent exchange buffers (no per-step allocation of the [N, width] tables)
        self.pull_events = []                       # (start, end) CUDA events around the pulls of each exchange (for bench.py)
        # peer pulls: copy engine (-1, default: no SMs taken from the GEMM running beside it) or the copy kernel on this many
        # CTAs (TFGK_DIST_PULL_CTAS > 0)
        self.pull_ctas = int(os.environ.get("TFGK_DIST_PULL_CTAS", "-1"))
        self.nvlink_bytes = 0                       # bytes pulled from / received from peers so far (accounting)

    @classmethod
    def from_global(cls, edge_index, edge_weight, num_nodes, rank=None, world_size=None, group=None, exchange=None):
        """Select this rank's in-edges from a full edge list (order preserved)."""
        rank = dist.get_rank(group) if rank is None else rank
        world_size = dist.get_world_size(group) if world_size is None else world_size
        edge_index = ops.as_device(edge_index, torch.int32)
        exchange = exchange or os.environ.get("TFGK_DIST_EXCHANGE") or (
            "p2p" if edge_index.is_cuda and world_size > 1 else "collective")
        part = RowPartition(num_nodes, world_size, rank, align=ROW_ALIGN if exchange.startswith("p2p") else 1)
        row = edge_index[0]
        mask = (row >= part.lo) & (row < part.hi)
        local = torch.stack([row[mask] - part.lo, edge_index[1][mask]]).contiguous()
        w = None
        if edge_weight is not None:
            w = ops.as_device(edge_weight, torch.float32, device=edge_index.device)[mask].contiguous()
        return cls(part, local, w, group, exchange)

    # ---- structure ------------------------------------------------------------------------------------------------
    def _with_self_loops(self, weight, fill):
        p = self.part
        dev = self.edge_index.device
        loc = torch.arange(p.n_local, dtype=torch.int32, device=dev)
        index = torch.cat([self.edge_index, torch.stack([loc, loc + p.lo])], dim=1).contiguous()
        if weight is None:
            weight = torch.ones((self.edge_index.shape[1],), dtype=torch.float32, device=dev)
        value = torch.cat([weight, torch.full((p.n_local,), fill, dtype=torch.float32, device=dev)]).contiguous()
        return index, value

    def csr(self, self_loops=False):
        key = "csr_loop" if self_loops else "csr"
        if key not in self.cache:
            index = self._with_self_loops(None, 1.0)[0] if self_loops else self.edge_index
            self.cache[key] = ops.csr_build(index[0].contiguous(), index[1].contiguous(), self.part.n_local,
                                            self.part.padded_nodes)
        return self.cache[key]

    def gcn_normed(self, renorm=True, improved=False):
        """Default GCN normalisation (norm='both', add_self_loop, sym=True; nn/conv/gcn.py:75-98) on the partition:
        row degrees are local, the column side needs deg^-1/2 of every node -> all-gather of one fp32 vector."""
        key = "gcn_normed_{}_{}".format(renorm, improved)
        if key in self.cache:
            return self.cache[key]
        p = self.part
        fill = 2.0 if improved else 1.0
        if renorm:
            index, value = self._with_self_loops(self.edge_weight, fill)
        else:
            index = self.edge_index
            value = self.edge_weight if self.edge_weight is not None else torch.ones(
                (index.shape[1],), dtype=torch.float32, device=index.device)
        csr = ops.csr_build(index[0].contiguous(), index[1].contiguous(), p.n_local, p.padded_nodes)
        deg = ops.csr_rowsum(csr, ops.permute(value, csr.perm))
        dis_local = ops.deg_inv(deg, ops.POW_INV_SQRT)
        dis_full = self.all_gather_rows(dis_local.unsqueeze(1)).squeeze(1).contiguous()
        normed = ops.scale_edges(index[0].contiguous(), index[1].contiguous(), value, dl=dis_local, dr=dis_full)
        if not renorm:
            index, normed = self._append_loops_after(index, normed, fill)
            csr = ops.csr_build(index[0].contiguous(), index[1].contiguous(), p.n_local, p.padded_nodes)
        self.cache[key] = (csr, ops.permute(normed, csr.perm))
        return self.cache[key]

    def _append_loops_after(self, index, value, fill):
        p = self.part
        loc = torch.arange(p.n_local, dtype=torch.int32, device=index.device)
        index = torch.cat([index, torch.stack([loc, loc + p.lo])], dim=1).contiguous()
        value = torch.cat([value, torch.full((p.n_local,), fill, dtype=torch.float32, device=value.device)]).contiguous()
        return index, value

    # ---- the exchange step -----------------------------------------------------------------------------------------
    def _row_exchange(self, width, device):
        """peer.RowExchange for rows of `width` floats, created on first use; None when peer mappings are unavailable
        on any rank (all ranks then agree on the collective path)."""
        if width in self._row_exchanges:
            return self._row_exchanges[width]
        from . import peer, _ffi
        ex, ok = None, 1
        try:
            ex = peer.RowExchange(self.part.block, width, device, self.group)
        except (_ffi.TfgkError, RuntimeError) as err:
            ok = 0
            self._peer_error = str(err)
        flag = torch.tensor([ok], dtype=torch.int32, device=device)
        dist.all_reduce(flag, op=dist.ReduceOp.MIN, group=self.group)
        if int(flag.item()) == 0:
            if ex is not None:
                ex.close()
            ex = None
            self.exchange = "collective"
        self._row_exchanges[width] = ex
        return ex

    def _workspace(self, name, shape, device):
        """Exchange buffers are kept across steps: they are consumed (projected / aggregated) before the next publication's
        pulls are enqueued behind it, and [N, width] tables of tens of GB must not bounce through the allocator."""
        buf = self._work.get(name)
        if buf is None or tuple(buf.shape) != tuple(shape) or buf.device != device:
            buf = torch.empty(shape, dtype=torch.float32, device=device)
            self._work[name] = buf
        return buf

    def new_step(self):
        """Forget which tensor was published last: the next layer call publishes its input again even if it is the same
        tensor object (bench.py calls this so that every timed step pays for the full exchange protocol)."""
        for ex in self._row_exchanges.values():
            if ex is not None:
                ex._published = None

    def project_all_rows(self, x_local, groups):
        """Dense projections of EVERY node's features, which each aggregation kernel then gathers from.
        groups: list of column groups, each a list of (weight [F, n], bias or None, act code); the projections of one
        group are laid side by side in one [padded_nodes, sum n] buffer (e.g. K | V).  Returns the list of buffers.
        p2p: peers' rows pulled over NVLink peer mappings on a side stream, blocks projected as they land (or, for wide
        inputs, the peers' projected rows pulled); collective: local projection + all-gather of the projected rows."""
        p = self.part
        dev = x_local.device
        widths = [sum(int(w.shape[1]) for w, _, _ in g) for g in groups]
        fused_ok = x_local.is_cuda and x_local.shape[1] % 4 == 0 and sum(widths) % 4 == 0        # 16-byte rows for the pulls
        if self.exchange == "p2p_fused":
            fused_ok = fused_ok and x_local.shape[1] <= ops.GEMM_PROJ_MAX_K                         # tfgk_gemm_proj_f32 limit
        if p.world_size == 1 or self.exchange not in ("p2p", "p2p_fused") or not fused_ok \
                or self._row_exchange(x_local.shape[1], dev) is None:
            send = torch.empty((p.block, sum(widths)), dtype=torch.float32, device=dev)
            if p.n_local < p.block:
                send[p.n_local:].zero_()
            _project_into(x_local, groups, send, p.n_local)
            full = self.all_gather_rows(send)
            if p.world_size > 1:
                self.nvlink_bytes += (p.world_size - 1) * p.block * sum(widths) * 4
            outs, c0 = [], 0
            for wd in widths:
                outs.append(full[:, c0:c0 + wd])
                c0 += wd
            return outs
        if self.exchange == "p2p_fused":
            # alternative: the GEMM's loads read the owners' rows in place (tfgk_gemm_proj_f32 a_parts).  Peer reads bypass
            # the local L2, so every column block re-reads the remote tile.
            ex = self._row_exchange(x_local.shape[1], dev)
            slot = ex.publish(x_local)
            outs = [torch.empty((p.padded_nodes, wd), dtype=torch.float32, device=dev) for wd in widths]
            pieces = _pieces(groups, outs)
            first = (p.rank + 1) % p.world_size
            for i in range(0, len(pieces), 4):
                ops.gemm_proj(ex.local_slot(slot), pieces[i:i + 4], a_parts=ex.slot_ptrs(slot), part_rows=p.block,
                              first_part=first, num_rows=p.num_nodes)
                self.nvlink_bytes += (p.num_nodes - p.n_local) * x_local.shape[1] * 4
            return outs
        main = torch.cuda.current_stream(dev)
        if self._pull_stream is None:
            self._pull_stream = torch.cuda.Stream(dev)
        side = self._pull_stream
        order = [(p.rank + k) % p.world_size for k in range(1, p.world_size)]       # every rank pulls from a different peer
        bounds = lambda r: (min(r * p.block, p.num_nodes), min((r + 1) * p.block, p.num_nodes))      # noqa: E731
        if x_local.shape[1] < sum(widths):
            # (1) the input is narrower than what is aggregated: publish x, pull the peers' blocks over NVLink into a local
            # [N, F] table on a side stream, and project every block as soon as it has landed - the pull of block j+1
            # travels while the tensor core works on block j; no collective, no halo of projected rows
            ex = self._row_exchange(x_local.shape[1], dev)
            slot = ex.publish(x_local)
            outs = [torch.empty((p.padded_nodes, wd), dtype=torch.float32, device=dev) for wd in widths]
            x_full = self._workspace("x_full", (p.padded_nodes, x_local.shape[1]), dev)
            side.wait_stream(main)
            events = []
            t0, t1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            with torch.cuda.stream(side):
                t0.record(side)
                for r in order:
                    lo, hi = bounds(r)
                    ex.pull(r, slot, hi - lo, x_full[lo:hi], max_ctas=self.pull_ctas)
                    ev = torch.cuda.Event()
                    ev.record(side)
                    events.append(ev)
                t1.record(side)
            self.pull_events.append((t0, t1))
            del self.pull_events[:-64]

            def project(rows, lo, hi):
                if hi <= lo:
                    return
                pieces = _pieces(groups, [o[lo:hi] for o in outs])
                for i in range(0, len(pieces), 4):
                    ops.gemm_proj(rows, pieces[i:i + 4])
            project(x_local, p.lo, p.hi)
            for r, ev in zip(order, events):
                main.wait_event(ev)
                lo, hi = bounds(r)
                project(x_full[lo:hi], lo, hi)
            self.nvlink_bytes += (p.num_nodes - p.n_local) * x_local.shape[1] * 4
            return outs
        # (2) the input is at least as wide as the projections: project the local rows straight into the published slot and
        # pull the peers' projected rows (no replicated GEMM)
        total = sum(widths)
        ex = self._row_exchange(total, dev)
        slot = ex.next_slot()
        mine = ex.local_slot(slot)
        _project_into(x_local, groups, mine, p.n_local)
        ex.commit(slot)
        full = self._workspace("rows_full_{}".format(total), (p.padded_nodes, total), dev)
        side.wait_stream(main)
        t0, t1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        with torch.cuda.stream(side):
            t0.record(side)
            for r in order:
                lo, hi = bounds(r)
                ex.pull(r, slot, hi - lo, full[lo:hi], max_ctas=self.pull_ctas)
            t1.record(side)
        self.pull_events.append((t0, t1))
        del self.pull_events[:-64]
        full[p.lo:p.hi].copy_(mine[:p.n_local])
        main.wait_stream(side)
        self.nvlink_bytes += (p.num_nodes - p.n_local) * total * 4
        outs, c0 = [], 0
        for wd in widths:
            outs.append(full[:, c0:c0 + wd])
            c0 += wd
        return outs

    def close(self):
        """Unmap the peers' buffers and free this rank's published buffers (collective: every rank calls it).  Optional -
        process exit releases them too."""
        for ex in self._row_exchanges.values():
            if ex is not None:
                ex.close()
        self._row_exchanges = {}
        self._work = {}

    def share(self, x_local, layers):
        """Publish x_local once and compute, in ONE fused launch sequence, the all-row projections of every layer in
        `layers` (tfg.layers.GCN / GAT ...).  Pass the result instead of x_local: layer([shared, partitioned_graph]).
        The result is meant to be consumed by those layers before the next share() / layer call on this graph: when the
        projected rows are pulled from the peers (input at least as wide as the projections) they live in an exchange buffer
        that the next exchange overwrites."""
        x_local = ops.as_device(x_local, torch.float32, device=self.edge_index.device)
        shared = SharedRows(x_local, self)
        groups, owners = [], []
        for layer in layers:
            layer._maybe_build([x_local])
            for key, group in layer.partitioned_projections():
                owners.append(key)
                groups.append(group)
        _forward_only("PartitionedGraph.share", x_local, *[t for group in groups for w, b, _ in group for t in (w, b)])
        if groups:
            for key, buf in zip(owners, self.project_all_rows(x_local, groups)):
                shared.projected[key] = buf
        return shared

    def all_gather_rows(self, local_rows, out=None, async_op=False):
        """[n_local, D] on every rank -> [R*B, D] indexed by global node id (rows >= N are padding).
        async_op=True returns (buffer, work): the collective runs on the communicator's stream and `work.wait()` makes the
        current stream wait for it - used to run the exchange under independent compute."""
        p = self.part
        d = local_rows.shape[1]
        if out is None:
            out = torch.empty((p.padded_nodes, d), dtype=local_rows.dtype, device=local_rows.device)
        if p.world_size == 1:
            out[:p.n_local].copy_(local_rows)
            return (out, None) if async_op else out
        send = local_rows
        if local_rows.shape[0] != p.block or not local_rows.is_contiguous():      # callers may pass block-padded rows
            send = torch.zeros((p.block, d), dtype=local_rows.dtype, device=local_rows.device)
            send[:local_rows.shape[0]].copy_(local_rows)
        work = dist.all_gather_into_tensor(out, send, group=self.group, async_op=async_op)
        return (out, work) if async_op else out


def _pieces(groups, outs):
    """(weight, bias, act, out view) per block of at most 128 columns, in buffer order."""
    pieces = []
    for group, out in zip(groups, outs):
        c0 = 0
        for w, b, act in group:
            for k0 in range(0, w.shape[1], 128):
                k1 = min(k0 + 128, w.shape[1])
                pieces.append((w[:, k0:k1], None if b is None else b[k0:k1], act, out[:, c0 + k0:c0 + k1]))
            c0 += w.shape[1]
    return pieces


def _project_into(x_local, groups, out, n_rows):
    outs, c0 = [], 0
    for g in groups:
        wd = sum(int(w.shape[1]) for w, _, _ in g)
        outs.append(out[:n_rows, c0:c0 + wd])
        c0 += wd
    pieces = _pieces(groups, outs)
    for i in range(0, len(pieces), 4):
        ops.gemm_proj(x_local, pieces[i:i + 4])


class SharedRows(object):
    """x_local plus the all-row projections computed for it by PartitionedGraph.share (keyed by weight identity)."""

    def __init__(self, x_local, pg):
        self.x, self.pg, self.projected = x_local, pg, {}
        self.shape, self.device, self.is_cuda = x_local.shape, x_local.device, x_local.is_cuda

    def __len__(self):
        return self.shape[0]

    def find(self, *weights):
        return self.projected.get(tuple(id(w) for w in weights))


def _forward_only(what, *tensors):
    """The partitioned path has no backward pass: fail loudly rather than return rows without a grad_fn (a trainable
    layer would silently receive no gradient)."""
    from . import autograd
    if autograd.needs_grad(*[t.x if isinstance(t, SharedRows) else t for t in tensors]):
        raise NotImplementedError("{}: the partitioned (multi-GPU) path is forward-only; call it under torch.no_grad() "
                                  "(or with layers created without trainable=True)".format(what))


def _unwrap(x_local, dev):
    if isinstance(x_local, SharedRows):
        return x_local.x, x_local
    return ops.as_device(x_local, torch.float32, device=dev), None


def gcn_partitioned(pg, x_local, kernel, bias=None, activation=None, renorm=True, improved=False):
    """tfg.nn.gcn on a PartitionedGraph: returns this rank's rows of act(norm(A) (x W) + b), or of act((norm(A) x) W + b)
    for the widths ops.spmm_proj takes, like the single-GPU layer."""
    dev = pg.edge_index.device
    _forward_only("gcn_partitioned", x_local, kernel, bias)
    x_local, shared = _unwrap(x_local, dev)
    csr, value_csr = pg.gcn_normed(renorm=renorm, improved=improved)
    act_code, leftover = ops.activation_code(activation)
    bias = None if bias is None else ops.as_device(bias, torch.float32, device=dev)
    if kernel is not None and x_local.is_cuda and ops.spmm_proj_shape(x_local.shape[1], kernel.shape[1]):
        # narrower input than output: gather x's rows and project each aggregate in the kernel's epilogue, as the
        # single-GPU layer does (same bits)
        out = ops.spmm_proj(csr, value_csr, pg.all_gather_rows(x_local),
                            ops.as_device(kernel, torch.float32, device=dev), bias=bias, act=act_code)
        return leftover(out) if leftover is not None else out
    h_full = shared.find(kernel) if shared is not None and kernel is not None else None
    if h_full is None:
        if kernel is None:
            h_full = pg.all_gather_rows(x_local)
        else:
            h_full = pg.project_all_rows(x_local, [[(ops.as_device(kernel, torch.float32, device=dev), None, ops.ACT_NONE)]])[0]
    out = ops.spmm(csr, value_csr, h_full, reduce="sum", bias=bias, act=act_code)
    return leftover(out) if leftover is not None else out


def gat_partitioned(pg, x_local, query_kernel, query_bias, query_activation, key_kernel, key_bias, key_activation,
                    kernel, bias=None, activation=None, num_heads=1):
    """tfg.nn.gat (split_value_heads=True) on a PartitionedGraph: Q stays local, K and V travel in ONE all-gather of a
    [n_local, A + U] buffer that both projections write into directly."""
    dev = pg.edge_index.device
    _forward_only("gat_partitioned", x_local, query_kernel, query_bias, key_kernel, key_bias, kernel, bias)
    x_local, shared = _unwrap(x_local, dev)
    f32 = lambda t: None if t is None else ops.as_device(t, torch.float32, device=dev)   # noqa: E731
    q_act, q_left = ops.activation_code(query_activation)
    k_act, k_left = ops.activation_code(key_activation)
    if q_left is not None or k_left is not None:
        raise NotImplementedError("partitioned GAT supports relu / None for the query and key activations")
    kv_full = shared.find(key_kernel, kernel) if shared is not None else None
    wq, wk, wv = f32(query_kernel), f32(key_kernel), f32(kernel)
    a = wk.shape[1]
    if kv_full is None:
        kv_full = pg.project_all_rows(x_local, [[(wk, f32(key_bias), k_act), (wv, None, ops.ACT_NONE)]])[0]
    Q = torch.empty((x_local.shape[0], wq.shape[1]), dtype=torch.float32, device=dev)
    _project_into(x_local, [[(wq, f32(query_bias), q_act)]], Q, x_local.shape[0])
    act_code, leftover = ops.activation_code(activation)
    out = ops.gat_fused(pg.csr(self_loops=True), Q, kv_full[:, :a], kv_full[:, a:], num_heads,
                        bias=None if bias is None else f32(bias), act=act_code)
    return leftover(out) if leftover is not None else out


def gcn_gat_overlapped(pg, x_local, gcn_kernel, gcn_bias, gcn_activation,
                       query_kernel, query_bias, key_kernel, key_bias, kernel, bias, gat_activation, num_heads):
    """One GCN layer and one GAT layer on the same partitioned graph with the two halo exchanges issued asynchronously:
    all projections run first, the all-gather of h (GCN) and of K|V (GAT) are queued back to back on the communicator
    stream, and the GCN aggregation runs while K|V is still travelling.  Results are identical to calling
    gcn_partitioned / gat_partitioned one after the other (relu query/key activations)."""
    dev = pg.edge_index.device
    _forward_only("gcn_gat_overlapped", x_local, gcn_kernel, gcn_bias, query_kernel, query_bias, key_kernel, key_bias, kernel, bias)
    x_local = ops.as_device(x_local, torch.float32, device=dev)
    f32 = lambda t: None if t is None else ops.as_device(t, torch.float32, device=dev)   # noqa: E731
    csr, value_csr = pg.gcn_normed()
    h_local = ops.gemm(x_local, f32(gcn_kernel))
    h_full, work_h = pg.all_gather_rows(h_local, async_op=True)
    wq, wk, wv = f32(query_kernel), f32(key_kernel), f32(kernel)
    a, u = wq.shape[1], wv.shape[1]
    Q = ops.gemm(x_local, wq, bias=f32(query_bias), act=ops.ACT_RELU)
    kv_local = torch.empty((x_local.shape[0], a + u), dtype=torch.float32, device=dev)
    ops.gemm(x_local, wk, bias=f32(key_bias), act=ops.ACT_RELU, out=kv_local[:, :a])
    ops.gemm(x_local, wv, out=kv_local[:, a:])
    kv_full, work_kv = pg.all_gather_rows(kv_local, async_op=True)
    if work_h is not None:
        work_h.wait()
    act_gcn, left_gcn = ops.activation_code(gcn_activation)
    out_gcn = ops.spmm(csr, value_csr, h_full, reduce="sum", bias=f32(gcn_bias), act=act_gcn)
    if left_gcn is not None:
        out_gcn = left_gcn(out_gcn)
    if work_kv is not None:
        work_kv.wait()
    act_gat, left_gat = ops.activation_code(gat_activation)
    out_gat = ops.gat_fused(pg.csr(self_loops=True), Q, kv_full[:, :a], kv_full[:, a:], num_heads, bias=f32(bias),
                            act=act_gat)
    if left_gat is not None:
        out_gat = left_gat(out_gat)
    return out_gcn, out_gat


# ---- bench.py --gpus N ------------------------------------------------------------------------------------------------

def _tolerance_fraction(got, want):
    """max |got - want| / (1e-4 * max|want| + 1e-4 * |want|): <= 1 means inside north_star's fp32 gate
    (allclose(rtol=1e-4, atol=1e-4 * max|ref|))."""
    bound = 1e-4 * want.abs().max() + 1e-4 * want.abs() + 1e-30
    return float(((got - want).abs() / bound).max())


def _sampled_row_check(pg, edge_index_global, n, x_hosts, gcn, gat, out_gcn, out_gat, heads, samples=48):
    """Independent float64 restatement (plain torch on the device, no kernel of this library) of GCN and GAT for a few
    of this rank's rows, from the GLOBAL edge list and the features of every rank: guards the path that is timed."""
    p = pg.part
    dev = out_gcn.device
    gen = torch.Generator(device="cpu")
    gen.manual_seed(7 + p.rank)
    rows = (torch.randint(0, max(p.n_local, 1), (samples,), generator=gen) + p.lo).to(dev)
    row_g, col_g = edge_index_global[0].long(), edge_index_global[1].long()
    deg = torch.bincount(row_g, minlength=n).double() + 1.0                   # renormalised: A + I
    x_all = torch.cat([h.to(dev) for h in x_hosts]).double()
    w_gcn = gcn.kernel.double()
    wq, wk, wv = gat.query_kernel.double(), gat.key_kernel.double(), gat.kernel.double()
    worst = 0.0
    for r in rows.tolist():
        nb = torch.cat([col_g[row_g == r], torch.tensor([r], device=dev)])
        # GCN: relu(sum_j d_r^-1/2 d_j^-1/2 (x_j W) + b)
        coef = (deg[r] ** -0.5) * (deg[nb] ** -0.5)
        want = torch.relu((coef[:, None] * (x_all[nb] @ w_gcn)).sum(0) + gcn.bias.double())
        got = out_gcn[r - p.lo].double()
        worst = max(worst, _tolerance_fraction(got, want))
        # GAT: per head softmax over the neighbours (self loop included) of <q_r, k_j> / sqrt(d)
        q = torch.relu(x_all[r] @ wq + gat.query_bias.double()).view(heads, -1)
        k = torch.relu(x_all[nb] @ wk + gat.key_bias.double()).view(len(nb), heads, -1)
        v = (x_all[nb] @ wv).view(len(nb), heads, -1)
        att = torch.softmax((k * q[None]).sum(-1) / (q.shape[1] ** 0.5), dim=0)
        want = torch.relu((att[:, :, None] * v).sum(0).reshape(-1) + gat.bias.double())
        got = out_gat[r - p.lo].double()
        worst = max(worst, _tolerance_fraction(got, want))
    return worst


def _hash_features(row0, n_rows, width, device):
    """Deterministic synthetic features as a function of the GLOBAL row id: any rank can recompute any row (cfg 5 never
    materialises the whole matrix on one GPU).  Values in [-1, 1)."""
    r = torch.arange(row0, row0 + n_rows, dtype=torch.int64, device=device).unsqueeze(1)
    c = torch.arange(width, dtype=torch.int64, device=device).unsqueeze(0)
    return (((r * 2654435761 + c * 40503 + 12345) % 2000003).float() / 1000001.5 - 1.0).contiguous()


def bench_papers(args, rank, world, device, metric, config):
    """BASELINE config 5: GCN(128, relu) forward at ogbn-papers100M shape (111,059,956 nodes / 1,615,685,872 directed edges /
    128 features), destination-partitioned.  With 8 ranks this is the configuration itself; with fewer ranks every rank keeps
    the per-GPU load of the 8-rank run (world/8 of the nodes and edges) and the line says so.  Edges are generated per
    partition on the device (seed 1000 + rank; the global graph never exists anywhere), features per owner."""
    import numpy as np
    import bench as B
    import tf_geometric_b200 as tfg
    from . import _ffi

    cfg = B.CONFIGS["cfg5"]
    F = cfg["features"]
    n_total = int(cfg["nodes"] * args.scale) * world // 8 if world != 8 else int(cfg["nodes"] * args.scale)
    e_total = int(cfg["edges"] * args.scale) * world // 8 if world != 8 else int(cfg["edges"] * args.scale)
    exchange = os.environ.get("TFGK_DIST_EXCHANGE") or ("p2p" if world > 1 else "collective")
    part = RowPartition(n_total, world, rank, align=ROW_ALIGN if exchange.startswith("p2p") else 1)
    e_local = e_total // world
    gen = torch.Generator(device=device)
    gen.manual_seed(1000 + rank)
    row_local = torch.randint(0, max(part.n_local, 1), (e_local,), generator=gen, device=device, dtype=torch.int32)
    col_global = torch.randint(0, n_total, (e_local,), generator=gen, device=device, dtype=torch.int32)
    pg = PartitionedGraph(part, torch.stack([row_local, col_global]).contiguous(), None, exchange=exchange)
    del row_local, col_global
    x = _hash_features(part.lo, part.n_local, F, device)
    gcn = tfg.layers.GCN(B.UNITS, activation=tfg.nn.relu, seed=2)

    def step(xd):
        pg.new_step()
        return (gcn([xd, pg]),)

    torch.cuda.synchronize()
    t0 = __import__("time").perf_counter()
    out = step(x)[0]
    torch.cuda.synchronize()
    t_cache = __import__("time").perf_counter() - t0

    # parity before timing: sampled destination rows from first principles in float64 (features recomputed from the
    # global ids, degrees from an all-gather of per-rank edge counts - nothing of the library's exchange is reused)
    counts = torch.bincount(pg.edge_index[0].long(), minlength=part.block).to(torch.int32)
    if counts.numel() < part.block:
        counts = torch.cat([counts, torch.zeros(part.block - counts.numel(), dtype=torch.int32, device=device)])
    deg_all = torch.empty((part.padded_nodes,), dtype=torch.int32, device=device)
    dist.all_gather_into_tensor(deg_all, counts[:part.block].contiguous())
    rows = torch.randint(0, max(part.n_local, 1), (32,), generator=torch.Generator(device="cpu").manual_seed(5 + rank))
    w64 = gcn.kernel.double()
    worst = 0.0
    erow, ecol = pg.edge_index[0], pg.edge_index[1].long()
    for r in rows.tolist():
        nb = torch.cat([ecol[erow == r], torch.tensor([r + part.lo], device=device)])
        d_r = float(deg_all[r + part.lo]) + 1.0
        coef = (d_r ** -0.5) * ((deg_all[nb].double() + 1.0) ** -0.5)
        xs = torch.cat([_hash_features(int(j), 1, F, device) for j in nb.tolist()]).double()
        want = torch.relu((coef[:, None] * (xs @ w64)).sum(0) + gcn.bias.double())
        got = out[r].double()
        worst = max(worst, _tolerance_fraction(got, want))
    check = torch.tensor([worst], dtype=torch.float64, device=device)
    dist.all_reduce(check, op=dist.ReduceOp.MAX)
    if float(check[0]) > 1.0:
        raise SystemExit("cfg5 parity check failed: sampled-row error is {:.3e} of the tolerance".format(float(check[0])))
    del deg_all, counts, out

    for _ in range(max(args.warmup, 3) - 1):
        step(x)
    trace = _ffi.CallTrace(timed=("tfgk_spmm_f32", "tfgk_gemm_proj_f32", "tfgk_gemm_f32"))
    _ffi.set_trace(trace)
    sampler = B.ClockSampler(device.index)
    sampler.start()
    nv0 = pg.nvlink_bytes
    del pg.pull_events[:]
    torch.cuda.synchronize(); dist.barrier(); torch.cuda.synchronize()
    ev = [torch.cuda.Event(enable_timing=True) for _ in range(2)]
    ev[0].record()
    for _ in range(args.steps):
        step(x)
    ev[1].record()
    torch.cuda.synchronize(); dist.barrier(); torch.cuda.synchronize()
    clocks = sampler.stop()
    _ffi.set_trace(None)
    nvlink_per_step = (pg.nvlink_bytes - nv0) / args.steps
    t = torch.tensor([ev[0].elapsed_time(ev[1]) / args.steps], dtype=torch.float64, device=device)
    dist.all_reduce(t, op=dist.ReduceOp.MAX)
    ms_step = float(t.item())
    pulls = [a.elapsed_time(b) for a, b in pg.pull_events[-args.steps:]]
    pull_ms = float(np.mean(pulls)) if pulls else 0.0
    spmm_ms = float(np.mean(trace.elapsed_ms("tfgk_spmm_f32")))
    proj_ms = float(np.sum(trace.elapsed_ms("tfgk_gemm_proj_f32")) + np.sum(trace.elapsed_ms("tfgk_gemm_f32"))) / args.steps
    e_loop = e_local + part.n_local
    spmm_bytes = e_loop * (4 * B.UNITS + 8) + part.n_local * (4 * B.UNITS + 8)
    peak, peak_src = B.measured_peak_gbs()
    mem = torch.cuda.max_memory_allocated(device) / 2 ** 30
    launches = sum(trace.counts.get(k, 0) for k in ("tfgk_spmm_f32", "tfgk_gemm_proj_f32", "tfgk_gemm_f32", "tfgk_peer_barrier"))
    if rank == 0:
        config = dict(config, nodes=n_total, edges=e_total, edges_per_step=e_total,
                      workload="{} ({} nodes, {} directed edges, {} features), uniform random directed edges generated per "
                               "partition{}".format(cfg["what"], n_total, e_total, F,
                                                    "" if world == 8 else " - PER-GPU SCALE: {}/8 of the 8-GPU configuration".format(world)),
                      parallelism="dst-partitioned x{}".format(world))
        line = {"metric": metric, "value": e_total / (ms_step * 1e-3), "unit": "edges/s", "n_gpus": world,
                "steps": args.steps, "warmup": max(args.warmup, 3), "ms_per_step": ms_step, "higher_is_better": True,
                "scaling": "weak", "vs_baseline": None, "dtype": "f32", "data": "synthetic", "config": config,
                "clocks": clocks, "e2e": None, "gpu_launches": launches,
                "roofline": {"bound": "hbm", "kernel": "spmm_tma4_kernel<false,3> (tfgk_spmm_f32), rank 0 partition",
                             "achieved": spmm_bytes / (spmm_ms * 1e-3) / 1e9, "peak": peak, "unit": "GB/s",
                             "frac": spmm_bytes / (spmm_ms * 1e-3) / 1e9 / peak, "traffic": None, "peak_source": peak_src,
                             "algorithmic_bytes": spmm_bytes, "kernel_ms": spmm_ms},
                "cpu_baseline": None,
                "breakdown_ms": {"gcn_spmm": spmm_ms, "projection_local_rows": proj_ms, "peer_pulls": pull_ms,
                                 "peer_pull_GBps": (nvlink_per_step / (pull_ms * 1e-3) / 1e9) if pull_ms > 0 else None,
                                 "first_call_incl_cache_s": t_cache},
                "parity": {"sampled_rows_error_as_fraction_of_tolerance_vs_float64": float(check[0]),
                           "tolerance": "allclose(rtol=1e-4, atol=1e-4*max|ref|)"},
                "max_memory_GiB_rank0": mem,
                "exchange": {"mode": pg.exchange, "nvlink_bytes_in_per_rank_per_step": nvlink_per_step,
                             "hbm_algorithmic_bytes_per_rank_per_step": spmm_bytes + part.n_local * B.UNITS * 4
                             + n_total * (F + B.UNITS) * 4,
                             "note": "the step is bound by the exchange: every rank needs almost every source row "
                                     "(uniform random sources), i.e. 7/8 of the [N, 128] table over NVLink per forward"}}
        B.emit(line)
    dist.destroy_process_group()


def bench_partitioned(args, rank, world, device, metric, config):
    """Strong scaling of the bench workload: the same synthetic graph, destination-partitioned over `world` ranks, driven
    through tfg.layers.GCN / GAT with [x_local, partitioned_graph] inputs.  Timed on the device with CUDA events between
    barriers; the reported time is the max over ranks."""
    import numpy as np
    import bench as B
    import tf_geometric_b200 as tfg
    from . import _ffi

    n = int(B.PRODUCTS_NODES * args.scale)
    pairs = int(B.PRODUCTS_UNDIRECTED * args.scale)
    edge_index = B.make_graph_device(n, pairs, 0, device)      # same seed on every rank -> identical global graph
    E = edge_index.shape[1]
    pg = PartitionedGraph.from_global(edge_index, None, n, rank, world)
    p = pg.part

    def features(r):
        part = RowPartition(n, world, r, align=ROW_ALIGN if pg.exchange.startswith("p2p") else 1)
        gen = torch.Generator(device="cpu")
        gen.manual_seed(100 + r)
        return torch.randn((part.n_local, B.FEATURES), generator=gen, dtype=torch.float32)

    x_host = features(rank).pin_memory()
    x = x_host.to(device)
    gcn = tfg.layers.GCN(B.UNITS, activation=tfg.nn.relu, seed=2)
    gat = tfg.layers.GAT(B.UNITS, num_heads=B.HEADS, activation=tfg.nn.relu, seed=3)

    def step(xd):
        pg.new_step()                                          # every step publishes and pulls its input again
        shared = pg.share(xd, [gcn, gat])                      # one fused all-gather -> projection launch for both layers
        return gcn([shared, pg]), gat([shared, pg])

    a, b = step(x)                                             # builds weights, CSRs, normalisation, peer mappings
    torch.cuda.synchronize()
    # parity of the path that is timed, before timing: (1) sampled rows against a float64 restatement,
    # (2) all rows bit-identical to the collective (NCCL all-gather) path
    err = _sampled_row_check(pg, edge_index, n, [features(r) for r in range(world)], gcn, gat, a, b, B.HEADS)
    del edge_index
    mode = pg.exchange
    identical = None
    if mode.startswith("p2p"):
        pg.exchange = "collective"
        a2, b2 = step(x)
        pg.exchange = mode
        identical = bool(torch.equal(a, a2) and torch.equal(b, b2))
        del a2, b2
    check = torch.tensor([err, 0.0 if identical in (None, True) else 1.0], dtype=torch.float64, device=device)
    dist.all_reduce(check, op=dist.ReduceOp.MAX)
    if float(check[0]) > 1.0 or float(check[1]) != 0.0:
        raise SystemExit("partitioned path failed its parity check: sampled-row error {:.3e} of the tolerance, p2p == collective: {}".format(
            float(check[0]), float(check[1]) == 0.0))
    del a, b
    torch.cuda.empty_cache()

    for _ in range(max(args.warmup, 3)):
        step(x)
    trace = _ffi.CallTrace(timed=("tfgk_gat_fused_f32", "tfgk_spmm_f32", "tfgk_gemm_proj_f32"))
    _ffi.set_trace(trace)
    sampler = B.ClockSampler(device.index)
    sampler.start()
    nv0 = pg.nvlink_bytes
    torch.cuda.synchronize()
    dist.barrier()
    torch.cuda.synchronize()
    ev = [torch.cuda.Event(enable_timing=True) for _ in range(2)]
    ev[0].record()
    for _ in range(args.steps):
        step(x)
    ev[1].record()
    torch.cuda.synchronize()
    dist.barrier()
    torch.cuda.synchronize()
    clocks = sampler.stop()
    _ffi.set_trace(None)
    nvlink_per_step = (pg.nvlink_bytes - nv0) / args.steps
    t = torch.tensor([ev[0].elapsed_time(ev[1]) / args.steps], dtype=torch.float64, device=device)
    dist.all_reduce(t, op=dist.ReduceOp.MAX)
    ms_step = float(t.item())

    e2e = None
    if not args.no_e2e:
        local = B.run_e2e(args, device, x_host, step, p.n_local, E, barrier=dist.barrier)
        t2 = torch.tensor([local["ms_per_step"]], dtype=torch.float64, device=device)
        dist.all_reduce(t2, op=dist.ReduceOp.MAX)
        e2e = dict(local, value=2.0 * E / (float(t2.item()) * 1e-3), ms_per_step=float(t2.item()),
                   h2d_bytes_per_step=n * B.FEATURES * 4, d2h_bytes_per_step=2 * n * B.UNITS * 4)

    gat_ms = float(np.mean(trace.elapsed_ms("tfgk_gat_fused_f32")))
    spmm_ms = float(np.mean(trace.elapsed_ms("tfgk_spmm_f32")))
    proj_ms = float(np.sum(trace.elapsed_ms("tfgk_gemm_proj_f32"))) / args.steps
    e_local = pg.csr(self_loops=True).nnz
    gat_bytes = e_local * (8 * B.UNITS + 4) + p.n_local * (8 * B.UNITS + 8)
    peak, peak_src = B.measured_peak_gbs()
    launching = ("tfgk_gat_fused_f32", "tfgk_spmm_f32", "tfgk_gemm_f32", "tfgk_gemm_proj_f32", "tfgk_peer_barrier")
    launches = sum(trace.counts.get(k, 0) for k in launching)
    if rank == 0:
        hbm_step = gat_bytes + e_local * (4 * B.UNITS + 8) + p.n_local * (4 * B.UNITS + 8) \
            + n * B.FEATURES * 4 + n * 3 * B.UNITS * 4
        line = {"metric": metric, "value": 2.0 * E / (ms_step * 1e-3), "unit": "edges/s", "n_gpus": world,
                "steps": args.steps, "warmup": max(args.warmup, 3), "ms_per_step": ms_step, "higher_is_better": True,
                "scaling": "strong", "vs_baseline": None, "dtype": "f32", "data": "synthetic", "config": config,
                "clocks": clocks, "e2e": e2e, "gpu_launches": launches,
                "roofline": {"bound": "hbm", "kernel": "gat_tma4_kernel<2> (tfgk_gat_fused_f32), rank 0 partition",
                             "achieved": gat_bytes / (gat_ms * 1e-3) / 1e9, "peak": peak, "unit": "GB/s",
                             "frac": gat_bytes / (gat_ms * 1e-3) / 1e9 / peak, "traffic": None, "peak_source": peak_src,
                             "algorithmic_bytes": gat_bytes, "kernel_ms": gat_ms},
                "cpu_baseline": None,
                "breakdown_ms": {"gat_fused": gat_ms, "gcn_spmm": spmm_ms, "projections_incl_exchange": proj_ms},
                "parity": {"sampled_rows_error_as_fraction_of_tolerance_vs_float64": float(check[0]),
                           "tolerance": "allclose(rtol=1e-4, atol=1e-4*max|ref|)",
                           "all_rows_bit_identical_to_collective_path": identical},
                "exchange": {"mode": mode,
                             "what": {"p2p": "x rows pulled block by block over NVLink peer mappings (tfgk_peer_pull on a side stream) "
                                             "while tfgk_gemm_proj_f32 projects the blocks that have landed; no collective",
                                      "p2p_fused": "x rows read over NVLink inside the projection GEMM (a_parts)",
                                      }.get(mode, "all_gather_into_tensor of the projected rows (NCCL)"),
                             "nvlink_bytes_in_per_rank_per_step": nvlink_per_step,
                             "hbm_algorithmic_bytes_per_rank_per_step": hbm_step}}
        B.emit(line)
    dist.destroy_process_group()
