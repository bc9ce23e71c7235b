# coding=utf-8
"""Neighbour samplers with the reference's interface (utils/graph_utils.py:630-846), on the device.

RandomNeighborSampler: the reference keeps a Python dict of neighbour arrays and loops over every node calling
np.random.choice (the bottleneck of demo/demo_graph_sage.py:53-55); here the dict is the stable row-sorted CSR and the
loop is one thread per row (tfgk_neighbor_sample_*).  UniformNeighborSampler: a Bernoulli flag per edge + compaction.
Randomness is counter-based (csrc/rng.cuh); pass `seed=` for reproducible draws.

RandomNeighborSampler.sample_neighborhood (an extension of the reference API) grows a seed-node mini-batch hop by hop
on the device: K13 samples the listed rows of the cached CSR and tfgk_frontier_i32 appends and relabels the new nodes, so
the work follows the batch, not the graph.

RandomNeighborSampler.sample_blocks (also an extension) samples the same neighbourhood as layer-wise bipartite blocks:
block i maps the hop_sizes[L - i] nodes of its input onto the hop_sizes[L - 1 - i] nodes the next layer reads, so every
layer computes only the rows it must.  The sizes stay on the device until the batch ends, which costs one host
synchronisation per batch.  sample_link_blocks seeds such a batch with the endpoints of target pairs and their
negatives (LinkBlocks), optionally with the targets excluded from the neighbourhoods their endpoints aggregate.

HostFeatureTable keeps an [N, F] float32, float16 or bfloat16 feature table in host memory (page-locked in place) and
gathers the rows a batch reads over the host link (tfgk_gather_rows_mapped_f32, or tfgk_gather_rows_mapped_16 for a
16-bit table, whose rows arrive widened to float32), so the table need not fit on the device.  With device_rows it also
keeps those rows in device memory, in the table's dtype, and reads them from there (tfgk_gather_rows_cached_f32 /
_16); rank_source_rows orders a graph's rows by how many sampled batches read them, to choose which rows to keep."""
import mmap
import threading

import numpy as np
import torch

from .. import ops, _rng
from ..sparse import SparseMatrix


def _split_node_index(sampled_node_index):
    if isinstance(sampled_node_index, tuple):
        return sampled_node_index
    return sampled_node_index, sampled_node_index


def _virtual_mapping(sampled_index, num_nodes, device, strict=True):
    """-1 everywhere, position-in-`sampled_index` at the sampled ids (graph_utils.py:792-800).  Ids outside
    [0, num_nodes) raise like numpy's fancy assignment does, unless strict=False (a symmetric node set applied to the
    narrower side of a rectangular edge list: such nodes simply have no edge there)."""
    idx = ops.as_device(sampled_index, torch.int32, device=device).reshape(-1)
    n_virtual = idx.numel()
    position = torch.arange(n_virtual, dtype=torch.int32, device=device)
    if n_virtual and (int(idx.max().item()) >= num_nodes or int(idx.min().item()) < 0):
        if strict:
            raise IndexError("sampled_node_index holds ids outside [0, {})".format(num_nodes))
        valid = (idx >= 0) & (idx < num_nodes)
        idx, position = idx[valid], position[valid]
    mapping = torch.full((num_nodes,), -1, dtype=torch.int32, device=device)
    mapping[idx.long()] = position
    return mapping, n_virtual


class _SamplerBase(object):

    def __init__(self, edge_index, edge_weight=None):
        self.edge_index = ops.as_device(edge_index, torch.int32)
        dev = self.edge_index.device
        E = self.edge_index.shape[1]
        self.num_edges = E
        self.edge_weight = torch.ones((E,), dtype=torch.float32, device=dev) if edge_weight is None \
            else ops.as_device(edge_weight, torch.float32, device=dev).reshape(-1)
        self._has_weights = edge_weight is not None
        self.row, self.col = self.edge_index[0].contiguous(), self.edge_index[1].contiguous()
        self.num_row_nodes = int(self.row.max().item()) + 1 if E else 0
        self.num_col_nodes = int(self.col.max().item()) + 1 if E else 0

    def _virtual_edges(self, sampled_node_index, bernoulli=ops.BERNOULLI_NONE, prob=0.0, seed=0):
        """Edges with both ends in the sampled sets, relabelled; optionally thinned by a Bernoulli rule in the same
        pass.  Returns (virtual_row, virtual_col, weight, num_virtual_rows, num_virtual_cols)."""
        rows, cols = _split_node_index(sampled_node_index)
        dev = self.edge_index.device
        row_map, n_vr = _virtual_mapping(rows, self.num_row_nodes, dev)
        if cols is rows and self.num_col_nodes == self.num_row_nodes:
            col_map, n_vc = row_map, n_vr
        else:
            col_map, n_vc = _virtual_mapping(cols, self.num_col_nodes, dev, strict=cols is not rows)
        flag = ops.edge_flags(self.row, self.col, self.num_edges, mode=ops.FLAG_MAPPED, row_map=row_map, col_map=col_map,
                              bernoulli=bernoulli, prob=prob, seed=seed)
        index = ops.select_flagged(flag)
        v_row = ops.gather_i32(row_map, ops.gather_i32(self.row, index))
        v_col = ops.gather_i32(col_map, ops.gather_i32(self.col, index))
        return v_row, v_col, ops.permute(self.edge_weight, index), n_vr, n_vc


class SampledNeighborhood(object):
    """A seed-node mini-batch (RandomNeighborSampler.sample_neighborhood).

    node_index: int32 [n] global ids; the seeds first, then every node reached, in first-occurrence order.
    edge_index_list / edge_weight_list: one edge list per layer, layer 0 nearest the input; rows and columns are positions
        in node_index.  Layer i's rows lie in node_index[:hop_sizes[-2 - i]] (the nodes whose neighbours it drew).
    hop_sizes: [number of seeds, list length after hop 1, ..., after the last hop] (the last one is n)."""

    __slots__ = ("node_index", "edge_index_list", "edge_weight_list", "hop_sizes")

    def __init__(self, node_index, edge_index_list, edge_weight_list, hop_sizes):
        self.node_index = node_index
        self.edge_index_list = edge_index_list
        self.edge_weight_list = edge_weight_list
        self.hop_sizes = hop_sizes


class Block(ops.SampledInput):
    """One layer of a SampledBlocks batch: a bipartite graph from num_src input rows to num_dst output rows, where the
    output rows are the first num_dst input rows (the same nodes).

    edge_index: int32 [2, S] local (row < num_dst, col < num_src), rows ascending and in draw order within a row.
    edge_weight: float32 [S].  global_col: int32 [S], the node id of every edge's column.
    csr: ops.CSR with n_rows = num_dst, n_cols = num_src; its perm is the identity (the edges are already in CSR order).
    fanout: the fan-out of the hop that drew the block (None: every neighbour, or a block built by hand); for a LABOR
    block, the k each row keeps in expectation.
    dst_ids: int32 [num_dst], the node id of every output row (a view of the batch's node_index; None for a block built
    by hand).  degrees: the sampler's full-graph degrees for with_gcn_norm(), a callable returning (rowptr int64, row
    sums float32), both indexed by node id (None for a block built by hand).  excluded: for a block of a link batch that
    excluded its target edges, (excl_off int64, n_excl): output row r < n_excl lost excl_off[r + 1] - excl_off[r] of its
    full-graph entries, which with_gcn_norm() leaves out of its scale (None otherwise, and for a block built by hand).
    weighted: whether the hop drew its fan-out in proportion to the edge weights (weighted=True of the samplers).
    labor: whether the hop drew by the layer-neighbour rule (labor=True of the samplers, integer fan-outs): its fanout is
    then k in expectation, and a row may hold up to all its neighbours.
    The transposed CSR that the backward needs is built on first use and kept on the block."""

    __slots__ = ("num_src", "num_dst", "edge_index", "edge_weight", "global_col", "csr", "fanout", "dst_ids", "degrees",
                 "excluded", "weighted", "labor", "_csr_t", "_w_t", "_looped", "_gcn")

    def __init__(self, num_src, num_dst, edge_index, edge_weight, global_col, csr, fanout=None, dst_ids=None,
                 degrees=None, excluded=None, weighted=False, labor=False):
        self.num_src, self.num_dst = int(num_src), int(num_dst)
        self.edge_index, self.edge_weight, self.global_col, self.csr = edge_index, edge_weight, global_col, csr
        self.fanout = None if fanout is None else int(fanout)
        self.dst_ids, self.degrees, self.excluded = dst_ids, degrees, excluded
        self.weighted = bool(weighted)
        self.labor = bool(labor)
        self._csr_t, self._w_t, self._looped, self._gcn = None, {}, None, None

    def with_self_loops(self):
        """The SelfLoopBlock of this block (GAT's input on a sampled block), made on first use and kept: one launch, and
        no synchronisation unless its rows are long enough for a work plan."""
        if self._looped is None:
            self._looped = SelfLoopBlock(self)
        return self._looped

    def with_gcn_norm(self):
        """The GcnBlock of this block (GCN's input on a sampled block), made on first use and kept; no device work until
        a configuration's values are first used.  A block built by hand carries no full-graph degrees: ValueError.
        A weighted block with an integer fan-out: NotImplementedError (the rescale n_g / k_r is the unbiased factor of
        uniform draws; a weighted sample would need every entry's inclusion probability)."""
        if self.weighted and self.fanout is not None:
            raise NotImplementedError("with_gcn_norm() rescales uniform draws; a block drawn with weighted=True would "
                                      "need inclusion probabilities")
        if self._gcn is None:
            if self.degrees is None or self.dst_ids is None:
                raise ValueError("with_gcn_norm() needs the full graph's degrees, which only a block from a sampler's "
                                 "sample_blocks carries")
            self._gcn = GcnBlock(self)
        return self._gcn

    def transposed(self, reduce=None, weighted=True):
        """(csr_t, w_t): the stable CSR of the edges keyed by local source (n_rows = num_src, n_cols = num_dst) and the
        edge weights (ones when not `weighted`) in its order, divided by their destination row's edge count for
        reduce="mean".  w_t is None for reduce=None and for an unweighted sum."""
        if self._csr_t is None:
            row, col = self.edge_index[0], self.edge_index[1]
            self._csr_t = ops.csr_build(col, row, self.num_src, self.num_dst, ids_in_range=True)
        if reduce is None or (reduce == "sum" and not weighted):
            return self._csr_t, None
        w_t = self._w_t.get((reduce, weighted))
        if w_t is None:
            w = self.edge_weight if weighted else torch.ones_like(self.edge_weight)
            if reduce == "mean":
                cnt = self.csr.degree_i64().clamp(min=1).to(torch.float32)
                w = ops.scale_edges(self.edge_index[0], None, w, dl=torch.reciprocal(cnt))
            w_t = self._w_t[(reduce, weighted)] = ops.permute(w, self._csr_t.perm)
        return self._csr_t, w_t


def _plan_for_fanout(k):
    """Whether a block CSR whose rows hold at most k edges (None: unbounded) can need a work plan: below
    DENSE_ROW_DEGREE every row is short and build_plan returns None."""
    return k is None or k >= ops.DENSE_ROW_DEGREE


class SelfLoopBlock(ops.SampledInput):
    """A Block with GAT's self loops (Block.with_self_loops()): the self loop of output row r is the edge (r, r), since
    output row r is input row r, appended after the row's sampled edges, where add_self_loop_edge puts self loops in the
    stable CSR of a full graph.  tfg.nn.gat and tfg.layers.GAT take it in place of an edge_index and add no self loops of
    their own; every other operator refuses it.

    edge_index: int32 [2, S + num_dst] local, in CSR order.  csr: ops.CSR with n_rows = num_dst, n_cols = num_src and an
    identity perm; it gets a work plan when its rows may be long (a fan-out of None or of DENSE_ROW_DEGREE - 1 or more,
    and every LABOR block).
    The transposed CSR that the backward needs is built on first use and kept."""

    __slots__ = ("num_src", "num_dst", "edge_index", "csr", "_csr_t")

    def __init__(self, block):
        self.num_src, self.num_dst = block.num_src, block.num_dst
        rowptr, self.edge_index = ops.block_self_loops(block.csr.rowptr, block.edge_index, block.num_dst)
        nnz = self.edge_index.shape[1]
        self.csr = ops.CSR(rowptr, self.edge_index[1], torch.arange(nnz, dtype=torch.int32, device=rowptr.device),
                           self.num_dst, self.num_src)
        if _plan_for_fanout(None if block.fanout is None or block.labor else block.fanout + 1):
            self.csr.plan = ops.build_plan(self.csr)
        self._csr_t = None

    def transposed(self):
        """The stable CSR of the looped edges keyed by local source (n_rows = num_src, n_cols = num_dst); its perm maps
        each of its slots to the looped CSR's position."""
        if self._csr_t is None:
            self._csr_t = ops.csr_build(self.edge_index[1], self.edge_index[0], self.num_src, self.num_dst,
                                        ids_in_range=True)
        return self._csr_t


def gcn_block_codes(norm, add_self_loop, sym, renorm, improved):
    """(norm code, loop code, deg_fill, fill) of tfgk_block_gcn_values_f32 for a gcn_norm_adj configuration; refuses the
    ones blocks do not support.  The degree takes the loops' fill when they are added before normalising (renorm, and
    always for left and right); with norm="both" and renorm=False the loops keep their fill unnormalised."""
    fill = 2.0 if improved else 1.0
    codes = {"both": ops.GCN_NORM_BOTH, "left": ops.GCN_NORM_LEFT, "right": ops.GCN_NORM_RIGHT}
    if norm not in codes:
        raise Exception("wrong GCN norm type: {}".format(norm))
    if norm == "both" and not sym:
        raise NotImplementedError("GCN on a sampled block needs sym=True with norm='both': column sums of the full graph "
                                  "are not kept by the sampler")
    if not add_self_loop:
        return codes[norm], ops.GCN_LOOP_NONE, 0.0, fill
    if norm == "both" and not renorm:
        return codes[norm], ops.GCN_LOOP_FILL, 0.0, fill
    return codes[norm], ops.GCN_LOOP_NORMED, fill, fill


class _BlockAdjacency(SparseMatrix):
    """A GcnBlock's normalised [num_dst, num_src] matrix: index, CSR and values in the block's CSR order (identity perm),
    and a transposed CSR that is the block's own, built on first use without an id check.  Matrices derived by dropout
    share it (SparseMatrix._pattern_of)."""

    def __init__(self, index, value, shape, csr, transposed):
        super().__init__(index, value, shape, _csr=csr, _value_csr=value)
        self._block_transposed = transposed

    def _transposed_csr(self):
        if self._csc is None:
            self._csc = self._block_transposed()
        return self._csc


class GcnBlock(ops.SampledInput):
    """A Block with GCN's normalisation (Block.with_gcn_norm()): every row, source-only rows included, is normalised with
    its degree in the sampler's full graph, and the sampled edges of output row r (global id g, k_r sampled of n_g) are
    scaled by s_r = n_g / k_r, so that each aggregate is an unbiased estimate of the full graph's row.  With every
    neighbour (fan-out None) s_r = 1 and the values are the full graph's gcn_norm_adj values for the same rows, bit for
    bit.  In a link batch that excluded x_r of row r's entries, s_r = (n_g - x_r) / k_r: the degrees stay the full
    graph's, and the aggregate estimates the full graph's row without the excluded terms (with fan-out None, exactly
    those values).  tfg.nn.gcn and tfg.layers.GCN take it in place of the adjacency; every other operator refuses it.

    normalized(norm, add_self_loop, sym, renorm, improved) gives the rectangular [num_dst, num_src] SparseMatrix of one
    configuration, made on first use (one launch of tfgk_block_gcn_values_f32) and kept.  With self loops its structure is
    block.with_self_loops()'s (CSR, plan and transposed CSR shared with GAT's view of the block), else the block's own."""

    __slots__ = ("num_src", "num_dst", "block", "_normed")

    def __init__(self, block):
        self.num_src, self.num_dst, self.block = block.num_src, block.num_dst, block
        self._normed = {}

    def normalized(self, norm="both", add_self_loop=True, sym=True, renorm=True, improved=False):
        from ..nn.conv.gcn import compute_cache_key         # nn imports this module
        key = compute_cache_key(norm, add_self_loop, sym, renorm, improved)
        normed = self._normed.get(key)
        if normed is None:
            normed = self._normed[key] = self._make(*gcn_block_codes(norm, add_self_loop, sym, renorm, improved))
        return normed

    def _make(self, norm, loop, deg_fill, fill):
        blk = self.block
        g_rowptr, g_rowsum = blk.degrees()
        if loop == ops.GCN_LOOP_NONE:
            index, csr = blk.edge_index, blk.csr

            def transposed():
                return blk.transposed()[0]
        else:
            looped = blk.with_self_loops()
            index, csr, transposed = looped.edge_index, looped.csr, looped.transposed
        args = (blk.csr.rowptr, blk.global_col, blk.edge_weight, blk.dst_ids, g_rowptr, g_rowsum, norm, loop, deg_fill,
                fill)
        value = ops.block_gcn_values(*args) if blk.excluded is None else \
            ops.block_gcn_values(*args, excluded=blk.excluded)
        return _BlockAdjacency(index, value, [self.num_dst, self.num_src], csr, transposed)


class SourceRows(ops.SampledInput):
    """Layer 0's input of a SampledBlocks batch taken from the global [N, F] feature table x without gathering it:
    mean and sum GraphSAGE aggregate straight from x through the block's global columns and gather only the self rows.
    shape is (num_src, F), the shape of the gathered table."""

    __slots__ = ("x", "node_index")

    def __init__(self, x, node_index):
        self.x, self.node_index = x, node_index

    @property
    def shape(self):
        return (self.node_index.numel(), self.x.shape[1])

    def gather(self, rows=None):
        """x[node_index[:rows]] (all source rows by default); differentiable when x requires grad."""
        from .. import autograd
        index = self.node_index if rows is None else self.node_index[:rows]
        if self.x.requires_grad and torch.is_grad_enabled():
            return autograd.TakeRows.apply(self.x, index)
        return ops.permute(self.x.detach(), index)


class SampledBlocks(object):
    """A seed-node mini-batch as layer-wise blocks (RandomNeighborSampler.sample_blocks).

    node_index, hop_sizes: those of sample_neighborhood with the same arguments.
    blocks: one Block per layer, layer 0 nearest the input; block i has num_src = hop_sizes[L - i] and num_dst =
        hop_sizes[L - 1 - i], and its edge_index / edge_weight are sample_neighborhood's edge_index_list[i] /
        edge_weight_list[i].
    num_nodes: the node count the sampler checked every id against (None for a batch built by hand)."""

    __slots__ = ("node_index", "hop_sizes", "blocks", "num_nodes")

    def __init__(self, node_index, hop_sizes, blocks, num_nodes=None):
        self.node_index, self.hop_sizes, self.blocks = node_index, hop_sizes, blocks
        self.num_nodes = None if num_nodes is None else int(num_nodes)

    def source_rows(self, x):
        """Layer 0's input for the global feature table x [N, F]: a float32 tensor (moved to the device when it is not
        there; any other dtype is converted to a float32 copy first), or a HostFeatureTable, whose rows node_index are
        gathered over the host link into a new float32 [num_src, F] device tensor on the current stream (a 16-bit
        table's rows widened exactly, so the rows are x.float()[node_index] bit for bit).  For a batch from
        sample_blocks the ids were checked by the sampler, so the table only needs num_nodes rows and the gather makes
        no host synchronisation; a batch built by hand takes the checked HostFeatureTable.gather."""
        if isinstance(x, HostFeatureTable):
            if self.num_nodes is None:
                return x.gather(self.node_index)
            if x.num_rows < self.num_nodes:
                raise ValueError("the feature table has {} rows; the sampler's graph has {} nodes".format(
                    x.num_rows, self.num_nodes))
            return x._gather(self.node_index)
        x = ops.as_device(x, torch.float32, device=self.node_index.device)
        return SourceRows(x, self.node_index)


# one registration per host buffer: base address -> [number of open tables over it, bytes, device address of the base]
_host_lock = threading.RLock()
_host_registered = {}


def _host_range(x, array):
    """(address, bytes) of the whole host buffer under x: its storage, or for a numpy view the array that owns the
    memory, so that tables over different views of one buffer share one registration."""
    st = x.untyped_storage()
    lo, size = st.data_ptr(), st.nbytes()
    if isinstance(array, np.ndarray):
        root = array
        while isinstance(root.base, np.ndarray):
            root = root.base
        if (root.flags.c_contiguous or root.flags.f_contiguous) and root.ctypes.data <= lo and \
                lo + size <= root.ctypes.data + root.nbytes:
            lo, size = root.ctypes.data, root.nbytes
    return lo, size


def _host_acquire(x, array=None):
    """Make the host buffer under the CPU tensor x readable by the device: (key, device address of x.data_ptr()).  The
    whole buffer (see _host_range) is page-locked in place once however many users share it, and counted; key is the
    registration to hand back to _host_release, or None when nothing was registered (pinned memory, which is mapped at its
    host address under unified addressing, or an empty x)."""
    base, nbytes = _host_range(x, array)
    if not x.numel():
        return None, x.data_ptr() - base
    with _host_lock:
        owner = next((b for b, (_, size, _) in _host_registered.items() if b <= base and base + nbytes <= b + size), None)
        if owner is not None:           # inside a buffer an open user registered: count one more user
            entry = _host_registered[owner]
            entry[0] += 1
            return owner, entry[2] + (base - owner) + (x.data_ptr() - base)
        if x.is_pinned():
            return None, x.data_ptr()
        dev_base = ops.host_register(base, nbytes)
        _host_registered[base] = [1, nbytes, dev_base]
        return base, dev_base + (x.data_ptr() - base)


def _host_release(key):
    """Drop one user of the registration `key` (from _host_acquire; None does nothing); the last one unregisters it,
    after the device's pending work."""
    if key is None:
        return
    with _host_lock:
        entry = _host_registered[key]
        entry[0] -= 1
        if entry[0] == 0:
            del _host_registered[key]
            ops.host_unregister(key)


class HostFeatureTable(object):
    """A feature table [N, F] kept in host memory, whose rows the device gathers over the host link.

    x: a CPU 2-D tensor or numpy array of `dtype` with unit column stride (numpy is wrapped without a copy).
    dtype: the storage type, torch.float32 (the default), torch.float16 or torch.bfloat16; anything else raises
    ValueError, and an x of another dtype raises TypeError: the table never converts or copies x, so a float32 table
    becomes a 16-bit one only by the caller's own copy (x.to(torch.bfloat16)).  numpy has no bfloat16, so a bfloat16
    table takes a torch tensor.  A 16-bit table moves half the bytes over the link and keeps twice the rows in the same
    device memory; its gathers still return float32, each element widened exactly.
    A pinned tensor is read as it is; otherwise the whole buffer under x (its storage, or the numpy array that owns the
    memory) is page-locked in place (no copy, so host memory is not doubled), once however many tables share it, and
    released when the last of them closes.  The table keeps a reference to x.  A host table is a constant: x must not require grad.

    device_rows: optional integer id vector (numpy, CPU or CUDA; int32 CUDA is used as it is) of rows to keep in device
    memory as well, on device_rows' device if it is a CUDA tensor, otherwise on the current device.  Those rows are
    copied once, by the same host gather, to a [C, F] device buffer in the table's dtype (a 16-bit table copies the
    rows' bit patterns), next to an int32 [N] map from row to buffer slot (-1: not cached).  A gather on that device reads cached rows from device memory and the rest over the host link, in
    one launch; a gather on another device reads every row over the link.  Either way the bits are x[index].  The ids
    are checked with one read-back: IndexError outside [0, N), ValueError for a repeated id or an array that is not a
    vector, TypeError for non-integer ids.  The constructor returns once the device rows are in place, so any stream
    may gather at once.  None or an empty vector keeps no rows on the device.  rank_source_rows chooses the rows.

    gather(index) and SampledBlocks.source_rows(table) return new float32 device tensors, bit-identical to
    x.float()[index] (x[index] for a float32 table).
    close() (or leaving a `with` block) drops the device rows and releases the registration after the current device's
    pending work; a table that is dropped without close() does both when it is collected."""

    def __init__(self, x, device_rows=None, dtype=torch.float32):
        self._closed = True                 # until registration succeeds: nothing for close() / __del__ to release
        self._key = None
        self._cache = self._slot = self._device_rows = None
        if dtype not in (torch.float32, torch.float16, torch.bfloat16):
            raise ValueError("HostFeatureTable stores torch.float32, torch.float16 or torch.bfloat16 (got dtype={})"
                             .format(dtype))
        array = x
        if isinstance(x, np.ndarray):
            x = torch.from_numpy(x)
        if not torch.is_tensor(x):
            raise TypeError("HostFeatureTable takes a CPU tensor or a numpy array (got {})".format(type(x).__name__))
        if x.is_cuda:
            raise TypeError("HostFeatureTable takes a table in host memory; a CUDA tensor goes to source_rows directly")
        if x.dim() != 2:
            raise TypeError("HostFeatureTable takes a 2-D [N, F] table (got {} dimensions)".format(x.dim()))
        if x.dtype != dtype:
            if dtype == torch.float32:
                raise TypeError("HostFeatureTable takes float32 features (got {})".format(x.dtype))
            raise TypeError("HostFeatureTable(dtype={}) takes {} features (got {}); the table does not convert "
                            "x".format(dtype, dtype, x.dtype))
        if x.requires_grad:
            raise ValueError("a host feature table is a constant: x must not require grad")
        n, F = x.shape
        if F > 1 and x.stride(1) != 1:
            raise ValueError("HostFeatureTable needs unit column stride (got strides {})".format(tuple(x.stride())))
        if n > 1 and x.stride(0) < F:
            raise ValueError("HostFeatureTable needs rows that do not overlap (got strides {})".format(tuple(x.stride())))
        rows = None if device_rows is None else _cached_ids(device_rows, n)
        self.x = x
        self._ld = max(F, x.stride(0))
        self._key, self._ptr = _host_acquire(x, array)
        self._closed = False
        if rows is not None:
            if dtype == torch.float32:
                self._cache = ops.gather_rows_mapped(self._ptr, self._ld, n, F, rows)
            else:                           # the rows' 16-bit patterns as they are
                self._cache = ops.gather_rows_mapped_16(self._ptr, dtype, self._ld, n, F, rows, out_dtype=dtype)
            slot = torch.full((n,), -1, dtype=torch.int32, device=rows.device)
            slot[rows.long()] = torch.arange(rows.numel(), dtype=torch.int32, device=rows.device)
            self._slot, self._device_rows = slot, rows
            # the cache and the map are private, so no caller can order a gather on another stream after their fill:
            # the table is ready for any stream when the constructor returns
            if rows.is_cuda:
                torch.cuda.current_stream(rows.device).synchronize()

    @property
    def num_rows(self):
        return self.x.shape[0]

    @property
    def num_features(self):
        return self.x.shape[1]

    @property
    def dtype(self):
        """The storage type of x: torch.float32, torch.float16 or torch.bfloat16 (gathers return float32)."""
        return self.x.dtype

    @property
    def device_rows(self):
        """The ids of the rows kept in device memory (int32 on the device, in cache order), or None."""
        return self._device_rows

    @property
    def device_bytes(self):
        """Device memory this table holds: the cached rows (C * F * itemsize) plus the row-to-slot map (4 * N), 0
        without device rows."""
        if self._cache is None:
            return 0
        return self._cache.numel() * self._cache.element_size() + self._slot.numel() * 4

    def _check_open(self):
        if self._closed:
            raise RuntimeError("this HostFeatureTable is closed")

    def _gather(self, index, out=None):
        """gather without the id check: index is an int32 device vector of ids in [0, num_rows)."""
        self._check_open()
        if index.numel() == 0 and out is None:
            return torch.empty((0, self.num_features), dtype=torch.float32, device=index.device)
        cached = self._cache is not None and index.device == self._cache.device
        if self.x.dtype != torch.float32:
            if cached:
                return ops.gather_rows_cached_16(self._ptr, self._ld, self.num_rows, self.num_features, self._cache,
                                                 self._slot, index.contiguous(), out)
            return ops.gather_rows_mapped_16(self._ptr, self.x.dtype, self._ld, self.num_rows, self.num_features,
                                             index.contiguous(), out)
        if cached:
            return ops.gather_rows_cached(self._ptr, self._ld, self.num_rows, self.num_features, self._cache, self._slot,
                                          index.contiguous(), out)
        return ops.gather_rows_mapped(self._ptr, self._ld, self.num_rows, self.num_features, index.contiguous(), out)

    def gather(self, index, out=None):
        """x[index] as a new contiguous float32 device tensor [len(index), F] (or into `out`, a float32 CUDA tensor of
        that shape), on the current stream; a 16-bit table's rows are widened exactly (x.float()[index]).  Ids: an
        integer vector (int32 on the device is used as it is); ids outside [0, num_rows) raise IndexError after one
        read-back of their range."""
        self._check_open()
        idx = ops.as_device(index).reshape(-1)
        if idx.dtype.is_floating_point or idx.dtype.is_complex or idx.dtype == torch.bool:
            raise TypeError("gather takes integer ids (got {})".format(idx.dtype))
        if idx.numel():
            lo, hi = torch.stack(torch.aminmax(idx)).tolist()
            if lo < 0 or hi >= self.num_rows:
                raise IndexError("index holds ids outside [0, {})".format(self.num_rows))
        return self._gather(idx.to(torch.int32), out)

    def close(self):
        """Drop the device rows and release the registration this table holds (the last table over a storage
        unregisters it).  Idempotent."""
        if self._closed:
            return
        self._closed = True
        self._cache = self._slot = self._device_rows = None
        key, self._key = self._key, None
        _host_release(key)

    def __enter__(self):
        return self

    def __exit__(self, *exc):
        self.close()

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass


def _cached_ids(device_rows, num_rows):
    """HostFeatureTable's device_rows as an int32 device vector of distinct ids in [0, num_rows), or None when empty;
    one read-back checks range and repeats."""
    ids = ops.as_device(device_rows)
    if ids.dim() != 1:
        raise ValueError("device_rows takes an id vector (got {} dimensions)".format(ids.dim()))
    if ids.numel() == 0:
        return None
    if ids.dtype.is_floating_point or ids.dtype.is_complex or ids.dtype == torch.bool:
        raise TypeError("device_rows takes integer ids (got {})".format(ids.dtype))
    lo, hi = torch.aminmax(ids)
    # ids clamped into range only so that the count is defined; an id outside the range is refused before it matters
    count = ops.segment_count(ids.clamp(0, max(num_rows - 1, 0)).to(torch.int32), max(num_rows, 1))
    lo, hi, most = torch.stack([lo.long(), hi.long(), count.max().long()]).tolist()
    if lo < 0 or hi >= num_rows:
        raise IndexError("device_rows holds ids outside [0, {})".format(num_rows))
    if most > 1:
        raise ValueError("device_rows holds a repeated id")
    return ids.to(torch.int32, copy=True)            # the table's own copy: the caller may reuse its buffer


def rank_source_rows(batches):
    """Rank a graph's rows by how often sampled batches read them, to choose HostFeatureTable's device_rows.

    batches: an iterable of SampledBlocks from sample_blocks (RandomNeighborSampler or HostNeighborSampler) over one
    graph; nothing is sampled here.  Returns (ids, counts), int32 on the batches' device: counts[j] is the number of
    batches whose node_index (layer 0's source rows) holds j, and ids lists every j with counts[j] > 0, most-read first,
    ties by smaller id.  One host read-back at the end.  ValueError for a batch built by hand (num_nodes None) or
    batches over different node counts.  An empty iterable gives two empty vectors."""
    counts = None
    num_nodes = None
    for b in batches:
        if b.num_nodes is None:
            raise ValueError("rank_source_rows takes batches from sample_blocks (this one was built by hand)")
        if counts is None:
            num_nodes = b.num_nodes
            counts = ops.segment_count(b.node_index, num_nodes)
            continue
        if b.num_nodes != num_nodes:
            raise ValueError("batches over {} and {} nodes: rank_source_rows takes batches of one graph".format(
                num_nodes, b.num_nodes))
        counts += ops.segment_count(b.node_index, num_nodes)
    if counts is None:
        empty = torch.empty((0,), dtype=torch.int32, device=ops.default_device())
        return empty, empty.clone()
    # radix keys ~count: read as unsigned, a larger count is a smaller key, and the stable sort keeps ties in id order
    order = ops.stable_argsort(torch.bitwise_not(counts), key_bits=32)
    read = int(torch.count_nonzero(counts).item())
    return order[:read], counts


_LINK_DOC = """Link-prediction mini-batch on blocks (an extension of the reference API, as DGL's edge data loaders and
        PyG's LinkNeighborLoader): the target pairs `edge_index` and their negatives are scored on the final embeddings
        of their endpoints, whose neighbourhoods are sampled as sample_blocks samples a seed list.

        Seeds: the distinct endpoints of the positive pairs, then of the negative pairs, pair by pair (source, then
        destination) in first-occurrence order; node_index[:hop_sizes[0]] is that list.  With exclude=None the batch is
        sample_blocks(that list, fanouts, padding, seed), bit for bit.
        Negatives: with num_negatives = q, negative pair b * q + j is (u_b, t), u_b the source of positive b and t drawn
        uniformly from all nodes (random_below64(seed, RNG_STREAM_LINK, b * q + j, N), tail corruption).  A negative may
        coincide with a true edge; for exact non-edges pass negative_edge_index (for example from
        negative_sampling_with_start_node) with num_negatives=0.  Both at once: ValueError.
        Exclusion: "self" removes every CSR entry (u, v) of every positive pair (u, v) from u's row (duplicates
        included), at every hop and before any draw; "reverse" also removes (v, u).  Negatives are never excluded, and a
        pair that is not an edge excludes nothing.  The batch equals sample_blocks on a sampler built over the edge list
        with those entries deleted (same order, weights following), for every fan-out rule; with_gcn_norm() keeps the
        full graph's degrees and rescales by the kept entries.
        Synchronisation: one host read-back per batch, one more for the exclusion lists' total, and one per hop of
        fan-out None or drawn by LABOR.  Calls on one sampler must be ordered on one CUDA stream.

        :param edge_index: int [2, B] target pairs (numpy, list or tensor)
        :param fanouts: as sample_blocks
        :param num_negatives: negatives drawn per positive pair
        :param negative_edge_index: int [2, M] negative pairs to use instead
        :param exclude: None, "self" or "reverse"
        :param weighted: draw every integer fan-out in proportion to edge_weight, as sample_blocks(weighted=True); the
            excluded entries are not candidates
        :param labor, layer_dependency: draw every integer fan-out by the layer-neighbour rule, as
            sample_blocks(labor=True); the excluded entries are not candidates (d counts the kept entries only)
        :return: LinkBlocks, on the device.  Ids outside [0, N) raise ValueError after the batch's read-back."""


def _with_link_doc(fn):
    fn.__doc__ = _LINK_DOC
    return fn


_ROW_BLOCK_DOC = """Every in-neighbour of the rows r0, ..., r1 - 1 as a one-block batch (layer-wise inference, as DGL's
        full-neighbour loaders and PyG's subgraph_loader): output rows are the nodes r0 .. r1 - 1 and hop_sizes is
        [r1 - r0, num_src].  The batch is sample_blocks(torch.arange(r0, r1), [None]), bit for bit (node list, edges,
        weights, CSR and work plan, degrees handle), so with_self_loops() and with_gcn_norm() apply unchanged.

        The range is one contiguous slice of the CSR, so its columns (and weights) are taken whole: in place on
        RandomNeighborSampler, by one asynchronous bulk copy per array from HostNeighborSampler's host CSR (an unweighted
        graph's ones are made on the device).  tfgk_row_block_i32 then relabels them.  Synchronisation: one read-back
        when the range has edges, plus the block's work plan.  Calls on one sampler must be ordered on one CUDA stream.

        :param r0, r1: the rows, 0 <= r0 <= r1 <= N; ValueError otherwise, or for a range of 2^31 - 1 edges or more
        :return: SampledBlocks with one Block, on the device"""


def _row_range(rp, r0, r1):
    """(r0, r1, e0, e1): the rows [r0, r1) of the host rowptr rp and their CSR positions [e0, e1); ValueError for rows
    outside [0, N), r0 > r1, or a range of 2^31 - 1 edges or more (tfgk_row_block_i32's int32 positions)."""
    N = rp.size - 1
    if not all(isinstance(r, (int, np.integer)) and not isinstance(r, bool) for r in (r0, r1)):
        raise TypeError("row_block takes integer rows (got {!r}, {!r})".format(r0, r1))
    r0, r1 = int(r0), int(r1)
    if r0 < 0 or r1 > N or r0 > r1:
        raise ValueError("row_block takes rows 0 <= r0 <= r1 <= {} (got r0={}, r1={})".format(N, r0, r1))
    e0, e1 = int(rp[r0]), int(rp[r1])
    if e1 - e0 >= (1 << 31) - 1:
        raise ValueError("rows [{}, {}) hold {} edges; a row block takes fewer than 2^31 - 1".format(r0, r1, e1 - e0))
    return r0, r1, e0, e1


def _row_block(sampler, r0, r1, staged=None):
    """row_block of either sampler; staged = (cols, w) when the caller staged the range's arrays itself."""
    r0, r1, e0, e1 = _row_range(sampler._host_rowptr(), r0, r1)
    cols, w = sampler._stage(e0, e1) if staged is None else staged
    rowptr, node_map, degrees = sampler._row_block_args()
    nodes, out_rowptr, row, local = ops.row_block(rowptr, r0, r1, cols, node_map)
    sizes = [r1 - r0, nodes.numel()]
    blocks = _blocks_of(rowptr.device, nodes, sizes, [(out_rowptr, row, local, cols, w)], [None], degrees)
    return SampledBlocks(nodes, sizes, blocks, num_nodes=node_map.numel())


class RandomNeighborSampler(_SamplerBase):
    """Per-node fan-out sampling (graph_utils.py:630-776)."""

    def __init__(self, edge_index, edge_weight=None):
        super().__init__(edge_index, edge_weight)
        self._csr = None
        self._w_csr = None
        self._rowptr_all = None
        self._node_map = None
        self._rowsum = None
        self._rowptr_host = None
        self._pos_deg = None

    def _structure(self):
        if self._csr is None:
            self._csr = ops.csr_build(self.row, self.col, self.num_row_nodes, max(self.num_col_nodes, 1))
            self._w_csr = ops.permute(self.edge_weight, self._csr.perm)
        return self._csr, self._w_csr

    def sample(self, k=None, ratio=None, sampled_node_index=None, padding=False, seed=None):
        """
        :param k: neighbours per node (all of them when the node has at most k and padding is False; k draws with
            replacement when padding is True and the node has at most k)
        :param ratio: instead of k, keep ceil(degree * ratio) neighbours per node, without replacement
        :param sampled_node_index: ids (or a (row_ids, col_ids) tuple): restrict to, and relabel into, this node set
        :return: (edge_index int32 [2, S], edge_weight float32 [S]) on the device, or (None, None) when S == 0
        """
        if k is not None and ratio is not None:
            raise Exception("k and ratio cannot be provided simultaneously")
        if sampled_node_index is None:
            csr, w_csr = self._structure()
        else:
            v_row, v_col, w, n_vr, n_vc = self._virtual_edges(sampled_node_index)
            if v_row.numel() == 0:
                return None, None
            csr = ops.csr_build(v_row, v_col, n_vr, max(n_vc, 1))
            w_csr = ops.permute(w, csr.perm)
        if csr.nnz == 0:
            return None, None
        out_row, out_pos, _ = ops.neighbor_sample(csr, k=k, ratio=ratio, padding=padding, seed=_rng.resolve_host(seed))
        if out_row.numel() == 0:
            return None, None
        return torch.stack([out_row, ops.gather_i32(csr.col, out_pos)]), ops.permute(w_csr, out_pos)

    def _neighborhood_structure(self):
        """The cached CSR with one row per node id (ids past the last source row have no neighbours), and the [N] id ->
        position map of the relabelling kernels, which is -1 everywhere between calls."""
        csr, w_csr = self._structure()
        if self._node_map is None:
            n = max(self.num_row_nodes, self.num_col_nodes)
            rowptr = csr.rowptr
            if n > csr.n_rows:
                rowptr = torch.cat([rowptr, rowptr[-1:].expand(n - csr.n_rows)])
            self._rowptr_all = rowptr
            self._node_map = torch.full((n,), -1, dtype=torch.int32, device=rowptr.device)
        return csr, w_csr, self._rowptr_all, self._node_map

    def _gcn_degrees(self):
        """(rowptr int64 [N + 1], row sums float32 [N]) of the cached CSR, one row per node id: the sequential fp32 sums
        of each row's weights (csr_rowsum, gcn_norm_adj's degrees before any self loop), made on first use and kept."""
        csr, w_csr, rowptr, node_map = self._neighborhood_structure()
        if self._rowsum is None:
            n = node_map.numel()
            rowsum = ops.csr_rowsum(csr, w_csr) if csr.n_rows else torch.zeros((0,), dtype=torch.float32,
                                                                              device=rowptr.device)
            if n > csr.n_rows:
                rowsum = torch.cat([rowsum, rowsum.new_zeros(n - csr.n_rows)])
            self._rowsum = rowsum
        return rowptr, self._rowsum

    def _positive_degrees(self):
        """int32 [N]: every row's entries of weight > 0 (the weighted rule's d+), made on the first weighted call and
        kept.  That call reads the count of invalid weights back once: ValueError for a negative, NaN or infinite weight,
        and for a sampler built without edge_weight."""
        if self._pos_deg is None:
            if not self._has_weights:
                raise ValueError("weighted=True draws in proportion to edge_weight; this sampler was built without one")
            csr, w_csr, rowptr, node_map = self._neighborhood_structure()
            pos_deg = torch.empty((node_map.numel(),), dtype=torch.int32, device=rowptr.device)
            n_invalid = torch.zeros((1,), dtype=torch.int32, device=rowptr.device)
            ops.csr_positive_degree(rowptr, w_csr, pos_deg, n_invalid)
            _check_weights(int(n_invalid.item()))
            self._pos_deg = pos_deg
        return self._pos_deg

    def sample_neighborhood(self, seed_node_index, fanouts, padding=False, seed=None, weighted=False):
        """Seed-node mini-batch sampling (an extension of the reference API).

        Hop h draws fanouts[-1 - h] neighbours (by sample()'s k rule and `padding`) for EVERY node already in the list, so
        one index space serves all layers; a node's draw depends only on the node and the hop's key, which is derived
        from `seed` and h.  The new nodes are appended in the order the sampled edges first reach them.
        Calls on one sampler must be ordered on one CUDA stream (they share the relabelling map).

        :param seed_node_index: distinct node ids (numpy, list or tensor); duplicates raise ValueError
        :param fanouts: neighbours per node for each layer, layer 0 nearest the input: sampling starts with fanouts[-1]
        :param weighted: draw every integer fan-out in proportion to edge_weight (sample_blocks' weighted rule)
        :return: SampledNeighborhood, on the device
        """
        from .graph_utils import _batch_seed         # graph_utils imports this module
        seed = _rng.resolve_host(seed)
        _check_weighted_padding(weighted, padding)
        csr, w_csr, rowptr, node_map = self._neighborhood_structure()
        wargs = {}
        if weighted:
            wargs = dict(weighted=(self._positive_degrees(), w_csr), rng_stream=ops.RNG_STREAM_WEIGHTED)
        dev = rowptr.device
        N = node_map.numel()
        nodes = ops.as_device(seed_node_index, torch.int32, device=dev).reshape(-1).contiguous()
        if nodes.numel():
            lo, hi = torch.aminmax(nodes)
            if int(lo) < 0 or int(hi) >= N:
                raise ValueError("seed_node_index holds node ids outside [0, {})".format(N))
        _, n_dup = ops.reindex(nodes, nodes[:0], node_map)
        if n_dup:
            raise ValueError("seed_node_index holds {} duplicate node ids".format(n_dup))
        n = nodes.numel()
        hop_sizes, hop_edges, hop_weights = [n], [], []
        for h, k in enumerate(reversed(list(fanouts))):
            out_row, out_pos, _ = ops.neighbor_sample_rows(rowptr, nodes[:n], k=None if k is None else int(k),
                                                           padding=padding, seed=_batch_seed(seed, h), **wargs)
            S = out_pos.numel()
            grown = torch.empty((n + S,), dtype=torch.int32, device=dev)
            grown[:n].copy_(nodes[:n])
            if S:
                local, n_new, _ = ops.frontier(grown, n, ops.gather_i32(csr.col, out_pos), node_map)
                weight = ops.permute(w_csr, out_pos)
            else:
                local, n_new = out_pos, 0
                weight = torch.empty((0,), dtype=torch.float32, device=dev)
            hop_edges.append(torch.stack([out_row, local]))
            hop_weights.append(weight)
            nodes, n = grown, n + n_new
            hop_sizes.append(n)
        return SampledNeighborhood(nodes[:n], hop_edges[::-1], hop_weights[::-1], hop_sizes)

    def sample_blocks(self, seed_node_index, fanouts, padding=False, seed=None, weighted=False, labor=False,
                      layer_dependency=False):
        """sample_neighborhood's batch as layer-wise bipartite blocks (an extension of the reference API); same arguments
        and the same node list and edges for the same key.  Integer fan-outs and device-resident seeds synchronise the
        host once per batch; a fan-out of None (every neighbour) adds one read-back for its hop.

        weighted=True (DGL's prob=, PyG's weight_attr=): every integer fan-out draws in proportion to the sampler's
        edge_weight, by the rule of include/tfgk.h ("weighted block sampler"): min(k, d+) entries without replacement by
        successive sampling, or with padding and k >= d+ k draws with replacement, P = w / W; entries of weight 0 are
        never drawn, and fan-out None takes every entry as without weights.  A sampler built without edge_weight, and
        padding="head", raise ValueError; the first weighted call makes the positive degrees and reads back once more.

        labor=True (layer-neighbour sampling, LABOR-0: Balin & Catalyurek, NeurIPS 2023; DGL's LaborSampler): every
        integer fan-out k draws by the rule of include/tfgk.h ("LABOR block sampler").  Each source node c gets one
        variate u_c per hop, and a row of d > k neighbours keeps its neighbour c iff u_c * d < k 2^32, so each row keeps
        every neighbour with probability pi = ceil(k 2^32 / d) / 2^32 (k in expectation, up to d), the kept set is uniform
        given its size, and rows that share a neighbour keep it together: a batch reaches fewer distinct source rows than
        with independent draws.  A row of d <= k keeps every neighbour; a row of d > k keeps none with probability
        (1 - pi)^d (over its distinct neighbours).  The mean and with_gcn_norm()'s n_g / k_r rescale stay unbiased given
        k_r >= 1.  layer_dependency=True uses hop 0's variates at every hop, so a node drawn at one hop is preferred at the
        next.  Fan-out None takes every neighbour as without LABOR.  padding (True or "head") and layer_dependency
        without labor raise ValueError, weighted=True raises NotImplementedError, all before any device work.  No
        capacity bounds a LABOR hop, so each one reads its edge total back and its block is planned as a fan-out None
        block (a work-plan build, one more read-back): a batch of L integer LABOR hops synchronises 1 + 2 L times.

        :return: SampledBlocks, on the device"""
        _check_rule(weighted, labor, layer_dependency, padding)
        csr, w_csr, rowptr, node_map = self._neighborhood_structure()
        pos_deg = self._positive_degrees() if weighted else None
        return _sample_blocks(lambda nodes, hop_fanouts, keys: ops.block_sample(
            rowptr, csr.col, w_csr, nodes, hop_fanouts, keys, node_map, padding=padding, **_rule_args(pos_deg, labor)),
            rowptr.device, node_map.numel(), seed_node_index, fanouts, seed, self._gcn_degrees, weighted, labor,
            layer_dependency)

    def row_block(self, r0, r1):
        return _row_block(self, r0, r1)

    row_block.__doc__ = _ROW_BLOCK_DOC

    def _host_rowptr(self):
        """The CSR's rowptr (one row per node id) as int64 numpy, read back once on first use."""
        if self._rowptr_host is None:
            self._rowptr_host = self._neighborhood_structure()[2].cpu().numpy()
        return self._rowptr_host

    def _stage(self, e0, e1):
        """The columns and weights of CSR positions [e0, e1): slices of the device CSR, read in place."""
        csr, w_csr, _, _ = self._neighborhood_structure()
        return csr.col[e0:e1], w_csr[e0:e1]

    def _row_block_args(self):
        _, _, rowptr, node_map = self._neighborhood_structure()
        return rowptr, node_map, self._gcn_degrees

    @_with_link_doc
    def sample_link_blocks(self, edge_index, fanouts, num_negatives=1, negative_edge_index=None, exclude=None,
                           padding=False, seed=None, weighted=False, labor=False, layer_dependency=False):
        _check_rule(weighted, labor, layer_dependency, padding)
        csr, w_csr, rowptr, node_map = self._neighborhood_structure()
        pos_deg = self._positive_degrees() if weighted else None
        return _sample_link_blocks(lambda pairs, n_pos, hop_fanouts, keys, exclude: ops.link_block_sample(
            rowptr, csr.col, w_csr, pairs, n_pos, hop_fanouts, keys, node_map, exclude=exclude, padding=padding,
            **_rule_args(pos_deg, labor)), rowptr.device, node_map.numel(), edge_index, fanouts, num_negatives,
            negative_edge_index, exclude, padding, seed, self._gcn_degrees, weighted, labor, layer_dependency)


def _check_weighted_padding(weighted, padding):
    if weighted and ops._padding_code(padding) == ops.SAMPLE_HEAD:
        raise ValueError("padding='head' takes the first entries of each row and draws nothing: it cannot be weighted")


def _check_weights(n_invalid):
    if n_invalid:
        raise ValueError("edge_weight holds {} negative, NaN or infinite weights; weighted=True draws in proportion to "
                         "weights >= 0".format(n_invalid))


def _check_rule(weighted, labor, layer_dependency, padding):
    """The samplers' refusals of a draw rule, before any device work."""
    _check_weighted_padding(weighted, padding)
    if layer_dependency and not labor:
        raise ValueError("layer_dependency=True reuses LABOR's variates across hops: it needs labor=True")
    if labor and ops._padding_code(padding):
        raise ValueError("labor=True draws without replacement: it takes no padding (True or 'head')")
    if labor and weighted:
        raise NotImplementedError("weighted LABOR is not implemented: it needs a per-row solve for the inclusion "
                                  "probabilities")


def _rule_args(pos_deg, labor=False):
    """The block samplers' keywords for a weighted batch (pos_deg not None), a LABOR batch or a uniform one."""
    if labor:
        return dict(labor=True, rng_stream=ops.RNG_STREAM_LABOR)
    return {} if pos_deg is None else dict(pos_deg=pos_deg, rng_stream=ops.RNG_STREAM_WEIGHTED)


def _hop_keys(fanouts, seed, layer_dependency=False):
    """(per-hop fan-outs in hop order, hop keys) of a batch with the resolved key `seed`; with layer_dependency every
    hop takes hop 0's key."""
    from .graph_utils import _batch_seed         # graph_utils imports this module
    hop_fanouts = [None if k is None else int(k) for k in reversed(list(fanouts))]
    return hop_fanouts, [_batch_seed(seed, 0 if layer_dependency else h) for h in range(len(hop_fanouts))]


def _blocks_of(dev, node_index, sizes, hops, hop_fanouts, degrees, excluded=None, weighted=False, labor=False):
    """The Blocks of a batch, layer 0 first, from the block sampler's hops.  A LABOR block's rows are not bounded by its
    fan-out, so it is planned as a block of fan-out None."""
    blocks = []
    for h, (k, (out_rowptr, row, local, gcol, w)) in enumerate(zip(hop_fanouts, hops)):
        n_dst, n_src = sizes[h], sizes[h + 1]
        S = row.numel()
        by_labor = labor and k is not None
        block_csr = ops.CSR(out_rowptr[:n_dst + 1], local, torch.arange(S, dtype=torch.int32, device=dev), n_dst, n_src)
        if _plan_for_fanout(None if by_labor else k):
            block_csr.plan = ops.build_plan(block_csr)
        blocks.append(Block(n_src, n_dst, torch.stack([row, local]), w, gcol, block_csr, fanout=k,
                            dst_ids=node_index[:n_dst], degrees=degrees, excluded=excluded, weighted=weighted,
                            labor=by_labor))
    return blocks[::-1]


def _sample_blocks(block_sample, dev, num_nodes, seed_node_index, fanouts, seed, degrees, weighted=False, labor=False,
                   layer_dependency=False):
    """sample_blocks of both samplers around their block sampler: block_sample(seeds int32, per-hop fan-outs in hop order,
    hop keys) returns ops.block_sample's (nodes, hop_sizes, hops, n_bad, n_dup); this refuses bad seeds and assembles
    the SampledBlocks.  degrees: the sampler's (rowptr, row sums) handle that every Block keeps for with_gcn_norm()."""
    seed = _rng.resolve_host(seed)
    nodes = ops.as_device(seed_node_index, torch.int32, device=dev).reshape(-1).contiguous()
    hop_fanouts, keys = _hop_keys(fanouts, seed, layer_dependency)
    node_index, sizes, hops, n_bad, n_dup = block_sample(nodes, hop_fanouts, keys)
    if n_bad:
        raise ValueError("seed_node_index holds node ids outside [0, {})".format(num_nodes))
    if n_dup:
        raise ValueError("seed_node_index holds {} duplicate node ids".format(n_dup))
    return SampledBlocks(node_index, sizes, _blocks_of(dev, node_index, sizes, hops, hop_fanouts, degrees,
                                                       weighted=weighted, labor=labor), num_nodes=num_nodes)


class LinkBlocks(SampledBlocks):
    """A link-prediction mini-batch as layer-wise blocks (sample_link_blocks of RandomNeighborSampler and
    HostNeighborSampler): a SampledBlocks seeded by the distinct endpoints of its pairs, so source_rows and
    rank_source_rows take it as they take any batch.

    pos_index: int32 [2, B], the target pairs relabelled to positions in node_index (all < hop_sizes[0]).
    neg_index: int32 [2, M], the negative pairs, relabelled the same way.
    predict_edge(h) scores both on the seeds' final embeddings."""

    __slots__ = ("pos_index", "neg_index", "_pairs", "_half_csr")

    def __init__(self, node_index, hop_sizes, blocks, num_nodes, pairs, num_pos):
        super().__init__(node_index, hop_sizes, blocks, num_nodes=num_nodes)
        self._pairs = pairs
        self.pos_index, self.neg_index = pairs[:, :num_pos], pairs[:, num_pos:]
        self._half_csr = None

    def predict_edge(self, h):
        """(pos_logits [B], neg_logits [M]): <h[u], h[v]> for every positive and negative pair (u, v), from one EdgeDot
        over [pos || neg]; h: [hop_sizes[0], D], the last layer's output.  Differentiable in h, with the deterministic
        backward of tfg.nn.predict_edge; its half-edge CSR is built without an id check (the local ids are in range by
        construction) and kept on the batch.  No host synchronisation."""
        from .. import autograd
        n = self.hop_sizes[0]
        if h.dim() != 2 or h.shape[0] != n:
            raise ValueError("predict_edge takes the seeds' embeddings, [{}, D] (got {})".format(n, tuple(h.shape)))
        if self._half_csr is None and h.requires_grad and torch.is_grad_enabled():
            self._half_csr = autograd._half_edge_csr(self._pairs, n, ids_in_range=True)
        logits = autograd.EdgeDot.apply(h, self._pairs)
        B = self.pos_index.shape[1]
        return logits[:B], logits[B:]


def _pair_tensor(pairs, dev, what):
    """`pairs` as an int32 [2, P] device tensor: ValueError for another shape, TypeError for non-integer ids."""
    t = ops.as_device(pairs, device=dev)
    if t.dim() != 2 or t.shape[0] != 2:
        raise ValueError("{} must have shape [2, B] (got {})".format(what, tuple(t.shape)))
    if t.dtype.is_floating_point or t.dtype.is_complex or t.dtype == torch.bool:
        raise TypeError("{} takes integer node ids (got {})".format(what, t.dtype))
    return t


def _sample_link_blocks(link_block_sample, dev, num_nodes, edge_index, fanouts, num_negatives, negative_edge_index,
                        exclude, padding, seed, degrees, weighted=False, labor=False, layer_dependency=False):
    """sample_link_blocks of both samplers around their link block sampler: link_block_sample(pairs int32 [2, P], n_pos,
    per-hop fan-outs, hop keys, exclude) returns ops.link_block_sample's outputs.  This checks the arguments, writes the
    pairs (positives, then negatives), refuses endpoints outside the graph and assembles the LinkBlocks."""
    pos = _pair_tensor(edge_index, dev, "edge_index")
    if isinstance(num_negatives, bool) or not isinstance(num_negatives, (int, np.integer)) or num_negatives < 0:
        raise ValueError("num_negatives must be an integer >= 0 (got {!r})".format(num_negatives))
    q = int(num_negatives)
    if negative_edge_index is not None and q > 0:
        raise ValueError("pass either num_negatives > 0 (negatives drawn here) or negative_edge_index, not both; "
                         "with negative_edge_index set num_negatives=0")
    if exclude not in (None, "self", "reverse"):
        raise ValueError("exclude must be None, 'self' or 'reverse' (got {!r})".format(exclude))
    neg = None if negative_edge_index is None else _pair_tensor(negative_edge_index, dev, "negative_edge_index")
    ops._check_block_fanouts(list(fanouts), padding)
    B = pos.shape[1]
    M = B * q if neg is None else neg.shape[1]
    if num_nodes == 0 and B + M:
        raise ValueError("the pairs hold node ids outside [0, 0): the graph has no nodes")
    seed = _rng.resolve_host(seed)
    hop_fanouts, keys = _hop_keys(fanouts, seed, layer_dependency)
    pairs = torch.empty((2, B + M), dtype=torch.int32, device=dev)
    pairs[:, :B].copy_(pos)
    if neg is not None:
        pairs[:, B:].copy_(neg)
    elif M:
        ops.link_tail_negatives(pairs[0, :B], q, num_nodes, seed, pairs[0, B:], pairs[1, B:])
    node_index, sizes, hops, n_bad, local, excluded = link_block_sample(pairs, B, hop_fanouts, keys, exclude)
    if n_bad:
        raise ValueError("the pairs hold {} node ids outside [0, {})".format(n_bad, num_nodes))
    blocks = _blocks_of(dev, node_index, sizes, hops, hop_fanouts, degrees, excluded, weighted, labor)
    return LinkBlocks(node_index, sizes, blocks, num_nodes, local, B)


class UniformNeighborSampler(_SamplerBase):
    """Independent Bernoulli(prob) edge sampling (graph_utils.py:775-846)."""

    def sample(self, prob, sampled_node_index=None, seed=None):
        seed = _rng.resolve_host(seed)
        if sampled_node_index is None:
            flag = ops.edge_flags(None, None, self.num_edges, bernoulli=ops.BERNOULLI_KEEP, prob=float(prob), seed=seed,
                                  device=self.edge_index.device)
            index = ops.select_flagged(flag)
            return (torch.stack([ops.gather_i32(self.row, index), ops.gather_i32(self.col, index)]),
                    ops.permute(self.edge_weight, index))
        v_row, v_col, w, _, _ = self._virtual_edges(sampled_node_index, bernoulli=ops.BERNOULLI_KEEP, prob=float(prob),
                                                    seed=seed)
        return torch.stack([v_row, v_col]), w


# Device bytes the host CSR build holds per edge and per row of a range (ops.mapped_csr_range at its peak, in the radix
# sort): the selected rows, columns and weights (12), csr_build's two key buffers, value buffer and histogram (12.25)
# and its sorted columns and permutation (8), without the 4 bytes of selected weights for an unweighted graph; per row,
# the range's counts and rowptr (12).  Besides the ranges the build holds the graph's rowptr and the selection's tile
# offsets (HOST_CSR_FIXED_BYTES plus 8 bytes per row of the graph and per 1024 edges).
HOST_CSR_EDGE_BYTES = 33
HOST_CSR_EDGE_BYTES_UNWEIGHTED = 29
HOST_CSR_ROW_BYTES = 12
HOST_CSR_FIXED_BYTES = 1 << 20

# Device bytes one chunk of layerwise_inference holds per edge and per output row of its range, as the code allocates
# them.  Row block, per edge: the staged columns and weights of this range and of the next one, staged while this one is
# computed (16); the relabelling's flags and offsets (8); the block's output rows and local columns (8), its edge_index
# (8) and CSR perm (4); the node list (4); the work plan's hub slices (1).  Per row: the rebased rowptr (8), the node list
# (4), the relabelling's map of row ids is the sampler's (0), the work plan's workspace (24) and task arrays, allocated at
# capacity and then cloned (2 x 28).  With self loops (GAT, and GCN's block values) the looped edge_index and perm (12
# per edge; per row one more edge, its rowptr and its own work plan: 12 + 8 + 80).  GCN's values: 4 per edge and per row.
ROW_BLOCK_EDGE_BYTES = 49
ROW_BLOCK_ROW_BYTES = 92
LOOPED_EDGE_BYTES = 12
LOOPED_ROW_BYTES = 100
GCN_VALUE_BYTES = 4
LAYERWISE_FIXED_BYTES = 16 << 20        # scan scratch, counters, per-call buffers and the allocator's rounding


def layerwise_chunk_bytes(layer, in_width):
    """(edge_bytes, row_bytes, out_width): the device bytes layerwise_inference counts per edge and per output row of a
    chunk of `layer` over an input of in_width features, and the layer's output width.  Every edge counts as a possible
    new source row, whose input row (in_width floats, gathered) and projections are held; every output row holds its own
    source row, its aggregates and projections, and two output rows (the chunk's, and the previous chunk's until its copy
    to host memory ends).  TypeError for a layer layerwise_inference does not take."""
    from .. import layers as L           # layers import this module
    F = int(in_width)
    eb, rb = ROW_BLOCK_EDGE_BYTES, ROW_BLOCK_ROW_BYTES
    if isinstance(layer, L.GCN):
        D = layer.units if layer.use_kernel else F
        src = F + D                                      # gathered row, its projection
        eb, rb = eb + LOOPED_EDGE_BYTES + GCN_VALUE_BYTES, rb + LOOPED_ROW_BYTES + GCN_VALUE_BYTES
        dst = src + D                                    # and its aggregate
    elif isinstance(layer, L.GAT):
        D = layer.units
        V = layer.units * (1 if layer.split_value_heads else layer.num_heads)
        src = F + 2 * layer.attention_units + V          # gathered row, query, key and value
        eb, rb = eb + LOOPED_EDGE_BYTES, rb + LOOPED_ROW_BYTES
        dst = src + V
    elif isinstance(layer, (L.MeanGraphSage, L.SumGraphSage)):
        D = layer.units
        src = F                                          # gathered row (a device x is read in place)
        dst = src + 2 * F + 2 * D                        # aggregate, self row, the two projections
    elif isinstance(layer, (L.MeanPoolGraphSage, L.MaxPoolGraphSage)):
        D = layer.units
        k = layer.units // 2 if layer.concat else layer.units
        src = F + 4 * k                                  # gathered row, its neighbour-MLP row
        dst = src + 4 * k + 2 * D                        # reduced row, the two projections
    else:
        raise TypeError("layerwise_inference takes tfg.layers.GCN, GAT, MeanGraphSage, SumGraphSage, MeanPoolGraphSage "
                        "and MaxPoolGraphSage layers (got {})".format(type(layer).__name__))
    return eb + 4 * src, rb + 4 * (dst + 2 * D), D


def _row_ranges(rowptr, budget, edge_bytes, row_bytes=HOST_CSR_ROW_BYTES):
    """Cut the rows of rowptr (int64 numpy [n + 1]) into consecutive ranges [r0, r1) of fewer than 2^31 edges whose
    working set edge_bytes * edges + row_bytes * (rows + 1) fits `budget` bytes, each as long as it can be.  Raises
    ValueError naming the row when one row alone does not fit, or holds 2^31 edges or more (the draws use a 32-bit
    degree)."""
    rowptr = np.asarray(rowptr, np.int64)
    n = rowptr.size - 1
    deg = np.diff(rowptr)
    if n and int(deg.max()) >= (1 << 31) - 1:
        r = int(deg.argmax())
        raise ValueError("row {} has {} edges; HostNeighborSampler takes rows of fewer than 2^31 - 1 edges".format(
            r, int(deg[r])))
    cost = edge_bytes * rowptr + row_bytes * np.arange(n + 1, dtype=np.int64)       # cost of [r0, r1) = cost[r1] - cost[r0] + row_bytes
    ranges, r0 = [], 0
    while r0 < n:
        r1 = int(np.searchsorted(cost, cost[r0] + budget - row_bytes, side="right")) - 1
        r1 = min(r1, int(np.searchsorted(rowptr, rowptr[r0] + (1 << 31) - 1, side="right")) - 1)
        if r1 <= r0:
            raise ValueError("row {} has {} edges, which need {} bytes of device memory to build; device_bytes leaves "
                             "{} for a range of rows".format(r0, int(deg[r0]), edge_bytes * int(deg[r0]) + 2 * row_bytes,
                                                             max(int(budget), 0)))
        ranges.append((r0, r1))
        r0 = r1
    return ranges


# cudaHostRegister page-locks whole pages, and a page can be in one registration only, so the sampler reads in place only
# arrays of at least this size: smaller allocations may share a page with other data (malloc serves them from its heap;
# glibc's threshold for giving an allocation pages of its own is at most 32 MiB).
HOST_IN_PLACE_BYTES = 32 << 20


def _page_array(n, dtype):
    """An empty numpy vector of n `dtype` entries on pages of its own (page-aligned, nothing else on its last page)."""
    page = mmap.PAGESIZE
    pages = -(-max(n * np.dtype(dtype).itemsize, 1) // page)
    raw = np.empty((pages + 1) * page, np.uint8)
    off = -raw.ctypes.data % page
    return raw[off:off + pages * page].view(dtype)[:n]


def _host_array(a, what, dtype, ndim):
    """`a` as a C-contiguous numpy array of `dtype` that can be page-locked on its own: `a` itself when it is one of at
    least HOST_IN_PLACE_BYTES, else a copy on pages of its own."""
    if torch.is_tensor(a):
        if a.is_cuda:
            raise TypeError("HostNeighborSampler takes {} in host memory; for a CUDA tensor use RandomNeighborSampler"
                            .format(what))
        if a.requires_grad:
            raise ValueError("{} must not require grad: the sampler's graph is a constant".format(what))
        a = a.detach().numpy()
    elif not isinstance(a, np.ndarray):
        raise TypeError("HostNeighborSampler takes {} as a CPU tensor or a numpy array (got {})".format(
            what, type(a).__name__))
    kind = np.dtype(dtype).kind
    if (a.dtype.kind not in "iu" if kind == "i" else a.dtype.kind not in "iuf"):
        raise TypeError("HostNeighborSampler takes {} of an {} dtype (got {})".format(
            what, "integer" if kind == "i" else "integer or floating", a.dtype))
    if a.ndim != ndim:
        raise ValueError("{} must have {} dimension(s) (got shape {})".format(what, ndim, a.shape))
    if a.dtype != dtype:
        if kind == "i" and a.size:
            lo, hi = int(a.min()), int(a.max())
            if lo < 0:
                raise ValueError("{} holds negative node ids".format(what))
            if hi >= (1 << 31):
                raise ValueError("{} holds node ids of 2^31 or more".format(what))
    elif a.flags.c_contiguous and a.nbytes >= HOST_IN_PLACE_BYTES:
        return a
    out = _page_array(a.size, dtype).reshape(a.shape)
    out[...] = a
    return out


class HostNeighborSampler(object):
    """RandomNeighborSampler.sample_blocks over a graph whose CSR stays in host memory (an extension of the reference
    API, for graphs whose edges do not fit on the device, such as ogbn-papers100M on one GPU).

    edge_index: int [2, E] as a CPU tensor or a numpy array; E may be 2^31 or more.  A C-contiguous int32 array (of 32 MiB
        or more) is read in place; any other integer array is converted once on the host, which makes an int32 copy of
        it.  Ids must be >= 0.  edge_weight: optional float32 [E], read in place or converted the same way (a copy).
    device_bytes: the most device memory the build may hold at once (default: half of the device's free memory when the
        build starts).  A row whose edges do not fit in it is refused with ValueError, as is a row of 2^31 - 1 edges or
        more.

    The constructor builds the stable row-sorted CSR of RandomNeighborSampler, bit for bit: the edge list is page-locked
    in place, its id range and row counts are found in streaming passes over the host link, and rows are processed in
    ranges that fit device_bytes (each range's edges selected in edge order, sorted stably by row, permuted and copied
    to host arrays, page-locked in place; an unweighted graph keeps no weights).  The edge list is released before the
    constructor returns; the sampler keeps no reference to it.  The device holds the int64 rowptr (one row per node id),
    the float32 row sums `rowsum` of the weights (GcnBlock's full-graph degrees, summed range by range during the build as
    csr_rowsum sums RandomNeighborSampler's CSR) and the [N] relabelling map; the int32 columns and float32 weights stay in host memory and each sampled edge reads
    them over the host link.

    Nodes: CSR rows = max(row) + 1, and the node count N (seeds, relabelling, SampledBlocks.num_nodes) is
    max(max row, max col) + 1, as RandomNeighborSampler.  sample_blocks has RandomNeighborSampler.sample_blocks'
    contract and returns the same batch for the same key, on the device.  sample, sample_neighborhood and the ratio rule
    are not offered: they take every sampled edge into one index space, which does not scale to such graphs.

    close() (or leaving a `with` block, or collection) releases the host CSR after the device's pending work; batches
    already returned stay valid (they hold device tensors only), and sampling after close() raises RuntimeError."""

    def __init__(self, edge_index, edge_weight=None, device_bytes=None):
        self._closed = True                 # until the build succeeds: nothing for close() / __del__ to release
        self._keys = []
        ei = _host_array(edge_index, "edge_index", np.int32, 2)
        if ei.shape[0] != 2:
            raise ValueError("edge_index must have shape [2, E] (got {})".format(ei.shape))
        E = ei.shape[1]
        w = None
        if edge_weight is not None:
            w = _host_array(edge_weight.reshape(-1) if hasattr(edge_weight, "reshape") else edge_weight, "edge_weight",
                            np.float32, 1)
            if w.shape[0] != E:
                raise ValueError("edge_weight has {} entries for {} edges".format(w.shape[0], E))
        dev = ops.default_device()
        if device_bytes is None:
            device_bytes = torch.cuda.mem_get_info(dev)[0] // 2
        self.num_edges = E
        self._device = dev
        self._has_weights = w is not None
        if E == 0:
            self.num_nodes, self.num_row_nodes = 0, 0
            self.rowptr = torch.zeros((1,), dtype=torch.int64, device=dev)
            self._rp = np.zeros((1,), np.int64)
            self.rowsum = torch.zeros((0,), dtype=torch.float32, device=dev)
            self._col_ptr, self._w_ptr, self._ranges = 0, None, []
            self._col = self._w = None
        else:
            self._build(ei, w, int(device_bytes))
        self._node_map = torch.full((self.num_nodes,), -1, dtype=torch.int32, device=dev)
        self._pos_deg = None
        rowptr, rowsum = self.rowptr, self.rowsum
        self._degrees = lambda: (rowptr, rowsum)      # the blocks' handle: device tensors only, not the sampler
        self._closed = False

    def _build(self, ei, w, device_bytes):
        E, dev = ei.shape[1], self._device
        edge_keys = []
        try:
            key, ei_ptr = _host_acquire(torch.from_numpy(ei))
            edge_keys.append(key)
            row_ptr, col_ptr = ei_ptr, ei_ptr + 4 * E
            w_ptr = None
            if w is not None:
                key, w_ptr = _host_acquire(torch.from_numpy(w))
                edge_keys.append(key)
            lo_r, hi_r, lo_c, hi_c = ops.mapped_id_range(row_ptr, col_ptr, E, dev)
            if min(lo_r, lo_c) < 0:
                raise ValueError("edge_index holds negative node ids")
            self.num_row_nodes = hi_r + 1
            self.num_nodes = N = max(hi_r, hi_c) + 1
            edge_bytes = HOST_CSR_EDGE_BYTES if w is not None else HOST_CSR_EDGE_BYTES_UNWEIGHTED
            budget = device_bytes - 8 * (N + 1) - 8 * (E // 1024 + 1) - HOST_CSR_FIXED_BYTES
            rowptr = ops.mapped_rowptr(row_ptr, E, N, dev)
            rp = rowptr.cpu().numpy()
            ranges = _row_ranges(rp, budget, edge_bytes)
            # ordinary host memory, page-locked in place (torch's pinned allocator would round each array up to a power
            # of two bytes); the CSR's registrations are the sampler's from here on
            col = _page_array(E, np.int32)
            key, col_dev = _host_acquire(torch.from_numpy(col))
            self._keys.append(key)
            cw, w_dev = None, None
            if w is not None:
                cw = _page_array(E, np.float32)
                key, w_dev = _host_acquire(torch.from_numpy(cw))
                self._keys.append(key)
            col_t = torch.from_numpy(col)
            w_t = None if cw is None else torch.from_numpy(cw)
            # the full graph's row sums (GcnBlock's degrees), from each range's weights while they are on the device
            rowsum = torch.zeros((N,), dtype=torch.float32, device=dev)
            for r0, r1 in ranges:
                e0, e1 = int(rp[r0]), int(rp[r1])
                if e1 == e0:
                    continue
                c, cwr = ops.mapped_csr_range(row_ptr, col_ptr, w_ptr, E, r0, r1, e1 - e0, N, dev)
                range_csr = ops.CSR(rowptr[r0:r1 + 1] - e0, c, None, r1 - r0, N)
                rowsum[r0:r1].copy_(ops.csr_rowsum(range_csr, torch.ones_like(c, dtype=torch.float32) if cwr is None
                                                   else cwr))
                col_t[e0:e1].copy_(c)
                if w_t is not None:
                    w_t[e0:e1].copy_(cwr)
                del c, cwr, range_csr
        except BaseException:
            for key in self._keys:
                _host_release(key)
            self._keys = []
            raise
        finally:
            for key in edge_keys:
                _host_release(key)
        self.rowptr, self.rowsum = rowptr, rowsum
        self._rp = rp                   # the host copy: each row block's CSR positions, and the chunks cut from them
        self._ranges = ranges
        self._col, self._w = col, cw
        self._col_ptr, self._w_ptr = col_dev, w_dev

    def _check_open(self):
        if self._closed:
            raise RuntimeError("this HostNeighborSampler is closed")

    def _positive_degrees(self):
        """RandomNeighborSampler._positive_degrees over the host CSR: tfgk_csr_positive_degree_f32 range by range over the
        build's row ranges, each range's weights (only they) copied to the device by one asynchronous bulk copy."""
        if self._pos_deg is None:
            if not self._has_weights:
                raise ValueError("weighted=True draws in proportion to edge_weight; this sampler was built without one")
            pos_deg = torch.zeros((self.num_nodes,), dtype=torch.int32, device=self._device)
            n_invalid = torch.zeros((1,), dtype=torch.int32, device=self._device)
            for r0, r1 in self._ranges:
                e0, e1 = int(self._rp[r0]), int(self._rp[r1])
                if e1 > e0:
                    w = torch.empty((e1 - e0,), dtype=torch.float32, device=self._device)
                    ops.copy_async(w, self._w.ctypes.data + 4 * e0, 4 * (e1 - e0))
                    ops.csr_positive_degree(self.rowptr[r0:r1 + 1], w, pos_deg[r0:r1], n_invalid, w_base=e0)
            _check_weights(int(n_invalid.item()))
            self._pos_deg = pos_deg
        return self._pos_deg

    def sample_blocks(self, seed_node_index, fanouts, padding=False, seed=None, weighted=False, labor=False,
                      layer_dependency=False):
        """RandomNeighborSampler.sample_blocks over the host CSR: same arguments, same batch for the same key (rows of
        the CSR are sampled in place over the host link).  A batch synchronises with the host once (plus one read-back
        per hop of fan-out None).  Calls on one sampler must be ordered on one CUDA stream.  weighted=True: as
        RandomNeighborSampler's; every candidate's weight is read over the host link.  labor=True, layer_dependency: as
        RandomNeighborSampler's (1 + 2 L read-backs for L integer hops); the columns of every row of d > k cross the host
        link twice, warp-wide, once to count and once to fill.

        :return: SampledBlocks, on the device"""
        self._check_open()
        _check_rule(weighted, labor, layer_dependency, padding)
        pos_deg = self._positive_degrees() if weighted else None
        return _sample_blocks(lambda nodes, hop_fanouts, keys: ops.block_sample_mapped(
            self.rowptr, self._col_ptr, self._w_ptr, nodes, hop_fanouts, keys, self._node_map, padding=padding,
            **_rule_args(pos_deg, labor)), self._device, self.num_nodes, seed_node_index, fanouts, seed, self._degrees,
            weighted, labor, layer_dependency)

    @_with_link_doc
    def sample_link_blocks(self, edge_index, fanouts, num_negatives=1, negative_edge_index=None, exclude=None,
                           padding=False, seed=None, weighted=False, labor=False, layer_dependency=False):
        self._check_open()
        _check_rule(weighted, labor, layer_dependency, padding)
        pos_deg = self._positive_degrees() if weighted else None
        return _sample_link_blocks(lambda pairs, n_pos, hop_fanouts, keys, exclude: ops.link_block_sample_mapped(
            self.rowptr, self._col_ptr, self._w_ptr, pairs, n_pos, hop_fanouts, keys, self._node_map, exclude=exclude,
            padding=padding, **_rule_args(pos_deg, labor)), self._device, self.num_nodes, edge_index, fanouts,
            num_negatives, negative_edge_index, exclude, padding, seed, self._degrees, weighted, labor,
            layer_dependency)

    def row_block(self, r0, r1):
        self._check_open()
        return _row_block(self, r0, r1)

    row_block.__doc__ = _ROW_BLOCK_DOC

    def _host_rowptr(self):
        return self._rp

    def _stage(self, e0, e1):
        """The columns and weights of CSR positions [e0, e1) in new device buffers, copied from the page-locked host CSR
        by one asynchronous bulk copy per array on the current stream (an unweighted graph's ones made on the device)."""
        self._check_open()
        S = e1 - e0
        cols = torch.empty((S,), dtype=torch.int32, device=self._device)
        if S:
            ops.copy_async(cols, self._col.ctypes.data + 4 * e0, 4 * S)
        if self._w is None:
            return cols, torch.ones((S,), dtype=torch.float32, device=self._device)
        w = torch.empty((S,), dtype=torch.float32, device=self._device)
        if S:
            ops.copy_async(w, self._w.ctypes.data + 4 * e0, 4 * S)
        return cols, w

    def _row_block_args(self):
        return self.rowptr, self._node_map, self._degrees

    def close(self):
        """Release the host CSR's registrations (after the device's pending work) and the arrays.  Idempotent."""
        if self._closed:
            return
        self._closed = True
        keys, self._keys = self._keys, []
        for key in keys:
            _host_release(key)
        self._col = self._w = None

    def __enter__(self):
        return self

    def __exit__(self, *exc):
        self.close()

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass
