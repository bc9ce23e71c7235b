# coding=utf-8
"""Typed wrappers over the C ABI (include/tfgk.h): torch CUDA tensors in, torch CUDA tensors out.

Nothing here computes with PyTorch: tensors are allocated with torch.empty and handed to libtfgk.so by pointer on
the current CUDA stream.  Every function requires CUDA tensors and raises otherwise (no CPU path).
"""
import ctypes

import numpy as np
import torch

from . import _ffi, _rng
from ._ffi import (REDUCE_SUM, REDUCE_MEAN, REDUCE_MAX, ACT_NONE, ACT_RELU, POW_INV_SQRT, POW_INV,  # noqa: F401
                   HEADS_SPLIT, HEADS_BROADCAST, HEADS_REDUCE, FLAG_ALL, FLAG_UPPER, FLAG_MAPPED,
                   BERNOULLI_NONE, BERNOULLI_DROPOUT, BERNOULLI_KEEP, SAMPLE_NO_PADDING, SAMPLE_PADDING, SAMPLE_HEAD,
                   GCN_NORM_BOTH, GCN_NORM_LEFT, GCN_NORM_RIGHT, GCN_LOOP_NONE, GCN_LOOP_NORMED, GCN_LOOP_FILL,
                   NEG_UPPER, NEG_START, PAD_ROW_MAJOR, PAD_STEP_MAJOR, SPGEMM_GRAD_LEFT, SPGEMM_GRAD_RIGHT)

_REDUCE_CODES = {"sum": REDUCE_SUM, "mean": REDUCE_MEAN, "max": REDUCE_MAX}


def _require_cuda():
    if not torch.cuda.is_available():
        raise RuntimeError("tf_geometric_b200 needs a CUDA device (H100 / sm_90a); there is no CPU fallback")


def default_device():
    _require_cuda()
    return torch.device("cuda", torch.cuda.current_device())


class SampledInput(object):
    """Base of the sampled-batch inputs (utils.sampling.Block, SelfLoopBlock, GcnBlock, SourceRows) that only the
    block-aware GraphSAGE aggregators, GAT and GCN take; as_device refuses them, so every other operator rejects them
    before any device work."""

    __slots__ = ()


def refuse_sampled(x):
    """TypeError for a SampledInput (the check as_device applies to every non-tensor input)."""
    if isinstance(x, SampledInput):
        raise TypeError("a {} is taken only by mean_graph_sage, sum_graph_sage, mean_pool_graph_sage and "
                        "max_pool_graph_sage (and their layers) on a Block, by gat (and GAT) on the SelfLoopBlock of "
                        "block.with_self_loops(), and by gcn (and GCN) on the GcnBlock of block.with_gcn_norm(); other "
                        "operators need a normalisation, self loops or padding that is not defined for a sampled "
                        "block".format(type(x).__name__))


def as_device(x, dtype=None, device=None):
    """numpy / list / torch (any device) -> contiguous CUDA tensor of `dtype` (reference casting rules are applied
    by the callers: int32 edge_index, float32 weights/features; data/graph.py:58-86).
    A conversion creates a NEW tensor on every call, and the CSR caches are keyed on tensor identity: for the warm path
    (no re-sort per forward) hand the layers an int32 CUDA edge_index - `Graph.to_device()` produces one - or pass
    `cache=graph.cache`."""
    if x is None:
        return None
    if not torch.is_tensor(x):
        refuse_sampled(x)
        x = torch.from_numpy(np.ascontiguousarray(x))
    if device is None:
        device = x.device if x.is_cuda else default_device()
    if dtype is not None and x.dtype != dtype:
        x = x.to(dtype)
    if x.device != device:
        x = x.to(device, non_blocking=True)
    return x.contiguous()


def _p(t):
    return None if t is None else ctypes.c_void_p(t.data_ptr())


def _stream(t):
    return ctypes.c_void_p(torch.cuda.current_stream(t.device).cuda_stream)


def _check(t, dtype, name):
    if not (torch.is_tensor(t) and t.is_cuda):
        raise TypeError("{} must be a CUDA tensor (got {})".format(name, type(t)))
    if t.dtype != dtype:
        raise TypeError("{} must be {} (got {})".format(name, dtype, t.dtype))
    if not t.is_contiguous():
        raise ValueError("{} must be contiguous".format(name))


def _row_major_2d(t, name):
    """Accept [N, D] tensors whose rows are contiguous (stride(1) == 1); returns the leading dimension."""
    if t.dim() != 2:
        raise ValueError("{} must be 2-D".format(name))
    if t.shape[1] > 1 and t.stride(1) != 1:
        raise ValueError("{} rows must be contiguous".format(name))
    return t.stride(0) if t.shape[0] > 1 else max(t.shape[1], t.stride(0))


HUB_THRESHOLD = 2048     # rows with more edges are cut into slices ...
HUB_CHUNK = 2048         # ... of this many edges (about the work of one ordinary 32-row task)
ROWS_PER_TASK = 32


class Plan(object):
    """Device-side work plan of a CSR with hub rows (struct tfgk_plan): task arrays + a scratch allocator."""

    def __init__(self, arrays, n_tasks, n_hubs, n_slots):
        self.arrays = arrays            # keeps the device tensors alive
        self.n_tasks, self.n_hubs, self.n_slots = n_tasks, n_hubs, n_slots
        self._scratch = None

    def struct(self, floats_per_slot, device):
        # the hub-slice scratch is allocated per call (the caching allocator makes that cheap and stream-ordered): a buffer
        # kept on the plan would be shared by launches on different streams that use the same cached CSR
        need = max(self.n_slots * floats_per_slot, 1)
        self._scratch = torch.empty((need,), dtype=torch.float32, device=device)
        a = self.arrays
        st = _ffi.PlanStruct(self.n_tasks, self.n_hubs, self.n_slots, HUB_CHUNK,
                             a["task_row"].data_ptr(), a["task_nrows"].data_ptr(), a["task_e0"].data_ptr(),
                             a["task_e1"].data_ptr(), a["task_slot"].data_ptr(), a["hub_row"].data_ptr(),
                             a["hub_slot0"].data_ptr(), a["hub_nslots"].data_ptr(), self._scratch.data_ptr(),
                             self._scratch.numel() * 4)
        return st


class CSR(object):
    """Destination-sorted CSR of a COO edge list (stable by row): rowptr int64 [n_rows+1], col int32 [nnz],
    perm int32 [nnz] (position of each CSR slot in the original edge list); `plan` is set when the graph has hub rows."""

    __slots__ = ("rowptr", "col", "perm", "n_rows", "n_cols", "nnz", "plan", "__weakref__")

    def __init__(self, rowptr, col, perm, n_rows, n_cols):
        self.rowptr, self.col, self.perm = rowptr, col, perm
        self.n_rows, self.n_cols = int(n_rows), int(n_cols)
        self.nnz = int(col.shape[0])
        self.plan = None

    def degree_i64(self):
        return self.rowptr[1:] - self.rowptr[:-1]


# ---- integer edge preprocessing ---------------------------------------------------------------------------------

def self_loops(edge_index, num_nodes):
    _check(edge_index, torch.int32, "edge_index")
    E = edge_index.shape[1] if edge_index.dim() == 2 else 0
    out = torch.empty((2, E + num_nodes), dtype=torch.int32, device=edge_index.device)
    _ffi.call("tfgk_self_loops_i32", _p(edge_index), E, num_nodes, _p(out), _stream(out))
    return out


def self_loop_weights(edge_weight, num_edges, num_nodes, fill_weight, device):
    if edge_weight is not None:
        _check(edge_weight, torch.float32, "edge_weight")
    out = torch.empty((num_edges + num_nodes,), dtype=torch.float32, device=device)
    _ffi.call("tfgk_self_loop_weights_f32", _p(edge_weight), num_edges, num_nodes, float(fill_weight), _p(out),
              _stream(out))
    return out


def segment_count(ids, num_segments):
    _check(ids, torch.int32, "index")
    out = torch.empty((num_segments,), dtype=torch.int32, device=ids.device)
    _ffi.call("tfgk_segment_count_i32", _p(ids), ids.numel(), num_segments, _p(out), _stream(out))
    return out


def csr_build(row, col, n_rows, n_cols=None, ids_in_range=False, plan=True):
    """ids_in_range=True: the ids are known to lie in [0, n_rows) x [0, n_cols) (tfgk_csr_build_in_range, which skips the
    check and its synchronisation; the work plan is still built).  plan=False builds no work plan, whose build reads its
    task counts back: with ids_in_range the build then makes no host synchronisation, and hub rows run unsplit."""
    _check(row, torch.int32, "row")
    _check(col, torch.int32, "col")
    n_cols = n_rows if n_cols is None else n_cols
    E = row.numel()
    dev = row.device
    need = ctypes.c_size_t()
    _ffi.call("tfgk_csr_workspace_bytes", E, n_rows, ctypes.byref(need))
    ws = torch.empty((max(need.value, 1),), dtype=torch.uint8, device=dev)
    rowptr = torch.empty((n_rows + 1,), dtype=torch.int64, device=dev)
    col_sorted = torch.empty((E,), dtype=torch.int32, device=dev)
    perm = torch.empty((E,), dtype=torch.int32, device=dev)
    _ffi.call("tfgk_csr_build_in_range" if ids_in_range else "tfgk_csr_build", _p(row), _p(col), E, n_rows, n_cols,
              _p(rowptr), _p(col_sorted), _p(perm),
              _p(ws), need.value, _stream(row))
    csr = CSR(rowptr, col_sorted, perm, n_rows, n_cols)
    csr.plan = build_plan(csr) if plan else None
    return csr


DENSE_ROW_DEGREE = 128   # average row length from which 32-row tasks starve the machine (few, long rows: pooling)
TASK_EDGE_TARGET = 512   # ... and the edges one task should then hold


def build_plan(csr):
    """Work plan: hub rows (> HUB_THRESHOLD edges) are cut into slices, and when the rows are few and long on average
    (graph pooling, set2set: one row per graph) the tasks shrink from 32 rows to about TASK_EDGE_TARGET edges so that
    there are enough warps to fill the GPU.  None when neither applies (the kernels then use their implicit 32-row
    tasks, which is also the fastest path for ordinary graphs)."""
    if csr.nnz == 0 or csr.n_rows == 0:
        return None
    avg = csr.nnz / float(csr.n_rows)
    rows_per_task = ROWS_PER_TASK if avg < DENSE_ROW_DEGREE else max(1, min(ROWS_PER_TASK, int(TASK_EDGE_TARGET // avg)))
    dev = csr.rowptr.device
    cap_t, cap_h = ctypes.c_int64(), ctypes.c_int64()
    _ffi.call("tfgk_plan_capacity", csr.nnz, csr.n_rows, HUB_THRESHOLD, HUB_CHUNK, rows_per_task, ctypes.byref(cap_t),
              ctypes.byref(cap_h))
    need = ctypes.c_size_t()
    _ffi.call("tfgk_plan_workspace_bytes", csr.n_rows, ctypes.byref(need))
    ws = torch.empty((need.value,), dtype=torch.uint8, device=dev)
    arrays = {k: torch.empty((cap_t.value,), dtype=torch.int32, device=dev) for k in ("task_row", "task_nrows", "task_slot")}
    arrays.update({k: torch.empty((cap_t.value,), dtype=torch.int64, device=dev) for k in ("task_e0", "task_e1")})
    arrays.update({k: torch.empty((cap_h.value,), dtype=torch.int32, device=dev) for k in ("hub_row", "hub_slot0", "hub_nslots")})
    counts = (ctypes.c_int32 * 3)()
    _ffi.call("tfgk_plan_build", _p(csr.rowptr), csr.n_rows, HUB_THRESHOLD, HUB_CHUNK, rows_per_task,
              _p(arrays["task_row"]), _p(arrays["task_nrows"]), _p(arrays["task_e0"]), _p(arrays["task_e1"]),
              _p(arrays["task_slot"]), _p(arrays["hub_row"]), _p(arrays["hub_slot0"]), _p(arrays["hub_nslots"]),
              cap_t.value, cap_h.value, counts, _p(ws), need.value, _stream(csr.rowptr))
    n_tasks, n_hubs, n_slots = int(counts[0]), int(counts[1]), int(counts[2])
    if n_hubs == 0 and rows_per_task == ROWS_PER_TASK:
        return None
    arrays = {k: v[:(n_tasks if k.startswith("task") else n_hubs)].clone() for k, v in arrays.items()}
    return Plan(arrays, n_tasks, n_hubs, n_slots)


def edge_unique(row, col, num_nodes):
    """Unique (row, col) pairs in first-occurrence order and, per edge, the index of its representative
    (merge_duplicated_edge's tf.unique step).  Returns (unique_edge_index int32 [2, U], unique_of_edge int32 [E])."""
    _check(row, torch.int32, "row")
    _check(col, torch.int32, "col")
    E = row.numel()
    dev = row.device
    need = ctypes.c_size_t()
    _ffi.call("tfgk_edge_unique_workspace_bytes", E, num_nodes, ctypes.byref(need))
    ws = torch.empty((max(need.value, 1),), dtype=torch.uint8, device=dev)
    uniq = torch.empty((2, max(E, 1)), dtype=torch.int32, device=dev)
    of_edge = torch.empty((E,), dtype=torch.int32, device=dev)
    n_unique = ctypes.c_int32()
    _ffi.call("tfgk_edge_unique", _p(row), _p(col), E, num_nodes, _p(uniq), _p(of_edge), ctypes.byref(n_unique), _p(ws),
              need.value, _stream(row))
    return uniq[:, :n_unique.value].contiguous(), of_edge


def directed_edges(upper_index):
    """upper edges followed by the mirrored non-self-loop upper edges; also the source column of every mirrored edge."""
    _check(upper_index, torch.int32, "upper_index")
    U = upper_index.shape[1]
    dev = upper_index.device
    need = ctypes.c_size_t()
    _ffi.call("tfgk_directed_workspace_bytes", U, ctypes.byref(need))
    ws = torch.empty((max(need.value, 1),), dtype=torch.uint8, device=dev)
    out = torch.empty((2, max(2 * U, 1)), dtype=torch.int32, device=dev)
    lower_src = torch.empty((max(U, 1),), dtype=torch.int32, device=dev)
    n_lower = ctypes.c_int32()
    _ffi.call("tfgk_directed_edges", _p(upper_index), U, U, _p(out), max(2 * U, 1), _p(lower_src), ctypes.byref(n_lower),
              _p(ws), need.value, _stream(upper_index))
    return out[:, :U + n_lower.value].contiguous(), lower_src[:n_lower.value]


def permute(src, perm, inverse=False):
    """COO-order values -> CSR order (dst[i] = src[perm[i]]), or back with inverse=True.  src: [E] or [E, W]."""
    _check(src, torch.float32, "src")
    _check(perm, torch.int32, "perm")
    width = 1 if src.dim() == 1 else src.shape[1]
    if inverse:
        if src.shape[0] != perm.numel():
            raise ValueError("unpermute: src must have one row per index")
        dst = torch.empty_like(src)
    else:                                    # a gather: one output row per index (perm may select a subset of src)
        dst = torch.empty((perm.numel(),) + tuple(src.shape[1:]), dtype=src.dtype, device=src.device)
    _ffi.call("tfgk_unpermute_f32" if inverse else "tfgk_permute_f32", _p(src), _p(perm), perm.numel(), width, _p(dst),
              _stream(src))
    return dst


# ---- feature tables in host memory (utils.HostFeatureTable) -------------------------------------------------------

def host_register(ptr, nbytes):
    """Page-lock the host range [ptr, ptr + nbytes) in place; returns the address the device reads it through."""
    dev = ctypes.c_void_p()
    _ffi.call("tfgk_host_register", ctypes.c_void_p(ptr), nbytes, ctypes.byref(dev))
    return dev.value


def host_unregister(ptr):
    """Release a registration made by host_register (ptr is the same host address)."""
    _ffi.call("tfgk_host_unregister", ctypes.c_void_p(ptr))


def gather_rows_mapped(table_ptr, ld, n_rows, num_features, index, out=None):
    """out[i] = table[index[i], :num_features] for a float32 table in mapped host memory at device address table_ptr
    (row stride ld floats, n_rows rows); ids outside [0, n_rows) give NaN rows.  index: int32 CUDA vector.  Returns out,
    a new [n, num_features] tensor on index's device unless given (rows contiguous, any row stride)."""
    _check(index, torch.int32, "index")
    n = index.numel()
    if out is None:
        out = torch.empty((n, num_features), dtype=torch.float32, device=index.device)
    elif not (torch.is_tensor(out) and out.is_cuda and out.dtype == torch.float32 and tuple(out.shape) == (n, num_features)):
        raise TypeError("out must be a float32 CUDA tensor of shape {}".format((n, num_features)))
    if n:
        ldo = _row_major_2d(out, "out")
        _ffi.call("tfgk_gather_rows_mapped_f32", ctypes.c_void_p(table_ptr), ld, n_rows, num_features, _p(index), n,
                  _p(out), ldo, _stream(out))
    return out


def gather_rows_cached(table_ptr, ld, n_rows, num_features, cache, slot, index, out=None):
    """gather_rows_mapped with a device cache of some rows: slot (int32 [n_rows]) maps row r to cache[slot[r]] when
    slot[r] >= 0, which is read from device memory instead of over the host link; -1 reads the host table.  cache:
    float32 [C, num_features] CUDA tensor (rows contiguous, any row stride).  cache, slot, index and out share one
    device.  The cache and the map are recorded on the stream the gather runs on, so dropping them while it is pending
    is safe."""
    _check(index, torch.int32, "index")
    _check(slot, torch.int32, "slot")
    if not (torch.is_tensor(cache) and cache.is_cuda and cache.dtype == torch.float32 and cache.dim() == 2
            and cache.shape[1] == num_features):
        raise TypeError("cache must be a float32 CUDA tensor of shape [C, {}]".format(num_features))
    if slot.numel() != n_rows:
        raise ValueError("slot must have one entry per table row ({} != {})".format(slot.numel(), n_rows))
    n = index.numel()
    if out is None:
        out = torch.empty((n, num_features), dtype=torch.float32, device=index.device)
    elif not (torch.is_tensor(out) and out.is_cuda and out.dtype == torch.float32 and tuple(out.shape) == (n, num_features)):
        raise TypeError("out must be a float32 CUDA tensor of shape {}".format((n, num_features)))
    if not (cache.device == slot.device == index.device == out.device):
        raise ValueError("cache, slot, index and out must be on one device")
    if n:
        ldc = _row_major_2d(cache, "cache")
        ldo = _row_major_2d(out, "out")
        stream = torch.cuda.current_stream(out.device)
        _ffi.call("tfgk_gather_rows_cached_f32", ctypes.c_void_p(table_ptr), ld, n_rows, num_features, _p(cache), ldc,
                  _p(slot), _p(index), n, _p(out), ldo, ctypes.c_void_p(stream.cuda_stream))
        cache.record_stream(stream)
        slot.record_stream(stream)
    return out


_DTYPE16_CODES = {torch.bfloat16: _ffi.DTYPE_BF16, torch.float16: _ffi.DTYPE_F16}


def _gather_out(out, n, num_features, dtype, device):
    if out is None:
        return torch.empty((n, num_features), dtype=dtype, device=device)
    if not (torch.is_tensor(out) and out.is_cuda and out.dtype == dtype and tuple(out.shape) == (n, num_features)):
        raise TypeError("out must be a {} CUDA tensor of shape {}".format(dtype, (n, num_features)))
    return out


def gather_rows_mapped_16(table_ptr, dtype, ld, n_rows, num_features, index, out=None, out_dtype=torch.float32):
    """gather_rows_mapped for a 16-bit table (dtype torch.bfloat16 or torch.float16; ld counted in elements): out[i] =
    table[index[i], :num_features] widened exactly to float32, bit-identical to the float32 table's gather; ids outside
    [0, n_rows) give NaN rows.  out_dtype=dtype copies the 16-bit patterns unchanged instead (a bad id then gives a
    16-bit NaN row), which fills a 16-bit device cache.  Returns out, a new [n, num_features] tensor of out_dtype on
    index's device unless given (rows contiguous, any row stride)."""
    if dtype not in _DTYPE16_CODES:
        raise ValueError("gather_rows_mapped_16 takes a torch.bfloat16 or torch.float16 table (got {})".format(dtype))
    if out_dtype not in (torch.float32, dtype):
        raise ValueError("out_dtype must be torch.float32 or the table's {} (got {})".format(dtype, out_dtype))
    _check(index, torch.int32, "index")
    n = index.numel()
    out = _gather_out(out, n, num_features, out_dtype, index.device)
    if n:
        ldo = _row_major_2d(out, "out")
        _ffi.call("tfgk_gather_rows_mapped_16", ctypes.c_void_p(table_ptr), _DTYPE16_CODES[dtype], ld, n_rows,
                  num_features, _p(index), n, _p(out), _ffi.DTYPE_F32 if out_dtype == torch.float32 else
                  _DTYPE16_CODES[dtype], ldo, _stream(out))
    return out


def gather_rows_cached_16(table_ptr, ld, n_rows, num_features, cache, slot, index, out=None):
    """gather_rows_cached for a 16-bit table: the table's dtype is cache's (torch.bfloat16 or torch.float16, [C,
    num_features], rows contiguous, any row stride), ld counts elements, and out is float32, each element widened
    exactly.  cache, slot, index and out share one device; the cache and the map are recorded on the gather's stream."""
    _check(index, torch.int32, "index")
    _check(slot, torch.int32, "slot")
    if not (torch.is_tensor(cache) and cache.is_cuda and cache.dtype in _DTYPE16_CODES and cache.dim() == 2
            and cache.shape[1] == num_features):
        raise TypeError("cache must be a bfloat16 or float16 CUDA tensor of shape [C, {}]".format(num_features))
    if slot.numel() != n_rows:
        raise ValueError("slot must have one entry per table row ({} != {})".format(slot.numel(), n_rows))
    n = index.numel()
    out = _gather_out(out, n, num_features, torch.float32, index.device)
    if not (cache.device == slot.device == index.device == out.device):
        raise ValueError("cache, slot, index and out must be on one device")
    if n:
        ldc = _row_major_2d(cache, "cache")
        ldo = _row_major_2d(out, "out")
        stream = torch.cuda.current_stream(out.device)
        _ffi.call("tfgk_gather_rows_cached_16", ctypes.c_void_p(table_ptr), _DTYPE16_CODES[cache.dtype], ld, n_rows,
                  num_features, _p(cache), ldc, _p(slot), _p(index), n, _p(out), ldo,
                  ctypes.c_void_p(stream.cuda_stream))
        cache.record_stream(stream)
        slot.record_stream(stream)
    return out


# ---- a CSR built from an edge list in host memory (utils.HostNeighborSampler) -------------------------------------
# row_ptr, col_ptr, w_ptr: device addresses of page-locked host arrays (host_register), int32 / int32 / float32 [E]

def mapped_id_range(row_ptr, col_ptr, num_edges, device):
    """(min row, max row, min col, max col) of an edge list in host memory with num_edges > 0 edges (synchronises)."""
    ws = torch.empty((16,), dtype=torch.uint8, device=device)
    out = (ctypes.c_int32 * 4)()
    _ffi.call("tfgk_mapped_id_range_i32", ctypes.c_void_p(row_ptr), ctypes.c_void_p(col_ptr), num_edges, out, _p(ws), 16,
              _stream(ws))
    return tuple(int(v) for v in out)


def mapped_rowptr(row_ptr, num_edges, n_rows, device):
    """int64 [n_rows + 1] device rowptr of the edge list in host memory (rows outside [0, n_rows) are not counted)."""
    need = ctypes.c_size_t()
    _ffi.call("tfgk_mapped_rowptr_workspace_bytes", n_rows, ctypes.byref(need))
    ws = torch.empty((need.value,), dtype=torch.uint8, device=device)
    rowptr = torch.empty((n_rows + 1,), dtype=torch.int64, device=device)
    _ffi.call("tfgk_mapped_rowptr_i32", ctypes.c_void_p(row_ptr), num_edges, n_rows, _p(rowptr), _p(ws), need.value,
              _stream(rowptr))
    return rowptr


def mapped_csr_range(row_ptr, col_ptr, w_ptr, num_edges, r0, r1, n_range, n_cols, device):
    """Rows [r0, r1) of the stable row-sorted CSR of the edge list in host memory, which hold n_range < 2^31 edges:
    (col int32 [n_range], weights float32 [n_range] or None when w_ptr is None), on the device.  The edges are selected in
    edge order (tfgk_mapped_select_rows_i32), sorted by row - r0 with the stable radix sort of csr_build and permuted."""
    need = ctypes.c_size_t()
    _ffi.call("tfgk_mapped_select_rows_workspace_bytes", num_edges, ctypes.byref(need))
    ws = torch.empty((max(need.value, 1),), dtype=torch.uint8, device=device)
    sel_row = torch.empty((n_range,), dtype=torch.int32, device=device)
    sel_col = torch.empty((n_range,), dtype=torch.int32, device=device)
    sel_w = None if w_ptr is None else torch.empty((n_range,), dtype=torch.float32, device=device)
    _ffi.call("tfgk_mapped_select_rows_i32", ctypes.c_void_p(row_ptr), ctypes.c_void_p(col_ptr),
              None if w_ptr is None else ctypes.c_void_p(w_ptr), num_edges, r0, r1, _p(sel_row), _p(sel_col), _p(sel_w),
              n_range, _p(ws), need.value, _stream(ws))
    del ws
    _ffi.call("tfgk_csr_workspace_bytes", n_range, r1 - r0, ctypes.byref(need))
    ws = torch.empty((max(need.value, 1),), dtype=torch.uint8, device=device)
    rowptr = torch.empty((r1 - r0 + 1,), dtype=torch.int64, device=device)
    col = torch.empty((n_range,), dtype=torch.int32, device=device)
    perm = torch.empty((n_range,), dtype=torch.int32, device=device)
    _ffi.call("tfgk_csr_build_in_range", _p(sel_row), _p(sel_col), n_range, r1 - r0, n_cols, _p(rowptr), _p(col),
              _p(perm), _p(ws), need.value, _stream(ws))
    del ws, sel_row, sel_col, rowptr
    return col, None if sel_w is None else permute(sel_w, perm)


def csr_rowsum(csr, w_csr):
    _check(w_csr, torch.float32, "w_csr")
    out = torch.empty((csr.n_rows,), dtype=torch.float32, device=w_csr.device)
    _ffi.call("tfgk_csr_rowsum_f32", _p(csr.rowptr), _p(w_csr), csr.n_rows, _p(out), _stream(out))
    return out


def deg_inv(deg, power):
    _check(deg, torch.float32, "deg")
    out = torch.empty_like(deg)
    _ffi.call("tfgk_deg_inv_f32", _p(deg), deg.numel(), power, _p(out), _stream(out))
    return out


def scale_edges(row, col, w, dl=None, dr=None):
    _check(w, torch.float32, "value")
    out = torch.empty_like(w)
    _ffi.call("tfgk_scale_edges_f32", _p(row), _p(col), _p(w), w.numel(), _p(dl), _p(dr), _p(out), _stream(out))
    return out


# ---- K1 ----------------------------------------------------------------------------------------------------------

def spmm(csr, w_csr, h, reduce="sum", alpha=1.0, addend=None, beta=0.0, bias=None, act=ACT_NONE, out=None, col=None,
         keep_layout=False, out_bf16=None):
    """out = epilogue(REDUCE_{e in row} w[e] * h[col[e]]); see tfgk_spmm_f32.  `col` overrides csr.col (used by the
    generic reducers, which gather message rows through csr.perm).  h may be bfloat16 (tfgk_spmm_bf16): the output is
    fp32 and bit-identical to the product over h.float(), also for strided or unaligned views of h.  With keep_layout=True
    a bf16 view is read in place, and the result is instead that of the fp32 product over a widened view with the same
    layout (the column chunks of SparseMatrix.matmul).
    out_bf16 (bf16 h only, tfgk_spmm_bf16_dual): a bfloat16 [n, D] tensor or view that receives the same result rounded
    to nearest even.  The fp32 result is then written only into an `out` passed explicitly: with out=None the call
    stores 2 bytes per element and returns out_bf16 (the intermediate hops of a propagation chain).  A bf16 h allocated
    by bf16_table() is read with its pad columns, which keeps every width on the ring kernels."""
    if isinstance(h, Fp8Table):
        if out_bf16 is not None:
            raise TypeError("spmm: an fp8 table takes no out_bf16")
        return _spmm_fp8(csr, w_csr, h, reduce, alpha, addend, beta, bias, act, out, col)
    if h.dtype not in (torch.float32, torch.bfloat16) or not h.is_cuda:
        raise TypeError("h must be a float32 or bfloat16 CUDA tensor")
    ldh = _row_major_2d(h, "h")
    n_dst, D = csr.n_rows, h.shape[1]
    plan = getattr(csr, "plan", None)
    if h.dtype == torch.bfloat16 and not keep_layout and plan is not None and plan.n_hubs > 0 and D % 4 == 0 and \
            32 <= D <= 512 and (ldh % 4 or h.data_ptr() % 8):
        # rows that are not 8-byte aligned take tfgk_spmm_bf16's scalar path, which sums hub rows strictly in order; the
        # fp32 kernel over h.float() (contiguous) slices them through the plan.  A dense copy takes the ring with the plan,
        # so that the result stays bit-identical to the product over h.float()
        h = h.clone(memory_format=torch.contiguous_format)
        ldh = _row_major_2d(h, "h")
    # a bf16 table with padded 16-byte rows (bf16_table) goes to the dual entry, which reads it with its pad columns on
    # the TMA ring: the same bits as tfgk_spmm_bf16, which would take the cp.async ring or the scalar path
    d8 = -(-D // 8) * 8
    padded = h.dtype == torch.bfloat16 and D % 8 != 0 and ldh % 8 == 0 and ldh >= d8 and h.data_ptr() % 16 == 0
    dual = out_bf16 is not None or padded
    if out_bf16 is not None:
        if h.dtype != torch.bfloat16:
            raise TypeError("spmm: out_bf16 needs a bfloat16 h")
        if not (out_bf16.is_cuda and out_bf16.dtype == torch.bfloat16 and tuple(out_bf16.shape) == (n_dst, D)):
            raise TypeError("spmm: out_bf16 must be a bfloat16 CUDA tensor of shape {}".format((n_dst, D)))
    elif out is None:
        out = torch.empty((n_dst, D), dtype=torch.float32, device=h.device)
    ldo = 0 if out is None else _row_major_2d(out, "out")
    ldob = 0 if out_bf16 is None else _row_major_2d(out_bf16, "out_bf16")
    lda = 0
    if addend is not None:
        lda = _row_major_2d(addend, "addend")
    if w_csr is not None:
        _check(w_csr, torch.float32, "w_csr")
    if bias is not None:
        _check(bias, torch.float32, "bias")
    code = _REDUCE_CODES[reduce] if isinstance(reduce, str) else reduce
    # the dual entry may read a padded table up to D rounded to 8 columns, hub slices included
    plan_struct = plan.struct(d8 if dual else D, h.device) if plan is not None else None
    plan_ref = ctypes.byref(plan_struct) if plan_struct is not None else None
    if dual:
        _ffi.call("tfgk_spmm_bf16_dual", _p(csr.rowptr), _p(csr.col if col is None else col), _p(w_csr), _p(h), ldh,
                  n_dst, D, code, float(alpha), _p(addend), lda, float(beta), _p(bias), act, _p(out), ldo, _p(out_bf16),
                  ldob, plan_ref, _stream(h))
        return out if out is not None else out_bf16
    _ffi.call("tfgk_spmm_bf16" if h.dtype == torch.bfloat16 else "tfgk_spmm_f32", _p(csr.rowptr),
              _p(csr.col if col is None else col), _p(w_csr), _p(h), ldh, n_dst, D,
              code, float(alpha), _p(addend), lda, float(beta), _p(bias), act, _p(out), ldo, plan_ref, _stream(h))
    return out


def spmm_proj_supported(x, W):
    """True when tfgk_spmm_proj_f32 takes x [n, F] and W [F, U]: fp32 CUDA tensors, 4 <= F < U <= 128, F % 4 == 0, and
    rows of x that are contiguous, 16-byte aligned and a multiple of 4 floats apart.  A shape-only condition."""
    if not (x.is_cuda and x.dtype == torch.float32 and x.dim() == 2 and W.dim() == 2):
        return False
    if W.shape[0] != x.shape[1] or not spmm_proj_shape(x.shape[1], W.shape[1]) or x.stride(1) != 1:
        return False
    return _row_major_2d(x, "x") % 4 == 0 and x.data_ptr() % 16 == 0


def spmm_proj_shape(F, U):
    """The widths tfgk_spmm_proj_f32 takes: 4 <= F < U <= 128, F % 4 == 0."""
    return 4 <= F < U <= 128 and F % 4 == 0


def spmm_proj(csr, w_csr, x, W, bias=None, act=ACT_NONE, out=None):
    """out = act((SUM_{e in row} w[e] * x[col[e]]) @ W + bias) with the aggregate never stored (tfgk_spmm_proj_f32, for
    x and W that spmm_proj_supported accepts): each aggregate is bit-identical to spmm(csr, w_csr, x)'s, and each output is
    an fmaf chain over the F columns of the aggregate from +0, then + bias, then the activation."""
    if not spmm_proj_supported(x, W):
        raise ValueError("spmm_proj: unsupported x {} / W {} (fp32 CUDA, 4 <= F < U <= 128, F % 4 == 0, aligned rows)".format(
            tuple(x.shape), tuple(W.shape)))
    W = W.to(torch.float32).contiguous()
    n_dst, F, U = csr.n_rows, x.shape[1], W.shape[1]
    if out is None:
        out = torch.empty((n_dst, U), dtype=torch.float32, device=x.device)
    elif not (out.is_cuda and out.dtype == torch.float32 and tuple(out.shape) == (n_dst, U)):
        raise TypeError("spmm_proj: out must be a float32 CUDA tensor of shape {}".format((n_dst, U)))
    if w_csr is not None:
        _check(w_csr, torch.float32, "w_csr")
    if bias is not None:
        _check(bias, torch.float32, "bias")
    plan = getattr(csr, "plan", None)
    plan_struct = plan.struct(F, x.device) if plan is not None else None
    _ffi.call("tfgk_spmm_proj_f32", _p(csr.rowptr), _p(csr.col), _p(w_csr), _p(x), _row_major_2d(x, "x"), n_dst, F, _p(W),
              U, _p(bias), act, _p(out), _row_major_2d(out, "out"),
              ctypes.byref(plan_struct) if plan_struct is not None else None, _stream(x))
    return out


def spmm_max(csr, w_csr, h):
    """(out, cnt): out[r] = max_{e in row r} w[e] * h[col[e]] (-FLT_MAX for an empty row), bit-identical to
    spmm(reduce="max"), and cnt[r, d] int32 = how many of those products equal out[r, d] (tfgk_spmm_max_f32, K11a)."""
    if h.dtype != torch.float32 or not h.is_cuda:
        raise TypeError("spmm_max: h must be a float32 CUDA tensor")
    ldh = _row_major_2d(h, "h")
    n, D = csr.n_rows, h.shape[1]
    if w_csr is not None:
        _check(w_csr, torch.float32, "w_csr")
    out = torch.empty((n, D), dtype=torch.float32, device=h.device)
    cnt = torch.empty((n, D), dtype=torch.int32, device=h.device)
    plan = getattr(csr, "plan", None)
    plan_struct = plan.struct(2 * D, h.device) if plan is not None else None
    _ffi.call("tfgk_spmm_max_f32", _p(csr.rowptr), _p(csr.col), _p(w_csr), _p(h), ldh, n, D, _p(out), max(D, 1), _p(cnt),
              max(D, 1), ctypes.byref(plan_struct) if plan_struct is not None else None, _stream(h))
    return out, cnt


def spmm_max_bwd(csr_t, w_t, h, out, cnt, g):
    """dh = d(spmm_max(...)[0]) / dh for upstream g, over the TRANSPOSED CSR csr_t (one row per source node; its `col`
    holds the destination row of every edge, w_t the weights in its order or None): tfgk_spmm_max_bwd_f32 (K11b).
    Bit-identical to the gradient of SegmentReduce(max) over the gathered messages summed by TakeRows."""
    for t, name in ((h, "h"), (out, "out"), (g, "g")):
        if t.dtype != torch.float32 or not t.is_cuda:
            raise TypeError("spmm_max_bwd: {} must be a float32 CUDA tensor".format(name))
    if cnt.dtype != torch.int32:
        raise TypeError("spmm_max_bwd: cnt must be int32")
    n_src, D = csr_t.n_rows, h.shape[1]
    n_dst = out.shape[0]
    if h.shape[0] != n_src or tuple(out.shape) != (n_dst, D) or tuple(cnt.shape) != (n_dst, D) or \
            tuple(g.shape) != (n_dst, D):
        raise ValueError("spmm_max_bwd: shapes h {}, out {}, cnt {}, g {} do not match {} sources".format(
            tuple(h.shape), tuple(out.shape), tuple(cnt.shape), tuple(g.shape), n_src))
    if w_t is not None:
        _check(w_t, torch.float32, "w_t")
    pk = torch.empty((n_dst, 2 * D), dtype=torch.float32, device=h.device)
    dh = torch.empty((n_src, D), dtype=torch.float32, device=h.device)
    plan = getattr(csr_t, "plan", None)
    plan_struct = plan.struct(D, h.device) if plan is not None else None
    _ffi.call("tfgk_spmm_max_bwd_f32", _p(csr_t.rowptr), _p(csr_t.col), _p(w_t), _p(h), _row_major_2d(h, "h"), n_src,
              n_dst, D, _p(out), _row_major_2d(out, "out"), _p(cnt), _row_major_2d(cnt, "cnt"), _p(g),
              _row_major_2d(g, "g"), _p(pk), _p(dh), max(D, 1), ctypes.byref(plan_struct) if plan_struct is not None else None,
              _stream(h))
    return dh


def _check_fp8_operand(t, name, n_grp, rows=None, device=None):
    """An Fp8Table the gather kernels can read: CUDA data and exponents on one device, and exponents as a dense
    [rows, n_grp] array (the kernels index them as row * n_grp + group).  A column block of a wider table (block()) is
    what gemm_proj and quantize_fp8 write into, but its exponents are strided: it is refused here rather than read with
    another row's exponents; gather from a table of its own."""
    if not isinstance(t, Fp8Table):
        raise TypeError("{} must be an Fp8Table".format(name))
    e = t.exps
    if e.shape[1] != n_grp or (n_grp > 1 and e.stride(1) != 1) or (e.shape[0] > 1 and e.stride(0) != n_grp):
        raise ValueError("{}: the exponents must be a dense [rows, {}] array (got shape {} with strides {}); a column block "
                         "of a wider table cannot be gathered".format(name, n_grp, tuple(e.shape), tuple(e.stride())))
    if rows is not None and t.data.shape[0] < rows:
        raise ValueError("{} has {} rows; the graph references {}".format(name, t.data.shape[0], rows))
    if not (t.data.is_cuda and e.is_cuda and e.device == t.data.device):
        raise TypeError("{}: data and exponents must be CUDA tensors on one device".format(name))
    if device is not None and t.data.device != device:
        raise ValueError("{} is on {}, the other operands on {}".format(name, t.data.device, device))
    _row_major_2d(t.data, name)


def _spmm_fp8(csr, w_csr, h, reduce, alpha, addend, beta, bias, act, out, col):
    """spmm over an fp8 table (tfgk_spmm_fp8): bit-identical to the fp32 product over the dequantised table with the same
    leading dimension wherever both take the work plan or neither does (tables up to 256 columns)."""
    n_dst, D = csr.n_rows, h.cols
    _check_fp8_operand(h, "h", max(-(-D // 128), 1), rows=csr.n_cols if col is None else None,
                       device=None if out is None else out.device)
    if out is None:
        out = torch.empty((n_dst, D), dtype=torch.float32, device=h.device)
    lda = 0 if addend is None else _row_major_2d(addend, "addend")
    if w_csr is not None:
        _check(w_csr, torch.float32, "w_csr")
    if bias is not None:
        _check(bias, torch.float32, "bias")
    code = _REDUCE_CODES[reduce] if isinstance(reduce, str) else reduce
    plan = getattr(csr, "plan", None)
    # the TMA ring reads the table with its pad columns, hub slices included
    plan_struct = plan.struct(-(-D // 16) * 16, h.device) if plan is not None else None
    _ffi.call("tfgk_spmm_fp8", _p(csr.rowptr), _p(csr.col if col is None else col), _p(w_csr), _p(h.data), h.ld, _p(h.exps), n_dst, D, code,
              float(alpha), _p(addend), lda, float(beta), _p(bias), act, _p(out), _row_major_2d(out, "out"),
              ctypes.byref(plan_struct) if plan_struct is not None else None, _stream(out))
    return out


class Fp8Table(object):
    """fp8 message rows in the format of include/tfgk.h: `data` a [rows, cols] uint8 view of e4m3fn bytes whose rows are
    16-byte aligned (the pad columns of the buffer zeroed), `exps` the int8 exponents, one column per group of 128
    columns ([rows, ceil(cols / 128)]; a GAT K | V table has two: the K group and the V group) and `cols` the logical
    width.  fp8_table() allocates one; block() is the view one K4 column block writes."""

    __slots__ = ("data", "exps", "cols")

    def __init__(self, data, exps, cols):
        if not (torch.is_tensor(data) and data.dtype == torch.uint8 and data.dim() == 2):
            raise TypeError("Fp8Table: data must be a 2-D uint8 tensor")
        if not (torch.is_tensor(exps) and exps.dtype == torch.int8 and exps.dim() == 2 and exps.shape[0] == data.shape[0]):
            raise TypeError("Fp8Table: exps must be a 2-D int8 tensor with one row per data row")
        if data.shape[1] != cols:
            raise ValueError("Fp8Table: data has {} columns, expected {}".format(data.shape[1], cols))
        self.data, self.exps, self.cols = data, exps, int(cols)

    dtype = torch.float8_e4m3fn

    @property
    def is_cuda(self):
        return self.data.is_cuda

    @property
    def device(self):
        return self.data.device

    @property
    def shape(self):
        return self.data.shape

    @property
    def ld(self):
        return _row_major_2d(self.data, "fp8 data")

    def block(self, c0, c1, group=None):
        """Columns [c0, c1) (at most one group of 128) with the exponent column `group` (default c0 // 128)."""
        g = c0 // 128 if group is None else int(group)
        if c1 - c0 > 128 or (group is None and c0 % 128):
            raise ValueError("Fp8Table.block: [{}, {}) is not inside one group of 128 columns".format(c0, c1))
        return Fp8Table(self.data[:, c0:c1], self.exps[:, g:g + 1], c1 - c0)


def fp8_table(rows, cols, device, groups=None):
    """An empty fp8 table (Fp8Table): rows padded to a multiple of 16 bytes with the pad columns zeroed, exponents
    [rows, groups] (default ceil(cols / 128))."""
    pitch = max(-(-int(cols) // 16) * 16, 16)
    buf = torch.empty((int(rows), pitch), dtype=torch.uint8, device=device)
    if pitch != cols:
        buf[:, cols:].zero_()
    n_grp = max(-(-int(cols) // 128), 1) if groups is None else int(groups)
    exps = torch.empty((int(rows), n_grp), dtype=torch.int8, device=device)
    return Fp8Table(buf[:, :cols], exps, cols)


def quantize_fp8(src, out=None):
    """fp8 table of a 2-D float32 CUDA tensor (tfgk_quantize_fp8): the bytes and exponents the K4 epilogue writes from
    the same values.  `out` may be an Fp8Table (or a block of one) of the same shape."""
    if not (torch.is_tensor(src) and src.is_cuda and src.dtype == torch.float32 and src.dim() == 2):
        raise TypeError("quantize_fp8: src must be a 2-D float32 CUDA tensor")
    if out is None:
        out = fp8_table(src.shape[0], src.shape[1], src.device)
    if not isinstance(out, Fp8Table) or tuple(out.shape) != tuple(src.shape):
        raise TypeError("quantize_fp8: out must be an Fp8Table of shape {}".format(tuple(src.shape)))
    if out.exps.shape[1] < -(-src.shape[1] // 128) or (out.exps.shape[1] > 1 and out.exps.stride(1) != 1):
        raise ValueError("quantize_fp8: out has {} exponent columns (column stride {}) for {} columns".format(
            out.exps.shape[1], out.exps.stride(1), src.shape[1]))
    if not (out.data.is_cuda and out.exps.is_cuda and out.data.device == src.device and out.exps.device == src.device):
        raise TypeError("quantize_fp8: out must live on the device of src ({})".format(src.device))
    _ffi.call("tfgk_quantize_fp8", _p(src), _row_major_2d(src, "src"), src.shape[0], src.shape[1], _p(out.data), out.ld,
              _p(out.exps), out.exps.stride(0), _stream(src))
    return out


def bf16_table(rows, cols, device):
    """An empty [rows, cols] bfloat16 table for message rows: a view of a row-major buffer whose rows are padded to a
    multiple of 8 elements (16 bytes), pad columns zeroed, so that tfgk_spmm_bf16_dual reads every width with its ring
    kernels."""
    pitch = -(-int(cols) // 8) * 8
    buf = torch.empty((int(rows), pitch), dtype=torch.bfloat16, device=device)
    if pitch != cols:
        buf[:, cols:].zero_()
    return buf[:, :cols]


def round_bf16_table(src):
    """bf16_table() holding src (2-D float32 CUDA) rounded to nearest even (tfgk_round_bf16)."""
    return round_bf16(src, out=bf16_table(src.shape[0], src.shape[1], src.device))


# ---- K3 ----------------------------------------------------------------------------------------------------------

def segment_softmax_csr(csr, score_csr):
    """score_csr: [E] or [E, H] in CSR order."""
    _check(score_csr, torch.float32, "score")
    H = 1 if score_csr.dim() == 1 else score_csr.shape[1]
    out = torch.empty_like(score_csr)
    _ffi.call("tfgk_segment_softmax_f32", _p(csr.rowptr), _p(score_csr), csr.n_rows, H, _p(out), _stream(out))
    return out


def gat_fused(csr, Q, K, V, num_heads, split_value_heads=True, bias=None, act=ACT_NONE, return_attention=False,
              att_buffer=None, out=None, scale=None):
    """Fused GAT attention (tfgk_gat_fused_f32).  K and V may both be bfloat16 (tfgk_gat_fused_bf16, inference only:
    no return_attention); Q and the output stay float32.  K may instead be an Fp8Table holding K | V ([N, 2A] bytes, two
    exponent columns) with V None (tfgk_gat_fused_fp8, inference only, the TMA ring's shapes)."""
    if isinstance(K, Fp8Table):
        return _gat_fused_fp8(csr, Q, K, V, num_heads, split_value_heads, bias, act, return_attention, out, scale)
    bf16 = K.dtype == torch.bfloat16
    for t, n, dt in ((Q, "Q", torch.float32), (K, "K", K.dtype), (V, "V", K.dtype)):
        if not (t.is_cuda and t.dtype == dt and dt in (torch.float32, torch.bfloat16)):
            raise TypeError("{} must be a {} CUDA tensor (Q float32; K and V both float32 or both bfloat16)".format(
                n, "float32" if n == "Q" else "float32 or bfloat16"))
    if bf16 and return_attention:
        raise NotImplementedError("gat_fused: bfloat16 K and V are an inference mode without attention coefficients")
    N = csr.n_rows
    H = int(num_heads)
    A, VW = Q.shape[1], V.shape[1]
    if A % H or VW % H or K.shape[1] != A:
        raise ValueError("attention units ({}) and value units ({}) must be divisible by num_heads ({})".format(A, VW, H))
    dqk, dv = A // H, VW // H
    out_w = VW if split_value_heads else dv
    if out is None:
        out = torch.empty((N, out_w), dtype=torch.float32, device=Q.device)
    att = att_buffer
    if att is not None and att.numel() < csr.nnz * H:
        att = None
    if att is None and return_attention:
        att = torch.empty((csr.nnz, H), dtype=torch.float32, device=Q.device)
    if bias is not None:
        _check(bias, torch.float32, "bias")
    # gat.py:78  scale = sqrt(cast(shape(Q_)[-1], float32)); set2set.py:37 uses raw dot products (scale = 1)
    scale = float(np.sqrt(np.float32(dqk))) if scale is None else float(scale)

    plan = getattr(csr, "plan", None)
    plan_struct = plan.struct(VW + 64, Q.device) if plan is not None else None

    def launch(att_buf):
        _ffi.call("tfgk_gat_fused_bf16" if bf16 else "tfgk_gat_fused_f32", _p(csr.rowptr), _p(csr.col), _p(Q),
                  _row_major_2d(Q, "Q"), _p(K),
                  _row_major_2d(K, "K"), _p(V), _row_major_2d(V, "V"), N, H, dqk, dv, scale,
                  1 if split_value_heads else 0, _p(bias), act, _p(att_buf), 1 if return_attention else 0, _p(out),
                  _row_major_2d(out, "out"), ctypes.byref(plan_struct) if plan_struct is not None else None, _stream(Q))

    try:
        launch(att)
    except _ffi.TfgkError as err:
        # the single-pass kernel needs no scratch; the two-pass / generic kernels ask for an [E, H] score buffer
        if err.code != _ffi.ERR_WORKSPACE or att is not None:
            raise
        att = torch.empty((csr.nnz, H), dtype=torch.float32, device=Q.device)
        launch(att)
    if return_attention:
        return out, att[:csr.nnz]
    return out


def _gat_fused_fp8(csr, Q, kv, V, num_heads, split_value_heads, bias, act, return_attention, out, scale):
    if V is not None:
        raise TypeError("gat_fused: an fp8 K | V table holds the values as well (pass V=None)")
    if return_attention or not split_value_heads:
        raise NotImplementedError("gat_fused: fp8 K | V concatenate the heads and return no attention coefficients")
    if not (torch.is_tensor(Q) and Q.dtype == torch.float32 and Q.dim() == 2):
        raise TypeError("Q must be a 2-D float32 CUDA tensor")
    H, A = int(num_heads), Q.shape[1]
    if kv.cols != 2 * A or A % H:
        raise ValueError("gat_fused: an fp8 K | V table has 2A columns, A divisible by num_heads")
    if Q.shape[0] != csr.n_rows:
        raise ValueError("gat_fused: Q has {} rows, the graph {}".format(Q.shape[0], csr.n_rows))
    _check_fp8_operand(kv, "K | V", 2, rows=csr.n_cols)
    if not (Q.is_cuda and Q.device == kv.device):
        raise TypeError("Q must be a CUDA tensor on the device of K | V ({})".format(kv.device))
    dqk = A // H
    if out is None:
        out = torch.empty((csr.n_rows, A), dtype=torch.float32, device=Q.device)
    if bias is not None:
        _check(bias, torch.float32, "bias")
    scale = float(np.sqrt(np.float32(dqk))) if scale is None else float(scale)
    plan = getattr(csr, "plan", None)
    plan_struct = plan.struct(A + 64, Q.device) if plan is not None else None
    _ffi.call("tfgk_gat_fused_fp8", _p(csr.rowptr), _p(csr.col), _p(Q), _row_major_2d(Q, "Q"), _p(kv.data), kv.ld,
              _p(kv.exps), csr.n_rows, H, dqk, scale, _p(bias), act, _p(out), _row_major_2d(out, "out"),
              ctypes.byref(plan_struct) if plan_struct is not None else None, _stream(Q))
    return out


def gat_packed_width(units):
    """Floats per slot of a packed key table for A = units (tfgk_gat_pack_keys_f32): V, the 4-float zero mask and at most A
    keys, rounded up to 32 floats so that every slot starts on a 128-byte boundary (288 = 1,152 bytes at A = 128; the
    fused kernel reads 128-byte aligned slots measurably faster than 64-byte aligned ones)."""
    return -(-(2 * int(units) + 4) // 32) * 32


def packed_key_table(num_nodes, units, device):
    """An empty packed key table [num_nodes, gat_packed_width(units)] float32 and its copy sizes [num_nodes] uint8; the
    V rows go into table[:, :units], then gat_pack_keys fills the rest."""
    table = torch.empty((int(num_nodes), gat_packed_width(units)), dtype=torch.float32, device=device)
    sizes = torch.empty((int(num_nodes),), dtype=torch.uint8, device=device)
    return table, sizes


def gat_pack_keys(K, table, sizes):
    """Writes K [N, A] (float32, A <= 128) into a packed key table: zero mask, non-zero entries in column order, copy size per
    node (tfgk_gat_pack_keys_f32).  Only the bit pattern 0x00000000 counts as zero."""
    if not (K.is_cuda and K.dtype == torch.float32 and K.dim() == 2):
        raise TypeError("gat_pack_keys: K must be a 2-D float32 CUDA tensor")
    _check(sizes, torch.uint8, "sizes")
    N, A = K.shape
    if table.dtype != torch.float32 or table.shape[0] != N or sizes.shape[0] != N:
        raise ValueError("gat_pack_keys: table and sizes must have {} rows".format(N))
    _ffi.call("tfgk_gat_pack_keys_f32", _p(K), _row_major_2d(K, "K"), N, A, _p(table), _row_major_2d(table, "table"),
              _p(sizes), _stream(K))
    return table, sizes


def gat_fused_packed(csr, Q, table, sizes, num_heads, bias=None, act=ACT_NONE, out=None, scale=None):
    """gat_fused with heads concatenated over a packed key table (tfgk_gat_fused_packed_f32): the same output bits as
    gat_fused(csr, Q, K, V, ...) for the K that gat_pack_keys packed and V = table[:, :A]."""
    _check(sizes, torch.uint8, "sizes")
    if not (Q.is_cuda and Q.dtype == torch.float32 and table.is_cuda and table.dtype == torch.float32):
        raise TypeError("gat_fused_packed: Q and table must be float32 CUDA tensors")
    N, H, A = csr.n_rows, int(num_heads), Q.shape[1]
    if A % H:
        raise ValueError("attention units ({}) must be divisible by num_heads ({})".format(A, H))
    if out is None:
        out = torch.empty((N, A), dtype=torch.float32, device=Q.device)
    if bias is not None:
        _check(bias, torch.float32, "bias")
    scale = float(np.sqrt(np.float32(A // H))) if scale is None else float(scale)
    plan = getattr(csr, "plan", None)
    plan_struct = plan.struct(A + 64, Q.device) if plan is not None else None
    _ffi.call("tfgk_gat_fused_packed_f32", _p(csr.rowptr), _p(csr.col), _p(Q), _row_major_2d(Q, "Q"), _p(table),
              _row_major_2d(table, "table"), _p(sizes), N, H, A // H, scale, _p(bias), act, _p(out), _row_major_2d(out, "out"),
              ctypes.byref(plan_struct) if plan_struct is not None else None, _stream(Q))
    return out


def gat_fused_stats(csr, Q, K, V, num_heads, bias=None, act=ACT_NONE, scale=None):
    """Training forward without the [E, H] coefficient table: returns (out, stats[N, 2H]) or None when the shape is not
    taken by the streaming kernel (tfgk_gat_fused_stats_f32)."""
    N, H = csr.n_rows, int(num_heads)
    A = Q.shape[1]
    if A % H or V.shape[1] != A or K.shape[1] != A:
        return None
    dqk = A // H
    scale = float(np.sqrt(np.float32(dqk))) if scale is None else float(scale)
    out = torch.empty((N, A), dtype=torch.float32, device=Q.device)
    stats = torch.empty((N, 2 * H), dtype=torch.float32, device=Q.device)
    plan = getattr(csr, "plan", None)
    plan_struct = plan.struct(A + 64, Q.device) if plan is not None else None
    try:
        _ffi.call("tfgk_gat_fused_stats_f32", _p(csr.rowptr), _p(csr.col), _p(Q), _row_major_2d(Q, "Q"), _p(K),
                  _row_major_2d(K, "K"), _p(V), _row_major_2d(V, "V"), N, H, dqk, dqk, scale, _p(bias), act, _p(out),
                  _row_major_2d(out, "out"), _p(stats), ctypes.byref(plan_struct) if plan_struct is not None else None, _stream(Q))
    except _ffi.TfgkError as err:
        if err.code != _ffi.ERR_UNSUPPORTED:
            raise
        return None
    return out, stats


def gat_backward_recompute(csr, csr_t, Q, K, V, G, Y, bias, act, stats, num_heads, scale):
    """(dQ, dK, dV) of the fused attention aggregation from (max, denominator) per row (tfgk_gat_bwd_*); None when the
    kernels do not take the shape."""
    N, H = csr.n_rows, int(num_heads)
    A = Q.shape[1]
    dqk = A // H
    GS = torch.empty((N, A + 32), dtype=torch.float32, device=Q.device)
    dQ, dK, dV = torch.empty_like(Q), torch.empty_like(K), torch.empty_like(V)
    try:
        _ffi.call("tfgk_gat_bwd_prepare_f32", _p(G), _row_major_2d(G, "G"), _p(Y), _row_major_2d(Y, "Y"), _p(bias), act,
                  _p(stats), N, H, dqk, _p(GS), A + 32, _stream(Q))
        _ffi.call("tfgk_gat_bwd_dst_f32", _p(csr.rowptr), _p(csr.col), _p(Q), _row_major_2d(Q, "Q"), _p(K),
                  _row_major_2d(K, "K"), _p(V), _row_major_2d(V, "V"), _p(GS), A + 32, N, H, dqk, float(scale), _p(dQ),
                  _row_major_2d(dQ, "dQ"), _stream(Q))
        # the transposed pass walks the SOURCE rows (set2set: nodes, while the forward rows are graphs)
        _ffi.call("tfgk_gat_bwd_src_f32", _p(csr_t.rowptr), _p(csr_t.col), _p(Q), _row_major_2d(Q, "Q"), _p(K),
                  _row_major_2d(K, "K"), _p(V), _row_major_2d(V, "V"), _p(GS), A + 32, csr_t.n_rows, H, dqk, float(scale), _p(dK),
                  _row_major_2d(dK, "dK"), _p(dV), _row_major_2d(dV, "dV"), _stream(Q))
    except _ffi.TfgkError as err:
        if err.code != _ffi.ERR_UNSUPPORTED:
            raise
        return None
    return dQ, dK, dV


# ---- training-mode extras: dropout, per-head aggregation, GAT softmax backward -----------------------------------

# rng_stream ids: independent draws for the same (seed, element); LINK = negative sampling and the edge split, WEIGHTED =
# the weighted fan-outs' keys (include/tfgk.h, "weighted block sampler"), LABOR = the layer-neighbour variates ("LABOR
# block sampler")
RNG_STREAM_DROPOUT, RNG_STREAM_SAMPLER, RNG_STREAM_LINK, RNG_STREAM_WEIGHTED, RNG_STREAM_LABOR = 0, 1, 2, 3, 4


def _keyed(entry, seed):
    """The entry and key arguments for `seed`: a host key, or an _rng.DeviceKey (CUDA-graph capture), which goes to the
    _devkey twin of the entry as (base pointer, slot)."""
    if isinstance(seed, _rng.DeviceKey):
        return entry[:-len("_f32")] + "_devkey_f32", (_p(seed.base), int(seed.slot))
    return entry, (int(seed),)


def dropout(x, rate, seed, rng_stream=RNG_STREAM_DROPOUT, out=None):
    """tf.nn.dropout with a counter-based mask: element i is kept iff u(seed, i) >= rate, kept values * 1/(1-rate).
    `seed` is a host key or an _rng.DeviceKey."""
    _check(x, torch.float32, "x")
    if out is None:
        out = torch.empty_like(x)
    entry, key = _keyed("tfgk_dropout_f32", seed)
    _ffi.call(entry, _p(x), x.numel(), float(rate), *key, int(rng_stream), _p(out), _stream(x))
    return out


def spmm_heads(csr, w, src, num_heads, mode=HEADS_SPLIT, emap=None, drop_rate=0.0, seed=0,
               rng_stream=RNG_STREAM_DROPOUT, alpha=1.0, bias=None, act=ACT_NONE, out=None):
    """Per-(edge, head) weighted aggregation over `csr`; see tfgk_spmm_heads_f32.  w: [E, H] (looked up through `emap`
    when the CSR is a transposed view of the structure w was computed on).  `seed` is a host key or an _rng.DeviceKey."""
    _check(w, torch.float32, "w")
    if not (src.is_cuda and src.dtype == torch.float32):
        raise TypeError("src must be a float32 CUDA tensor")
    if emap is not None:
        _check(emap, torch.int32, "emap")
    H = int(num_heads)
    lds = _row_major_2d(src, "src")
    if mode == HEADS_BROADCAST:
        dh = src.shape[1]
        out_w = H * dh
    else:
        if src.shape[1] % H:
            raise ValueError("spmm_heads: {} source columns are not divisible by {} heads".format(src.shape[1], H))
        dh = src.shape[1] // H
        out_w = dh if mode == HEADS_REDUCE else H * dh
    if out is None:
        out = torch.empty((csr.n_rows, out_w), dtype=torch.float32, device=src.device)
    if bias is not None:
        _check(bias, torch.float32, "bias")
    entry, key = _keyed("tfgk_spmm_heads_f32", seed)
    _ffi.call(entry, _p(csr.rowptr), _p(csr.col), _p(emap), _p(w), _p(src), lds, csr.n_rows, H, dh, int(mode),
              float(drop_rate), *key, int(rng_stream), float(alpha), _p(bias), act, _p(out), _row_major_2d(out, "out"),
              _stream(src))
    return out


def gat_softmax_bwd(csr, att, G, V, num_heads, split_value_heads=True, drop_rate=0.0, seed=0,
                    rng_stream=RNG_STREAM_DROPOUT):
    """d loss / d scaled scores [E, H] (CSR order) from G = d loss / d aggregated rows; see tfgk_gat_softmax_bwd_f32.
    `seed` is a host key or an _rng.DeviceKey."""
    _check(att, torch.float32, "att")
    H = int(num_heads)
    dv = V.shape[1] // H
    ds = torch.empty((csr.nnz, H), dtype=torch.float32, device=att.device)
    entry, key = _keyed("tfgk_gat_softmax_bwd_f32", seed)
    _ffi.call(entry, _p(csr.rowptr), _p(csr.col), _p(att), _p(G), _row_major_2d(G, "G"), _p(V), _row_major_2d(V, "V"),
              csr.n_rows, H, dv, 1 if split_value_heads else 0, float(drop_rate), *key, int(rng_stream), _p(ds),
              _stream(att))
    return ds


# ---- device-side edge sampling -----------------------------------------------------------------------------------

def edge_flags(row, col, num_edges, mode=FLAG_ALL, row_map=None, col_map=None, bernoulli=BERNOULLI_NONE, prob=0.0,
               seed=0, rng_stream=RNG_STREAM_SAMPLER, device=None):
    """int32 [E] keep flags: structural rule AND Bernoulli rule (tfgk_edge_flags_i32)."""
    for t, n in ((row, "row"), (col, "col"), (row_map, "row_map"), (col_map, "col_map")):
        if t is not None:
            _check(t, torch.int32, n)
    dev = device if row is None else row.device
    flag = torch.empty((num_edges,), dtype=torch.int32, device=dev)
    _ffi.call("tfgk_edge_flags_i32", _p(row), _p(col), num_edges, int(mode), _p(row_map), _p(col_map), int(bernoulli),
              float(prob), int(seed), int(rng_stream), _p(flag), _stream(flag))
    return flag


def select_flagged(flag):
    """Ascending positions of the non-zero flags (tf.boolean_mask(tf.range(n), flag)), int32 [n_selected]."""
    _check(flag, torch.int32, "flag")
    n = flag.numel()
    need = ctypes.c_size_t()
    _ffi.call("tfgk_select_workspace_bytes", n, ctypes.byref(need))
    ws = torch.empty((max(need.value, 1),), dtype=torch.uint8, device=flag.device)
    out = torch.empty((max(n, 1),), dtype=torch.int32, device=flag.device)
    n_out = ctypes.c_int64()
    _ffi.call("tfgk_select_flagged_i32", _p(flag), n, _p(out), ctypes.byref(n_out), _p(ws), need.value, _stream(flag))
    return out[:n_out.value]


def gather_i32(src, index):
    """src[index] for int32 vectors: a bit copy through tfgk_permute_f32 (the kernel moves 4-byte words)."""
    _check(src, torch.int32, "src")
    return permute(src.view(torch.float32), index).view(torch.int32)


def sort_keys_f32(score, descending=False):
    """Order-preserving int32 bit patterns of float32 scores (to be sorted as unsigned numbers)."""
    _check(score, torch.float32, "score")
    keys = torch.empty((score.numel(),), dtype=torch.int32, device=score.device)
    _ffi.call("tfgk_sort_keys_f32", _p(score), score.numel(), 1 if descending else 0, _p(keys), _stream(score))
    return keys


def stable_argsort(keys, key_bits=32):
    """Stable argsort of int32 bit patterns read as unsigned numbers (LSD radix, ceil(key_bits / 8) passes)."""
    _check(keys, torch.int32, "keys")
    n = keys.numel()
    need = ctypes.c_size_t()
    _ffi.call("tfgk_argsort_workspace_bytes", n, ctypes.byref(need))
    ws = torch.empty((max(need.value, 1),), dtype=torch.uint8, device=keys.device)
    perm = torch.empty((n,), dtype=torch.int32, device=keys.device)
    _ffi.call("tfgk_stable_argsort_u32", _p(keys), n, int(key_bits), _p(perm), _p(ws), need.value, _stream(keys))
    return perm


def _padding_code(padding):
    if padding == "head" or (not isinstance(padding, bool) and padding == SAMPLE_HEAD):
        return SAMPLE_HEAD
    return SAMPLE_PADDING if padding else SAMPLE_NO_PADDING


def neighbor_sample(csr, k=None, ratio=None, padding=False, seed=0, rng_stream=RNG_STREAM_SAMPLER):
    """Fan-out sampling over the rows of `csr` (tfgk_neighbor_sample_*).  Returns (row int32 [S], pos int32 [S],
    out_rowptr int64 [n_rows+1]): the row of every sampled edge and the CSR position it was drawn from.
    padding: False | True | SAMPLE_HEAD (deterministic: the first k / ceil(degree*ratio) entries of every row)."""
    dev = csr.rowptr.device
    kk = -1 if k is None else int(k)
    rr = -1.0 if ratio is None else float(ratio)
    padding = _padding_code(padding)
    need = ctypes.c_size_t()
    _ffi.call("tfgk_neighbor_sample_workspace_bytes", csr.n_rows, ctypes.byref(need))
    ws = torch.empty((max(need.value, 1),), dtype=torch.uint8, device=dev)
    out_rowptr = torch.empty((csr.n_rows + 1,), dtype=torch.int64, device=dev)
    total = ctypes.c_int64()
    _ffi.call("tfgk_neighbor_sample_count", _p(csr.rowptr), csr.n_rows, kk, rr, padding, _p(out_rowptr),
              ctypes.byref(total), _p(ws), need.value, _stream(out_rowptr))
    S = total.value
    out_row = torch.empty((S,), dtype=torch.int32, device=dev)
    out_pos = torch.empty((S,), dtype=torch.int32, device=dev)
    if S:
        _ffi.call("tfgk_neighbor_sample_fill", _p(csr.rowptr), csr.n_rows, kk, rr, padding, int(seed),
                  int(rng_stream), _p(out_rowptr), _p(out_row), _p(out_pos), _stream(out_rowptr))
    return out_row, out_pos, out_rowptr


def neighbor_sample_rows(rowptr, rows, k=None, ratio=None, padding=False, seed=0, rng_stream=RNG_STREAM_SAMPLER,
                         weighted=None):
    """K13: fan-out sampling of the listed rows of a CSR (tfgk_neighbor_sample_rows_*).  rowptr int64 [n_rows+1] is read in
    place; rows int32 [R] are global row ids (repeats allowed).  Returns (list position of each sampled edge's row int32 [S],
    CSR position int32 [S], out_rowptr int64 [R+1]); row t's positions are the ones neighbor_sample draws for row rows[t].
    weighted = (pos_deg int32 [n_rows], w_csr float32): an integer k draws by the weighted rule (the _weighted entries);
    k None takes every entry, as without weights."""
    _check(rowptr, torch.int64, "rowptr")
    _check(rows, torch.int32, "rows")
    dev = rowptr.device
    n_rows, R = rowptr.numel() - 1, rows.numel()
    kk = -1 if k is None else int(k)
    rr = -1.0 if ratio is None else float(ratio)
    padding = _padding_code(padding)
    if weighted is not None and k is not None:
        pos_deg, w_csr = weighted
        _check(pos_deg, torch.int32, "pos_deg")
        _check(w_csr, torch.float32, "w_csr")
        if ratio is not None or padding == SAMPLE_HEAD or kk < 0:
            raise ValueError("neighbor_sample_rows: the weighted rule takes a fan-out k >= 0, no ratio and no head rule")
    need = ctypes.c_size_t()
    _ffi.call("tfgk_neighbor_sample_workspace_bytes", R, ctypes.byref(need))
    ws = torch.empty((max(need.value, 1),), dtype=torch.uint8, device=dev)
    out_rowptr = torch.empty((R + 1,), dtype=torch.int64, device=dev)
    total = ctypes.c_int64()
    if weighted is not None and k is not None:
        _ffi.call("tfgk_neighbor_sample_rows_count_weighted", _p(rowptr), n_rows, _p(rows), R, kk, padding, _p(pos_deg),
                  _p(w_csr), _p(out_rowptr), ctypes.byref(total), _p(ws), need.value, _stream(rowptr))
    else:
        _ffi.call("tfgk_neighbor_sample_rows_count", _p(rowptr), n_rows, _p(rows), R, kk, rr, padding, _p(out_rowptr),
                  ctypes.byref(total), _p(ws), need.value, _stream(rowptr))
    S = total.value
    out_row = torch.empty((S,), dtype=torch.int32, device=dev)
    out_pos = torch.empty((S,), dtype=torch.int32, device=dev)
    if S and weighted is not None and k is not None:
        _ffi.call("tfgk_neighbor_sample_rows_fill_weighted", _p(rowptr), n_rows, _p(rows), R, kk, padding, _p(pos_deg),
                  _p(w_csr), int(seed), int(rng_stream), _p(out_rowptr), _p(out_row), _p(out_pos), _stream(rowptr))
    elif S:
        _ffi.call("tfgk_neighbor_sample_rows_fill", _p(rowptr), n_rows, _p(rows), R, kk, rr, padding, int(seed),
                  int(rng_stream), _p(out_rowptr), _p(out_row), _p(out_pos), _stream(rowptr))
    return out_row, out_pos, out_rowptr


def csr_positive_degree(rowptr, w, pos_deg, n_invalid, w_base=0):
    """tfgk_csr_positive_degree_f32: pos_deg int32 [n] = the entries of weight > 0 of the n rows of rowptr int64 [n + 1],
    whose weights are w[p - w_base] (float32, device); adds the number of negative, NaN and infinite weights to n_invalid
    (int32 [1], device).  Asynchronous."""
    _check(rowptr, torch.int64, "rowptr")
    _check(w, torch.float32, "w")
    _check(pos_deg, torch.int32, "pos_deg")
    _check(n_invalid, torch.int32, "n_invalid")
    n = rowptr.numel() - 1
    if pos_deg.numel() != n:
        raise ValueError("csr_positive_degree: {} outputs for {} rows".format(pos_deg.numel(), n))
    _ffi.call("tfgk_csr_positive_degree_f32", _p(rowptr), n, _p(w), int(w_base), _p(pos_deg), _p(n_invalid),
              _stream(rowptr))


def _relabel_workspace(n, device):
    need = ctypes.c_size_t()
    _ffi.call("tfgk_relabel_workspace_bytes", n, ctypes.byref(need))
    return torch.empty((need.value,), dtype=torch.uint8, device=device), need.value


def reindex(nodes, ids, node_map):
    """Position of every id of `ids` in the list `nodes` (-1 when absent), through `node_map` (int32 [N], all -1 before
    and after).  Returns (positions int32 [n_ids], number of repeated entries in `nodes`)."""
    _check(nodes, torch.int32, "nodes")
    _check(ids, torch.int32, "ids")
    _check(node_map, torch.int32, "node_map")
    out = torch.empty((ids.numel(),), dtype=torch.int32, device=ids.device)
    ws, nbytes = _relabel_workspace(0, ids.device)
    n_dup = ctypes.c_int32()
    _ffi.call("tfgk_reindex_i32", _p(nodes), nodes.numel(), _p(ids), ids.numel(), node_map.numel(), _p(node_map), _p(out),
              ctypes.byref(n_dup), _p(ws), nbytes, _stream(ids))
    return out, n_dup.value


def frontier(nodes, n_nodes, cols, node_map):
    """Grow the node list nodes[:n_nodes] (int32, room for cols.numel() more) by the ids of `cols` it lacks, in
    first-occurrence order, and relabel `cols` into it.  Returns (local cols int32 [S], new ids, repeated list entries)."""
    _check(nodes, torch.int32, "nodes")
    _check(cols, torch.int32, "cols")
    _check(node_map, torch.int32, "node_map")
    S = cols.numel()
    if nodes.numel() < n_nodes + S:
        raise ValueError("frontier: the node buffer holds {} ids, {} needed".format(nodes.numel(), n_nodes + S))
    local = torch.empty((S,), dtype=torch.int32, device=cols.device)
    ws, nbytes = _relabel_workspace(S, cols.device)
    n_new, n_dup = ctypes.c_int32(), ctypes.c_int32()
    _ffi.call("tfgk_frontier_i32", _p(cols), S, node_map.numel(), _p(nodes), int(n_nodes), _p(node_map), _p(local),
              ctypes.byref(n_new), ctypes.byref(n_dup), _p(ws), nbytes, _stream(cols))
    return local, n_new.value, n_dup.value


def block_capacities(n_listed, k, limit):
    """(edges, listed rows after the hop) that a hop of fan-out k over at most n_listed rows can produce, with at most
    `limit` rows in any list, or (None, None) when that is not known in advance (k None: every neighbour) or the edges
    reach 2^31."""
    if k is None or n_listed * k >= (1 << 31) - 1:
        return None, None
    return n_listed * k, min(limit, n_listed * (1 + k))


def _block_workspace(cap_list, cap_edges, device, entry="tfgk_block_sample_workspace_bytes"):
    need = ctypes.c_size_t()
    _ffi.call(entry, cap_list, cap_edges, ctypes.byref(need))
    return torch.empty((need.value,), dtype=torch.uint8, device=device), need.value


def block_sample(rowptr, col, w_csr, seeds, fanouts, keys, node_map, padding=False, rng_stream=RNG_STREAM_SAMPLER,
                 pos_deg=None, labor=False):
    """The block sampler (tfgk_block_sample_*): the hops of neighbor_sample_rows + frontier for every listed row, with the
    sizes kept on the device.  A hop whose capacity block_capacities cannot bound reads its edge total back; otherwise
    the batch synchronises once, in tfgk_block_sample_end, which also leaves node_map clean.
    rowptr int64 [N + 1], col int32, w_csr float32: the CSR (one row per node id) and its weights; seeds int32 [n];
    fanouts: one k (or None) per hop, in hop order; keys: the hop keys.
    Returns (nodes, hop_sizes, hops, n_bad, n_dup): nodes int32 [hop_sizes[-1]]; hops[h] = (out_rowptr int64 [>= n_h + 1],
    list position of each edge's row, its local column, its global column (int32 [S_h]), its weight float32 [S_h]);
    n_bad / n_dup count seeds outside [0, N) and repeated seeds (the lists are then meaningless).
    pos_deg: int32 [N], the CSR's positive degrees (csr_positive_degree), or None.  Given, every integer fan-out draws by
    the weighted rule (tfgk_block_sample_*_weighted; pass rng_stream=RNG_STREAM_WEIGHTED) and fan-out None as without it.
    labor: every integer fan-out draws by the LABOR rule (tfgk_block_sample_*_labor; pass rng_stream=RNG_STREAM_LABOR,
    and the same key for every hop for layer dependency), fan-out None as without it; no padding, no pos_deg.  No
    capacity bounds a LABOR hop, so each one reads its edge total back, as a hop of fan-out None does.
    Every argument the entries would refuse is refused before the map is touched, and a failure between the first and
    the last entry (an allocation, a hop past 2^31 edges) resets the map before it propagates."""
    padding = _check_block_fanouts(fanouts, padding, pos_deg, labor)
    _check(col, torch.int32, "col")
    _check(w_csr, torch.float32, "w_csr")
    return _block_sample(rowptr, _p(col), _p(w_csr), seeds, fanouts, keys, node_map, padding, rng_stream, False,
                         pos_deg=pos_deg, labor=labor)


def block_sample_mapped(rowptr, col_ptr, w_ptr, seeds, fanouts, keys, node_map, padding=False,
                        rng_stream=RNG_STREAM_SAMPLER, pos_deg=None, labor=False):
    """block_sample over a CSR in host memory (tfgk_block_sample_fill_mapped): col_ptr and w_ptr are the device addresses
    of its page-locked int32 columns and float32 weights (w_ptr None: every weight 1.0), at int64 positions; rowptr stays
    on the device.  Same arguments otherwise, and the same outputs as block_sample over the same CSR."""
    padding = _check_block_fanouts(fanouts, padding, pos_deg, labor)
    return _block_sample(rowptr, ctypes.c_void_p(col_ptr), None if w_ptr is None else ctypes.c_void_p(w_ptr), seeds,
                         fanouts, keys, node_map, padding, rng_stream, True, pos_deg=pos_deg, labor=labor)


def _check_block_fanouts(fanouts, padding, pos_deg=None, labor=False):
    # the fan-out rules of check_sample_mode, here so that no entry refuses a hop once the map holds the seeds
    padding = _padding_code(padding)
    if any(k is not None and int(k) < 0 for k in fanouts):
        raise ValueError("block_sample: fan-outs must be >= 0 or None")
    if padding == SAMPLE_HEAD and any(k is None for k in fanouts):
        raise ValueError("block_sample: the head rule needs an integer fan-out for every hop")
    if labor:
        if padding:
            raise ValueError("block_sample: the LABOR rule draws without replacement and takes no padding")
        if pos_deg is not None:
            raise NotImplementedError("block_sample: weighted LABOR is not implemented")
    if pos_deg is not None:
        _check(pos_deg, torch.int32, "pos_deg")
        if padding == SAMPLE_HEAD:
            raise ValueError("block_sample: the head rule takes no weights")
    return padding


def link_block_sample(rowptr, col, w_csr, pairs, n_pos, fanouts, keys, node_map, exclude=None, padding=False,
                      rng_stream=RNG_STREAM_SAMPLER, pos_deg=None, labor=False):
    """block_sample seeded by the endpoints of node pairs (tfgk_block_sample_begin_pairs): pairs int32 [2, P] (contiguous
    rows), whose distinct endpoints, taken pair by pair (source, then destination) in first-occurrence order, are the
    seeds.  exclude: None, "self" (every CSR entry (u, v) of the first n_pos pairs leaves u's row, at every hop) or
    "reverse" (and every entry (v, u)); the exclusion lists take one more host synchronisation (their total).
    Returns (nodes, hop_sizes, hops, n_bad, local, excluded): block_sample's outputs, with n_bad counting endpoints outside
    [0, N); local int32 [2, P], the pairs relabelled to positions in nodes; excluded = (excl_off int64, n_excl): row
    t < n_excl of every list had excl_off[t + 1] - excl_off[t] entries excluded (None without exclusion).
    pos_deg, labor: as block_sample's; a LABOR row's candidates are its entries less the excluded ones."""
    padding = _check_block_fanouts(fanouts, padding, pos_deg, labor)
    _check(col, torch.int32, "col")
    _check(w_csr, torch.float32, "w_csr")
    return _block_sample(rowptr, _p(col), _p(w_csr), None, fanouts, keys, node_map, padding, rng_stream, False,
                         pairs=(pairs, int(n_pos), exclude), pos_deg=pos_deg, labor=labor)


def link_block_sample_mapped(rowptr, col_ptr, w_ptr, pairs, n_pos, fanouts, keys, node_map, exclude=None, padding=False,
                             rng_stream=RNG_STREAM_SAMPLER, pos_deg=None, labor=False):
    """link_block_sample over a CSR in host memory (block_sample_mapped's arguments); the exclusion lists read the
    targeted rows' columns over the host link."""
    padding = _check_block_fanouts(fanouts, padding, pos_deg, labor)
    return _block_sample(rowptr, ctypes.c_void_p(col_ptr), None if w_ptr is None else ctypes.c_void_p(w_ptr), None,
                         fanouts, keys, node_map, padding, rng_stream, True, pairs=(pairs, int(n_pos), exclude),
                         pos_deg=pos_deg, labor=labor)


def link_tail_negatives(src, q, num_nodes, seed, out_row, out_col, rng_stream=RNG_STREAM_LINK):
    """Tail-corrupted negatives (tfgk_link_tail_negatives_i32): pair b * q + j is (src[b], random_below64(seed,
    rng_stream, b * q + j, num_nodes)), written to out_row / out_col int32 [len(src) * q]."""
    _check(src, torch.int32, "src")
    _check(out_row, torch.int32, "out_row")
    _check(out_col, torch.int32, "out_col")
    n = src.numel() * int(q)
    if out_row.numel() != n or out_col.numel() != n:
        raise ValueError("link_tail_negatives: outputs of {} and {} entries for {} pairs".format(
            out_row.numel(), out_col.numel(), n))
    _ffi.call("tfgk_link_tail_negatives_i32", _p(src), src.numel(), int(q), int(num_nodes), int(seed), int(rng_stream),
              _p(out_row), _p(out_col), _stream(src))


def _exclusion_lists(rowptr, col, nodes, cap, local, pairs, n_pos, exclude, mapped):
    """(excl_off int64 [cap + 1], excl_pos): the CSR positions the first n_pos pairs exclude from the rows of the list's
    first cap entries (tfgk_block_exclusion_*).  The targets (local source, global destination) are sorted by two stable
    radix passes, destination first."""
    dev = rowptr.device
    ts, td = local[0, :n_pos], pairs[1, :n_pos]
    if exclude == "reverse":
        ts, td = torch.cat([ts, local[1, :n_pos]]), torch.cat([td, pairs[0, :n_pos]])
    ts, td = ts.contiguous(), td.contiguous()
    if ts.numel():
        order = stable_argsort(td)
        ts, td = gather_i32(ts, order), gather_i32(td, order)
        order = stable_argsort(ts)
        ts, td = gather_i32(ts, order), gather_i32(td, order)
    need = ctypes.c_size_t()
    _ffi.call("tfgk_block_exclusion_workspace_bytes", cap, ctypes.byref(need))
    ws = torch.empty((max(need.value, 1),), dtype=torch.uint8, device=dev)
    excl_off = torch.empty((cap + 1,), dtype=torch.int64, device=dev)
    total = ctypes.c_int64()
    n_rows = rowptr.numel() - 1
    _ffi.call("tfgk_block_exclusion_count", _p(rowptr), n_rows, col, _p(nodes), cap, _p(ts), _p(td), ts.numel(),
              _p(excl_off), ctypes.byref(total), _p(ws), need.value, _stream(rowptr))
    excl_pos = torch.empty((max(total.value, 1),), dtype=torch.int64 if mapped else torch.int32, device=dev)
    _ffi.call("tfgk_block_exclusion_fill_mapped" if mapped else "tfgk_block_exclusion_fill", _p(rowptr), n_rows, col,
              _p(nodes), cap, _p(td), _p(excl_off), _p(excl_pos), _p(ws), need.value, _stream(rowptr))
    return excl_off, excl_pos


def _block_sample(rowptr, col, w_csr, seeds, fanouts, keys, node_map, padding, rng_stream, mapped, pairs=None,
                  pos_deg=None, labor=False):
    """block_sample's hops; col and w_csr are the fill's pointer arguments, to host memory when `mapped`.  The batch
    begins from the seed list `seeds`, or with pairs = (pair tensor, n_pos, exclude) from link_block_sample's pairs.
    pos_deg (not None): integer fan-outs by the weighted rule; labor: by the LABOR rule, each read back as a None hop."""
    _check(rowptr, torch.int64, "rowptr")
    _check(node_map, torch.int32, "node_map")
    if pairs is None:
        _check(seeds, torch.int32, "seeds")
        n_begin = seeds.numel()
    else:
        pair_t, n_pos, exclude = pairs
        _check(pair_t, torch.int32, "pairs")
        if pair_t.dim() != 2 or pair_t.shape[0] != 2 or not 0 <= n_pos <= pair_t.shape[1]:
            raise ValueError("link_block_sample: pairs must be [2, P] with n_pos <= P (got {}, n_pos {})".format(
                tuple(pair_t.shape), n_pos))
        if exclude not in (None, "self", "reverse"):
            raise ValueError("link_block_sample: exclude must be None, 'self' or 'reverse' (got {!r})".format(exclude))
        n_begin = 2 * pair_t.shape[1]                 # hop 0's capacity: every endpoint
    dev = rowptr.device
    n_rows, N, L = rowptr.numel() - 1, node_map.numel(), len(fanouts)
    ks = [-1 if k is None else int(k) for k in fanouts]
    bounds = [None if labor else k for k in fanouts]      # a LABOR row keeps up to all its entries
    # a list holds each id once, plus the repeated or invalid seeds of a batch that will be refused (a pair list holds
    # its distinct valid endpoints only)
    limit = N + (n_begin if pairs is None else 0)
    cap_nodes = n_begin
    for k in bounds:
        cap_nodes = block_capacities(cap_nodes, k, limit)[1]
        if cap_nodes is None:
            cap_nodes = limit
            break
    nodes = torch.empty((max(cap_nodes, 1),), dtype=torch.int32, device=dev)
    state = torch.empty((4 + 2 * L,), dtype=torch.int32, device=dev)
    # the device route passes no entry, so that a replacement of _block_workspace with the plain signature still fits
    ws_entry = ("tfgk_block_sample_mapped_workspace_bytes",) if mapped else ()
    fill = "tfgk_block_sample_fill_mapped" if mapped else "tfgk_block_sample_fill"
    st = _stream(rowptr)
    local = excluded = None
    if pairs is None:
        _ffi.call("tfgk_block_sample_begin", _p(seeds), seeds.numel(), N, _p(nodes), _p(node_map), _p(state), L, st)
    try:
        excl_args = ()
        if pairs is not None:
            P = pair_t.shape[1]
            local = torch.empty((2, P), dtype=torch.int32, device=dev)
            need = ctypes.c_size_t()
            _ffi.call("tfgk_block_pairs_workspace_bytes", P, ctypes.byref(need))
            ws = torch.empty((max(need.value, 1),), dtype=torch.uint8, device=dev)
            _ffi.call("tfgk_block_sample_begin_pairs", _p(pair_t[0]), _p(pair_t[1]), P, N, _p(nodes), _p(node_map),
                      _p(state), L, _p(local), _p(ws), need.value, st)
        if pairs is not None and exclude is not None:
            excl_off, excl_pos = _exclusion_lists(rowptr, col, nodes, n_begin, local, pair_t, n_pos, exclude, mapped)
            excluded = (excl_off, n_begin)
            excl_args = (_p(excl_off), _p(excl_pos), n_begin)
            fill += "_excl"
        cap_list, hops = n_begin, []
        for h, k in enumerate(ks):
            cap_edges, cap_next = block_capacities(cap_list, bounds[h], limit)
            ws, nbytes = _block_workspace(cap_list, 0 if cap_edges is None else cap_edges, dev, *ws_entry)
            out_rowptr = torch.empty((cap_list + 1,), dtype=torch.int64, device=dev)
            weighted = pos_deg is not None and k >= 0
            by_labor = labor and k >= 0
            if by_labor:
                _ffi.call("tfgk_block_sample_count_labor" + ("_mapped_excl" if mapped else "_excl") * bool(excl_args),
                          _p(rowptr), n_rows, col, _p(nodes), _p(state), h, L, cap_list, k, int(keys[h]),
                          int(rng_stream), *excl_args, _p(out_rowptr), _p(ws), nbytes, st)
            elif weighted and excl_args:
                _ffi.call("tfgk_block_sample_count_weighted_mapped_excl" if mapped else
                          "tfgk_block_sample_count_weighted_excl", _p(rowptr), n_rows, _p(nodes), _p(state), h, L,
                          cap_list, k, padding, _p(pos_deg), w_csr, excl_args[0], excl_args[1], excl_args[2],
                          _p(out_rowptr), _p(ws), nbytes, st)
            elif weighted:
                _ffi.call("tfgk_block_sample_count_weighted", _p(rowptr), n_rows, _p(nodes), _p(state), h, L, cap_list, k,
                          padding, _p(pos_deg), w_csr, _p(out_rowptr), _p(ws), nbytes, st)
            elif excl_args:
                _ffi.call("tfgk_block_sample_count_excl", _p(rowptr), n_rows, _p(nodes), _p(state), h, L, cap_list, k,
                          padding, excl_args[0], excl_args[2], _p(out_rowptr), _p(ws), nbytes, st)
            else:
                _ffi.call("tfgk_block_sample_count", _p(rowptr), n_rows, _p(nodes), _p(state), h, L, cap_list, k,
                          padding, _p(out_rowptr), _p(ws), nbytes, st)
            if cap_edges is None:
                n_list, total = ctypes.c_int32(), ctypes.c_int64()
                _ffi.call("tfgk_block_sample_read_total", _p(state), h, _p(out_rowptr), cap_list, ctypes.byref(n_list),
                          ctypes.byref(total), st)
                cap_edges, cap_next = total.value, min(limit, n_list.value + total.value)
                ws, nbytes = _block_workspace(cap_list, cap_edges, dev, *ws_entry)
            out = [torch.empty((max(cap_edges, 1),), dtype=torch.int32, device=dev) for _ in range(3)]
            out_w = torch.empty((max(cap_edges, 1),), dtype=torch.float32, device=dev)
            if by_labor:
                _ffi.call(fill.replace("tfgk_block_sample_fill", "tfgk_block_sample_fill_labor"), _p(rowptr), n_rows, col,
                          w_csr, N, _p(nodes), _p(node_map), _p(state), h, L, cap_list, cap_edges, k, int(keys[h]),
                          int(rng_stream), _p(out_rowptr), _p(out[0]), _p(out[1]), _p(out[2]), _p(out_w), *excl_args,
                          _p(ws), nbytes, st)
            elif weighted:
                wfill = fill.replace("tfgk_block_sample_fill", "tfgk_block_sample_fill_weighted")
                _ffi.call(wfill, _p(rowptr), n_rows, col, w_csr, _p(pos_deg), N, _p(nodes), _p(node_map),
                          _p(state), h, L, cap_list, cap_edges, k, padding, int(keys[h]), int(rng_stream),
                          _p(out_rowptr), _p(out[0]), _p(out[1]), _p(out[2]), _p(out_w), *excl_args, _p(ws), nbytes, st)
            else:
                _ffi.call(fill, _p(rowptr), n_rows, col, w_csr, N, _p(nodes), _p(node_map),
                          _p(state), h, L, cap_list, cap_edges, k, padding, int(keys[h]), int(rng_stream),
                          _p(out_rowptr), _p(out[0]), _p(out[1]), _p(out[2]), _p(out_w), *excl_args, _p(ws), nbytes,
                          st)
            hops.append((out_rowptr, out[0], out[1], out[2], out_w))
            cap_list = cap_next
        host = (ctypes.c_int32 * (4 + 2 * L))()
        _ffi.call("tfgk_block_sample_end", _p(nodes), cap_nodes, N, _p(node_map), _p(state), L, host, st)
    except BaseException:
        node_map.fill_(-1)            # the map is shared by every call on this sampler: leave it clean
        raise
    sizes = [int(v) for v in host[3:4 + L]]
    edges = [int(v) for v in host[4 + L:4 + 2 * L]]
    hops = [(rp, row[:S], loc[:S], gcol[:S], w[:S]) for (rp, row, loc, gcol, w), S in zip(hops, edges)]
    if pairs is not None:
        return nodes[:sizes[-1]], sizes, hops, int(host[0]), local, excluded
    return nodes[:sizes[-1]], sizes, hops, int(host[0]), int(host[1])


def block_self_loops(rowptr, edge_index, n_dst):
    """A block's CSR with the self loop (r, r) appended to every row r < n_dst (tfgk_block_self_loops_i32): rowptr int64
    [>= n_dst + 1] and edge_index int32 [2, S] in CSR order.  Returns (rowptr int64 [n_dst + 1], edge_index int32
    [2, S + n_dst]), in CSR order; one launch, no synchronisation."""
    _check(rowptr, torch.int64, "rowptr")
    _check(edge_index, torch.int32, "edge_index")
    S, n_dst = edge_index.shape[1], int(n_dst)
    if rowptr.numel() < n_dst + 1:
        raise ValueError("block_self_loops: rowptr has {} entries for {} rows".format(rowptr.numel(), n_dst))
    out_rowptr = torch.empty((n_dst + 1,), dtype=torch.int64, device=rowptr.device)
    out = torch.empty((2, S + n_dst), dtype=torch.int32, device=rowptr.device)
    _ffi.call("tfgk_block_self_loops_i32", _p(rowptr), _p(edge_index[0]), _p(edge_index[1]), S, n_dst, _p(out_rowptr),
              _p(out[0]), _p(out[1]), _stream(rowptr))
    return out_rowptr, out


def row_block(rowptr, r0, r1, cols, node_map):
    """The block sampler's one-hop batch for the seeds r0, ..., r1 - 1 with fan-out None (tfgk_row_block_i32), from the
    range's columns: rowptr int64 [N + 1] of the graph's CSR on the device, cols int32 [S], the columns
    [rowptr[r0], rowptr[r1]) staged on the device, node_map the sampler's int32 [N] map (-1 before and after).
    Returns (nodes int32 [num_src], out_rowptr int64 [n + 1], out_row int32 [S], out_local int32 [S]) with n = r1 - r0.
    One host read-back when S > 0."""
    _check(rowptr, torch.int64, "rowptr")
    _check(cols, torch.int32, "cols")
    _check(node_map, torch.int32, "node_map")
    N, S, n = node_map.numel(), cols.numel(), int(r1) - int(r0)
    if rowptr.numel() != N + 1:
        raise ValueError("row_block: rowptr has {} entries for {} nodes".format(rowptr.numel(), N))
    if not 0 <= r0 <= r1 <= N:
        raise ValueError("row_block: rows [{}, {}) are not a range of [0, {})".format(r0, r1, N))
    dev = rowptr.device
    nodes = torch.empty((max(min(N, n + S), 1),), dtype=torch.int32, device=dev)
    out_rowptr = torch.empty((n + 1,), dtype=torch.int64, device=dev)
    out_row = torch.empty((S,), dtype=torch.int32, device=dev)
    out_local = torch.empty((S,), dtype=torch.int32, device=dev)
    ws, nbytes = _relabel_workspace(S, dev)
    num_src = ctypes.c_int32()
    try:
        _ffi.call("tfgk_row_block_i32", _p(rowptr), N, int(r0), int(r1), _p(cols), S, _p(nodes), _p(node_map),
                  _p(out_rowptr), _p(out_row), _p(out_local), ctypes.byref(num_src), _p(ws), nbytes, _stream(rowptr))
    except BaseException:
        node_map.fill_(-1)            # the map is shared by every call on the sampler: leave it clean
        raise
    return nodes[:num_src.value], out_rowptr, out_row, out_local


def copy_async(dst, src_address, nbytes):
    """Copy nbytes from the address src_address (device memory, or page-locked host memory) into the CUDA tensor dst on
    the current stream, asynchronously (tfgk_copy_async).  dst may also be a CPU tensor over page-locked memory, with a
    device tensor's address as src_address."""
    if not dst.is_contiguous() or dst.numel() * dst.element_size() < nbytes:
        raise ValueError("copy_async: the destination holds {} contiguous bytes, {} needed".format(
            dst.numel() * dst.element_size() if dst.is_contiguous() else 0, nbytes))
    st = torch.cuda.current_stream().cuda_stream
    _ffi.call("tfgk_copy_async", _p(dst) if nbytes else None, ctypes.c_void_p(src_address) if nbytes else None,
              int(nbytes), ctypes.c_void_p(st))


def block_gcn_values(rowptr, gcol, w, dst, g_rowptr, g_rowsum, norm, loop, deg_fill, fill, excluded=None):
    """GCN's normalised values on a sampled block (tfgk_block_gcn_values_f32): the block's rowptr int64 [>= n_dst + 1],
    global columns int32 [S] and weights float32 [S] (or None: ones), its output rows' global ids dst int32 [n_dst], and
    the full graph's rowptr int64 and sequential row sums float32, indexed by global id.  norm: GCN_NORM_*; loop:
    GCN_LOOP_*; deg_fill is added to every row sum, fill is the self loops' weight.  Returns float32 [S + n_dst] in
    block_self_loops' layout with a loop mode, else [S] in the block's order; one launch, no synchronisation.
    excluded: (excl_off int64, n_excl) of a link batch's block (tfgk_block_gcn_values_excl_f32): output row r < n_excl
    had excl_off[r + 1] - excl_off[r] of its full-graph entries excluded, which its scale leaves out."""
    _check(rowptr, torch.int64, "rowptr")
    _check(gcol, torch.int32, "gcol")
    _check(dst, torch.int32, "dst")
    _check(g_rowptr, torch.int64, "g_rowptr")
    _check(g_rowsum, torch.float32, "g_rowsum")
    if w is not None:
        _check(w, torch.float32, "w")
        if w.numel() != gcol.numel():
            raise ValueError("block_gcn_values: {} weights for {} edges".format(w.numel(), gcol.numel()))
    S, n_dst = gcol.numel(), dst.numel()
    if rowptr.numel() < n_dst + 1:
        raise ValueError("block_gcn_values: rowptr has {} entries for {} rows".format(rowptr.numel(), n_dst))
    out = torch.empty((S + (n_dst if loop != GCN_LOOP_NONE else 0),), dtype=torch.float32, device=rowptr.device)
    if excluded is None:
        _ffi.call("tfgk_block_gcn_values_f32", _p(rowptr), _p(gcol), _p(w), S, _p(dst), n_dst, _p(g_rowptr),
                  _p(g_rowsum), int(norm), int(loop), float(deg_fill), float(fill), _p(out), _stream(rowptr))
        return out
    excl_off, n_excl = excluded
    _check(excl_off, torch.int64, "excl_off")
    if excl_off.numel() < int(n_excl) + 1:
        raise ValueError("block_gcn_values: {} exclusion offsets for {} rows".format(excl_off.numel(), n_excl))
    _ffi.call("tfgk_block_gcn_values_excl_f32", _p(rowptr), _p(gcol), _p(w), S, _p(dst), n_dst, _p(g_rowptr),
              _p(g_rowsum), int(norm), int(loop), float(deg_fill), float(fill), _p(excl_off), int(n_excl), _p(out),
              _stream(rowptr))
    return out


# ---- link prediction: K6 edge scoring, negative sampling ----------------------------------------------------------

def edge_dot(h, row, col, out=None):
    """out[e] = <h[row_e], h[col_e]> in fp32 (K6, tfgk_edge_dot_f32); an id outside [0, N) gives NaN."""
    if not (h.is_cuda and h.dtype == torch.float32 and h.dim() == 2):
        raise TypeError("h must be a 2-D float32 CUDA tensor")
    _check(row, torch.int32, "row")
    _check(col, torch.int32, "col")
    E = row.numel()
    if col.numel() != E:
        raise ValueError("edge_dot: row and col differ in length")
    if out is None:
        out = torch.empty((E,), dtype=torch.float32, device=h.device)
    _ffi.call("tfgk_edge_dot_f32", _p(h), _row_major_2d(h, "h"), h.shape[0], _p(row), _p(col), E, h.shape[1], _p(out),
              _stream(h))
    return out


def neg_offsets(csr, mode):
    """(offsets int64 [N+1], C): candidates before each row of the implicit negative list (tfgk_neg_offsets)."""
    dev = csr.rowptr.device
    need = ctypes.c_size_t()
    _ffi.call("tfgk_neg_offsets_workspace_bytes", csr.n_rows, ctypes.byref(need))
    ws = torch.empty((max(need.value, 1),), dtype=torch.uint8, device=dev)
    offsets = torch.empty((csr.n_rows + 1,), dtype=torch.int64, device=dev)
    total = ctypes.c_int64()
    _ffi.call("tfgk_neg_offsets", _p(csr.rowptr), csr.n_rows, int(mode), _p(offsets), ctypes.byref(total), _p(ws),
              need.value, _stream(offsets))
    return offsets, total.value


def neg_draw(C, n, seed, round=0, index=None, out=None, device=None, rng_stream=RNG_STREAM_LINK):
    """k[s] = random_below64(seed, rng_stream, round << 32 | s, C) for s < n, or only for s in `index` (into `out`)."""
    if index is not None:
        _check(index, torch.int32, "index")
    k = out if out is not None else torch.empty((n,), dtype=torch.int64, device=device)
    count = n if index is None else index.numel()
    if count:
        _ffi.call("tfgk_neg_draw", int(C), _p(index), count, int(seed), int(rng_stream), int(round), _p(k), _stream(k))
    return k


def neg_dup_flags(k, order):
    """int32 flags of the later duplicates of k, given a stable argsort `order` of k."""
    _check(k, torch.int64, "k")
    _check(order, torch.int32, "order")
    flag = torch.empty((k.numel(),), dtype=torch.int32, device=k.device)
    _ffi.call("tfgk_neg_dup_flags", _p(k), _p(order), k.numel(), _p(flag), _stream(k))
    return flag


def neg_decode(csr, offsets, mode, k):
    """Candidate indices k (int64) -> int32 [2, S] node pairs of the implicit negative list (tfgk_neg_decode)."""
    _check(k, torch.int64, "k")
    S = k.numel()
    out = torch.empty((2, S), dtype=torch.int32, device=k.device)
    _ffi.call("tfgk_neg_decode", _p(csr.rowptr), _p(csr.col), _p(offsets), csr.n_rows, int(mode), _p(k), S, _p(out[0]),
              _p(out[1]), _stream(k))
    return out


def neg_sample_start(csr, start, seed, rng_stream=RNG_STREAM_LINK):
    """One uniform candidate per start node over a TFGK_NEG_START structure (tfgk_neg_sample_start); -1 where none."""
    _check(start, torch.int32, "start")
    out = torch.empty((start.numel(),), dtype=torch.int32, device=start.device)
    _ffi.call("tfgk_neg_sample_start", _p(csr.rowptr), _p(csr.col), csr.n_rows, _p(start), start.numel(), int(seed),
              int(rng_stream), _p(out), _stream(start))
    return out


def random_pairs(num_nodes, num_samples, seed, device, rng_stream=RNG_STREAM_LINK):
    """int32 [2, S] uniform node ids (np.random.randint(0, N, [2, S]) with the counter-based generator)."""
    out = torch.empty((2, num_samples), dtype=torch.int32, device=device)
    _ffi.call("tfgk_random_pairs_i32", int(num_nodes), int(num_samples), int(seed), int(rng_stream), _p(out), _stream(out))
    return out


# ---- K7: edge-weight gradients ----------------------------------------------------------------------------------

def sddmm_csr(csr, G, X, row_scale=None, alpha=1.0, edge_order=True, out=None):
    """out[e] = alpha * row_scale[r] * <G[r], X[col_e]> for every CSR slot of row r (K7, tfgk_sddmm_csr_f32): the gradient
    of K1's output with respect to its edge weights.  edge_order=True writes slot p to out[csr.perm[p]], the order of
    the edge list (or SparseMatrix values) the CSR was built from; False keeps CSR order.  G: [n_rows, D], X: [*, D]
    (column slices are fine); row_scale: float32 [n_rows] or None."""
    for t, n in ((G, "G"), (X, "X")):
        if not (t.is_cuda and t.dtype == torch.float32 and t.dim() == 2):
            raise TypeError("{} must be a 2-D float32 CUDA tensor".format(n))
    D = G.shape[1]
    if X.shape[1] != D or G.shape[0] != csr.n_rows:
        raise ValueError("sddmm_csr: G is {} and X is {} for a CSR of {} rows".format(tuple(G.shape), tuple(X.shape),
                                                                                  csr.n_rows))
    if row_scale is not None:
        _check(row_scale, torch.float32, "row_scale")
    if out is None:
        out = torch.empty((csr.nnz,), dtype=torch.float32, device=G.device)
    _check(out, torch.float32, "out")
    if csr.nnz:
        _ffi.call("tfgk_sddmm_csr_f32", _p(csr.rowptr), _p(csr.col), _p(csr.perm) if edge_order else None, csr.n_rows,
                  _p(G), _row_major_2d(G, "G"), _p(X), _row_major_2d(X, "X"), D, _p(row_scale), float(alpha), _p(out),
                  _stream(G))
    return out


# ---- K8: per-graph dense algebra of DiffPool / MinCutPool ----------------------------------------------------------

def _float_2d(t, name):
    if not (torch.is_tensor(t) and t.is_cuda and t.dtype == torch.float32 and t.dim() == 2):
        raise TypeError("{} must be a 2-D float32 CUDA tensor".format(name))
    return _row_major_2d(t, name)


def graph_tmm(S, Y, gptr, num_graphs, gnodes=None, out=None):
    """out[g*C + c] = sum_{n in graph g} S[n, c] * Y[n] (K8a, tfgk_graph_tmm_f32): the per-graph S_g^T Y_g in block
    layout [G*C, D].  gptr int64 [G+1] delimits the node-list positions of every graph, gnodes int32 [N] maps positions to
    node ids (None: positions are node ids, i.e. graph-major nodes).  S: [N, C], Y: [N, D]; column slices are fine."""
    lds, ldy = _float_2d(S, "S"), _float_2d(Y, "Y")
    N, C = S.shape
    D = Y.shape[1]
    G = int(num_graphs)
    if Y.shape[0] != N:
        raise ValueError("graph_tmm: S has {} rows and Y {}".format(N, Y.shape[0]))
    if C < 1:
        raise ValueError("graph_tmm: S needs at least one cluster column")
    _check(gptr, torch.int64, "gptr")
    if gptr.numel() != G + 1:
        raise ValueError("graph_tmm: gptr has {} entries for {} graphs".format(gptr.numel(), G))
    if gnodes is not None:
        _check(gnodes, torch.int32, "gnodes")
    if out is None:
        out = torch.empty((G * C, D), dtype=torch.float32, device=S.device)
    ldo = _float_2d(out, "out")
    need = ctypes.c_size_t()
    _ffi.call("tfgk_graph_tmm_workspace_bytes", G, N, C, D, ctypes.byref(need))
    ws = torch.empty((max(need.value, 1),), dtype=torch.uint8, device=S.device)
    _ffi.call("tfgk_graph_tmm_f32", _p(S), lds, _p(Y), ldy, N, C, D, _p(gptr), _p(gnodes), G, _p(out), ldo, _p(ws),
              need.value, _stream(S))
    return out


def graph_rmm(Y, B, node_graph, num_clusters, trans=False, beta=0.0, out=None):
    """Every row times its graph's [C, K] block of the block-layout matrix B [G*C, K] (K8b, tfgk_graph_rmm_f32):
    trans=False: out[n] = beta * out[n] + Y[n, :C] @ B_g          (out [N, K])
    trans=True : out[n] = beta * out[n] + Y[n, :K] @ B_g^T        (out [N, C])
    with g = node_graph[n] (int32 [N])."""
    ldy, ldb = _float_2d(Y, "Y"), _float_2d(B, "B")
    C = int(num_clusters)
    N = Y.shape[0]
    if C < 1 or B.shape[0] % C:
        raise ValueError("graph_rmm: B has {} rows, not a multiple of {} clusters".format(B.shape[0], C))
    G, K = B.shape[0] // C, B.shape[1]
    if Y.shape[1] != (K if trans else C):
        raise ValueError("graph_rmm: Y has {} columns, {} expected".format(Y.shape[1], K if trans else C))
    _check(node_graph, torch.int32, "node_graph")
    if node_graph.numel() != N:
        raise ValueError("graph_rmm: node_graph has {} entries for {} rows".format(node_graph.numel(), N))
    if out is None:
        if beta != 0.0:
            raise ValueError("graph_rmm: beta != 0 needs `out`")
        out = torch.empty((N, C if trans else K), dtype=torch.float32, device=Y.device)
    ldo = _float_2d(out, "out")
    _ffi.call("tfgk_graph_rmm_f32", _p(Y), ldy, _p(node_graph), N, _p(B), ldb, G, C, K, 1 if trans else 0, float(beta),
              _p(out), ldo, _stream(Y))
    return out


# ---- K9: padded row gather of lstm_graph_sage / convert_x_to_3d -------------------------------------------------------

def pad_rows(csr, X, K, src=None, step_major=False, slot_index=False, out=None):
    """out[r, j] = X[src[rowptr[r] + j]] for j < min(deg r, K), zeros up to K (K9, tfgk_pad_rows_f32): [R, K, D], or
    [K, R, D] with step_major.  src is csr.col (default: neighbour rows) or csr.perm (the data rows of a segment-id CSR).
    slot_index=True also returns, per CSR slot, its flat output row (r*K + j, or j*R + r step-major; -1 past K), which
    needs K * R < 2^31.  X: [NX, D], column slices are fine."""
    ldx = _float_2d(X, "X")
    R, K, D = csr.n_rows, int(K), X.shape[1]
    src = csr.col if src is None else src
    _check(src, torch.int32, "src")
    if slot_index and K * R >= 2 ** 31:
        raise ValueError("pad_rows: K * R = {} does not fit the int32 slot index".format(K * R))
    shape = (K, R, D) if step_major else (R, K, D)
    if out is None:
        out = torch.empty(shape, dtype=torch.float32, device=X.device)
    elif tuple(out.shape) != shape or not out.is_contiguous() or out.dtype != torch.float32:
        raise ValueError("pad_rows: out must be a contiguous float32 tensor of shape {}".format(shape))
    slot = torch.empty((csr.nnz,), dtype=torch.int32, device=X.device) if slot_index else None
    _ffi.call("tfgk_pad_rows_f32", _p(csr.rowptr), _p(src), R, K, PAD_STEP_MAJOR if step_major else PAD_ROW_MAJOR,
              _p(X), ldx, X.shape[0], D, _p(out), _p(slot), _stream(X))
    return (out, slot) if slot_index else out


def unpad_rows(csr, G, out=None):
    """Backward of pad_rows with src = csr.perm (row-major): out[perm[p]] = G[r, j] for j = p - rowptr[r] < K, else 0
    (tfgk_unpad_rows_f32).  G: dense [R, K, D]; out: [csr.nnz, D], every row written."""
    if not (torch.is_tensor(G) and G.is_cuda and G.dtype == torch.float32 and G.dim() == 3 and G.is_contiguous()):
        raise TypeError("G must be a contiguous 3-D float32 CUDA tensor")
    R, K, D = G.shape
    if R != csr.n_rows:
        raise ValueError("unpad_rows: G has {} groups, the CSR {} rows".format(R, csr.n_rows))
    n = csr.nnz
    if out is None:
        out = torch.empty((n, D), dtype=torch.float32, device=G.device)
    elif tuple(out.shape) != (n, D) or not out.is_contiguous() or out.dtype != torch.float32:
        raise ValueError("unpad_rows: out must be a contiguous float32 tensor of shape {}".format((n, D)))
    _ffi.call("tfgk_unpad_rows_f32", _p(csr.rowptr), _p(csr.perm), R, K, _p(G), D, _p(out), n, _stream(G))
    return out


# ---- K10: CSR x CSR product -----------------------------------------------------------------------------------------

SPGEMM_BUDGET = 1 << 24    # products expanded per launch; the big rows among them need 24 bytes of workspace each


def _spgemm_chunks(prod_ptr, budget):
    """Row ranges [r0, r1) whose products fit `budget` (a row with more products is a range on its own)."""
    M = len(prod_ptr) - 1
    chunks, r0 = [], 0
    while r0 < M:
        r1 = int(np.searchsorted(prod_ptr, prod_ptr[r0] + budget, side="right")) - 1
        r1 = min(max(r1, r0 + 1), M)
        chunks.append((r0, r1))
        r0 = r1
    return chunks


def spgemm(a_rowptr, a_col, a_val, b_rowptr, b_col, b_val, n_cols, budget=SPGEMM_BUDGET):
    """C = A B for two CSR matrices (K10, tfgk_spgemm_*): A [M, K] and B [K, n_cols] as (rowptr int64, col int32,
    val float32).  Returns C's (rowptr int64 [M+1], col int32, val float32) with ascending columns per row; every entry is
    the fp32 sum of its products in Gustavson order, so the bits do not depend on `budget`, which bounds the products
    expanded per launch (and with it the workspace of the rows too large for shared memory)."""
    for t, n, dt in ((a_rowptr, "a_rowptr", torch.int64), (a_col, "a_col", torch.int32), (a_val, "a_val", torch.float32),
                     (b_rowptr, "b_rowptr", torch.int64), (b_col, "b_col", torch.int32), (b_val, "b_val", torch.float32)):
        _check(t, dt, n)
    if a_col.numel() != a_val.numel() or b_col.numel() != b_val.numel():
        raise ValueError("spgemm: column and value arrays differ in length")
    M, K = a_rowptr.numel() - 1, b_rowptr.numel() - 1
    dev, st = a_rowptr.device, _stream(a_rowptr)
    need = ctypes.c_size_t()
    _ffi.call("tfgk_spgemm_plan_workspace_bytes", M, ctypes.byref(need))
    ws = torch.empty((need.value,), dtype=torch.uint8, device=dev)
    prod_ptr = torch.empty((M + 1,), dtype=torch.int64, device=dev)
    big_ptr = torch.empty((M + 1,), dtype=torch.int64, device=dev)
    prod_host = np.empty((M + 1,), np.int64)
    big_host = np.empty((M + 1,), np.int64)
    _ffi.call("tfgk_spgemm_plan", _p(a_rowptr), _p(a_col), M, K, _p(b_rowptr), _p(b_col), int(n_cols), _p(prod_ptr),
              _p(big_ptr), prod_host.ctypes.data_as(ctypes.c_void_p), big_host.ctypes.data_as(ctypes.c_void_p), _p(ws),
              need.value, st)
    chunks = _spgemm_chunks(prod_host, max(int(budget), 0))
    big = [int(big_host[r1] - big_host[r0]) for r0, r1 in chunks]
    rows_ws = ctypes.c_size_t()
    _ffi.call("tfgk_spgemm_rows_workspace_bytes", max(big, default=0), ctypes.byref(rows_ws))
    rws = torch.empty((max(rows_ws.value, 1),), dtype=torch.uint8, device=dev)
    c_count = torch.empty((max(M, 1),), dtype=torch.int64, device=dev)
    for (r0, r1), nb in zip(chunks, big):
        _ffi.call("tfgk_spgemm_count", _p(a_rowptr), _p(a_col), _p(b_rowptr), _p(b_col), r0, r1, _p(prod_ptr),
                  _p(big_ptr), nb, _p(c_count), _p(rws), rows_ws.value, st)
    c_rowptr = torch.empty((M + 1,), dtype=torch.int64, device=dev)
    nnz = ctypes.c_int64()
    _ffi.call("tfgk_spgemm_rowptr", _p(c_count), M, _p(c_rowptr), ctypes.byref(nnz), _p(ws), need.value, st)
    c_col = torch.empty((nnz.value,), dtype=torch.int32, device=dev)
    c_val = torch.empty((nnz.value,), dtype=torch.float32, device=dev)
    if nnz.value:
        for (r0, r1), nb in zip(chunks, big):
            _ffi.call("tfgk_spgemm_fill_f32", _p(a_rowptr), _p(a_col), _p(a_val), _p(b_rowptr), _p(b_col), _p(b_val), r0,
                      r1, _p(prod_ptr), _p(big_ptr), nb, _p(c_rowptr), _p(c_col), _p(c_val), _p(rws), rows_ws.value, st)
    return c_rowptr, c_col, c_val


_SPGEMM_GRAD_MODES = {"left": SPGEMM_GRAD_LEFT, "right": SPGEMM_GRAD_RIGHT}


def spgemm_grad(mode, x_rowptr, x_col, y_rowptr, y_col, y_val, c_rowptr, c_col, grad_c, m, k, n, perm=None):
    """The gradient of K10's C = A B (A [m, k], B [k, n]) with respect to the values of one operand (K12,
    tfgk_spgemm_grad_*), given C's (rowptr, col) and grad_c = dL/dC in C's value order:
      mode "left":  X = A's CSR, Y = B's CSR (with values):    dA[(i, kk)] = sum_q B.val[q] * dC(i, B.col[q]) over B.row(kk)
      mode "right": X = B's CSR, Y = A^T's CSR (with values):  dB[(kk, j)] = sum_q At.val[q] * dC(At.col[q], j) over At.row(kk)
    Returns one float32 per entry of X, in X's CSR order, or at perm[p] (X's CSR slot -> COO position) when perm is given.
    A C entry that is missing contributes 0.  The bits depend only on the inputs (summation order in include/tfgk.h)."""
    if mode not in _SPGEMM_GRAD_MODES:
        raise ValueError("spgemm_grad: mode must be 'left' or 'right' (got {!r})".format(mode))
    for t, name, dt in ((x_rowptr, "x_rowptr", torch.int64), (x_col, "x_col", torch.int32), (y_rowptr, "y_rowptr", torch.int64),
                        (y_col, "y_col", torch.int32), (y_val, "y_val", torch.float32), (c_rowptr, "c_rowptr", torch.int64),
                        (c_col, "c_col", torch.int32), (grad_c, "grad_c", torch.float32)):
        _check(t, dt, name)
    if y_col.numel() != y_val.numel() or c_col.numel() != grad_c.numel():
        raise ValueError("spgemm_grad: column and value arrays differ in length")
    m, k, n = int(m), int(k), int(n)
    x_rows = m if mode == "left" else k
    for t, rows, name in ((x_rowptr, x_rows, "x_rowptr"), (y_rowptr, k, "y_rowptr"), (c_rowptr, m, "c_rowptr")):
        if t.numel() != rows + 1:
            raise ValueError("spgemm_grad: {} has {} entries, {} expected".format(name, t.numel(), rows + 1))
    nnz_x = x_col.numel()
    if perm is not None:
        _check(perm, torch.int32, "perm")
        if perm.numel() != nnz_x:
            raise ValueError("spgemm_grad: perm has {} entries for {} entries of X".format(perm.numel(), nnz_x))
    code = _SPGEMM_GRAD_MODES[mode]
    dev, st = x_rowptr.device, _stream(x_rowptr)
    need = ctypes.c_size_t()
    _ffi.call("tfgk_spgemm_grad_workspace_bytes", nnz_x, ctypes.byref(need))
    ws = torch.empty((need.value,), dtype=torch.uint8, device=dev)
    slice_ptr = torch.empty((nnz_x + 1,), dtype=torch.int64, device=dev)
    n_slices = ctypes.c_int64()
    _ffi.call("tfgk_spgemm_grad_plan", code, _p(x_rowptr), _p(x_col), nnz_x, _p(y_rowptr), _p(y_col), m, k, n,
              _p(slice_ptr), ctypes.byref(n_slices), _p(ws), need.value, st)
    partial = torch.empty((max(n_slices.value, 1),), dtype=torch.float32, device=dev)
    out = torch.empty((nnz_x,), dtype=torch.float32, device=dev)
    _ffi.call("tfgk_spgemm_grad_f32", code, _p(x_rowptr), _p(x_col), _p(perm), nnz_x, _p(y_rowptr), _p(y_col), _p(y_val),
              m, k, n, _p(c_rowptr), _p(c_col), _p(grad_c), _p(slice_ptr), n_slices.value, _p(partial), _p(out), st)
    return out


# ---- K4 ----------------------------------------------------------------------------------------------------------

# Largest K that tfgk_gemm_proj_f32 (the tensor-core kernel) accepts: W (hi | lo, 1024 bytes per K rounded up to 8) has to
# fit in shared memory next to at least two A stages.  Larger K goes to the exact-fp32 SIMT kernel.
GEMM_PROJ_MAX_K = 184

def gemm(a, b, bias=None, act=ACT_NONE, trans_a=False, trans_b=False, beta=0.0, out=None):
    """act(op(a) @ op(b) + bias + beta*out) in fp32."""
    for t, n in ((a, "a"), (b, "b")):
        if not (t.is_cuda and t.dtype == torch.float32 and t.dim() == 2):
            raise TypeError("{} must be a 2-D float32 CUDA tensor".format(n))
    M = a.shape[1] if trans_a else a.shape[0]
    Ka = a.shape[0] if trans_a else a.shape[1]
    Kb = b.shape[1] if trans_b else b.shape[0]
    N = b.shape[0] if trans_b else b.shape[1]
    if Ka != Kb:
        raise ValueError("gemm: inner dimensions differ ({} vs {})".format(Ka, Kb))
    if out is None:
        if beta != 0.0:
            raise ValueError("gemm: beta != 0 needs `out`")
        out = torch.empty((M, N), dtype=torch.float32, device=a.device)
    if bias is not None:
        _check(bias, torch.float32, "bias")
    need = ctypes.c_size_t()
    _ffi.call("tfgk_gemm_workspace_bytes", M, N, Ka, ctypes.byref(need))
    ws = torch.empty((need.value,), dtype=torch.uint8, device=a.device) if need.value else None
    _ffi.call("tfgk_gemm_f32", _p(a), _row_major_2d(a, "a"), int(trans_a), _p(b), _row_major_2d(b, "b"), int(trans_b),
              _p(bias), act, float(beta), M, N, Ka, _p(out), _row_major_2d(out, "out"), _p(ws), need.value, _stream(a))
    return out


def gemm_proj(a, blocks, a_parts=None, part_rows=0, first_part=0, max_ctas=0, num_rows=None):
    """Several projections of the same rows in ONE launch (tfgk_gemm_proj_f32): `blocks` is a list of
    (weight [K, n<=128], bias or None, act code, out [M, n] view); returns the list of outputs.  An `out` may be bfloat16
    (tfgk_gemm_proj_mixed, single-part input): it receives the fp32 result rounded to nearest even.
    With `a_parts` (device pointers of the row blocks of A, `part_rows` rows each, e.g. the other ranks' copies of x
    mapped through peer memory) the rows are pulled from where they live; `a` then only supplies lda / K / the stream.
    Shapes the tensor-core kernel does not take fall back to one tfgk_gemm_f32 per block (single-part input only)."""
    if not (a.is_cuda and a.dtype == torch.float32 and a.dim() == 2):
        raise TypeError("a must be a 2-D float32 CUDA tensor")
    lda = _row_major_2d(a, "a")
    M = int(a.shape[0] if num_rows is None else num_rows)
    K = a.shape[1]
    fields = []
    outs = []
    for i, blk in enumerate(blocks):
        w, bias, act, out = blk[:4]
        trans_b = bool(blk[4]) if len(blk) > 4 else False          # weight given as [n, K]: C = A @ w^T
        k_dim, n_dim = (1, 0) if trans_b else (0, 1)
        if not (w.is_cuda and w.dtype == torch.float32 and w.dim() == 2 and w.shape[k_dim] == K):
            raise TypeError("gemm_proj: weight {} must be a float32 CUDA tensor with inner dimension {}".format(i, K))
        n_cols = w.shape[n_dim]
        if out is None:
            out = torch.empty((M, n_cols), dtype=torch.float32, device=a.device)
        if isinstance(out, Fp8Table):
            if out.cols != n_cols or out.data.shape[0] < M or out.exps.shape[1] != 1:
                raise TypeError("gemm_proj: fp8 out {} must be a block of {} columns with one exponent column".format(
                    i, n_cols))
            if not (out.data.is_cuda and out.exps.is_cuda and out.data.device == a.device and out.exps.device == a.device):
                raise TypeError("gemm_proj: fp8 out {} must live on the device of a ({})".format(i, a.device))
        elif not (out.is_cuda and out.dtype in (torch.float32, torch.bfloat16)):
            raise TypeError("gemm_proj: out {} must be a float32 or bfloat16 CUDA tensor".format(i))
        if bias is not None:
            _check(bias, torch.float32, "bias")
        c = out.data if isinstance(out, Fp8Table) else out
        fields.append((w.data_ptr(), _row_major_2d(w, "weight"), n_cols, 1 if trans_b else 0,
                       None if bias is None else bias.data_ptr(), int(act), c.data_ptr(), _row_major_2d(c, "out")))
        outs.append(out)
    mixed = any(out.dtype == torch.bfloat16 for out in outs)
    fp8 = any(isinstance(out, Fp8Table) for out in outs)
    if fp8:
        if a_parts is not None:
            raise ValueError("gemm_proj: fp8 outputs need a single-part input")
        structs = (_ffi.ProjBlockFp8 * len(blocks))(*[
            _ffi.ProjBlockFp8(*(f + ((_ffi.DTYPE_FP8_E4M3, out.exps.data_ptr(), out.exps.stride(0))
                                     if isinstance(out, Fp8Table) else
                                     (_ffi.DTYPE_BF16 if out.dtype == torch.bfloat16 else _ffi.DTYPE_F32, None, 0))))
            for f, out in zip(fields, outs)])
    elif mixed:
        if a_parts is not None:
            raise ValueError("gemm_proj: bfloat16 outputs need a single-part input")
        structs = (_ffi.ProjBlockOut * len(blocks))(*[
            _ffi.ProjBlockOut(*(f + (_ffi.DTYPE_BF16 if out.dtype == torch.bfloat16 else _ffi.DTYPE_F32,)))
            for f, out in zip(fields, outs)])
    else:
        structs = (_ffi.ProjBlock * len(blocks))(*[_ffi.ProjBlock(*f) for f in fields])
    if a_parts is None:
        parts = (ctypes.c_void_p * 1)(a.data_ptr())
        n_parts = 1
    else:
        parts = (ctypes.c_void_p * len(a_parts))(*[int(q) for q in a_parts])
        n_parts = len(a_parts)
    try:
        _ffi.call("tfgk_gemm_proj_fp8" if fp8 else "tfgk_gemm_proj_mixed" if mixed else "tfgk_gemm_proj_f32", parts, n_parts, int(part_rows), lda, M, K,
                  structs, len(blocks), int(first_part), int(max_ctas), _stream(a))
    except _ffi.TfgkError as err:
        if err.code != _ffi.ERR_UNSUPPORTED or n_parts != 1:
            raise
        for blk, out in zip(blocks, outs):
            tb = bool(blk[4]) if len(blk) > 4 else False
            if isinstance(out, Fp8Table):       # the fp32 product, then quantised as the epilogue would
                quantize_fp8(gemm(a[:M], blk[0], bias=blk[1], act=blk[2], trans_b=tb), out=out)
            elif out.dtype == torch.bfloat16:   # the fp32 product, then rounded to nearest even
                round_bf16(gemm(a[:M], blk[0], bias=blk[1], act=blk[2], trans_b=tb), out=out)
            else:
                gemm(a[:M], blk[0], bias=blk[1], act=blk[2], trans_b=tb, out=out)
    return outs


def round_bf16(src, out=None):
    """bfloat16 copy of a 2-D float32 CUDA tensor, rounded to nearest even (tfgk_round_bf16); `out` may be a view."""
    if not (src.is_cuda and src.dtype == torch.float32 and src.dim() == 2):
        raise TypeError("round_bf16: src must be a 2-D float32 CUDA tensor")
    if out is None:
        out = torch.empty(tuple(src.shape), dtype=torch.bfloat16, device=src.device)
    if not (out.is_cuda and out.dtype == torch.bfloat16 and tuple(out.shape) == tuple(src.shape)):
        raise TypeError("round_bf16: out must be a bfloat16 CUDA tensor of shape {}".format(tuple(src.shape)))
    _ffi.call("tfgk_round_bf16", _p(src), _row_major_2d(src, "src"), src.shape[0], src.shape[1], _p(out),
              _row_major_2d(out, "out"), _stream(src))
    return out


def message_dtype(value):
    """Storage type of the rows a layer gathers along edges: None / torch.float32 -> None (fp32, the default path),
    torch.bfloat16 / "bfloat16" -> torch.bfloat16; anything else raises ValueError."""
    if value is None or value is torch.float32 or value == "float32":
        return None
    if value is torch.bfloat16 or value == "bfloat16":
        return torch.bfloat16
    raise ValueError("message_dtype must be None, torch.float32 or torch.bfloat16 (got {!r})".format(value))


def conv_message_dtype(value):
    """message_dtype of GCN and GAT, which also take fp8 message rows: None / torch.float32 -> None, torch.bfloat16 /
    "bfloat16" -> torch.bfloat16, torch.float8_e4m3fn / "float8_e4m3fn" -> torch.float8_e4m3fn; anything else (e5m2
    included) raises ValueError.  The other convolutions validate with message_dtype(), which refuses fp8."""
    if value is torch.float8_e4m3fn or value == "float8_e4m3fn":
        return torch.float8_e4m3fn
    try:
        return message_dtype(value)
    except ValueError:
        raise ValueError("message_dtype must be None, torch.float32, torch.bfloat16 or torch.float8_e4m3fn (got {!r})".format(
            value)) from None


def colsum(x):
    """Column sums of a [N, D] float32 matrix (bias gradients), deterministic."""
    if not (x.is_cuda and x.dtype == torch.float32 and x.dim() == 2):
        raise TypeError("colsum: x must be a 2-D float32 CUDA tensor")
    ldx = _row_major_2d(x, "x")
    n, d = x.shape
    need = ctypes.c_size_t()
    _ffi.call("tfgk_colsum_workspace_bytes", n, d, ctypes.byref(need))
    ws = torch.empty((max(need.value, 4),), dtype=torch.uint8, device=x.device)
    out = torch.empty((d,), dtype=torch.float32, device=x.device)
    _ffi.call("tfgk_colsum_f32", _p(x), ldx, n, d, _p(out), _p(ws), need.value, _stream(x))
    return out


def l2_normalize(x, out=None):
    if out is None:
        out = torch.empty_like(x)
    _ffi.call("tfgk_l2_normalize_f32", _p(x), _row_major_2d(x, "x"), x.shape[0], x.shape[1], _p(out),
              _row_major_2d(out, "out"), _stream(x))
    return out


def device_info():
    sm, major, minor = ctypes.c_int(), ctypes.c_int(), ctypes.c_int()
    _ffi.call("tfgk_device_info", ctypes.byref(sm), ctypes.byref(major), ctypes.byref(minor))
    return {"sm_count": sm.value, "cc": (major.value, minor.value)}


def activation_code(activation):
    """Map an activation callable to a fused epilogue code; returns (code, leftover_callable)."""
    if activation is None:
        return ACT_NONE, None
    if activation in (torch.relu, torch.nn.functional.relu) or getattr(activation, "_tfgk_act", None) == "relu" \
            or isinstance(activation, torch.nn.ReLU):
        return ACT_RELU, None
    return ACT_NONE, activation


def relu(x):
    """Stand-in for tf.nn.relu in the reference's layer defaults (layers/conv/gat.py:15-16, graph_sage.py:13)."""
    return torch.relu(x)


relu._tfgk_act = "relu"
