# coding=utf-8
"""Layer-wise inference over every node of a graph (an extension of the reference API, as DGL's model.inference over a
full-neighbour loader and PyG's subgraph_loader): a trained model's output for all N nodes, one layer at a time, in
chunks of consecutive rows whose row blocks (sampler.row_block) fit a device budget, so that neither the graph nor an
[N, D] table need fit on the device."""
import numpy as np
import torch

from .. import ops
from .sampling import (HostFeatureTable, HostNeighborSampler, RandomNeighborSampler, LAYERWISE_FIXED_BYTES,
                       _host_acquire, _host_release, _page_array, _row_block, _row_ranges, layerwise_chunk_bytes)


def _adapt(layer, block):
    """The block as the layer takes it: self-looped for GAT, GCN-normalised (with the layer's own configuration, chosen
    by the layer) for GCN, as it is for GraphSAGE."""
    from .. import layers as L           # layers import this package
    if isinstance(layer, L.GAT):
        return block.with_self_loops()
    if isinstance(layer, L.GCN):
        return block.with_gcn_norm()
    return block


def _plan_layer(rp, device_bytes, edge_bytes, row_bytes, out_bytes):
    """(ranges, on_device): the layer's output stays on the device when it fits device_bytes next to the chunks' working
    sets; otherwise it goes to host memory and the chunks take the whole budget.  ValueError naming a row that does not
    fit either way."""
    budget = device_bytes - LAYERWISE_FIXED_BYTES
    if out_bytes <= budget:
        try:
            return _row_block_ranges(rp, _row_ranges(rp, budget - out_bytes, edge_bytes, row_bytes)), True
        except ValueError:
            pass
    return _row_block_ranges(rp, _row_ranges(rp, budget, edge_bytes, row_bytes)), False


def _row_block_ranges(rp, ranges):
    """_row_ranges' ranges hold at most 2^31 - 1 edges, a row block fewer: such a range loses its last row to a range
    of its own (a row alone has fewer, _row_ranges refuses the others)."""
    out = []
    for r0, r1 in ranges:
        if rp[r1] - rp[r0] >= (1 << 31) - 1:
            out += [(r0, r1 - 1), (r1 - 1, r1)]
        else:
            out.append((r0, r1))
    return out


def _run_layer(sampler, h, layer, ranges, rp, on_device, dev, side=None):
    """One layer over every row: returns the [N, D] output, a device tensor or, off the device, a float32 numpy array on
    pages of its own with its registration key (page-locked, so that the copies into it are asynchronous).  side: the
    stream of the staging and of the copies to host memory (default: a new stream; passing the current stream runs them
    in line with the compute, which tools/bench_layerwise.py uses to measure their overlap)."""
    N = rp.size - 1
    main = torch.cuda.current_stream(dev)
    side = torch.cuda.Stream(dev) if side is None else side
    out = key = None

    def stage(c):
        # the range's columns on the side stream; main waits for its event before the row block reads them
        r0, r1 = ranges[c]
        with torch.cuda.stream(side):
            cols, w = sampler._stage(int(rp[r0]), int(rp[r1]))
            ev = side.record_event()
        cols.record_stream(main)
        w.record_stream(main)
        return cols, w, ev

    try:
        nxt = stage(0) if ranges else None
        for c, (r0, r1) in enumerate(ranges):
            cols, w, ev = nxt
            if c + 1 < len(ranges):
                nxt = stage(c + 1)
            main.wait_event(ev)
            batch = _row_block(sampler, r0, r1, staged=(cols, w))
            del cols, w
            with torch.no_grad():
                y = layer([batch.source_rows(h), _adapt(layer, batch.blocks[0])], training=False).contiguous()
            if out is None:
                D = y.shape[1]
                if on_device:
                    out = torch.empty((N, D), dtype=torch.float32, device=dev)
                else:
                    out = _page_array(N * D, np.float32).reshape(N, D)
                    key, _ = _host_acquire(torch.from_numpy(out))
            if on_device:
                out[r0:r1].copy_(y)
            else:
                # chunk c's rows go to host memory on the side stream while chunk c + 1 is computed
                side.wait_event(main.record_event())
                with torch.cuda.stream(side):
                    ops.copy_async(torch.from_numpy(out[r0:r1]), y.data_ptr(), y.numel() * 4)
                y.record_stream(side)
            del batch, y
        main.wait_stream(side)
    except BaseException:
        main.wait_stream(side)
        _host_release(key)
        raise
    return out, key


def layerwise_inference(sampler, x, layers, device_bytes=None):
    """layers[-1](... layers[0](x) ...) for every node of the sampler's graph, one layer at a time.

    sampler: a RandomNeighborSampler or a HostNeighborSampler.  x: a float32 [N, F] device tensor or a HostFeatureTable
    of any of its dtypes (at least N rows; a 16-bit table's rows reach the first layer widened exactly to float32).  layers: tfg.layers.GCN, GAT, MeanGraphSage, SumGraphSage, MeanPoolGraphSage or
    MaxPoolGraphSage, already built (trained); anything else raises TypeError before any device work.

    Each layer cuts the rows into consecutive ranges (_row_ranges) whose working set, layerwise_chunk_bytes per edge and
    per row, fits device_bytes (default: half of the device's free memory when the call starts).  For each range the
    sampler's row_block is adapted to the layer (with_self_loops() for GAT, with_gcn_norm() for GCN, as it is for
    GraphSAGE) and the layer runs as layer([batch.source_rows(h), block], training=False) under torch.no_grad(); its rows
    go to rows [r0, r1) of the layer's output.  So each output row is what the layer computes on the full graph.
    While a chunk is computed, the next range's columns are staged and the previous chunk's output rows are copied to
    host memory on a side stream, ordered by events.

    device_bytes bounds what the call allocates on the device at once: a layer's chunk working set, its output when that
    stays on the device, and the previous layer's output while it is this layer's input.  A layer's [N, D] output stays
    on the device when it fits next to one chunk's working set; otherwise it goes to page-locked host memory and the
    next layer reads it as a HostFeatureTable, closed when that layer is done.
    Synchronisation: at most three host read-backs per chunk, whatever its size (the row block's source-row count, the
    block's work plan and, for GAT and GCN, the looped block's work plan).  A row whose edges alone do not fit the
    budget raises ValueError naming it.

    :return: the last layer's output, float32 [N, D]: a CUDA tensor, or a CPU tensor when it went to host memory."""
    from .. import layers as L           # layers import this package
    if not isinstance(sampler, (RandomNeighborSampler, HostNeighborSampler)):
        raise TypeError("layerwise_inference takes a RandomNeighborSampler or a HostNeighborSampler (got {})".format(
            type(sampler).__name__))
    layers = list(layers)
    supported = (L.GCN, L.GAT, L.MeanGraphSage, L.SumGraphSage, L.MeanPoolGraphSage, L.MaxPoolGraphSage)
    for layer in layers:
        if not isinstance(layer, supported):
            layerwise_chunk_bytes(layer, 1)                 # the TypeError naming the supported layers
    if not layers:
        raise ValueError("layerwise_inference takes at least one layer")
    if isinstance(sampler, HostNeighborSampler):
        sampler._check_open()
        dev = sampler._device
    else:
        dev = sampler.edge_index.device
    rp = sampler._host_rowptr()
    N = rp.size - 1
    if isinstance(x, HostFeatureTable):
        x._check_open()
        rows, F = x.num_rows, x.num_features
    else:
        if not (torch.is_tensor(x) and x.is_cuda and x.dtype == torch.float32 and x.dim() == 2):
            raise TypeError("layerwise_inference takes x as a float32 [N, F] CUDA tensor or a HostFeatureTable")
        rows, F = x.shape
    if rows < N:
        raise ValueError("x has {} rows; the sampler's graph has {} nodes".format(rows, N))
    if device_bytes is None:
        device_bytes = torch.cuda.mem_get_info(dev)[0] // 2
    h, table, key = x, None, None
    try:
        for i, layer in enumerate(layers):
            eb, rb, D = layerwise_chunk_bytes(layer, F)
            held = 4 * N * F if h is not x and torch.is_tensor(h) else 0     # the previous layer's device output
            ranges, on_device = _plan_layer(rp, int(device_bytes) - held, eb, rb, 4 * N * D)
            out, key = _run_layer(sampler, h, layer, ranges, rp, on_device, dev)
            if table is not None:
                table.close()
                table = None
            if out is None:                                  # a graph without nodes
                out = torch.empty((0, D), dtype=torch.float32, device=dev)
            last = i + 1 == len(layers)
            if isinstance(out, np.ndarray):
                if last:
                    _host_release(key)                      # waits for the device's copies
                    key = None
                    return torch.from_numpy(out)
                h = table = HostFeatureTable(torch.from_numpy(out))     # one more user of the registration
                _host_release(key)
                key = None
            else:
                h = out
            F = D
        return h
    finally:
        if table is not None:
            table.close()
        _host_release(key)
