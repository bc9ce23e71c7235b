#!/usr/bin/env python
# coding=utf-8
"""Layer-wise inference over every node at the products shape (2 449 029 nodes, 123.7 M edges, x of 100 features), for
MeanGraphSage(256) -> (256) -> (47), GCN(256) -> (256) -> (47) and GAT(128, 4 heads) -> (128, 4) -> (47):
  (a) the full-graph layers on the device;
  (b) layerwise_inference over RandomNeighborSampler with a device x, at the default budget and at a budget that cuts
      each layer into about 10 chunks;
  (c) over HostNeighborSampler + HostFeatureTable, with the outputs on the device and with them forced to host memory
      (a budget smaller than one layer's output);
  (d) the composition available without it: the same chunks through HostNeighborSampler.sample_blocks(arange, [None]).
Every arm's output is checked within 1e-5 (relative to its largest entry) of arm (a) before timing; the arms alternate.
Reports wall time per model and per layer (median over rounds), peak allocated memory, and for arm (c) a probe pass
over one layer's chunks timed with CUDA events: staging (GB/s, next to a plain bulk copy of the same bytes from pinned
memory), row-block build (edges/s), source-row gather (GB/s), layer compute and the output copy to host memory.  The
host-output arm's budget is below every layer's output, and the placement of each layer's output is reported.  Overlap:
the same layer loop runs with its staging and host copies on a side stream and on the compute stream, alternating with
the other arms; the time of page-locking a fresh [N, D] output is reported too.  The card's name and power limit.  --papers: the papers100M shape over the host sampler (arm (c), host outputs), or a message when
the host lacks the memory.
    python tools/bench_layerwise.py [--rounds 3] [--papers] [--nodes N --edges E]"""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np
import torch

sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), ".."))
import bench                                   # noqa: E402
import tf_geometric_b200 as tfg                # noqa: E402
from tf_geometric_b200 import ops              # noqa: E402
from tf_geometric_b200.utils import sampling   # noqa: E402
from tf_geometric_b200.utils.layerwise import _adapt, _plan_layer, _run_layer   # noqa: E402

CLASSES = 47
PAPERS_NODES, PAPERS_PAIRS, PAPERS_F = 111_059_956, 1_615_685_872, 128


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                       text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 and q.stdout.strip() else torch.cuda.get_device_name()


def available_host_bytes():
    with open("/proc/meminfo") as f:
        for line in f:
            if line.startswith("MemAvailable:"):
                return int(line.split()[1]) * 1024
    return 0


def models():
    L, relu = tfg.layers, tfg.nn.relu
    return {"MeanGraphSage": [L.MeanGraphSage(256, activation=relu, seed=1), L.MeanGraphSage(256, activation=relu, seed=2),
                              L.MeanGraphSage(CLASSES, activation=None, concat=False, seed=3)],
            "GCN": [L.GCN(256, activation=relu, seed=1), L.GCN(256, activation=relu, seed=2), L.GCN(CLASSES, seed=3)],
            "GAT": [L.GAT(128, num_heads=4, activation=relu, seed=1), L.GAT(128, num_heads=4, activation=relu, seed=2),
                    L.GAT(CLASSES, num_heads=1, seed=3)]}


def full_graph(layers, x, ei, adj):
    h = x
    with torch.no_grad():
        for layer in layers:
            if isinstance(layer, tfg.layers.GAT):
                h = layer([h, ei])
            elif isinstance(layer, tfg.layers.GCN):
                h = layer([h, adj], cache=adj_cache)
            else:
                h = layer([h, ei])
    return h


adj_cache = {}


def composed(sampler, x, layers, device_bytes):
    """(d): layerwise_inference's chunks through sample_blocks(arange(r0, r1), [None]), outputs on the device."""
    rp = sampler._host_rowptr()
    N = rp.size - 1
    h, F = x, x.num_features if isinstance(x, tfg.utils.HostFeatureTable) else x.shape[1]
    for layer in layers:
        eb, rb, D = sampling.layerwise_chunk_bytes(layer, F)
        ranges, _ = _plan_layer(rp, device_bytes, eb, rb, 4 * N * D)
        out = torch.empty((N, D), device="cuda")
        for r0, r1 in ranges:
            b = sampler.sample_blocks(torch.arange(r0, r1, dtype=torch.int32, device="cuda"), [None])
            with torch.no_grad():
                out[r0:r1] = layer([b.source_rows(h), _adapt(layer, b.blocks[0])], training=False)
        h, F = out, D
    return h


def timed(fn):
    torch.cuda.synchronize()
    torch.cuda.reset_peak_memory_stats()
    base = torch.cuda.memory_allocated()
    t0 = time.perf_counter()
    out = fn()
    torch.cuda.synchronize()
    return out, (time.perf_counter() - t0) * 1e3, (torch.cuda.max_memory_allocated() - base) / 1e9


def per_layer_ms(sampler, x, layers, device_bytes):
    """Wall time of each layer of layerwise_inference (each layer runs alone on the previous layer's output; a host
    output is wrapped in a HostFeatureTable that is closed once the next layer is done)."""
    times, h, table = [], x, None
    for layer in layers:
        inp = h if isinstance(h, tfg.utils.HostFeatureTable) or h.is_cuda else tfg.utils.HostFeatureTable(h)
        h, ms, _ = timed(lambda: tfg.utils.layerwise_inference(sampler, inp, [layer], device_bytes=device_bytes))
        if table is not None:
            table.close()
        table = inp if inp is not x and isinstance(inp, tfg.utils.HostFeatureTable) else None
        times.append(round(ms, 1))
    if table is not None:
        table.close()
    return times


def placements(sampler, x, layers, device_bytes):
    """Where layerwise_inference puts each layer's output at device_bytes, and its chunk count (its own rule)."""
    rp = sampler._host_rowptr()
    N = rp.size - 1
    F = x.num_features if isinstance(x, tfg.utils.HostFeatureTable) else x.shape[1]
    held, out = 0, []
    for layer in layers:
        eb, rb, D = sampling.layerwise_chunk_bytes(layer, F)
        ranges, on_device = _plan_layer(rp, device_bytes - held, eb, rb, 4 * N * D)
        out.append({"output": "device" if on_device else "host", "chunks": len(ranges)})
        held, F = (4 * N * D if on_device else 0), D
    return out


def layers_on_streams(sampler, x, layers, device_bytes, serial):
    """layerwise_inference's layer loop with its staging and host copies on a side stream, or (serial) on the current
    stream, in line with the compute: the two differ only in the stream, so their times show the overlap."""
    rp = sampler._host_rowptr()
    N = rp.size - 1
    F = x.num_features if isinstance(x, tfg.utils.HostFeatureTable) else x.shape[1]
    h, table, held = x, None, 0
    side = torch.cuda.current_stream() if serial else None
    for layer in layers:
        eb, rb, D = sampling.layerwise_chunk_bytes(layer, F)
        ranges, on_device = _plan_layer(rp, device_bytes - held, eb, rb, 4 * N * D)
        out, key = _run_layer(sampler, h, layer, ranges, rp, on_device, torch.device("cuda", 0), side=side)
        if table is not None:
            table.close()
            table = None
        if key is not None:
            h = table = tfg.utils.HostFeatureTable(torch.from_numpy(out))
            sampling._host_release(key)
        else:
            h = out
        held, F = (4 * N * D if on_device else 0), D
    if table is not None:                       # the last output: closing releases it after the device's copies
        h = table.x
        table.close()
    return h


def registration_ms(N, D):
    """A fresh [N, D] float32 array on pages of its own, page-locked and released, as each host output is."""
    t0 = time.perf_counter()
    a = sampling._page_array(N * D, np.float32)
    t1 = time.perf_counter()
    key, _ = sampling._host_acquire(torch.from_numpy(a))
    t2 = time.perf_counter()
    sampling._host_release(key)
    t3 = time.perf_counter()
    return {"allocate_ms": round((t1 - t0) * 1e3, 1), "register_ms": round((t2 - t1) * 1e3, 1),
            "unregister_ms": round((t3 - t2) * 1e3, 1)}


def probe(sampler, table, layer, device_bytes):
    """CUDA-event times of each step of arm (c)'s chunks for one layer, run serially on one stream."""
    rp = sampler._host_rowptr()
    N = rp.size - 1
    eb, rb, D = sampling.layerwise_chunk_bytes(layer, table.num_features)
    ranges, _ = _plan_layer(rp, device_bytes, eb, rb, 4 * N * D)
    host_out = torch.empty((N, D), pin_memory=True)
    tot = {k: 0.0 for k in ("stage", "plain_copy", "build", "gather", "compute", "out_copy")}
    nbytes = {"stage": 0, "gather": 0, "out": 0}
    edges = 0
    for r0, r1 in ranges:
        S = int(rp[r1] - rp[r0])
        stage_bytes = 4 * S * (1 if sampler._w is None else 2)       # an unweighted graph stages its columns only
        ev = [torch.cuda.Event(enable_timing=True) for _ in range(7)]
        pinned = torch.empty((stage_bytes // 4,), dtype=torch.int32, pin_memory=True)
        dst = torch.empty((stage_bytes // 4,), dtype=torch.int32, device="cuda")
        ev[0].record()
        cols, w = sampler._stage(int(rp[r0]), int(rp[r1]))
        ev[1].record()
        ops.copy_async(dst, pinned.data_ptr(), stage_bytes)
        ev[2].record()
        batch = sampling._row_block(sampler, r0, r1, staged=(cols, w))
        ev[3].record()
        src = batch.source_rows(table)
        ev[4].record()
        with torch.no_grad():
            y = layer([src, _adapt(layer, batch.blocks[0])], training=False).contiguous()
        ev[5].record()
        ops.copy_async(host_out[r0:r1], y.data_ptr(), y.numel() * 4)
        ev[6].record()
        torch.cuda.synchronize()
        for i, k in enumerate(tot):
            tot[k] += ev[i].elapsed_time(ev[i + 1])
        nbytes["stage"] += stage_bytes
        nbytes["gather"] += 4 * src.numel()
        nbytes["out"] += 4 * y.numel()
        edges += S
    return {"chunks": len(ranges), "edges": edges, "ms": {k: round(v, 2) for k, v in tot.items()},
            "stage_gb_per_s": round(nbytes["stage"] / tot["stage"] / 1e6, 1),
            "plain_copy_gb_per_s": round(nbytes["stage"] / tot["plain_copy"] / 1e6, 1),
            "build_medges_per_s": round(edges / tot["build"] / 1e3, 1),
            "gather_gb_per_s": round(nbytes["gather"] / tot["gather"] / 1e6, 1),
            "out_copy_gb_per_s": round(nbytes["out"] / tot["out_copy"] / 1e6, 1),
            "serial_sum_ms": round(sum(tot.values()) - tot["plain_copy"], 1)}


def products(args, res):
    dev = torch.device("cuda", 0)
    N = args.nodes or bench.PRODUCTS_NODES
    ei_dev = bench.make_graph_device(N, args.edges or bench.PRODUCTS_UNDIRECTED, 0, dev)
    ei = ei_dev.cpu().numpy()
    gen = torch.Generator(device="cpu").manual_seed(0)
    x_host = torch.randn((N, 100), generator=gen)
    x = x_host.cuda()
    res.update({"nodes": N, "edges": int(ei.shape[1]), "features": 100})
    dsamp = tfg.utils.RandomNeighborSampler(ei_dev)
    hsamp = tfg.utils.HostNeighborSampler(ei)
    table = tfg.utils.HostFeatureTable(x_host)
    adj = tfg.SparseMatrix(ei_dev, None, [N, N])
    free = torch.cuda.mem_get_info(dev)[0] // 2
    out = {}
    for name, layers in models().items():
        adj_cache.clear()
        want, _, _ = timed(lambda: full_graph(layers, x, ei_dev, adj))
        scale = float(want.abs().max())
        ten = max(sampling.layerwise_chunk_bytes(l, f)[0] * ei.shape[1] // 10 + 4 * N * 256 * 2
                  for l, f in zip(layers, (100, 256, 256))) + sampling.LAYERWISE_FIXED_BYTES
        host_out = sampling.LAYERWISE_FIXED_BYTES + 4 * N * CLASSES - 1     # below every output, [N, 47] the narrowest
        arms = {"a_full_graph": lambda: full_graph(layers, x, ei_dev, adj),
                "b_device_default": lambda: tfg.utils.layerwise_inference(dsamp, x, layers),
                "b_device_10_chunks": lambda: tfg.utils.layerwise_inference(dsamp, x, layers, device_bytes=ten),
                "c_host_device_out": lambda: tfg.utils.layerwise_inference(hsamp, table, layers, device_bytes=free),
                "c_host_host_out": lambda: tfg.utils.layerwise_inference(hsamp, table, layers, device_bytes=host_out),
                "c_host_host_out_side_stream": lambda: layers_on_streams(hsamp, table, layers, host_out, False),
                "c_host_host_out_one_stream": lambda: layers_on_streams(hsamp, table, layers, host_out, True),
                "d_sample_blocks": lambda: composed(hsamp, table, layers, free)}
        err = {}
        for arm, fn in arms.items():                   # checked (and warmed) before timing
            got, _, _ = timed(fn)
            err[arm] = float((got.cuda() - want).abs().max()) / scale
            assert err[arm] <= 1e-5, (name, arm, err[arm])
            del got
        ms = {arm: [] for arm in arms}
        peak = {}
        for _ in range(args.rounds):
            for arm, fn in arms.items():
                got, t, p = timed(fn)
                ms[arm].append(t)
                peak[arm] = max(peak.get(arm, 0.0), p)
                del got
        out[name] = {"ms": {a: round(float(np.median(v)), 1) for a, v in ms.items()},
                     "ms_all": {a: [round(t, 1) for t in v] for a, v in ms.items()},
                     "placement": {"c_host_device_out": placements(hsamp, table, layers, free),
                                   "c_host_host_out": placements(hsamp, table, layers, host_out)},
                     "peak_gb": {a: round(v, 2) for a, v in peak.items()}, "max_rel_err": err,
                     "per_layer_ms": {"b_device_default": per_layer_ms(dsamp, x, layers, None),
                                      "c_host_host_out": per_layer_ms(hsamp, table, layers, host_out)},
                     "probe_c_layer0": probe(hsamp, table, layers[0], host_out)}
        print(json.dumps({name: out[name]}), flush=True)
    res["models"] = out
    res["host_output_registration"] = {"N x 256": registration_ms(N, 256), "N x 47": registration_ms(N, CLASSES)}
    table.close()
    hsamp.close()


def papers(args, res):
    E = 2 * PAPERS_PAIRS
    need = 4 * 2 * E + 4 * E + 4 * PAPERS_NODES * PAPERS_F + 4 * PAPERS_NODES * 256
    res.update({"nodes": PAPERS_NODES, "edges": E, "features": PAPERS_F, "host_bytes_needed_gb": round(need / 1e9, 1)})
    avail = available_host_bytes()
    if avail < need + (16 << 30):
        res["skipped"] = "needs about {:.0f} GB of host memory plus 16 GiB of headroom; {:.0f} GB available".format(
            need / 1e9, avail / 1e9)
        return
    dev = torch.device("cuda", 0)
    ei = np.empty((2, E), np.int32)
    chunk = 1 << 27
    for c0 in range(0, PAPERS_PAIRS, chunk):
        n = min(chunk, PAPERS_PAIRS - c0)
        part = bench.make_graph_device(PAPERS_NODES, n, c0 // chunk, dev).cpu().numpy()
        ei[:, c0:c0 + n] = part[:, :n]
        ei[:, PAPERS_PAIRS + c0:PAPERS_PAIRS + c0 + n] = part[:, n:]
        del part
    s = tfg.utils.HostNeighborSampler(ei)
    del ei
    x = np.random.RandomState(0).randn(PAPERS_NODES, PAPERS_F).astype(np.float32)
    with tfg.utils.HostFeatureTable(x) as table:
        layers = models()["MeanGraphSage"]
        _, ms, peak = timed(lambda: tfg.utils.layerwise_inference(s, table, layers))
    res["MeanGraphSage_host"] = {"ms": round(ms, 1), "peak_gb": round(peak, 2)}
    s.close()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--papers", action="store_true")
    ap.add_argument("--nodes", type=int, default=None)
    ap.add_argument("--edges", type=int, default=None, help="undirected pairs (mirrored)")
    args = ap.parse_args()
    res = {"card": card(), "shape": "papers100M" if args.papers else "products"}
    (papers if args.papers else products)(args, res)
    print(json.dumps(res))


if __name__ == "__main__":
    main()
