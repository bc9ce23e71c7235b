# coding=utf-8
"""K9 (padded row gather) and LSTMGraphSage on the device: per-launch CUDA-event times of K9 (both layouts) and of the
K1 backward of the neighbour case against their byte floors as a share of 3.35 TB/s; LSTMGraphSage(256) forward +
backward, alternating between the layer (step-major K9 feeding cuDNN directly), the same layer on a row-major K9 with a
batch_first LSTM, and a torch composition (x_pad[neighbor_matrix], batch_first LSTM, autograd's scatter-add backward),
after checking that their outputs are equal; and a torch.profiler breakdown of the layer's step by kernel family.

Workloads (sampled with RandomNeighborSampler, as demo/demo_graph_sage.py does):
  demo   2 500 nodes of average degree 28 (a PPI graph), 50 features: layer 1 at k = 25, layer 2 (256 features) at k = 10
  large  250 000 nodes of average degree 20, 128 features, k = 10 (at 1 000 000 nodes cuDNN's LSTM forward alone asks
         for a 108.7 GiB allocation on the 80 GB card, so the layer cannot run there)

    python tools/bench_padded.py [--steps 10] [--warmup 3] [--workloads demo,large]
"""
import argparse
import json
import os
import subprocess
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import tf_geometric_b200 as tfg                       # noqa: E402
from tf_geometric_b200 import autograd, ops, _structure   # noqa: E402
from tf_geometric_b200.nn.conv.graph_sage import _lstm_sage   # noqa: E402

HBM = 3.35e12
DEV = "cuda"


def card():
    try:
        return subprocess.check_output(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                                       text=True, timeout=30).strip().splitlines()[0]
    except Exception as err:                            # the number is reported as unknown, never guessed
        return "unknown ({})".format(err)


def event_ms(fn, reps, warmup):
    for _ in range(warmup):
        fn()
    times = []
    for _ in range(reps):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        fn()
        b.record()
        b.synchronize()
        times.append(a.elapsed_time(b))
    return float(np.median(times)), float(np.min(times)), float(np.max(times))


def sampled_graph(n, avg_degree, seed):
    g = torch.Generator(device=DEV)
    g.manual_seed(seed)
    e = n * avg_degree
    ei = torch.randint(0, n, (2, e), device=DEV, generator=g, dtype=torch.int64).to(torch.int32)
    return tfg.utils.RandomNeighborSampler(ei)


def torch_neighbor_matrix(ei, n):
    """The reference's index matrix with torch ops (graph_sage.py:316-331): pad id n, stable by row."""
    row, col = ei[0].long(), ei[1].long()
    row, order = torch.sort(row, stable=True)
    col = col[order]
    degree = torch.bincount(row, minlength=n)
    K = int(degree.max())
    before = torch.cumsum(degree, 0) - degree
    j = torch.arange(row.numel(), device=DEV) - before[row]
    m = torch.full((n, K), n, dtype=torch.long, device=DEV)
    m[row, j] = col
    return m


class Variants(object):
    """The layer and two alternatives sharing its weights."""

    def __init__(self, f, seed):
        self.layer = tfg.layers.LSTMGraphSage(256, activation=tfg.nn.relu, trainable=True, seed=seed)
        self.layer.build([(None, f)], device=torch.device(DEV))
        self.layer.built = True
        self.bf = torch.nn.LSTM(f, 128, batch_first=True, device=DEV)
        self.bf.load_state_dict(self.layer.lstm.state_dict())

    def params(self):
        return list(self.layer.parameters()) + list(self.bf.parameters())

    def step_major(self, x, ei):
        return self.layer([x, ei], training=True)

    def row_major(self, x, ei):
        L = self.layer
        return _lstm_sage(x, ei, lambda p: autograd.run_lstm_fp32(self.bf, p).mean(dim=1), False, L.self_kernel,
                          L.neighbor_kernel, L.bias, L.activation, True, False)

    def torch_composition(self, x, m):
        L = self.layer
        xp = torch.cat([x, x.new_zeros((1, x.shape[1]))])
        h = autograd.run_lstm_fp32(self.bf, xp[m]).mean(dim=1)
        return torch.relu(torch.cat([x @ L.self_kernel, h @ L.neighbor_kernel], 1) + L.bias)


def kernel_family(name):
    if "tfgk" in name:
        for key, fam in (("pad_rows", "K9"), ("spmm", "K1"), ("gemm", "K4")):
            if key in name:
                return fam
        return "other tfgk"
    low = name.lower()
    if "rnn" in low or "lstm" in low or "xmma" in low or "cutlass" in low or "gemm" in low or "gemv" in low:
        return "cuDNN"
    if "reduce" in low:
        return "mean (reduce)"
    return "torch elementwise / copies"


def run_layer(name, f, k, n, avg_degree, steps, warmup, seed, graph_seed, x=None):
    sampler = sampled_graph(n, avg_degree, graph_seed)
    ei, _ = sampler.sample(k=k, seed=seed)
    ei = ei.contiguous()
    if x is None:
        x = torch.randn(n, f, device=DEV)
    x = x.detach().requires_grad_(True)
    csr, _ = _structure.csr_for_edge_index(ei, n)
    K = int(csr.degree_i64().max())
    nnz = csr.nnz
    res = {"workload": name, "nodes": n, "sampled_edges": nnz, "features": f, "K": K}

    # K9 alone, both layouts, and the K1 backward of the neighbour case
    floor = n * K * f * 4 + nnz * (4 * f + 4) + n * 8
    for tag, step in (("step_major", True), ("row_major", False)):
        t = event_ms(lambda: ops.pad_rows(csr, x.detach(), K, step_major=step), steps, warmup)
        res["k9_%s_ms" % tag] = t[0]
        res["k9_%s_hbm_share" % tag] = floor / (t[0] * 1e-3) / HBM
    res["k9_bytes"] = floor
    _, slot = ops.pad_rows(csr, x.detach(), K, step_major=True, slot_index=True)
    csr_t, emap = autograd._transposed_of_csr(csr, ei)
    slot_col = ops.gather_i32(slot, emap)
    g = torch.randn(K * n, f, device=DEV)
    k1_floor = nnz * (4 * f + 4) + n * (4 * f + 8)
    t = event_ms(lambda: ops.spmm(csr_t, None, g, reduce="sum", col=slot_col), steps, warmup)
    res.update(k1_bwd_ms=t[0], k1_bwd_bytes=k1_floor, k1_bwd_hbm_share=k1_floor / (t[0] * 1e-3) / HBM)
    del g

    # the three variants: equal outputs first, then alternating forward + backward steps
    v = Variants(f, seed)
    m = torch_neighbor_matrix(ei, n)
    with torch.no_grad():
        outs = [v.step_major(x, ei), v.row_major(x, ei), v.torch_composition(x, m)]
    ref = outs[2].double()
    scale = float(ref.abs().max())
    res["max_abs_diff_vs_torch"] = [float((o.double() - ref).abs().max()) for o in outs[:2]]
    res["max_abs_ref"] = scale
    assert all(d <= 1e-4 * scale + 1e-4 for d in res["max_abs_diff_vs_torch"]), res
    del outs, ref
    fns = {"layer_step_major": lambda: v.step_major(x, ei), "layer_row_major": lambda: v.row_major(x, ei),
           "torch_composition": lambda: v.torch_composition(x, m)}
    params = [x] + v.params()

    def fwd_bwd(fn):
        out = fn()
        out.backward(torch.ones_like(out))
        for p in params:
            p.grad = None
    times = {key: [] for key in fns}
    for key, fn in fns.items():
        for _ in range(warmup):
            fwd_bwd(fn)
    for _ in range(steps):
        for key, fn in fns.items():
            a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            a.record()
            fwd_bwd(fn)
            b.record()
            b.synchronize()
            times[key].append(a.elapsed_time(b))
    for key, ts in times.items():
        res["%s_fwd_bwd_ms" % key] = [float(np.median(ts)), float(np.min(ts)), float(np.max(ts))]

    # breakdown of the layer's step by kernel family, in a run of its own
    from torch.profiler import profile, ProfilerActivity
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        fwd_bwd(fns["layer_step_major"])
        torch.cuda.synchronize()
    fam = {}
    for evt in prof.key_averages():
        us = getattr(evt, "device_time_total", None)
        if us is None:
            us = getattr(evt, "cuda_time_total", 0)
        if us and evt.key and not evt.key.startswith("aten::") and not evt.key.startswith("cuda"):
            fam[kernel_family(evt.key)] = fam.get(kernel_family(evt.key), 0.0) + us / 1e3
    res["layer_step_major_breakdown_ms"] = {k_: round(v_, 3) for k_, v_ in sorted(fam.items())}
    out = v.step_major(x, ei).detach()
    del v, m, csr_t, slot_col, slot
    return res, out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--workloads", default="demo,large")
    args = ap.parse_args()
    torch.manual_seed(0)
    dev_card = card()
    for w in args.workloads.split(","):
        if w == "demo":
            r1, h = run_layer("demo layer 1", 50, 25, 2500, 28, args.steps, args.warmup, 1, 0)
            r2, _ = run_layer("demo layer 2", 256, 10, 2500, 28, args.steps, args.warmup, 2, 0, x=h)
            rows = [r1, r2]
        elif w == "large":
            rows = [run_layer("large", 128, 10, 250000, 20, args.steps, args.warmup, 3, 1)[0]]
        else:
            raise SystemExit("unknown workload " + w)
        for r in rows:
            r["card"] = dev_card
            print(json.dumps(r), flush=True)
        torch.cuda.empty_cache()


if __name__ == "__main__":
    main()
