# coding=utf-8
"""K11 (max aggregation with tie counts and its transposed-CSR backward) on the device: CUDA-event times of K11a and K11b
at the products shape with D = 512 (the neighbour-MLP width of MaxPoolGraphSage(256)) against their byte floors as a
share of 3.35 TB/s; one MaxPoolGraphSage(256) forward + backward step at the products shape with its peak allocated
memory; and at 1 M nodes / 20 M edges, MaxPoolGraphSage(64) forward + backward through NeighborMax and through the
composition it replaces (TakeRows + SegmentReduce over [E, 256] messages), alternating, after checking that the output
and every gradient agree bit for bit.  Prints the card's name and power limit and one JSON line.

    python tools/bench_max_agg.py [--steps 5] [--warmup 2]
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

HBM = 3.35e12
DEV = "cuda"
N_PRODUCTS, E_PRODUCTS, F_PRODUCTS = 2449029, 123718280, 100


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


def random_edges(n, e, seed):
    gen = torch.Generator(device=DEV).manual_seed(seed)
    return torch.randint(0, n, (2, e), dtype=torch.int32, device=DEV, generator=gen)


def kernels(steps, warmup, D=512):
    n, e = N_PRODUCTS, E_PRODUCTS
    ei = random_edges(n, e, 0)
    csr, _ = _structure.csr_for_edge_index(ei, n)
    csr_t, _ = autograd._max_transposed(ei, n, None)
    gen = torch.Generator(device=DEV).manual_seed(1)
    h = torch.relu(torch.randn((n, D), device=DEV, generator=gen))
    g = torch.randn((n, D), device=DEV, generator=gen)
    res = {}
    state = {}

    def fwd():
        state["out"], state["cnt"] = ops.spmm_max(csr, None, h)

    t_a = event_ms(fwd, steps, warmup)
    k1 = ops.spmm(csr, None, h, reduce="max")
    assert torch.equal(k1.view(torch.int32), state["out"].view(torch.int32)), "K11a differs from K1 MAX"
    del k1
    floor_a = e * (4 * D + 4) + n * (8 * D + 8)
    res["k11a"] = dict(ms=t_a[0], min_ms=t_a[1], max_ms=t_a[2], floor_gb=floor_a / 1e9,
                       floor_share=floor_a / (t_a[0] * 1e-3) / HBM)
    t_b = event_ms(lambda: ops.spmm_max_bwd(csr_t, None, h, state["out"], state["cnt"], g), steps, warmup)
    floor_b = e * (8 * D + 4) + n * (8 * D + 8)
    res["k11b"] = dict(ms=t_b[0], min_ms=t_b[1], max_ms=t_b[2], floor_gb=floor_b / 1e9,
                       floor_share=floor_b / (t_b[0] * 1e-3) / HBM,
                       floor_share_with_pack_pass=(floor_b + 20 * D * n) / (t_b[0] * 1e-3) / HBM)
    res["ties_per_output"] = float(state["cnt"].float().mean())
    res["plan_hubs"] = 0 if csr.plan is None else csr.plan.n_hubs
    res["plan_hubs_transposed"] = 0 if csr_t.plan is None else csr_t.plan.n_hubs
    return res


def sage_step(n, e, f, units, seed):
    """(step closure, layer, x): MaxPoolGraphSage(units) forward + backward of sum(out * gout)."""
    ei = random_edges(n, e, seed)
    gen = torch.Generator(device=DEV).manual_seed(seed + 1)
    x = torch.randn((n, f), device=DEV, generator=gen).requires_grad_()
    w = torch.ones(e, device=DEV)
    layer = tfg.layers.MaxPoolGraphSage(units, activation=tfg.nn.relu, trainable=True, seed=seed)
    layer.build([(n, f)], device=x.device)
    layer.built = True
    gout = torch.randn((n, units), device=DEV, generator=gen)

    def step():
        x.grad = None
        for p in layer.parameters():
            p.grad = None
        out = layer([x, ei, w])
        (out * gout).sum().backward()
        return out
    return step, layer, x


def products_step(steps, warmup):
    step, _, _ = sage_step(N_PRODUCTS, E_PRODUCTS, F_PRODUCTS, 256, 3)
    step()
    torch.cuda.synchronize()
    torch.cuda.reset_peak_memory_stats()
    t = event_ms(step, steps, warmup)
    return dict(ms=t[0], min_ms=t[1], max_ms=t[2], peak_gb=torch.cuda.max_memory_allocated() / 1e9)


class _Composition(object):
    """Device tensors take TakeRows + SegmentReduce("max") inside the block (the route NeighborMax replaces)."""

    def __enter__(self):
        self.prev = autograd._is_device
        autograd._is_device = lambda t: False

    def __exit__(self, *exc):
        autograd._is_device = self.prev
        return False


def alternating(steps, warmup, n=1000000, e=20000000):
    step, layer, x = sage_step(n, e, F_PRODUCTS, 64, 5)

    def run(old):
        if old:
            with _Composition():
                out = step()
        else:
            out = step()
        return [out.detach().clone(), x.grad.clone()] + [p.grad.clone() for p in layer.parameters()]

    new, old = run(False), run(True)
    same = all(torch.equal(a.view(torch.int32), b.view(torch.int32)) for a, b in zip(new, old))
    del new, old
    times = {"k11": [], "composition": []}
    for i in range(warmup + steps):
        for name in ("k11", "composition"):
            a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            a.record()
            if name == "composition":
                with _Composition():
                    step()
            else:
                step()
            b.record()
            b.synchronize()
            if i >= warmup:
                times[name].append(a.elapsed_time(b))
    return dict(nodes=n, edges=e, bit_identical=bool(same),
                k11_ms=float(np.median(times["k11"])), composition_ms=float(np.median(times["composition"])))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=2)
    args = ap.parse_args()
    torch.cuda.set_device(0)
    res = {"card": card()}
    print("card (name, power limit):", res["card"], flush=True)
    res["kernels_products_D512"] = kernels(args.steps, args.warmup)
    print(json.dumps(res["kernels_products_D512"]), flush=True)
    _structure.clear()
    torch.cuda.empty_cache()
    res["products_max_pool_graph_sage_256"] = products_step(args.steps, args.warmup)
    print(json.dumps(res["products_max_pool_graph_sage_256"]), flush=True)
    _structure.clear()
    torch.cuda.empty_cache()
    res["alternating_1m_20m_max_pool_graph_sage_64"] = alternating(args.steps, args.warmup)
    print(json.dumps(res))


if __name__ == "__main__":
    main()
