# coding=utf-8
"""What K1 (tfgk_spmm_f32) and K3 (tfgk_gat_fused_f32) must compute on every kernel path, called through the raw ABI so
that no wrapper can route around a kernel.  The host models are in tests/k1k3_ref.py.

Dispatch, pinned by test_dispatch_table (kernel names recorded by torch.profiler):
  K1  D < 32 (float4 rows)                       spmm_kernel<4, ...>
      32 <= D <= 256, float4 rows                spmm_tma4_kernel<IS_MAX, 3, ...>
      256 < D <= 512, float4 rows                spmm_async_kernel<3|4, ...>
      D > 512                                    one launch per 512 columns, the last chunk by its own width
      D % 4 != 0 or a misaligned view            spmm_kernel<1, ...>, 128 columns per launch
      with a plan that has hub rows              the ring kernel + spmm_hub_fixup_kernel
  K3  heads concatenated, H and dqk / 4 powers of two, H <= 32, dqk == dv, H dqk <= 128:
        K | V adjacent in one buffer             gat_tma4_kernel<2, float>
        K and V apart                            gat_async_kernel<2, 3>
        with a plan that has hub rows            + gat_hub_fixup_kernel
      the same shapes up to A = 512, or return_attention                              gat_online_kernel
      dqk != dv with dv % 4 == 0                                                      gat_fast_kernel
      dv % 4 != 0, dqk / 4 not a power of two, averaged heads                         gat_generic_kernel
  Only the shape picks the kernel.  The plan is only read by the K1 rings (the whole width in one launch: float4 rows,
  32 <= D <= 512; k1k3_ref.k1_takes_plan) and by the two K3 rings.  The kernels never read plan->chunk, so a plan
  built by tfgk_plan_build with a threshold of 5 and a chunk of 3 is a valid plan with thousands of 1- to 3-edge slices.

K1 is compared bit for bit (assert equal) with k1k3_ref.k1_expected on every width, reducer and plan: the widths reach
every K1 kernel; rows are sequential fp32 sums in CSR order, hub rows sequential per slice and folded in slice order.

K3 is compared with float64 attention computed from the fp32 inputs.  Per output entry
    |got - ref| <= (2 delta + C (deg + n_slices + 8) 2^-24) S + 2^-23 |ref|,      S = sum_e alpha_e |v_e|,
with delta = (dqk + 2) 2^-24 max_e sum_j |q_j k_ej| / scale the fp32 score error (dqk - 1 roundings of the dot product
with or without FMA, one of the divide), and C = 10 (k1k3_ref.C_GAT), derived, with u = 2^-24 and expf within 2 ulp
(= 4u relative; the build has no fast-math):
  * a score error of at most delta moves every exp(s - m) and the denominator by a factor within e^(+-delta), so
    every alpha_e by e^(+-2 delta): 2 delta S to first order;
  * the online softmax (and the fix-up across slices) carries every partial sum through at most deg + n_slices later
    steps, each one fma rounding (u) and possibly a rescale by an expf (4u): 5u per step for the numerator and 5u for
    the denominator, whose relative error multiplies the whole output: C = 10 per step;
  * the constant 8 C u covers what every term pays once: its own expf (4u) and product (u), the denominator's expf (4u),
    the +1e-8 and the reciprocal (2u), and the argument roundings of the exponentials, whose sum along a term's chain
    telescopes to |s_e - m| u for the numerator and to at most ln(deg) u on average for the denominator: with the test
    inputs |s| <= 16 (asserted), so these stay below 2 * 32 u;
  * the final a * inv + bias is one rounding of the result: 2^-23 |ref|.  ReLU is 1-Lipschitz.
The two-pass and generic kernels round fewer times per edge (the exact max, a per-lane then butterfly denominator, one
divide and one multiply-add per edge); averaged heads add H + 1 roundings, under the constant for H <= 8.
The stats forward keeps (m, Z): |m_got - m| <= delta_h and |Z_got - Z| <= (2 delta_h + C (deg + n_slices + 8) u) Z.
tests/test_k1k3_ref_host.py shows the bound is tight enough: dropping the largest-alpha edge of a row, or giving one
edge its neighbour's V row, falls outside it on that row.
"""
import ctypes
import json
import os
import subprocess
import sys

import numpy as np
import pytest
import torch

import k1k3_ref as ref
from tf_geometric_b200 import _ffi, ops

pytestmark = pytest.mark.gpu

REDUCE = {"sum": ops.REDUCE_SUM, "mean": ops.REDUCE_MEAN, "max": ops.REDUCE_MAX}


def dev(a):
    return ops.as_device(a)


def stream():
    return ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)


def ptr(t):
    return None if t is None else ctypes.c_void_p(t.data_ptr())


def ld(t):
    return t.stride(0)


# ---- raw plan ------------------------------------------------------------------------------------------------------

class RawPlan(object):
    """A plan built by tfgk_plan_capacity + tfgk_plan_build with any (threshold, chunk, rows_per_task)."""

    def __init__(self, rowptr, thr, chunk, rpt, cap_tasks=None):
        rowptr = np.asarray(rowptr, np.int64)
        self.N, self.E = len(rowptr) - 1, int(rowptr[-1])
        self.thr, self.chunk, self.rpt = thr, chunk, rpt
        cap_t, cap_h = ctypes.c_int64(), ctypes.c_int64()
        _ffi.call("tfgk_plan_capacity", self.E, self.N, thr, chunk, rpt, ctypes.byref(cap_t), ctypes.byref(cap_h))
        self.capacity = (cap_t.value, cap_h.value)
        need = ctypes.c_size_t()
        _ffi.call("tfgk_plan_workspace_bytes", self.N, ctypes.byref(need))
        ws = torch.empty((max(need.value, 1),), dtype=torch.uint8, device="cuda")
        ct = self.capacity[0] if cap_tasks is None else cap_tasks
        self.t = {k: torch.empty((max(ct, 1),), dtype=torch.int32, device="cuda") for k in ("task_row", "task_nrows", "task_slot")}
        self.t.update({k: torch.empty((max(ct, 1),), dtype=torch.int64, device="cuda") for k in ("task_e0", "task_e1")})
        self.t.update({k: torch.empty((max(cap_h.value, 1),), dtype=torch.int32, device="cuda")
                       for k in ("hub_row", "hub_slot0", "hub_nslots")})
        self.rowptr = dev(rowptr)
        counts = (ctypes.c_int32 * 3)()
        _ffi.call("tfgk_plan_build", ptr(self.rowptr), self.N, thr, chunk, rpt, *[ptr(self.t[k]) for k in ref.PLAN_KEYS],
                  ct, cap_h.value, counts, ptr(ws), need.value, stream())
        torch.cuda.synchronize()
        self.n_tasks, self.n_hubs, self.n_slots = int(counts[0]), int(counts[1]), int(counts[2])
        self.host = {k: self.t[k].cpu().numpy()[:(self.n_tasks if k.startswith("task") else self.n_hubs)] for k in ref.PLAN_KEYS}
        self.host.update(n_tasks=self.n_tasks, n_hubs=self.n_hubs, n_slots=self.n_slots)
        self._scratch = None

    def struct(self, floats_per_slot, slots=None):
        """_ffi.PlanStruct with a scratch of `slots` (default n_slots) slots of floats_per_slot floats."""
        slots = self.n_slots if slots is None else slots
        self._scratch = torch.empty((max(slots * floats_per_slot, 1),), dtype=torch.float32, device="cuda")
        return _ffi.PlanStruct(self.n_tasks, self.n_hubs, self.n_slots, self.chunk,
                               *[self.t[k].data_ptr() for k in ref.PLAN_KEYS], self._scratch.data_ptr(),
                               slots * floats_per_slot * 4)


# ---- A. plan builder -----------------------------------------------------------------------------------------------

def _check_plan(rowptr, thr, chunk, rpt):
    p = RawPlan(rowptr, thr, chunk, rpt)
    assert p.capacity == ref.plan_capacity_model(int(rowptr[-1]), len(rowptr) - 1, thr, chunk, rpt)
    want = ref.plan_model(rowptr, thr, chunk, rpt)
    assert (p.n_tasks, p.n_hubs, p.n_slots) == (want["n_tasks"], want["n_hubs"], want["n_slots"])
    for k in ref.PLAN_KEYS:
        np.testing.assert_array_equal(p.host[k], want[k], err_msg=k)
    ref.check_plan_invariants(p.host, rowptr, thr, chunk, rpt, p.capacity)
    return p


@pytest.mark.parametrize("rpt", [1, 3, 32])
@pytest.mark.parametrize("case", sorted(ref.plan_degree_cases()))
def test_plan_builder_matches_the_definition(case, rpt):
    deg, thr, chunk = ref.plan_degree_cases()[case]
    _check_plan(np.concatenate([[0], np.cumsum(deg)]), thr, chunk, rpt)


@pytest.mark.parametrize("plan_name", [k for k, (_, p) in ref.K1_PLANS.items() if p is not None])
def test_plan_builder_on_the_contract_graphs(plan_name):
    rowptr, _ = ref.GRAPHS[ref.K1_PLANS[plan_name][0]]()
    _check_plan(rowptr, *ref.plan_params(plan_name, rowptr))


def test_plan_builder_refuses_a_short_capacity():
    """The counts are checked on the host before the fill kernel runs: one task short of the count is ERR_WORKSPACE."""
    rowptr, _ = ref.k1_main_graph()
    n_tasks = ref.plan_model(rowptr, 5, 3, 32)["n_tasks"]
    with pytest.raises(_ffi.TfgkError) as err:
        RawPlan(rowptr, 5, 3, 32, cap_tasks=n_tasks - 1)
    assert err.value.code == _ffi.ERR_WORKSPACE
    RawPlan(rowptr, 5, 3, 32, cap_tasks=n_tasks)


# ---- B. K1 ---------------------------------------------------------------------------------------------------------

K1_WIDTHS = (1, 3, 4, 28, 32, 36, 64, 124, 128, 132, 196, 256, 260, 384, 508, 512, 516, 1024)


def spmm_raw(rowptr, col, w, h, n_dst, reduce, out, plan_struct=None, alpha=1.0, addend=None, beta=0.0, bias=None,
             act=ops.ACT_NONE):
    _ffi.call("tfgk_spmm_f32", ptr(rowptr), ptr(col), ptr(w), ptr(h), ld(h), n_dst, h.shape[1], REDUCE[reduce],
              float(alpha), ptr(addend), 0 if addend is None else ld(addend), float(beta), ptr(bias), act, ptr(out), ld(out),
              None if plan_struct is None else ctypes.byref(plan_struct), stream())
    return out


def aligned4(*ts):
    return all(t is None or (t.data_ptr() % 16 == 0 and (t.dim() == 1 or t.shape[0] <= 1 or t.stride(0) % 4 == 0))
               for t in ts)


K1_REDUCERS = (("sum", True), ("sum", False), ("mean", True), ("max", True))
_GRAPH_CACHE = {}


def k1_graph(name):
    if name not in _GRAPH_CACHE:
        rowptr, col = ref.GRAPHS[name]()
        w = (np.random.RandomState(len(col)).rand(len(col)) + 0.1).astype(np.float32)
        _GRAPH_CACHE[name] = (rowptr, col, w, dev(rowptr), dev(col), dev(w))
    return _GRAPH_CACHE[name]


def _mismatch(got, want, what):
    got = got.cpu().numpy()
    bad = np.argwhere(~((got == want) | (np.isnan(got) & np.isnan(want))))
    return "{}: {} entries differ, first at {}: got {!r}, want {!r}".format(what, len(bad), tuple(bad[0]), got[tuple(bad[0])],
                                                                           want[tuple(bad[0])])


@pytest.mark.parametrize("plan_name", list(ref.K1_PLANS))
@pytest.mark.parametrize("D", K1_WIDTHS)
def test_k1_shape_dispatch_is_bit_exact(D, plan_name):
    graph, params = ref.K1_PLANS[plan_name]
    rowptr, col, w, rp_d, col_d, w_d = k1_graph(graph)
    n_dst = len(rowptr) - 1
    h = np.random.RandomState(D).randn(3001, D).astype(np.float32)
    h_d = dev(h)
    plan = RawPlan(rowptr, *ref.plan_params(plan_name, rowptr)) if params is not None else None
    sliced = plan is not None and ref.k1_takes_plan(D, D % 4 == 0)
    out = torch.empty((n_dst, D), dtype=torch.float32, device="cuda")
    for reduce, weighted in K1_REDUCERS:
        wts, wts_d = (w, w_d) if weighted else (None, None)
        want = ref.k1_expected(rowptr, col, wts, h, reduce, plan=plan.host if sliced else None)
        out.fill_(float("nan"))
        spmm_raw(rp_d, col_d, wts_d, h_d, n_dst, reduce, out, None if plan is None else plan.struct(D))
        torch.cuda.synchronize()
        assert torch.equal(out, dev(want)), _mismatch(out, want, "D={} {}{} plan={}".format(
            D, reduce, "" if weighted else " unweighted", plan_name))


LAYOUT_WIDTHS = (4, 32, 100, 128, 196, 256, 384, 512, 1024)


@pytest.mark.parametrize("layout", ["dense", "strided", "offset"])
@pytest.mark.parametrize("plan_name", ["none", "hub", "tiny5x3", "short"])
@pytest.mark.parametrize("reduce,relu", [("sum", True), ("mean", False), ("max", True)])
def test_k1_epilogue_and_views(reduce, relu, plan_name, layout):
    """alpha acc + beta addend, bias and ReLU; h, out and addend as strided views ("strided": 16-byte aligned, wider leading
    dimensions; "offset": every base one column in, which takes the scalar path without the plan); columns outside the
    output view stay untouched."""
    graph, params = ref.K1_PLANS[plan_name]
    rowptr, col, w, rp_d, col_d, w_d = k1_graph(graph)
    n_dst = len(rowptr) - 1
    plan = RawPlan(rowptr, *ref.plan_params(plan_name, rowptr)) if params is not None else None
    c0 = {"dense": 0, "strided": 4, "offset": 1}[layout]
    pad = 0 if layout == "dense" else 12
    for D in LAYOUT_WIDTHS:
        rs = np.random.RandomState(D + 1)
        hbuf = rs.randn(3001, D + pad).astype(np.float32)
        abuf = rs.randn(n_dst, D + pad + 4).astype(np.float32)
        bias = rs.randn(D).astype(np.float32)
        h_d = dev(hbuf)[:, c0:c0 + D]
        add_d = dev(abuf)[:, c0:c0 + D]
        obuf = torch.full((n_dst, D + pad + 8), 7.0, dtype=torch.float32, device="cuda")
        out = obuf[:, c0:c0 + D]
        sliced = plan is not None and ref.k1_takes_plan(D, D % 4 == 0 and aligned4(h_d, add_d, out))
        assert sliced == (plan is not None and layout != "offset" and 32 <= D <= 512)
        epi = dict(alpha=0.75, addend=abuf[:, c0:c0 + D], beta=-1.25, bias=bias, relu=relu)
        want = ref.k1_expected(rowptr, col, w, hbuf[:, c0:c0 + D], reduce, epilogue=epi, plan=plan.host if sliced else None)
        spmm_raw(rp_d, col_d, w_d, h_d, n_dst, reduce, out, None if plan is None else plan.struct(D), alpha=0.75,
                 addend=add_d, beta=-1.25, bias=dev(bias), act=ops.ACT_RELU if relu else ops.ACT_NONE)
        torch.cuda.synchronize()
        assert torch.equal(out, dev(want)), _mismatch(out, want, "D={} {} {} plan={}".format(D, reduce, layout, plan_name))
        rest = torch.cat([obuf[:, :c0], obuf[:, c0 + D:]], dim=1)
        assert bool((rest == 7.0).all()), "columns outside the output view were written"


@pytest.mark.parametrize("D", [32, 128, 384])
def test_k1_refuses_a_plan_scratch_one_slot_short(D):
    rowptr, col, w, rp_d, col_d, w_d = k1_graph("main")
    plan = RawPlan(rowptr, 5, 3, 32)
    out = torch.full((len(rowptr) - 1, D), 7.0, device="cuda")
    with pytest.raises(_ffi.TfgkError) as err:
        spmm_raw(rp_d, col_d, w_d, dev(np.ones((3001, D), np.float32)), len(rowptr) - 1, "sum", out,
                 plan.struct(D, slots=plan.n_slots - 1))
    assert err.value.code == _ffi.ERR_INVALID_ARGUMENT
    torch.cuda.synchronize()
    assert bool((out == 7.0).all())


# ---- C. K3 ---------------------------------------------------------------------------------------------------------

def gat_main_graph():
    """2001 rows, degrees 0 to 16, empty rows, a 3000-edge hub and a 2100-edge hub at the last row."""
    rs = np.random.RandomState(201)
    deg = rs.randint(0, 17, 2001)
    deg[:3] = 0
    deg[900:905] = 0
    deg[500] = 3000
    deg[-1] = 2100
    return ref.csr_from_degrees(deg, 2001, 202)


def gat_short_graph():
    """41 rows of 100 to 180 edges (the short-task plan), an empty row and a 2300-edge hub, from 2001 sources."""
    rs = np.random.RandomState(203)
    deg = rs.randint(100, 180, 41)
    deg[3] = 0
    deg[20] = 2300
    return ref.csr_from_degrees(deg, 2001, 204)


K3_PLANS = {"none": ("main", None), "hub": ("main", (ref.HUB_THRESHOLD, ref.HUB_CHUNK, 32)),
            "tiny5x3": ("main", (5, 3, 32)), "short": ("short", "short")}
K3_GRAPHS = {"main": gat_main_graph, "short": gat_short_graph}
FUSED_SHAPES = [(H, dqk) for H in (1, 2, 4, 8, 16, 32) for dqk in (4, 8, 16, 32, 64, 128) if H * dqk <= 128]
STATS_SHAPES = [(H, dqk) for H, dqk in FUSED_SHAPES if H <= 8]
_K3_CACHE = {}


def k3_graph(name):
    if name not in _K3_CACHE:
        rowptr, col = K3_GRAPHS[name]()
        _K3_CACHE[name] = (rowptr, col, dev(rowptr), dev(col))
    return _K3_CACHE[name]


def k3_plan(plan_name):
    graph, params = K3_PLANS[plan_name]
    if params is None:
        return None
    rowptr = k3_graph(graph)[0]
    if params == "short":
        params = (ref.HUB_THRESHOLD, ref.HUB_CHUNK, ref.short_task_rows(len(rowptr) - 1, int(rowptr[-1])))
    return RawPlan(rowptr, *params)


def gat_inputs(n_dst, H, dqk, dv, seed):
    rs = np.random.RandomState(seed)
    Q = rs.randn(n_dst, H * dqk).astype(np.float32)
    K = rs.randn(2001, H * dqk).astype(np.float32)
    V = rs.randn(2001, H * dv).astype(np.float32)
    bias = rs.randn(H * dv).astype(np.float32)
    return Q, K, V, bias


def gat_raw(rp_d, col_d, Q, K, V, n_dst, H, dqk, dv, out, plan_struct=None, split=True, bias=None, act=ops.ACT_NONE,
            att=None, write_att=False, scale=None):
    scale = float(np.sqrt(np.float32(dqk))) if scale is None else scale
    _ffi.call("tfgk_gat_fused_f32", ptr(rp_d), ptr(col_d), ptr(Q), ld(Q), ptr(K), ld(K), ptr(V), ld(V), n_dst, H, dqk, dv,
              scale, 1 if split else 0, ptr(bias), act, ptr(att), 1 if write_att else 0, ptr(out), ld(out),
              None if plan_struct is None else ctypes.byref(plan_struct), stream())
    return out


_WORST = {}


@pytest.fixture(scope="module", autouse=True)
def report_worst_ratio():
    yield
    if _WORST:
        print("\nK3 largest |got - ref| / bound: " + ", ".join("{}: {:.4f}".format(k, v) for k, v in sorted(_WORST.items())))


def check_gat(got, r, n_slices, what):
    got = got.cpu().numpy() if torch.is_tensor(got) else got
    assert r["max_abs_score"] <= ref.MAX_ABS_SCORE
    bound = ref.gat_bound(r, n_slices)
    bad = ref.outside_bound(got, r["ref"], bound)
    kind = what.split(" ")[0].split(":")[0]
    err = np.abs(got.astype(np.float64) - r["ref"])
    _WORST[kind] = max(_WORST.get(kind, 0.0), float(np.max(np.where(bound > 0, err / np.maximum(bound, 1e-300), 0.0))))
    if bad.any():
        i = tuple(np.argwhere(bad)[0])
        raise AssertionError("{}: {} of {} entries outside the bound, first at {}: got {!r}, ref {!r}, bound {:.3e}, "
                             "largest err / bound {:.3g}".format(what, int(bad.sum()), bad.size, i, got[i], r["ref"][i],
                                                                 bound[i], np.nanmax(err / np.maximum(bound, 1e-300))))


_REF_CACHE = {}


def _refs(graph, H, dqk, dv, bias_on, seed, split=True, relu=False):
    """Inputs (bias of the output width) and their float64 reference, kept for the other plans of the same graph."""
    key = (graph, H, dqk, dv, bias_on, seed, split, relu)
    if key not in _REF_CACHE:
        if len(_REF_CACHE) > 8:
            _REF_CACHE.clear()
        rowptr, col, _, _ = k3_graph(graph)
        Q, K, V, bias = gat_inputs(len(rowptr) - 1, H, dqk, dv, seed)
        bias = bias if split else bias[:dv]
        r = ref.gat_reference(rowptr, col, Q, K, V, H, dqk, dv, np.sqrt(np.float32(dqk)), split=split,
                              bias=bias if bias_on else None, relu=relu)
        _REF_CACHE[key] = ((Q, K, V, bias), r)
    return _REF_CACHE[key]


@pytest.mark.parametrize("H,dqk", FUSED_SHAPES)
def test_k3_fused_rings_within_the_bound(H, dqk):
    """Every power-of-two (H, dqk) with H dqk <= 128 through the TMA ring (K | V adjacent) and the cp.async ring (K and V
    in separate buffers), without a plan, with the production hub plan, a threshold-5 chunk-3 plan and the short-task
    plan."""
    A = H * dqk
    for plan_name in K3_PLANS:
        graph = K3_PLANS[plan_name][0]
        rowptr, col, rp_d, col_d = k3_graph(graph)
        n = len(rowptr) - 1
        (Q, K, V, bias), r = _refs(graph, H, dqk, dqk, True, H * 1000 + dqk)
        plan = k3_plan(plan_name)
        ns = ref.slices_per_row(None if plan is None else plan.host, n)
        Qd, kv = dev(Q), dev(np.concatenate([K, V], axis=1))
        Kd, Vd, bd = dev(K), dev(V), dev(bias)
        out = torch.empty((n, A), dtype=torch.float32, device="cuda")
        for name, k_, v_ in (("tma", kv[:, :A], kv[:, A:]), ("async", Kd, Vd)):
            out.fill_(float("nan"))
            gat_raw(rp_d, col_d, Qd, k_, v_, n, H, dqk, dqk, out, None if plan is None else plan.struct(A + 64), bias=bd)
            torch.cuda.synchronize()
            check_gat(out, r, ns, "{} H={} dqk={} plan={}".format(name, H, dqk, plan_name))


@pytest.mark.parametrize("H,dqk", [(2, 128), (8, 32), (4, 128), (16, 32)])
def test_k3_online_kernel_wide_rows(H, dqk):
    """A = 256 and 512 take gat_online_kernel (the plan is not used there: hub rows run in one warp).  A = 384 cannot
    reach it: H and dqk / 4 are powers of two."""
    rowptr, col, rp_d, col_d = k3_graph("main")
    n, A = len(rowptr) - 1, H * dqk
    (Q, K, V, bias), r = _refs("main", H, dqk, dqk, True, A + H)
    plan = k3_plan("hub")
    out = torch.full((n, A), float("nan"), device="cuda")
    gat_raw(rp_d, col_d, dev(Q), dev(K), dev(V), n, H, dqk, dqk, out, plan.struct(A + 64), bias=dev(bias))
    check_gat(out, r, None, "online H={} dqk={}".format(H, dqk))


OTHER_KERNELS = [
    # name, H, dqk, dv, split, write_att
    ("online_writes_attention", 8, 16, 16, True, True),
    ("fast_dqk_ne_dv", 4, 32, 16, True, False),
    ("fast_dqk_ne_dv_wide", 8, 64, 48, True, True),
    ("generic_dv_not_multiple_of_4", 8, 4, 2, True, True),
    ("generic_averaged_heads", 4, 16, 12, False, False),
    ("generic_3_heads", 3, 12, 12, True, True),
]


@pytest.mark.parametrize("name,H,dqk,dv,split,write_att", OTHER_KERNELS, ids=[c[0] for c in OTHER_KERNELS])
def test_k3_other_kernels_within_the_bound(name, H, dqk, dv, split, write_att):
    rowptr, col, rp_d, col_d = k3_graph("main")
    n = len(rowptr) - 1
    (Q, K, V, bias), r = _refs("main", H, dqk, dv, True, 7 * H + dqk + dv, split=split, relu=True)
    out_w = H * dv if split else dv
    out = torch.full((n, out_w), float("nan"), device="cuda")
    att = torch.full((len(col), H), float("nan"), device="cuda")
    gat_raw(rp_d, col_d, dev(Q), dev(K), dev(V), n, H, dqk, dv, out, split=split, bias=dev(bias), act=ops.ACT_RELU,
            att=att, write_att=write_att)
    torch.cuda.synchronize()
    check_gat(out, r, None, name)
    if write_att:
        a = r["alpha"]
        deg = np.diff(rowptr)[ref.csr_rows(rowptr)].astype(np.float64)
        bound = (2 * r["delta_h"][ref.csr_rows(rowptr)] + ref.C_GAT * (deg[:, None] + 8) * ref.U) * a
        got = att.cpu().numpy()
        assert not ref.outside_bound(got, a, bound).any(), "{}: attention coefficients outside the bound".format(name)


@pytest.mark.parametrize("H,dqk", STATS_SHAPES)
def test_k3_stats_forward_with_hub_slices(H, dqk):
    """tfgk_gat_fused_stats_f32 on every shape gat_recompute_shape accepts, with hub rows cut into slices: the output and
    (max, denominator) of the hub rows come from the fix-up."""
    A = H * dqk
    for plan_name in ("hub", "tiny5x3", "short"):
        graph = K3_PLANS[plan_name][0]
        rowptr, col, rp_d, col_d = k3_graph(graph)
        n = len(rowptr) - 1
        (Q, K, V, bias), r = _refs(graph, H, dqk, dqk, True, H * 77 + dqk)
        plan = k3_plan(plan_name)
        ns = ref.slices_per_row(plan.host, n)
        kv, Qd, bd = dev(np.concatenate([K, V], axis=1)), dev(Q), dev(bias)
        for name, k_, v_ in (("tma", kv[:, :A], kv[:, A:]), ("async", dev(K), dev(V))):
            out = torch.full((n, A), float("nan"), device="cuda")
            stats = torch.full((n, 2 * H), float("nan"), device="cuda")
            _ffi.call("tfgk_gat_fused_stats_f32", ptr(rp_d), ptr(col_d), ptr(Qd), A, ptr(k_), ld(k_), ptr(v_), ld(v_), n,
                      H, dqk, dqk, float(np.sqrt(np.float32(dqk))), ptr(bd), ops.ACT_NONE, ptr(out), A, ptr(stats),
                      ctypes.byref(plan.struct(A + 64)), stream())
            torch.cuda.synchronize()
            what = "stats {} H={} dqk={} plan={}".format(name, H, dqk, plan_name)
            check_gat(out, r, ns, what)
            st = stats.cpu().numpy().astype(np.float64)
            m, Z, deg = st[:, :H], st[:, H:], np.diff(rowptr)
            live = deg > 0
            assert np.all(m[~live] == -ref.FLT_MAX) and np.all(Z[~live] == np.float32(1e-8)), what + ": empty rows"
            dh = r["delta_h"][live]
            assert np.all(np.abs(m[live] - r["m"][live]) <= dh), what + ": maximum"
            zb = (2 * dh + ref.C_GAT * (deg[live] + ns[live] + 8)[:, None] * ref.U) * r["Z"][live]
            assert np.all(np.abs(Z[live] - r["Z"][live]) <= zb), what + ": denominator"


@pytest.mark.parametrize("impl", ["tma", "async"])
def test_k3_relu_empty_rows_and_strided_operands(impl):
    """Bias and ReLU; rows without edges give act(bias); Q, K, V and out as strided views of wider buffers."""
    H, dqk = 8, 16
    A = H * dqk
    rowptr, col, rp_d, col_d = k3_graph("main")
    n = len(rowptr) - 1
    (Q, K, V, bias), r = _refs("main", H, dqk, dqk, True, 5, relu=True)
    plan = k3_plan("tiny5x3")
    qd = dev(np.pad(Q, ((0, 0), (4, 8))))[:, 4:4 + A]
    if impl == "tma":
        buf = dev(np.pad(np.concatenate([K, V], axis=1), ((0, 0), (8, 4))))
        k_, v_ = buf[:, 8:8 + A], buf[:, 8 + A:8 + 2 * A]
    else:
        k_, v_ = dev(np.pad(K, ((0, 0), (4, 12))))[:, 4:4 + A], dev(np.pad(V, ((0, 0), (12, 4))))[:, 12:12 + A]
    obuf = torch.full((n, A + 8), 7.0, device="cuda")
    out = obuf[:, 4:4 + A]
    gat_raw(rp_d, col_d, qd, k_, v_, n, H, dqk, dqk, out, plan.struct(A + 64), bias=dev(bias), act=ops.ACT_RELU)
    torch.cuda.synchronize()
    check_gat(out, r, ref.slices_per_row(plan.host, n), "strided " + impl)
    empty = np.diff(rowptr) == 0
    np.testing.assert_array_equal(out.cpu().numpy()[empty], np.tile(np.maximum(bias, 0), (int(empty.sum()), 1)))
    assert bool((obuf[:, :4] == 7.0).all()) and bool((obuf[:, 4 + A:] == 7.0).all())


def test_k3_refuses_a_plan_scratch_one_slot_short():
    H, dqk = 8, 16
    A = H * dqk
    rowptr, col, rp_d, col_d = k3_graph("main")
    n = len(rowptr) - 1
    plan = k3_plan("tiny5x3")
    x = dev(np.ones((2001, A), np.float32))
    out = torch.full((n, A), 7.0, device="cuda")
    with pytest.raises(_ffi.TfgkError) as err:
        gat_raw(rp_d, col_d, x[:n], x, x, n, H, dqk, dqk, out, plan.struct(A + 64, slots=plan.n_slots - 1))
    assert err.value.code == _ffi.ERR_INVALID_ARGUMENT
    torch.cuda.synchronize()
    assert bool((out == 7.0).all())


@pytest.mark.parametrize("H", [1, 5, 32])
def test_segment_softmax_within_the_bound(H):
    """tfgk_segment_softmax_f32: segments longer than a warp, a 1000-entry segment, empty segments."""
    rs = np.random.RandomState(H)
    deg = rs.randint(0, 100, 300)
    deg[::7] = 0
    deg[150] = 1000
    rowptr, _ = ref.csr_from_degrees(deg, 1, H)
    score = (rs.randn(int(rowptr[-1]), H) * 4).astype(np.float32)
    out = torch.full(score.shape, float("nan"), device="cuda")
    rp_d, score_d = dev(rowptr), dev(score)
    _ffi.call("tfgk_segment_softmax_f32", ptr(rp_d), ptr(score_d), 300, H, ptr(out), stream())
    torch.cuda.synchronize()
    want, gap = ref.segment_softmax_reference(rowptr, score)
    bad = ref.outside_bound(out.cpu().numpy(), want, ref.segment_softmax_bound(rowptr, want, gap))
    assert not bad.any(), "{} coefficients outside the bound".format(int(bad.sum()))


# ---- D. dispatch ---------------------------------------------------------------------------------------------------

def _launched(fn):
    from torch.profiler import ProfilerActivity, profile
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        fn()
        torch.cuda.synchronize()
    evs = [e for e in prof.events() if "tfgk::" in e.name]
    evs.sort(key=lambda e: e.time_range.start)
    return [e.name for e in evs]


def _k1_case(D, plan_name="none", offset=0, reduce="sum"):
    def run():
        graph, params = ref.K1_PLANS[plan_name]
        rowptr, col, w, rp_d, col_d, w_d = k1_graph(graph)
        n = len(rowptr) - 1
        h = dev(np.ones((3001, D + offset), np.float32))[:, offset:offset + D]
        out = torch.empty((n, D), device="cuda")
        plan = RawPlan(rowptr, *ref.plan_params(plan_name, rowptr)) if params is not None else None
        st = None if plan is None else plan.struct(D)
        return _launched(lambda: spmm_raw(rp_d, col_d, w_d, h, n, reduce, out, st))
    return run


def _k3_case(H, dqk, dv=None, adjacent=True, plan_name="none", split=True, write_att=False, stats=False):
    dv = dqk if dv is None else dv

    def run():
        rowptr, col, rp_d, col_d = k3_graph("main")
        n, A, VW = len(rowptr) - 1, H * dqk, H * dv
        kv = dev(np.random.RandomState(0).randn(2001, A + VW).astype(np.float32))
        k_, v_ = (kv[:, :A], kv[:, A:]) if adjacent else (kv[:, :A].contiguous(), kv[:, A:].contiguous())
        q = dev(np.ones((n, A), np.float32))
        out = torch.empty((n, VW if split else dv), device="cuda")
        att = torch.empty((len(col), H), device="cuda")
        plan = k3_plan(plan_name)
        st = None if plan is None else plan.struct(VW + 64)
        if stats:
            s = torch.empty((n, 2 * H), device="cuda")
            return _launched(lambda: _ffi.call(
                "tfgk_gat_fused_stats_f32", ptr(rp_d), ptr(col_d), ptr(q), A, ptr(k_), ld(k_), ptr(v_), ld(v_), n, H,
                dqk, dqk, float(np.sqrt(dqk)), None, 0, ptr(out), A, ptr(s), None if st is None else ctypes.byref(st),
                stream()))
        return _launched(lambda: gat_raw(rp_d, col_d, q, k_, v_, n, H, dqk, dv, out, st, split=split, att=att,
                                         write_att=write_att))
    return run


FIXUP = "spmm_hub_fixup_kernel<false, false>"
DISPATCH = [
    ("k1 D=28", _k1_case(28), ["spmm_kernel<4, 8, 1, false,"]),
    ("k1 D=32", _k1_case(32), ["spmm_tma4_kernel<false, 3, float, false>"]),
    ("k1 D=256", _k1_case(256), ["spmm_tma4_kernel<false, 3, float, false>"]),
    ("k1 D=256 max", _k1_case(256, reduce="max"), ["spmm_tma4_kernel<true, 3, float, false>"]),
    ("k1 D=260", _k1_case(260), ["spmm_async_kernel<3, false, 4, 3, float, false>"]),
    ("k1 D=512", _k1_case(512), ["spmm_async_kernel<4, false, 2, 4, float, false>"]),
    ("k1 D=516", _k1_case(516), ["spmm_async_kernel<4, false, 2, 4, float, false>", "spmm_kernel<4, 1, 1, false,"]),
    ("k1 D=1024", _k1_case(1024), ["spmm_async_kernel<4, false, 2, 4, float, false>"] * 2),
    ("k1 D=128 misaligned", _k1_case(128, offset=1), ["spmm_kernel<1, 32, 4, false,"]),
    ("k1 D=300 misaligned", _k1_case(300, offset=1), ["spmm_kernel<1, 32, 4, false,"] * 2 + ["spmm_kernel<1, 32, 2, false,"]),
    ("k1 D=128 hub plan", _k1_case(128, plan_name="hub"), ["spmm_tma4_kernel<false, 3, float, false>", FIXUP]),
    ("k1 D=384 hub plan", _k1_case(384, plan_name="hub"), ["spmm_async_kernel<3, false, 4, 3, float, false>", FIXUP]),
    ("k1 D=128 short plan", _k1_case(128, plan_name="short"), ["spmm_tma4_kernel<false, 3, float, false>", FIXUP]),
    ("k3 adjacent", _k3_case(8, 16), ["gat_tma4_kernel<2, float>"]),
    ("k3 separate", _k3_case(8, 16, adjacent=False), ["gat_async_kernel<2, 3>"]),
    ("k3 adjacent hub plan", _k3_case(8, 16, plan_name="tiny5x3"), ["gat_tma4_kernel<2, float>", "gat_hub_fixup_kernel"]),
    ("k3 separate hub plan", _k3_case(8, 16, adjacent=False, plan_name="hub"), ["gat_async_kernel<2, 3>",
                                                                                 "gat_hub_fixup_kernel"]),
    ("k3 stats hub plan", _k3_case(8, 16, plan_name="hub", stats=True), ["gat_tma4_kernel<2, float>", "gat_hub_fixup_kernel"]),
    ("k3 A=256", _k3_case(8, 32, plan_name="hub"), ["gat_online_kernel<2, 2, float>"]),
    ("k3 A=512", _k3_case(4, 128), ["gat_online_kernel<4, 2, float>"]),
    ("k3 return_attention", _k3_case(8, 16, plan_name="hub", write_att=True), ["gat_online_kernel<1, 4, float>"]),
    ("k3 dqk != dv", _k3_case(4, 32, dv=16), ["gat_fast_kernel<1, 1, 4>"]),
    ("k3 dv % 4 != 0", _k3_case(8, 4, dv=2), ["gat_generic_kernel<float>"]),
    ("k3 averaged heads", _k3_case(4, 16, split=False), ["gat_generic_kernel<float>"]),
    ("k3 H=3 dqk=12", _k3_case(3, 12), ["gat_generic_kernel<float>"]),
]


def _record_dispatch():
    """{entry: launched kernel names} for every DISPATCH entry, one profiler session each."""
    return {name: run() for name, run, _ in DISPATCH}


@pytest.fixture(scope="module")
def dispatch_record():
    """The table is recorded in a fresh interpreter: a torch.profiler session earlier in the same process (another test
    file may open one) can leave later sessions without some or all of their kernel records."""
    here = os.path.dirname(os.path.abspath(__file__))
    code = ("import json, sys; sys.path[:0] = [{!r}, {!r}]; import test_gpu_k1k3_contract as t; "
            "print('@@' + json.dumps(t._record_dispatch()))").format(here, os.path.dirname(here))
    # the child ignores the user's site-packages exactly when this interpreter does
    flags = ["-I"] if sys.flags.isolated else ["-s"] if sys.flags.no_user_site else []
    res = subprocess.run([sys.executable] + flags + ["-c", code], capture_output=True, text=True, timeout=900)
    assert res.returncode == 0, res.stdout[-2000:] + res.stderr[-4000:]
    return json.loads([line for line in res.stdout.splitlines() if line.startswith("@@")][-1][2:])


@pytest.mark.parametrize("name,want", [(d[0], d[2]) for d in DISPATCH], ids=[d[0] for d in DISPATCH])
def test_dispatch_table(name, want, dispatch_record):
    """The kernels each entry launches, in order (demangled names recorded by torch.profiler).  A profiler that records no
    kernel fails the test: the contract above would otherwise hold for unknown kernels."""
    got = dispatch_record[name]
    assert got, "{}: the profiler recorded no tfgk kernel".format(name)
    assert len(got) == len(want) and all(p in g for p, g in zip(want, got)), \
        "{}: launched {}, expected {}".format(name, got, want)
