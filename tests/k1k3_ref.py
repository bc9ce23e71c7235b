# coding=utf-8
"""Host models of K1 (tfgk_spmm_f32), K3 (tfgk_gat_fused_f32) and their work plan (tfgk_plan_build), in numpy and the
C oracle.  No GPU is needed; tests/test_k1k3_ref_host.py checks the models, tests/test_gpu_k1k3_contract.py holds the
kernels to them.

* plan_model(rowptr, thr, chunk, rpt): the task arrays of the definition in include/tfgk.h.  Rows are visited in order; a
  row with more than `thr` edges is a hub and becomes ceil(deg / chunk) one-row tasks of `chunk` edges (the last one
  shorter), each with its own scratch slot, slots numbered in row order; a run of light rows starts at every multiple of
  `rpt` and right after a hub, and ends before the next multiple of `rpt`, the next hub or the end.
* k1_expected(...): the exact fp32 answer of K1.  A row that is not sliced is summed (or maxed) strictly in CSR order from
  0 (-FLT_MAX) with separate multiply and add roundings: the C oracle's aggregate.  A hub row that the kernel slices is
  the same sequential reduction per slice, the slices then folded in slice order from 0 (-FLT_MAX), as
  spmm_hub_fixup_kernel does.  The epilogue follows in float32, one rounding per operation, in the kernels' order: mean
  divide by max(deg, 1), then alpha acc + beta addend (alpha acc without an addend), then bias, then ReLU.
* gat_reference / gat_bound: float64 attention from the fp32 inputs and the per-entry bound of the module
  docstring of tests/test_gpu_k1k3_contract.py.
"""
import numpy as np

from oracle import c_oracle

U = 2.0 ** -24                               # unit roundoff of fp32
FLT_MAX = float(np.finfo(np.float32).max)

# ops.build_plan's production parameters and its short-task rule (average degree >= DENSE_ROW_DEGREE)
HUB_THRESHOLD, HUB_CHUNK, ROWS_PER_TASK = 2048, 2048, 32
DENSE_ROW_DEGREE, TASK_EDGE_TARGET = 128, 512


def short_task_rows(n_rows, nnz):
    """rows_per_task of ops.build_plan."""
    avg = nnz / float(n_rows)
    return ROWS_PER_TASK if avg < DENSE_ROW_DEGREE else max(1, min(ROWS_PER_TASK, int(TASK_EDGE_TARGET // avg)))


# ---- work plan --------------------------------------------------------------------------------------------------------

PLAN_KEYS = ("task_row", "task_nrows", "task_e0", "task_e1", "task_slot", "hub_row", "hub_slot0", "hub_nslots")


def plan_model(rowptr, thr, chunk, rpt):
    """The plan of include/tfgk.h as a dict of the eight arrays plus n_tasks, n_hubs, n_slots."""
    rowptr = np.asarray(rowptr, np.int64)
    n = len(rowptr) - 1
    deg = np.diff(rowptr)
    hub = deg > thr
    out = {k: [] for k in PLAN_KEYS}
    n_slots = 0
    for r in range(n):
        if hub[r]:
            ns = int(-(-deg[r] // chunk))
            out["hub_row"].append(r)
            out["hub_slot0"].append(n_slots)
            out["hub_nslots"].append(ns)
            for j in range(ns):
                out["task_row"].append(r)
                out["task_nrows"].append(1)
                out["task_e0"].append(rowptr[r] + j * chunk)
                out["task_e1"].append(min(rowptr[r + 1], rowptr[r] + (j + 1) * chunk))
                out["task_slot"].append(n_slots + j)
            n_slots += ns
        elif r % rpt == 0 or (r > 0 and hub[r - 1]):
            r2 = r + 1
            while r2 < n and r2 % rpt != 0 and not hub[r2]:
                r2 += 1
            out["task_row"].append(r)
            out["task_nrows"].append(r2 - r)
            out["task_e0"].append(rowptr[r])
            out["task_e1"].append(rowptr[r2])
            out["task_slot"].append(-1)
    plan = {k: np.asarray(v, np.int64 if k in ("task_e0", "task_e1") else np.int32) for k, v in out.items()}
    plan.update(n_tasks=len(out["task_row"]), n_hubs=len(out["hub_row"]), n_slots=n_slots)
    return plan


def plan_capacity_model(E, N, thr, chunk, rpt):
    """(max_tasks, max_hubs) that tfgk_plan_capacity promises: at most E / (thr + 1) rows can be hubs, every hub adds at
    most one run after it and ceil(deg / chunk) <= deg / chunk + 1 slices."""
    hubs = E // (thr + 1) + 1
    return -(-N // rpt) + hubs + (E // chunk + hubs) + 2, hubs


def check_plan_invariants(plan, rowptr, thr, chunk, rpt, capacity=None):
    """What any valid plan satisfies, independently of plan_model; raises AssertionError."""
    rowptr = np.asarray(rowptr, np.int64)
    n, E = len(rowptr) - 1, int(rowptr[-1])
    deg = np.diff(rowptr)
    nt, nh = plan["n_tasks"], plan["n_hubs"]
    row, nrows, e0, e1, slot = (plan[k][:nt].astype(np.int64) for k in ("task_row", "task_nrows", "task_e0", "task_e1",
                                                                           "task_slot"))
    hub_row, slot0, nslots = (plan[k][:nh].astype(np.int64) for k in ("hub_row", "hub_slot0", "hub_nslots"))
    # the [e0, e1) ranges tile [0, E) in task order
    if nt:
        assert e0[0] == 0 and e1[-1] == E, "edge ranges do not start at 0 and end at E"
        assert np.array_equal(e0[1:], e1[:-1]), "edge ranges leave a gap or overlap"
    assert np.all(e1 >= e0)
    # every row is covered exactly once: by one light task or by its hub slices
    covered = np.zeros(n, np.int64)
    light = slot < 0
    assert np.all(nrows[light] >= 1) and np.all(nrows[light] <= rpt), "a light task holds 0 or more than rpt rows"
    for r, k in zip(row[light], nrows[light]):
        covered[r:r + k] += 1
    assert np.array_equal(hub_row, np.sort(hub_row)) and len(np.unique(hub_row)) == nh
    covered[hub_row] += 1
    assert np.all(covered == 1), "rows covered {} times".format(sorted(set(covered.tolist())))
    assert np.array_equal(e0[light], rowptr[row[light]]) and np.array_equal(e1[light], rowptr[row[light] + nrows[light]])
    # hubs are exactly the rows above the threshold, sliced into consecutive slots of at most `chunk` edges
    assert np.array_equal(hub_row, np.nonzero(deg > thr)[0])
    assert np.all(nrows[~light] == 1) and np.all(e1[~light] - e0[~light] >= 1) and np.all(e1[~light] - e0[~light] <= chunk)
    assert np.array_equal(slot[~light], np.arange(plan["n_slots"])), "slots are not numbered in task order"
    if nh:
        assert np.array_equal(slot0, np.concatenate([[0], np.cumsum(nslots)[:-1]])), "hub slots not in row order"
    assert int(nslots.sum()) == plan["n_slots"]
    for h in range(nh):
        t = np.nonzero(slot == slot0[h])[0][0]
        ts = slice(t, t + nslots[h])
        assert np.all(row[ts] == hub_row[h]) and e0[t] == rowptr[hub_row[h]] and e1[t + nslots[h] - 1] == rowptr[hub_row[h] + 1]
    if capacity is not None:
        assert nt <= capacity[0] and nh <= capacity[1], "counts {} / {} beyond capacity {}".format(nt, nh, capacity)


def plan_degree_cases():
    """name -> (degrees, hub_threshold, chunk): the boundaries of the plan definition."""
    rs = np.random.RandomState(7)
    thr, chunk = 5, 3
    mixed = rs.randint(0, 12, 40)
    cases = {
        "degree_at_thr_thr_plus_1": (np.array([thr, thr + 1, thr, thr + 1, 0, thr + 1, thr]), thr, chunk),
        "degree_k_chunk_and_k_chunk_plus_1": (np.array([2 * chunk, 2 * chunk + 1, 3 * chunk, 3 * chunk + 1, 1, 4 * chunk,
                                                        4 * chunk + 1]), thr, chunk),
        "hub_first_and_last_row": (np.concatenate([[20], mixed[:9] % (thr + 1), [31]]), thr, chunk),
        "consecutive_hubs": (np.array([1, 9, 10, 11, 12, 2, 3, 8, 8, 0, 1]), thr, chunk),
        "every_row_a_hub": (np.full(13, thr + 1 + 2), thr, chunk),
        "empty_rows_between_hubs": (np.array([0, 9, 0, 0, 9, 0, 9, 0, 0, 0, 0, 9, 0]), thr, chunk),
        "single_row_light": (np.array([3]), thr, chunk),
        "single_row_hub": (np.array([17]), thr, chunk),
        "single_empty_row": (np.array([0]), thr, chunk),
        "mixed_40": (mixed, thr, chunk),
        "chunk_1": (rs.randint(0, 5, 50), 2, 1),
        # several 256-row blocks of plan_count_kernel and five 4096-entry scan tiles
        "large_20011": (np.where(rs.rand(20011) < 0.02, rs.randint(30, 200, 20011), rs.randint(0, 12, 20011)), 24, 16),
    }
    return cases


# ---- K1 -------------------------------------------------------------------------------------------------------------

def k1_takes_plan(D, aligned):
    """spmm.cu tfgk_spmm_f32: the plan is used when the whole width runs in one launch of a ring kernel, i.e. float4 rows
    (`aligned`: D % 4 == 0, ldh / ldo / ld_addend multiples of 4, 16-byte aligned pointers) and 32 <= D <= 512."""
    return aligned and 32 <= D <= 512


def csr_rows(rowptr):
    rowptr = np.asarray(rowptr, np.int64)
    return np.repeat(np.arange(len(rowptr) - 1, dtype=np.int32), np.diff(rowptr))


def k1_reduce(rowptr, col, w, h, reduce, plan=None):
    """The accumulators before the epilogue (sum for "sum" and "mean", max for "max"), hub rows of `plan` sliced."""
    rowptr = np.asarray(rowptr, np.int64)
    n = len(rowptr) - 1
    op = "max" if reduce == "max" else "sum"
    seg = csr_rows(rowptr)
    if plan is None or plan["n_hubs"] == 0:
        return c_oracle.aggregate(seg, col, w, h, n, op)
    nt = plan["n_tasks"]
    slot, e0, e1 = plan["task_slot"][:nt], plan["task_e0"][:nt], plan["task_e1"][:nt]
    seg = seg.copy()
    for s, a, b in zip(slot[slot >= 0], e0[slot >= 0], e1[slot >= 0]):
        seg[a:b] = n + s                                  # every slice is a segment of its own
    parts = c_oracle.aggregate(seg, col, w, h, n + plan["n_slots"], op)
    acc = parts[:n].copy()
    nh = plan["n_hubs"]
    hub_row, slot0, nslots = plan["hub_row"][:nh], plan["hub_slot0"][:nh], plan["hub_nslots"][:nh]
    fold = np.full((nh, h.shape[1]), -FLT_MAX if op == "max" else 0.0, np.float32)
    for j in range(int(nslots.max())):                    # slice order, as spmm_hub_fixup_kernel
        live = nslots > j
        part = parts[n + slot0[live] + j]
        fold[live] = np.maximum(fold[live], part) if op == "max" else fold[live] + part
    acc[hub_row] = fold
    return acc


def k1_epilogue(acc, rowptr, reduce, alpha=1.0, addend=None, beta=0.0, bias=None, relu=False):
    a = np.array(acc, np.float32)
    if reduce == "mean":
        a = a / np.maximum(np.diff(np.asarray(rowptr, np.int64)), 1).astype(np.float32)[:, None]
    if addend is not None:
        a = a * np.float32(alpha) + np.asarray(addend, np.float32) * np.float32(beta)
    elif alpha != 1.0:
        a = a * np.float32(alpha)
    if bias is not None:
        a = a + np.asarray(bias, np.float32)
    if relu:
        a = np.maximum(a, np.float32(0))
    return a.astype(np.float32)


def k1_expected(rowptr, col, w, h, reduce, epilogue=None, plan=None):
    """K1's exact output: `plan` is the plan the kernel actually uses (None when k1_takes_plan is false); `epilogue` a dict
    of k1_epilogue's keyword arguments."""
    return k1_epilogue(k1_reduce(rowptr, col, w, h, reduce, plan), rowptr, reduce, **(epilogue or {}))


# ---- graphs shared by the host and the GPU tests --------------------------------------------------------------------------

def csr_from_degrees(deg, n_src, seed):
    rs = np.random.RandomState(seed)
    deg = np.asarray(deg, np.int64)
    rowptr = np.concatenate([[0], np.cumsum(deg)]).astype(np.int64)
    col = rs.randint(0, n_src, int(rowptr[-1])).astype(np.int32)
    return rowptr, col


def k1_main_graph():
    """3001 rows (no task size divides it), about 31 500 edges: degrees 0 to 20, runs of empty rows, a 5000-edge hub
    (three production slices) in the middle and a 2500-edge hub at the last row, rows of exactly 5, 6, 40, 41, 47 and 48
    edges around the tiny-threshold plans."""
    rs = np.random.RandomState(101)
    n = 3001
    deg = rs.randint(0, 21, n)
    deg[:4] = 0
    deg[700:709] = 0
    deg[1234] = 5000
    deg[-1] = 2500
    deg[[10, 11, 12, 13, 14, 15]] = [5, 6, 40, 41, 47, 48]
    deg[16:20] = [7, 0, 7, 0]
    return csr_from_degrees(deg, n, 102)


def k1_short_graph():
    """61 long rows gathering from 3001 sources (average degree >= 128: the short-task plan with rows_per_task = 3), an
    empty row and a 2600-edge hub row."""
    rs = np.random.RandomState(103)
    deg = rs.randint(70, 130, 61)
    deg[7] = 0
    deg[30] = 2600
    return csr_from_degrees(deg, 3001, 104)


# name -> (graph, hub_threshold, chunk, rows_per_task); None: no plan
K1_PLANS = {
    "none": ("main", None),
    "hub": ("main", (HUB_THRESHOLD, HUB_CHUNK, ROWS_PER_TASK)),
    "tiny5x3": ("main", (5, 3, ROWS_PER_TASK)),
    "tiny40x16r3": ("main", (40, 16, 3)),
    "short": ("short", "short"),
}
GRAPHS = {"main": k1_main_graph, "short": k1_short_graph}


def plan_params(plan_name, rowptr):
    graph, params = K1_PLANS[plan_name]
    if params == "short":
        return HUB_THRESHOLD, HUB_CHUNK, short_task_rows(len(rowptr) - 1, int(rowptr[-1]))
    return params


# ---- K3 -------------------------------------------------------------------------------------------------------------

C_GAT = 10     # see the derivation in tests/test_gpu_k1k3_contract.py
MAX_ABS_SCORE = 16.0


def _segment(fn, x, rowptr, empty):
    """fn.reduceat over the CSR rows of x (first axis); rows without edges get `empty`."""
    rowptr = np.asarray(rowptr, np.int64)
    n = len(rowptr) - 1
    out = np.full((n,) + x.shape[1:], empty, np.float64)
    nz = np.nonzero(np.diff(rowptr) > 0)[0]
    if len(nz):
        out[nz] = fn.reduceat(x, rowptr[nz], axis=0)
    return out


def gat_reference(rowptr, col, Q, K, V, H, dqk, dv, scale, split=True, bias=None, relu=False, vcol=None):
    """float64 attention from the fp32 inputs: s = q.k / scale, alpha = exp(s - m) / (sum exp(s - m) + 1e-8),
    out = act(sum alpha v + bias).  `vcol` (default col) picks the V rows, to plant faults.  Returns a dict with
    ref (output), S = sum alpha |v| (per output entry), delta (the score error bound per output entry), m and Z
    (per row and head), alpha [E, H], deg."""
    rowptr = np.asarray(rowptr, np.int64)
    n = len(rowptr) - 1
    seg = csr_rows(rowptr)
    col = np.asarray(col, np.int64)
    vcol = col if vcol is None else np.asarray(vcol, np.int64)
    scale = float(np.float32(scale))
    qk = Q.astype(np.float64).reshape(Q.shape[0], H, dqk)[seg] * K.astype(np.float64).reshape(K.shape[0], H, dqk)[col]
    s = qk.sum(-1) / scale                                                        # [E, H]
    absdot = np.abs(qk).sum(-1) / scale
    m = _segment(np.maximum, s, rowptr, -np.inf)
    p = np.exp(s - m[seg])
    Z = _segment(np.add, p, rowptr, 0.0) + 1e-8
    alpha = p / Z[seg]
    v = V.astype(np.float64).reshape(V.shape[0], H, dv)[vcol]                     # [E, H, dv]
    out = _segment(np.add, alpha[:, :, None] * v, rowptr, 0.0)                   # [n, H, dv]
    S = _segment(np.add, alpha[:, :, None] * np.abs(v), rowptr, 0.0)
    delta = (dqk + 2) * U * _segment(np.maximum, absdot, rowptr, 0.0)             # [n, H]
    if split:
        out, S = out.reshape(n, H * dv), S.reshape(n, H * dv)
        delta = np.repeat(delta, dv, axis=1)
    else:
        out, S, delta = out.mean(1), S.mean(1), np.repeat(delta.max(1, keepdims=True), dv, axis=1)
    pre = out + (0.0 if bias is None else bias.astype(np.float64))
    return dict(ref=np.maximum(pre, 0.0) if relu else pre, S=S, delta=delta, m=m, Z=Z, alpha=alpha, s=s,
                delta_h=(dqk + 2) * U * _segment(np.maximum, absdot, rowptr, 0.0),
                deg=np.diff(rowptr), max_abs_score=float(np.abs(s).max()) if s.size else 0.0)


def gat_bound(r, n_slices=None):
    """|got - ref| <= (2 delta + C_GAT (deg + n_slices + 8) 2^-24) S + 2^-23 |ref| per entry."""
    cnt = r["deg"].astype(np.float64) + (0 if n_slices is None else n_slices) + 8
    return (2 * r["delta"] + C_GAT * cnt[:, None] * U) * r["S"] + 2.0 ** -23 * np.abs(r["ref"])


def slices_per_row(plan, n):
    """Number of hub slices of every row under `plan` (0 for rows that are not sliced, and without a plan)."""
    out = np.zeros(n, np.int64)
    if plan is not None and plan["n_hubs"]:
        nh = plan["n_hubs"]
        out[plan["hub_row"][:nh]] = plan["hub_nslots"][:nh]
    return out


def outside_bound(got, ref, bound):
    """Boolean mask of the entries where |got - ref| > bound (a NaN is outside)."""
    err = np.abs(np.asarray(got, np.float64) - ref)
    return ~(err <= bound)


def segment_softmax_reference(rowptr, score):
    """float64 exp(s - max) / (sum + 1e-8) per CSR segment and column of score [E, H]."""
    seg = csr_rows(rowptr)
    s = score.astype(np.float64)
    m = _segment(np.maximum, s, rowptr, -np.inf)
    p = np.exp(s - m[seg])
    Z = _segment(np.add, p, rowptr, 0.0) + 1e-8
    return p / Z[seg], (s - m[seg])


def segment_softmax_bound(rowptr, ref, gap):
    """(C_GAT (deg + 8) + |s - m|) 2^-24 ref: expf within 2 ulp, the rounded argument s - m, the per-lane and butterfly
    sums of the denominator (fewer than deg + 8 roundings) and the divide."""
    deg = np.diff(np.asarray(rowptr, np.int64))[csr_rows(rowptr)].astype(np.float64)
    return (C_GAT * (deg[:, None] + 8) + np.abs(gap)) * U * ref
