# coding=utf-8
"""CPU checks of the host models in tests/k1k3_ref.py: the plan model, the sliced-sum model of K1 and the K3 bound.
A model that is wrong in the same way as a kernel would let the GPU contract pass, so each model is checked here
against hand-worked cases, an independent restatement or planted faults."""
import numpy as np
import pytest

import k1k3_ref as ref
from oracle import c_oracle


# ---- plan model ---------------------------------------------------------------------------------------------------

def test_plan_model_hand_worked_case():
    """deg [0, 6, 2, 7, 1], threshold 5, chunk 3, two rows per task: a run at every even row and after every hub."""
    rowptr = np.array([0, 0, 6, 8, 15, 16])
    p = ref.plan_model(rowptr, 5, 3, 2)
    assert (p["n_tasks"], p["n_hubs"], p["n_slots"]) == (8, 2, 5)
    np.testing.assert_array_equal(p["task_row"], [0, 1, 1, 2, 3, 3, 3, 4])
    np.testing.assert_array_equal(p["task_nrows"], [1, 1, 1, 1, 1, 1, 1, 1])
    np.testing.assert_array_equal(p["task_e0"], [0, 0, 3, 6, 8, 11, 14, 15])
    np.testing.assert_array_equal(p["task_e1"], [0, 3, 6, 8, 11, 14, 15, 16])
    np.testing.assert_array_equal(p["task_slot"], [-1, 0, 1, -1, 2, 3, 4, -1])
    np.testing.assert_array_equal(p["hub_row"], [1, 3])
    np.testing.assert_array_equal(p["hub_slot0"], [0, 2])
    np.testing.assert_array_equal(p["hub_nslots"], [2, 3])


def test_plan_model_light_runs_end_at_multiples_of_rows_per_task():
    p = ref.plan_model(np.arange(8), 5, 3, 3)                    # seven rows of one edge
    np.testing.assert_array_equal(p["task_row"], [0, 3, 6])
    np.testing.assert_array_equal(p["task_nrows"], [3, 3, 1])
    np.testing.assert_array_equal(p["task_e0"], [0, 3, 6])
    np.testing.assert_array_equal(p["task_e1"], [3, 6, 7])
    assert p["n_hubs"] == 0 and p["n_slots"] == 0


@pytest.mark.parametrize("rpt", [1, 3, 32])
@pytest.mark.parametrize("case", sorted(ref.plan_degree_cases()))
def test_plan_model_satisfies_the_invariants(case, rpt):
    deg, thr, chunk = ref.plan_degree_cases()[case]
    rowptr = np.concatenate([[0], np.cumsum(deg)])
    p = ref.plan_model(rowptr, thr, chunk, rpt)
    ref.check_plan_invariants(p, rowptr, thr, chunk, rpt, ref.plan_capacity_model(int(rowptr[-1]), len(deg), thr, chunk, rpt))


def test_plan_invariants_catch_a_short_last_slice():
    """The invariant check is what the GPU plan comparison leans on besides the model: a hub slice one edge short fails."""
    rowptr = np.array([0, 0, 6, 8, 15, 16])
    p = ref.plan_model(rowptr, 5, 3, 2)
    p["task_e1"] = p["task_e1"].copy()
    p["task_e1"][2] -= 1
    with pytest.raises(AssertionError):
        ref.check_plan_invariants(p, rowptr, 5, 3, 2)


@pytest.mark.parametrize("thr,chunk,rpt", [(1, 1, 1), (2, 1, 32), (5, 3, 3), (7, 2, 5)])
def test_capacity_covers_the_densest_plans(thr, chunk, rpt):
    """Every row a hub of thr + 1 edges (the most hubs per edge), alternating with empty rows (a run after every hub)."""
    deg = np.tile([thr + 1, 0], 500)
    rowptr = np.concatenate([[0], np.cumsum(deg)])
    p = ref.plan_model(rowptr, thr, chunk, rpt)
    cap = ref.plan_capacity_model(int(rowptr[-1]), len(deg), thr, chunk, rpt)
    assert p["n_tasks"] <= cap[0] and p["n_hubs"] <= cap[1]


# ---- K1 model -----------------------------------------------------------------------------------------------------

def _h(n, d, seed):
    return np.random.RandomState(seed).randn(n, d).astype(np.float32)


def _w(e, seed):
    return (np.random.RandomState(seed).rand(e) + 0.1).astype(np.float32)


def test_k1_sequential_model_is_the_oracle():
    """Without a plan the model is c_oracle.aggregate over the CSR, mean included."""
    rowptr, col = ref.k1_main_graph()
    h, w = _h(3001, 8, 1), _w(len(col), 2)
    rows = ref.csr_rows(rowptr)
    for reduce in ("sum", "mean", "max"):
        np.testing.assert_array_equal(ref.k1_expected(rowptr, col, w, h, reduce),
                                      c_oracle.aggregate(rows, col, w, h, len(rowptr) - 1, reduce))


@pytest.mark.parametrize("plan_name", [k for k, (_, p) in ref.K1_PLANS.items() if p is not None])
def test_k1_sliced_sums_differ_from_sequential(plan_name):
    """Bit-equality with the sliced model proves the slicing ran only if slicing changes bits: it does for every plan with
    hub rows, for the weighted sum.  The max is the same either way (fmaxf is exact), and so is every row that is not a
    hub."""
    graph, _ = ref.K1_PLANS[plan_name]
    rowptr, col = ref.GRAPHS[graph]()
    thr, chunk, rpt = ref.plan_params(plan_name, rowptr)
    plan = ref.plan_model(rowptr, thr, chunk, rpt)
    assert plan["n_hubs"] > 0
    h, w = _h(3001, 32, 3), _w(len(col), 4)
    hub = np.zeros(len(rowptr) - 1, bool)
    hub[plan["hub_row"]] = True
    seq = ref.k1_expected(rowptr, col, w, h, "sum")
    sliced = ref.k1_expected(rowptr, col, w, h, "sum", plan=plan)
    assert not np.array_equal(seq[hub], sliced[hub])
    np.testing.assert_array_equal(seq[~hub], sliced[~hub])
    np.testing.assert_allclose(sliced, seq, rtol=1e-4, atol=1e-3)
    np.testing.assert_array_equal(ref.k1_expected(rowptr, col, w, h, "max", plan=plan),
                                  ref.k1_expected(rowptr, col, w, h, "max"))


def test_k1_short_task_plan_has_short_tasks():
    rowptr, _ = ref.k1_short_graph()
    thr, chunk, rpt = ref.plan_params("short", rowptr)
    assert rpt == 3 and (len(rowptr) - 1) % rpt != 0
    p = ref.plan_model(rowptr, thr, chunk, rpt)
    assert p["n_hubs"] == 1 and p["task_nrows"].max() == 3


def test_k1_fixup_order_is_visible():
    """Folding the slices in reverse order changes the bits of a hub row: a tolerance would hide that, equality does not."""
    rowptr, col = ref.k1_main_graph()
    plan = ref.plan_model(rowptr, 5, 3, 32)
    rev = dict(plan)
    nh = plan["n_hubs"]
    # the same slices, numbered backwards inside every hub: the fold then runs from the last slice to the first
    slot = plan["task_slot"].copy()
    for s0, ns in zip(plan["hub_slot0"][:nh], plan["hub_nslots"][:nh]):
        idx = np.nonzero((slot >= s0) & (slot < s0 + ns))[0]
        slot[idx] = slot[idx][::-1]
    rev["task_slot"] = slot
    h, w = _h(3001, 32, 5), _w(len(col), 6)
    assert not np.array_equal(ref.k1_expected(rowptr, col, w, h, "sum", plan=plan),
                              ref.k1_expected(rowptr, col, w, h, "sum", plan=rev))


def test_k1_epilogue_order():
    """mean divide, then alpha acc + beta addend, then bias, then ReLU, each rounded to fp32."""
    acc = np.array([[3.0, -7.0]], np.float32)
    rowptr = np.array([0, 3])
    got = ref.k1_epilogue(acc, rowptr, "mean", alpha=0.75, addend=np.array([[1.5, 2.0]], np.float32), beta=-1.25,
                          bias=np.array([0.5, 0.25], np.float32), relu=True)
    a = np.float32(3.0) / np.float32(3)
    want0 = np.float32(np.float32(a * np.float32(0.75)) + np.float32(np.float32(1.5) * np.float32(-1.25))) + np.float32(0.5)
    assert got[0, 0] == np.maximum(want0, np.float32(0)) and got[0, 1] == 0.0


@pytest.mark.parametrize("D,aligned,want", [
    (4, True, False), (31, True, False), (32, True, True), (128, True, True), (256, True, True), (512, True, True),
    (516, True, False), (1024, True, False), (128, False, False), (512, False, False)])
def test_k1_takes_plan(D, aligned, want):
    assert ref.k1_takes_plan(D, aligned) == want


# ---- K3 bound -----------------------------------------------------------------------------------------------------

def _gat_problem(H=4, dqk=8, dv=8, seed=11):
    rs = np.random.RandomState(seed)
    deg = rs.randint(1, 13, 300)
    deg[5], deg[77], deg[200:203] = 150, 40, 0
    rowptr, col = ref.csr_from_degrees(deg, 300, seed + 1)
    Q, K = rs.randn(300, H * dqk).astype(np.float32), rs.randn(300, H * dqk).astype(np.float32)
    V = rs.randn(300, H * dv).astype(np.float32)
    return rowptr, col, Q, K, V, H, dqk, dv, float(np.sqrt(np.float32(dqk)))


def _fp32_two_pass(rowptr, col, Q, K, V, H, dqk, dv, scale):
    """The reference order in plain fp32 (numpy): an honest fp32 computation, which must sit inside the bound."""
    f = np.float32
    seg = ref.csr_rows(rowptr)
    s = ((Q.reshape(-1, H, dqk)[seg] * K.reshape(-1, H, dqk)[col]).sum(-1, dtype=f) / f(scale)).astype(f)
    n = len(rowptr) - 1
    out = np.zeros((n, H, dv), f)
    for r in range(n):
        a, b = rowptr[r], rowptr[r + 1]
        if a == b:
            continue
        p = np.exp(s[a:b] - s[a:b].max(0)).astype(f)
        den = (p.sum(0, dtype=f) + f(1e-8)).astype(f)
        alpha = (p / den).astype(f)
        acc = np.zeros((H, dv), f)
        for e in range(a, b):
            acc = (acc + (V[col[e]].reshape(H, dv) * alpha[e - a][:, None]).astype(f)).astype(f)
        out[r] = acc
    return out.reshape(n, H * dv)


def test_gat_fp32_computation_is_inside_the_bound():
    prob = _gat_problem()
    r = ref.gat_reference(*prob)
    got = _fp32_two_pass(*prob)
    assert not ref.outside_bound(got, r["ref"], ref.gat_bound(r)).any()


@pytest.mark.parametrize("row", [5, 77])
def test_gat_bound_rejects_a_missing_edge(row):
    """The largest-alpha edge of a long row removed from the reference: outside the bound on that row."""
    rowptr, col, Q, K, V, H, dqk, dv, scale = _gat_problem()
    r = ref.gat_reference(rowptr, col, Q, K, V, H, dqk, dv, scale)
    a, b = rowptr[row], rowptr[row + 1]
    e = a + int(np.argmax(r["alpha"][a:b].max(1)))
    keep = np.ones(len(col), bool)
    keep[e] = False
    rp2 = rowptr.copy()
    rp2[row + 1:] -= 1
    bad = ref.gat_reference(rp2, col[keep], Q, K, V, H, dqk, dv, scale)
    out = ref.outside_bound(bad["ref"], r["ref"], ref.gat_bound(r, ref.slices_per_row(ref.plan_model(rowptr, 5, 3, 32),
                                                                                       len(rowptr) - 1)))
    assert out[row].any()
    assert not np.delete(out, row, axis=0).any()


@pytest.mark.parametrize("row", [5, 77])
def test_gat_bound_rejects_a_swapped_value_row(row):
    """One neighbour's V row replaced by the next neighbour's (K untouched): outside the bound on that row."""
    rowptr, col, Q, K, V, H, dqk, dv, scale = _gat_problem()
    r = ref.gat_reference(rowptr, col, Q, K, V, H, dqk, dv, scale)
    a, b = rowptr[row], rowptr[row + 1]
    e = a + int(np.argmax(r["alpha"][a:b - 1].max(1)))
    vcol = col.copy()
    vcol[e] = col[e + 1]
    bad = ref.gat_reference(rowptr, col, Q, K, V, H, dqk, dv, scale, vcol=vcol)
    out = ref.outside_bound(bad["ref"], r["ref"], ref.gat_bound(r))
    assert out[row].any()
    assert not np.delete(out, row, axis=0).any()


def test_gat_reference_rows_without_edges_are_bias():
    prob = _gat_problem()
    bias = np.random.RandomState(3).randn(prob[5] * prob[7]).astype(np.float32)
    r = ref.gat_reference(*prob, bias=bias, relu=True)
    np.testing.assert_array_equal(r["ref"][200:203], np.tile(np.maximum(bias, 0), (3, 1)))
    assert (r["S"][200:203] == 0).all()


def test_segment_softmax_bound_rejects_a_wrong_denominator():
    rs = np.random.RandomState(4)
    rowptr, _ = ref.csr_from_degrees(rs.randint(0, 80, 50), 1, 5)
    score = (rs.randn(int(rowptr[-1]), 5) * 4).astype(np.float32)
    want, gap = ref.segment_softmax_reference(rowptr, score)
    bound = ref.segment_softmax_bound(rowptr, want, gap)
    got = c_oracle.segment_softmax(score, ref.csr_rows(rowptr), 50)
    assert not ref.outside_bound(got, want, bound).any()
    seg = ref.csr_rows(rowptr)
    off = got * np.float32(1 + 2.0 ** -10)                              # every coefficient 1e-3 too large
    assert ref.outside_bound(off, want, bound).all(axis=1)[np.diff(rowptr)[seg] > 0].all()
