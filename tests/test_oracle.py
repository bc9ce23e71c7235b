# coding=utf-8
"""Pins the CPU oracle: reference fixtures / known answers, independent float64 dense model, numpy-vs-C agreement."""
import os

import numpy as np
import pytest

from oracle import tfg_oracle as o
from oracle import c_oracle
from conftest import assert_close, random_graph, glorot

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")


def test_readme_graph_to_directed():
    """README.md:31-59 / tutorial_intro.py:23-30 5-node graph; the README golden is from an older sorted
    implementation, so it is compared as an edge SET; the current code's order is upper || lower."""
    ei = np.array([[0, 0, 1, 3], [1, 2, 2, 1]])
    w = np.array([0.9, 0.8, 0.1, 0.2], dtype=np.float32)
    d, (dw,) = o.convert_edge_to_directed(ei, [w])
    assert d.tolist() == [[0, 0, 1, 1, 1, 2, 2, 3], [1, 2, 2, 3, 0, 0, 1, 1]]
    readme = {(0, 1), (0, 2), (1, 0), (1, 2), (1, 3), (2, 0), (2, 1), (3, 1)}
    assert set(zip(d[0].tolist(), d[1].tolist())) == readme
    np.testing.assert_array_equal(dw, np.array([.9, .8, .1, .2, .9, .8, .1, .2], dtype=np.float32))


def test_derived_kat_gcn_norm():
    """SURVEY.md section 8c derived known-answer vector (5 nodes, node 4 isolated)."""
    ei = np.array([[0, 0, 1, 1, 1, 2, 2, 3], [1, 2, 2, 3, 0, 0, 1, 1]])
    w = np.array([.9, .8, .1, .2, .9, .8, .1, .2], dtype=np.float32)
    n = o.gcn_norm_adj(o.SparseMatrix(ei, w, [5, 5]))
    assert n.index.tolist() == [[0, 0, 1, 1, 1, 2, 2, 3, 0, 1, 2, 3, 4], [1, 2, 2, 3, 0, 0, 1, 1, 0, 1, 2, 3, 4]]
    want = [0.36927447, 0.3532086, 0.0489116, 0.1230915, 0.36927447, 0.3532086, 0.0489116, 0.1230915, 0.37037033,
            0.45454547, 0.52631575, 0.8333334, 1.0]
    np.testing.assert_allclose(n.value, np.array(want, dtype=np.float32), rtol=2e-7)
    deg = o.SparseMatrix(ei, w, [5, 5]).add_diag(1.0).segment_sum()
    np.testing.assert_allclose(deg, np.array([2.7, 2.2, 1.9000001, 1.2, 1.0], dtype=np.float32), rtol=1e-7)


def test_adj_norm_edge_equals_gcn_norm_adj_default():
    """utils/graph_utils.py:914-943 is the tf_sparse-free twin of gcn_norm_adj(renorm=True, sym=True)."""
    ei = random_graph(50, 400, seed=3, symmetric=True)
    w = np.random.RandomState(1).rand(ei.shape[1]).astype(np.float32)
    i1, v1 = o.adj_norm_edge(ei, 50, w, add_self_loop=True)
    n = o.gcn_norm_adj(o.SparseMatrix(ei, w, [50, 50]))
    np.testing.assert_array_equal(i1, n.index)
    np.testing.assert_array_equal(v1, n.value)


def test_segment_semantics():
    ids = np.array([2, 0, 2, 2, -1], dtype=np.int32)
    data = np.array([[1., 2.], [3., 4.], [5., 6.], [-7., 8.], [100., 100.]], dtype=np.float32)
    s = o.unsorted_segment_sum(data, ids, 4)
    np.testing.assert_array_equal(s, [[3, 4], [0, 0], [-1, 16], [0, 0]])            # negative id dropped, empty -> 0
    m = o.unsorted_segment_mean(data[:4], ids[:4], 4)
    np.testing.assert_allclose(m[2], [-1 / 3, 16 / 3], rtol=1e-6)
    assert (m[1] == 0).all()
    mx = o.unsorted_segment_max(data[:4], ids[:4], 4)
    assert mx[1, 0] == np.finfo(np.float32).min and mx[2].tolist() == [5, 8]
    assert o.segment_count(np.array([0, 2, 2, 5], dtype=np.int32)).tolist() == [1, 0, 2, 0, 0, 1]
    assert o.segment_count(np.array([0, 2, 2, 5], dtype=np.int32)).dtype == np.int32


def test_sequential_rounding_of_segment_sum():
    """unsorted_segment_sum on CPU adds in input order: (1e8 + 1) + (-1e8) = 0 in fp32, not 1."""
    data = np.array([1e8, 1.0, -1e8], dtype=np.float32)
    assert o.unsorted_segment_sum(data, np.zeros(3, dtype=np.int32), 1)[0] == 0.0
    data = np.array([1e8, -1e8, 1.0], dtype=np.float32)
    assert o.unsorted_segment_sum(data, np.zeros(3, dtype=np.int32), 1)[0] == 1.0


def test_tf_unique_first_occurrence_order():
    u, idx = o.tf_unique(np.array([7, 3, 7, 1, 3]))
    assert u.tolist() == [7, 3, 1] and idx.tolist() == [0, 1, 0, 2, 1]


def test_merge_duplicated_edge_modes():
    ei = np.array([[0, 1, 0, 2, 1], [1, 2, 1, 0, 2]], dtype=np.int32)
    w = np.array([1., 2., 3., 4., 5.], dtype=np.float32)
    for mode, want in (("sum", [4, 7, 4]), ("min", [1, 2, 4]), ("max", [3, 5, 4]), ("mean", [2, 3.5, 4])):
        idx, (mw,) = o.merge_duplicated_edge(ei, [w], [mode])
        assert idx.tolist() == [[0, 1, 2], [1, 2, 0]]
        np.testing.assert_allclose(mw, want)


def test_add_self_loop_edge_appends_without_dedup():
    ei = np.array([[0, 1, 1], [1, 1, 0]], dtype=np.int32)       # holds the loop (1,1) already
    idx, w = o.add_self_loop_edge(ei, 3, np.ones(3, np.float32), fill_weight=2.0)
    assert idx.tolist() == [[0, 1, 1, 0, 1, 2], [1, 1, 0, 0, 1, 2]]
    assert w.tolist() == [1, 1, 1, 2, 2, 2] and idx.dtype == np.int32 and w.dtype == np.float32


@pytest.mark.parametrize("norm,loop,sym,renorm,improved", [
    ("both", True, True, True, False), ("both", True, True, False, False), ("both", True, False, True, True),
    ("both", False, False, False, False), ("left", True, False, True, False), ("right", True, False, True, False),
    ("left", False, False, True, False)])
def test_gcn_norm_against_dense_float64(norm, loop, sym, renorm, improved):
    n = 40
    ei = random_graph(n, 300, seed=11, symmetric=sym, isolated=2)
    w = (np.random.RandomState(5).rand(ei.shape[1]) + 0.1).astype(np.float32)
    normed = o.gcn_norm_adj(o.SparseMatrix(ei, w, [n, n]), norm, loop, sym, renorm, improved)
    a = np.zeros((n, n))
    np.add.at(a, (ei[0], ei[1]), w.astype(np.float64))
    fill = 2.0 if improved else 1.0
    eye = np.eye(n) * fill

    def inv_pow(d, p):
        with np.errstate(divide="ignore"):
            r = np.power(d, p)
        r[~np.isfinite(r)] = 0
        return r
    if norm == "both":
        if loop and renorm:
            a = a + eye
        dr = inv_pow(a.sum(1), -0.5)
        dc = dr if sym else inv_pow(a.sum(0), -0.5)
        want = dr[:, None] * a * dc[None, :]
        if loop and not renorm:
            want = want + eye
    else:
        if loop:
            a = a + eye
        d = inv_pow(a.sum(1), -1.0)
        want = d[:, None] * a if norm == "left" else a * d[None, :]
    assert_close(normed.to_dense(), want, rtol=1e-5, atol_scale=1e-6, what="gcn_norm " + norm)


def test_gat_against_dense_float64():
    rs = np.random.RandomState(0)
    n, f, a, u, heads = 30, 12, 16, 8, 4
    ei = random_graph(n, 200, seed=2)
    x = rs.randn(n, f).astype(np.float32)
    wq, wk, wv = glorot(rs, f, a), glorot(rs, f, a), glorot(rs, f, u)
    bq, bk, b = rs.randn(a).astype(np.float32) * .1, rs.randn(a).astype(np.float32) * .1, rs.randn(u).astype(np.float32)
    got = o.gat(x, ei, wq, bq, o.relu, wk, bk, o.relu, wv, b, o.relu, num_heads=heads)
    x64 = x.astype(np.float64)
    q = np.maximum(x64 @ wq + bq, 0)
    k = np.maximum(x64 @ wk + bk, 0)
    v = x64 @ wv
    full = np.concatenate([ei, np.stack([np.arange(n), np.arange(n)])], axis=1)
    want = np.zeros((n, u))
    dq, dv = a // heads, u // heads
    for h in range(heads):
        for r in range(n):
            es = np.where(full[0] == r)[0]
            s = np.array([q[r, h * dq:(h + 1) * dq] @ k[full[1][e], h * dq:(h + 1) * dq] for e in es]) / np.sqrt(dq)
            p = np.exp(s - s.max())
            p = p / p.sum()
            want[r, h * dv:(h + 1) * dv] = sum(p[i] * v[full[1][e], h * dv:(h + 1) * dv] for i, e in enumerate(es))
    want = np.maximum(want + b, 0)
    assert_close(got, want, rtol=1e-4, atol_scale=1e-5, what="gat oracle vs dense f64")


def test_spmm_oracle_against_dense_float64():
    rs = np.random.RandomState(3)
    ei = random_graph(64, 700, seed=4)
    w = rs.rand(ei.shape[1]).astype(np.float32)
    h = rs.randn(64, 10).astype(np.float32)
    got = o.SparseMatrix(ei, w, [64, 64]).matmul(h)
    assert_close(got, o.dense_spmm_f64(ei, w, [64, 64], h), rtol=1e-5, atol_scale=1e-6, what="spmm")


def test_c_oracle_is_bit_identical_to_numpy_oracle():
    rs = np.random.RandomState(7)
    n, e, d = 500, 9000, 19
    ei = random_graph(n, e, seed=8, isolated=5, hub=(17, 600))
    w = rs.rand(ei.shape[1]).astype(np.float32)
    h = rs.randn(n, d).astype(np.float32)
    msg = o.gcn_mapper(None, h[ei[1]], w)
    for red, fn in (("sum", o.sum_reducer), ("mean", o.mean_reducer), ("max", o.max_reducer)):
        np.testing.assert_array_equal(c_oracle.aggregate(ei[0], ei[1], w, h, n, red), fn(msg, ei[0], n))
    np.testing.assert_array_equal(c_oracle.aggregate(ei[0], ei[1], None, h, n, "sum"), o.sum_reducer(h[ei[1]], ei[0], n))
    for a, b in zip(c_oracle.csr_build(ei[0], ei[1], n), o.csr_build(ei[0], ei[1], n)):
        np.testing.assert_array_equal(a, b)
    s = rs.randn(ei.shape[1], 4).astype(np.float32)
    want = np.stack([o.segment_softmax(s[:, i], ei[0], n) for i in range(4)], axis=1)
    np.testing.assert_allclose(c_oracle.segment_softmax(s, ei[0], n), want, rtol=1e-6, atol=1e-9)


def test_c_gat_core_matches_numpy_gat():
    rs = np.random.RandomState(9)
    n, f, a, u, heads = 80, 10, 32, 32, 8
    ei = random_graph(n, 600, seed=10)
    x = rs.randn(n, f).astype(np.float32)
    wq, wk, wv = glorot(rs, f, a), glorot(rs, f, a), glorot(rs, f, u)
    zeros = np.zeros(a, np.float32)
    for split in (True, False):
        wv_ = wv if split else glorot(rs, f, u * heads)
        want, att = o.gat(x, ei, wq, zeros, o.relu, wk, zeros, o.relu, wv_, None, None, num_heads=heads,
                          split_value_heads=split, return_attention=True)
        full, _ = o.add_self_loop_edge(ei, n)
        q = o.relu((x @ wq).astype(np.float32))
        k = o.relu((x @ wk).astype(np.float32))
        v = (x @ wv_).astype(np.float32)
        got, att_c = c_oracle.gat_core(full[0], full[1], q, k, v, heads, split, return_attention=True)
        assert_close(got, want, rtol=1e-5, atol_scale=1e-6, what="gat core")
        np.testing.assert_allclose(att_c, att, rtol=1e-5, atol=1e-8)


def test_gat_attention_reference_matches_c_oracle_and_port():
    """port.gat_attention, the float64 reference of tests/test_gpu_gat_backward.py: its forward is the C oracle's attention
    core and the core of port.gat_forward, it takes destination rows without edges and fewer destinations than sources
    (the set2set layout), and its autograd gradients agree with finite differences."""
    import torch
    from oracle import torch_cpu_port as port
    rs = np.random.RandomState(11)
    n, f = 90, 10
    full, _ = o.add_self_loop_edge(random_graph(n, 700, seed=12, isolated=3), n)
    row, col = torch.from_numpy(full[0].astype(np.int64)), torch.from_numpy(full[1].astype(np.int64))
    t = lambda a: torch.from_numpy(np.asarray(a, np.float64))       # noqa: E731
    for heads, a, u in ((8, 32, 32), (4, 16, 24), (1, 8, 8)):
        x = rs.randn(n, f).astype(np.float32)
        wq, wk, wv = glorot(rs, f, a), glorot(rs, f, a), glorot(rs, f, u)
        bq, bk, bias = (rs.randn(k).astype(np.float32) * .1 for k in (a, a, u))
        q = o.relu((x @ wq + bq).astype(np.float32))
        k = o.relu((x @ wk + bk).astype(np.float32))
        v = (x @ wv).astype(np.float32)
        got = port.gat_attention(t(q), t(k), t(v), row, col, n, heads).numpy()
        assert_close(got, c_oracle.gat_core(full[0], full[1], q, k, v, heads), rtol=1e-5, atol_scale=1e-6,
                     what="gat_attention vs C gat core")
        x64 = t(x)
        want = port.gat_forward(x64, row, col, t(wq), t(bq), t(wk), t(bk), t(wv), t(bias), heads, relu=True)
        got = port.gat_attention(torch.relu(x64 @ t(wq) + t(bq)), torch.relu(x64 @ t(wk) + t(bk)), x64 @ t(wv), row, col, n,
                                 heads, bias=t(bias), relu=True)
        np.testing.assert_allclose(got.numpy(), want.numpy(), rtol=1e-12, atol=1e-12)

    # 4 destinations over 7 sources, destination 2 without edges, source 6 never gathered; H = 2, dqk = 2, dv = 3
    row = torch.tensor([0, 0, 1, 1, 1, 3, 3, 3, 0])
    col = torch.tensor([0, 3, 1, 2, 5, 4, 0, 3, 3])
    args = tuple(torch.tensor(rs.randn(*s), requires_grad=True) for s in ((4, 4), (7, 4), (7, 6), (6,)))
    out = port.gat_attention(*args[:3], row, col, 4, 2, bias=args[3]).detach().numpy()
    np.testing.assert_allclose(out[2], args[3].detach().numpy(), rtol=0, atol=0)
    torch.autograd.gradcheck(lambda Q, K, V, b: port.gat_attention(Q, K, V, row, col, 4, 2, scale=0.7, bias=b), args)


def test_graph_sage_quirks():
    rs = np.random.RandomState(1)
    n, f, u = 20, 6, 4
    ei = random_graph(n, 90, seed=12, symmetric=True)
    x = rs.randn(n, f).astype(np.float32)
    w = rs.rand(ei.shape[1]).astype(np.float32) + 0.5
    ws, wn, b = glorot(rs, f, u), glorot(rs, f, u), rs.randn(2 * u).astype(np.float32)
    # the pooling variants ignore the VALUES of edge_weight (replaced by ones) but crash on None
    wm, bm, wk = glorot(rs, f, 4 * u), rs.randn(4 * u).astype(np.float32), glorot(rs, 4 * u, u)
    a = o.max_pool_graph_sage(x, ei, w, ws, wm, wk, bm, b, o.relu)
    bb = o.max_pool_graph_sage(x, ei, np.ones_like(w), ws, wm, wk, bm, b, o.relu)
    np.testing.assert_array_equal(a, bb)
    with pytest.raises(Exception):
        o.mean_pool_graph_sage(x, ei, None, ws, wm, wk, bm, b, o.relu)
    # gcn_graph_sage: cache=None -> renorm False (normalise, THEN add I); non-empty dict -> renorm trick
    k = glorot(rs, f, u)
    no_cache = o.gcn_graph_sage(x, ei, w, k, cache=None)
    with_cache = o.gcn_graph_sage(x, ei, w, k, cache={"x": 1})
    assert np.abs(no_cache - with_cache).max() > 1e-3
    ones = np.ones(ei.shape[1], np.float32)
    adj = o.SparseMatrix(ei, ones, [n, n])
    want = (o.gcn_norm_adj(adj, renorm=False).matmul(x) @ k).astype(np.float32)
    assert_close(no_cache, want, rtol=1e-6, atol_scale=1e-7, what="gcn_graph_sage renorm quirk")


def test_golden_reference_execution_files_match_oracle():
    """tests/golden/ref_exec_*.npz were produced by running the reference's own Python functions over a numpy shim of
    the TF ops (tools/gen_golden_from_reference.py).  The oracle must reproduce them."""
    files = sorted(f for f in os.listdir(GOLDEN) if f.startswith("ref_exec_") and f.endswith(".npz")) \
        if os.path.isdir(GOLDEN) else []
    if not files:
        pytest.skip("golden files not generated yet")
    from golden_cases import replay_with_oracle
    for f in files:
        data = np.load(os.path.join(GOLDEN, f), allow_pickle=False)
        replay_with_oracle(f, data)


def test_fixture_generator_shim_is_independent_of_the_oracle():
    """The ref_exec_* fixtures pin the oracle only if the TF / tf_sparse stand-ins that executed the reference were written
    without it: tools/ref_shim must not import (or name) the checker, and loading it must not pull `oracle` into the
    interpreter.  Checked in a fresh interpreter."""
    import subprocess
    import sys
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    shim = os.path.join(root, "tools", "ref_shim")
    for name in os.listdir(shim):
        if name.endswith(".py"):
            text = open(os.path.join(shim, name)).read()
            assert "import oracle" not in text and "from oracle" not in text and "tfg_oracle" not in text, name
    code = ("import sys; sys.path.insert(0, {!r}); import ref_shim; "
            "bad = [m for m in sys.modules if m == 'oracle' or m.startswith('oracle.') or m.startswith('tf_geometric_b200')]; "
            "print(bad); sys.exit(1 if bad else 0)").format(os.path.join(root, "tools"))
    res = subprocess.run([sys.executable, "-c", code], capture_output=True, text=True, cwd=root)
    assert res.returncode == 0, res.stdout + res.stderr


def test_philox_known_answers_and_uniform_draws():
    """Philox4x32-10 against the Random123 known-answer vectors (counter, key -> output); the kernels in
    tf_geometric_b200/csrc/rng.cuh implement the same function and are compared with the oracle bit for bit on the GPU."""
    counter = np.array([[0, 0, 0, 0], [0xFFFFFFFF] * 4, [0x243F6A88, 0x85A308D3, 0x13198A2E, 0x03707344]], np.uint32)
    key = np.array([[0, 0], [0xFFFFFFFF] * 2, [0xA4093822, 0x299F31D0]], np.uint32)
    want = np.array([[0x6627E8D5, 0xE169C58D, 0xBC57AC4C, 0x9B00DBD8], [0x408F276D, 0x41C83B0E, 0xA20BC7C6, 0x6D5451FD],
                     [0xD16CFE09, 0x94FDCCEB, 0x5001E420, 0x24126EA1]], np.uint32)
    np.testing.assert_array_equal(o.philox4x32(counter, key), want)
    idx = np.arange(200000, dtype=np.uint64)
    u = o.random_uniform(42, 0, idx)
    assert u.dtype == np.float32 and u.min() >= 0.0 and u.max() < 1.0
    assert abs(u.mean() - 0.5) < 5e-3 and abs((u < 0.1).mean() - 0.1) < 5e-3
    assert abs(np.corrcoef(u[:-1], u[1:])[0, 1]) < 0.01
    assert not np.array_equal(u, o.random_uniform(43, 0, idx)) and not np.array_equal(u, o.random_uniform(42, 1, idx))
    np.testing.assert_array_equal(o.random_u32(42, 0, idx[4:8]), o.philox4x32(np.array([[1, 0, 0, 0]], np.uint32),
                                                                            np.array([[42, 0]], np.uint32))[0])
    b = o.random_below(7, 1, idx, 10)
    assert b.min() == 0 and b.max() == 9 and abs(np.bincount(b).std() / np.bincount(b).mean()) < 0.02


def test_dropout_and_drop_edge_semantics():
    x = np.random.RandomState(0).randn(50000).astype(np.float32)
    y = o.dropout(x, 0.2, seed=9)
    kept = y != 0
    assert abs(kept.mean() - 0.8) < 0.01
    np.testing.assert_array_equal(y[kept], (x * (np.float32(1) / np.float32(0.8)))[kept])
    np.testing.assert_array_equal(o.dropout(x, 0.0, seed=9), x)
    ei = np.array([[0, 1, 1, 2, 3, 0], [1, 0, 2, 1, 3, 3]], np.int32)
    out = o.drop_edge([ei, np.arange(6)], 0.0, force_undirected=True, training=True)
    np.testing.assert_array_equal(out[0], [[0, 1, 0, 1, 2, 3], [1, 2, 3, 0, 1, 0]])       # row<col edges, then mirrored
    np.testing.assert_array_equal(out[1], [0, 2, 5, 0, 2, 5])
    assert o.drop_edge([ei], 0.5, training=False)[0] is ei


def test_sampler_draws_are_uniform_like_numpy_choice():
    """Statistical parity with np.random.choice (graph_utils.py:756): without replacement every neighbour of a node is kept
    with probability k/degree and no neighbour twice; with replacement every draw is uniform over the neighbours."""
    deg, k, trials = 10, 3, 4000
    ei = np.stack([np.zeros(deg, np.int32), np.arange(100, 100 + deg, dtype=np.int32)])
    hits = np.zeros(deg)
    for seed in range(trials):
        si, _ = o.random_neighbor_sample(ei, None, k=k, seed=seed)
        cols = si[1] - 100
        assert len(set(cols.tolist())) == k
        hits[cols] += 1
    # membership is uniform; the ORDER inside a row is that of the reservoir slots, not a uniform permutation like
    # np.random.choice's (documented deviation: order-insensitive aggregators - mean / sum / max - cannot see it)
    assert np.abs(hits / trials - k / deg).max() < 0.03, hits / trials
    draws = np.zeros(deg)
    for seed in range(1000):
        si, _ = o.random_neighbor_sample(ei, None, k=12, padding=True, seed=seed)    # k >= degree: 12 draws with replacement
        assert si.shape[1] == 12
        np.add.at(draws, si[1] - 100, 1)
    assert np.abs(draws / draws.sum() - 1.0 / deg).max() < 0.01, draws / draws.sum()
    # different rows of one call are independent streams
    ei2 = np.stack([np.repeat(np.arange(200, dtype=np.int32), deg), np.tile(np.arange(deg, dtype=np.int32), 200)])
    si, _ = o.random_neighbor_sample(ei2, None, k=1, seed=5)
    assert np.abs(np.bincount(si[1], minlength=deg) / 200.0 - 0.1).max() < 0.08


def test_gat_softmax_bwd_restatement_against_autograd():
    """oracle.gat_softmax_bwd + spmm_heads are the building blocks the GPU backward is compared with; here they are checked
    against torch autograd over the reference's formulation (segment softmax, weighted segment sum)."""
    import torch
    from oracle import torch_cpu_port as port
    rs = np.random.RandomState(4)
    n, e, H, dv = 40, 300, 3, 5
    row = np.sort(rs.randint(0, n, e)).astype(np.int64)
    col = rs.randint(0, n, e).astype(np.int64)
    rowptr = np.concatenate([[0], np.cumsum(np.bincount(row, minlength=n))])
    s = torch.tensor(rs.randn(e, H), requires_grad=True)
    V = torch.tensor(rs.randn(n, H * dv))
    G = rs.randn(n, H * dv)
    rows_t = torch.from_numpy(row)
    att = torch.stack([port.segment_softmax(s[:, h], rows_t, n) for h in range(H)], dim=1)          # [e, H]
    out = torch.zeros((n, H * dv), dtype=torch.float64)
    msg = (V[torch.from_numpy(col)].reshape(e, H, dv) * att.unsqueeze(-1)).reshape(e, H * dv)
    out = out.index_add(0, rows_t, msg)
    (out * torch.tensor(G)).sum().backward()
    got = o.gat_softmax_bwd(rowptr, col, att.detach().numpy().astype(np.float32), G.astype(np.float32),
                            V.numpy().astype(np.float32), H, True)
    assert_close(got, s.grad.numpy(), rtol=1e-4, atol_scale=1e-5, what="d loss / d scores")
    agg = o.spmm_heads(rowptr, col, att.detach().numpy().astype(np.float32), V.numpy().astype(np.float32), H, "split")
    assert_close(agg, out.detach().numpy(), rtol=1e-5, atol_scale=1e-6, what="per-head aggregation")
