#!/usr/bin/env python
# coding=utf-8
"""Generate tests/golden/ref_exec_*.npz, link_exec.npz, cluster_pool_exec.npz, padded_exec.npz and asap_exec.npz by EXECUTING the reference's own Python (a read-only checkout of
CrawlScript/tf_geometric named by $TFG_REFERENCE) over the numpy shims in tools/ref_shim.  The tests never need the
reference: the resulting small fixtures are committed.  Re-run:  TFG_REFERENCE=<checkout> python tools/gen_golden_from_reference.py
"""
import importlib
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))
REFERENCE = os.environ.get("TFG_REFERENCE")
if not REFERENCE:
    raise SystemExit("set TFG_REFERENCE to a checkout of CrawlScript/tf_geometric")
OUT = os.path.join(ROOT, "tests", "golden")

import ref_shim  # noqa: E402

T = ref_shim.install(REFERENCE)
tf = sys.modules["tensorflow"]
tfs = sys.modules["tf_sparse"]
seg = importlib.import_module("tf_geometric.nn.kernel.segment")
mr = importlib.import_module("tf_geometric.nn.kernel.map_reduce")
gu = importlib.import_module("tf_geometric.utils.graph_utils")
gcn_m = importlib.import_module("tf_geometric.nn.conv.gcn")
gat_m = importlib.import_module("tf_geometric.nn.conv.gat")
sage_m = importlib.import_module("tf_geometric.nn.conv.graph_sage")
appnp_m = importlib.import_module("tf_geometric.nn.conv.appnp")
sgc_m = importlib.import_module("tf_geometric.nn.conv.sgc")
ssgc_m = importlib.import_module("tf_geometric.nn.conv.ssgc")
tagcn_m = importlib.import_module("tf_geometric.nn.conv.tagcn")
gin_m = importlib.import_module("tf_geometric.nn.conv.gin")
le_m = importlib.import_module("tf_geometric.nn.conv.le_conv")
sys.modules["tf_geometric.nn.pool"] = type(sys)("tf_geometric.nn.pool")
sys.modules["tf_geometric.nn.pool"].__path__ = [os.path.join(REFERENCE, "tf_geometric", "nn", "pool")]
pool_m = importlib.import_module("tf_geometric.nn.pool.common_pool")
cheb_m = importlib.import_module("tf_geometric.nn.conv.chebynet")


def glorot(rs, a, b):
    lim = np.sqrt(6.0 / (a + b))
    return rs.uniform(-lim, lim, (a, b)).astype(np.float32)


def graph(n, e, seed, symmetric):
    rs = np.random.RandomState(seed)
    if symmetric:
        u, v = rs.randint(0, n, e // 2), rs.randint(0, n, e // 2)
        keep = u != v
        u, v = u[keep], v[keep]
        return np.stack([np.concatenate([u, v]), np.concatenate([v, u])]).astype(np.int32)
    ei = rs.randint(0, n, (2, e)).astype(np.int32)
    ei[0][ei[0] < 3] = 3            # nodes 0..2 have no in-edges (empty segments)
    return ei


def save(name, **arrays):
    os.makedirs(OUT, exist_ok=True)
    np.savez_compressed(os.path.join(OUT, "ref_exec_{}.npz".format(name)),
                        **{k: np.asarray(v) for k, v in arrays.items() if v is not None})
    print("wrote ref_exec_{}.npz: {}".format(name, ", ".join(sorted(arrays))))


def main():
    rs = np.random.RandomState(1234)

    # ---- README fixture (README.md:31-35) + a random multigraph through the integer preprocessing -----------------
    readme_ei = np.array([[0, 0, 1, 3], [1, 2, 2, 1]], np.int32)
    readme_w = np.array([0.9, 0.8, 0.1, 0.2], np.float32)
    d_i, (d_w,) = gu.convert_edge_to_directed(T(readme_ei), [T(readme_w)], merge_modes=["sum"])
    multi = rs.randint(0, 12, (2, 80)).astype(np.int32)
    multi_w = rs.rand(80).astype(np.float32)
    out = {"readme_ei": readme_ei, "readme_w": readme_w, "readme_directed_index": d_i, "readme_directed_w": d_w,
           "multi_ei": multi, "multi_w": multi_w}
    for mode in ("sum", "min", "max", "mean"):
        m_i, (m_w,) = gu.merge_duplicated_edge(T(multi), [T(multi_w)], merge_modes=[mode])
        dd_i, (dd_w,) = gu.convert_edge_to_directed(T(multi), [T(multi_w)], merge_modes=[mode])
        out["merge_{}_index".format(mode)], out["merge_{}_w".format(mode)] = m_i, m_w
        out["directed_{}_index".format(mode)], out["directed_{}_w".format(mode)] = dd_i, dd_w
    sl_i, sl_w = gu.add_self_loop_edge(T(multi), 12, T(multi_w), fill_weight=2.0)
    rm_i, rm_w = gu.remove_self_loop_edge(T(multi), T(multi_w))
    an_i, an_w = gu.adj_norm_edge(T(multi), 12, T(multi_w), add_self_loop=True)
    out.update(self_loop_index=sl_i, self_loop_w=sl_w, no_loop_index=rm_i, no_loop_w=rm_w, adj_norm_index=an_i,
               adj_norm_w=an_w)
    save("graph_utils", **out)

    # ---- segment ops + aggregate_neighbors -----------------------------------------------------------------------------
    n, e, d = 60, 700, 9
    ei = graph(n, e, 5, False)
    x = rs.randn(n, d).astype(np.float32)
    w = rs.rand(ei.shape[1]).astype(np.float32)
    scores = (rs.randn(ei.shape[1]) * 3).astype(np.float32)
    out = {"ei": ei, "x": x, "w": w, "scores": scores, "n": n,
           "segment_softmax": seg.segment_softmax(T(scores), T(ei[0]), n),
           "segment_count": seg.segment_count(T(ei[0]), n)}
    reducers = {"sum": mr.sum_reducer, "mean": mr.mean_reducer, "max": mr.max_reducer}
    for rname, red in reducers.items():
        out["agg_identity_{}_sumupd".format(rname)] = mr.aggregate_neighbors(T(x), T(ei), None, mr.identity_mapper, red,
                                                                             mr.sum_updater, num_nodes=n)
        out["agg_gcn_{}_idupd".format(rname)] = mr.aggregate_neighbors(T(x), T(ei), T(w), gcn_m.gcn_mapper, red,
                                                                        mr.identity_updater, num_nodes=n)
    out["agg_count"] = mr.aggregate_neighbors(T(x), T(ei), None, mr.neighbor_count_mapper, mr.sum_reducer,
                                              mr.identity_updater, num_nodes=n)
    save("kernel", **out)

    # ---- gcn_norm_adj variants and gcn ---------------------------------------------------------------------------------
    n, f, u = 50, 14, 6
    ei_sym, ei_dir = graph(n, 500, 7, True), graph(n, 500, 8, False)
    w_sym = rs.rand(ei_sym.shape[1]).astype(np.float32) + 0.1
    # symmetric weights: mirror halves share a weight
    half = ei_sym.shape[1] // 2
    w_sym[half:] = w_sym[:half]
    w_dir = rs.rand(ei_dir.shape[1]).astype(np.float32) + 0.1
    x = rs.randn(n, f).astype(np.float32)
    kernel, bias = glorot(rs, f, u), rs.randn(u).astype(np.float32)
    out = {"n": n, "ei_sym": ei_sym, "w_sym": w_sym, "ei_dir": ei_dir, "w_dir": w_dir, "x": x, "kernel": kernel, "bias": bias}
    configs = [("both", True, True, True, False), ("both", True, True, True, True), ("both", True, True, False, False),
               ("both", True, False, True, False), ("both", False, False, True, False), ("left", True, False, True, False),
               ("right", True, False, True, False), ("left", False, False, True, False)]
    out["configs"] = np.array(["{}|{}|{}|{}|{}".format(*c) for c in configs])
    for i, (norm, loop, sym, renorm, improved) in enumerate(configs):
        ei_, w_ = (ei_sym, w_sym) if sym else (ei_dir, w_dir)
        adj = tfs.SparseMatrix(T(ei_), T(w_), [n, n])
        cache = {}
        normed = gcn_m.gcn_norm_adj(adj, norm, loop, sym, renorm, improved, cache=cache)
        key = gcn_m.compute_cache_key(norm, loop, sym, renorm, improved)
        assert list(cache.keys()) == [key]
        out["norm{}_index".format(i)], out["norm{}_value".format(i)] = normed.index, normed.value
        out["norm{}_cache_key".format(i)] = np.array(key)
        out["gcn{}_out".format(i)] = gcn_m.gcn(T(x), adj, T(kernel), T(bias), activation=tf.nn.relu, norm=norm,
                                                add_self_loop=loop, sym=sym, renorm=renorm, improved=improved)
    out["gcn_no_kernel"] = gcn_m.gcn(T(x), tfs.SparseMatrix(T(ei_sym), T(w_sym), [n, n]), None, None)
    save("gcn", **out)

    # ---- gat -----------------------------------------------------------------------------------------------------------
    n, f = 40, 10
    ei = graph(n, 300, 9, False)
    ei = np.concatenate([ei, np.array([[5, 5], [5, 5]], np.int32)], axis=1)     # pre-existing self loop, twice
    x = rs.randn(n, f).astype(np.float32)
    out = {"n": n, "ei": ei, "x": x}
    for tag, a, u, heads, split in (("h8", 32, 16, 8, True), ("h4avg", 16, 12, 4, False), ("h1", 8, 8, 1, True),
                                    ("demo", 8, 64, 8, True)):
        wq, wk = glorot(rs, f, a), glorot(rs, f, a)
        wv = glorot(rs, f, u if split else u * heads)
        bq, bk, b = (rs.randn(a) * .1).astype(np.float32), (rs.randn(a) * .1).astype(np.float32), rs.randn(u).astype(np.float32)
        res = gat_m.gat(T(x), T(ei), T(wq), T(bq), tf.nn.relu, T(wk), T(bk), tf.nn.relu, T(wv), T(b), tf.nn.relu,
                        num_heads=heads, split_value_heads=split)
        out.update({tag + "_wq": wq, tag + "_wk": wk, tag + "_wv": wv, tag + "_bq": bq, tag + "_bk": bk, tag + "_b": b,
                    tag + "_heads": heads, tag + "_split": int(split), tag + "_out": res})
    save("gat", **out)

    # ---- graph_sage ----------------------------------------------------------------------------------------------------
    n, f, u = 45, 12, 8
    ei = graph(n, 400, 10, True)
    w = rs.rand(ei.shape[1]).astype(np.float32) + 0.2
    x = rs.randn(n, f).astype(np.float32)
    ws, wn = glorot(rs, f, u), glorot(rs, f, u)
    b2, b1 = rs.randn(2 * u).astype(np.float32), rs.randn(u).astype(np.float32)
    wm, bm, wnk = glorot(rs, f, 4 * u), rs.randn(4 * u).astype(np.float32), glorot(rs, 4 * u, u)
    kernel = glorot(rs, f, u)
    out = {"n": n, "ei": ei, "w": w, "x": x, "ws": ws, "wn": wn, "b2": b2, "b1": b1, "wm": wm, "bm": bm, "wnk": wnk,
           "kernel": kernel}
    out["mean_w_concat_norm"] = sage_m.mean_graph_sage(T(x), T(ei), T(w), T(ws), T(wn), T(b2), tf.nn.relu, True, True)
    out["mean_now_add"] = sage_m.mean_graph_sage(T(x), T(ei), None, T(ws), T(wn), T(b1), tf.nn.relu, False, False)
    out["sum_w_concat"] = sage_m.sum_graph_sage(T(x), T(ei), T(w), T(ws), T(wn), T(b2), None, True, False)
    out["gcn_sage_nocache"] = sage_m.gcn_graph_sage(T(x), T(ei), T(w), T(kernel), T(b1), tf.nn.relu, False, cache=None)
    out["gcn_sage_cache"] = sage_m.gcn_graph_sage(T(x), T(ei), T(w), T(kernel), T(b1), tf.nn.relu, True, cache={"k": 1})
    out["mean_pool"] = sage_m.mean_pool_graph_sage(T(x), T(ei), T(w), T(ws), T(wm), T(wnk), T(bm), T(b2), tf.nn.relu)
    out["max_pool"] = sage_m.max_pool_graph_sage(T(x), T(ei), T(w), T(ws), T(wm), T(wnk), T(bm), T(b2), tf.nn.relu)
    save("graph_sage", **out)

    # ---- appnp ---------------------------------------------------------------------------------------------------------
    n, f = 40, 11
    ei = graph(n, 360, 11, True)
    w = np.ones(ei.shape[1], np.float32)
    x = rs.randn(n, f).astype(np.float32)
    k0, k1 = glorot(rs, f, 16), glorot(rs, 16, 5)
    b0, b1 = rs.randn(16).astype(np.float32), rs.randn(5).astype(np.float32)
    out = {"n": n, "ei": ei, "w": w, "x": x, "k0": k0, "k1": k1, "b0": b0, "b1": b1}
    out["k10"] = appnp_m.appnp(T(x), T(ei), T(w), [T(k0), T(k1)], [T(b0), T(b1)], k=10, alpha=0.1)
    out["k2_relu"] = appnp_m.appnp(T(x), T(ei), T(w), [T(k0), T(k1)], [T(b0), T(b1)], activation=tf.nn.relu, k=2, alpha=0.3)
    save("appnp", **out)

    # ---- sgc / ssgc / tagcn / gin / le_conv (SURVEY.md 8f-1) ------------------------------------------------------------
    n, f, u = 48, 9, 6
    ei = graph(n, 420, 13, True)
    w = rs.rand(ei.shape[1]).astype(np.float32) + 0.3
    w[len(w) // 2:] = w[:len(w) // 2]
    x = rs.randn(n, f).astype(np.float32)
    kernel, bias = glorot(rs, f, u), rs.randn(u).astype(np.float32)
    k0, b0, k1, b1 = glorot(rs, f, 12), rs.randn(12).astype(np.float32), glorot(rs, 12, u), rs.randn(u).astype(np.float32)
    tag_kernel = glorot(rs, f * 4, u)
    mlp_w = glorot(rs, f, u)
    ws, bs = glorot(rs, f, u), rs.randn(u).astype(np.float32)
    wa, ba, wn = glorot(rs, f, u), rs.randn(u).astype(np.float32), glorot(rs, f, u)
    out = {"n": n, "ei": ei, "w": w, "x": x, "kernel": kernel, "bias": bias, "k0": k0, "b0": b0, "k1": k1, "b1": b1,
           "tag_kernel": tag_kernel, "mlp_w": mlp_w, "ws": ws, "bs": bs, "wa": wa, "ba": ba, "wn": wn}
    out["sgc_k2"] = sgc_m.sgc(T(x), T(ei), T(w), 2, T(kernel), T(bias), tf.nn.relu)
    out["sgc_k1_improved"] = sgc_m.sgc(T(x), T(ei), T(w), 1, T(kernel), None, None, renorm=True, improved=True)
    out["ssgc_k5"] = ssgc_m.ssgc(T(x), T(ei), T(w), [T(k0), T(k1)], [T(b0), T(b1)], k=5, alpha=0.2)
    out["ssgc_nokernel"] = ssgc_m.ssgc(T(x), T(ei), T(w), None, None, k=3, alpha=0.1, activation=tf.nn.relu)
    out["tagcn_k3"] = tagcn_m.tagcn(T(x), T(ei), T(w), 3, T(tag_kernel), T(bias), tf.nn.relu)
    mlp = lambda h, training=None: tf.nn.relu(h @ T(mlp_w))      # noqa: E731
    out["gin_eps"] = gin_m.gin(T(x), T(ei), mlp, eps=0.25)
    out["le_conv"] = le_m.le_conv(T(x), T(ei), T(w), T(ws), T(bs), T(wa), T(ba), T(wn), None, tf.nn.relu)
    out["le_conv_now"] = le_m.le_conv(T(x), T(ei), None, T(ws), None, T(wa), None, T(wn), None, None)
    save("propagation", **out)

    # ---- graph pooling (SURVEY.md 8f-2) ----------------------------------------------------------------------------------
    n, d, g = 300, 7, 12
    gi = np.sort(rs.randint(0, g, n)).astype(np.int32)
    gi[gi == 5] = 6                                   # graph 5 is empty
    x = rs.randn(n, d).astype(np.float32)
    out = {"x": x, "gi": gi, "g": g}
    for name in ("mean_pool", "sum_pool", "max_pool", "min_pool"):
        out[name] = getattr(pool_m, name)(T(x), T(gi), g)
    out["mean_pool_auto"] = pool_m.mean_pool(T(x), T(gi))
    save("pool", **out)

    # ---- chebynet ------------------------------------------------------------------------------------------------------------
    n, f, u = 44, 8, 5
    ei = graph(n, 380, 17, True)
    ei = np.concatenate([ei, np.array([[3, 9], [3, 9]], np.int32)], axis=1)      # self loops, removed by chebynet_norm_edge
    w = rs.rand(ei.shape[1]).astype(np.float32) + 0.2
    half = (ei.shape[1] - 2) // 2
    w[half:2 * half] = w[:half]
    x = rs.randn(n, f).astype(np.float32)
    ks = [glorot(rs, f, u) for _ in range(4)]
    bias = rs.randn(u).astype(np.float32)
    out = {"n": n, "ei": ei, "w": w, "x": x, "bias": bias, "k0": ks[0], "k1": ks[1], "k2": ks[2], "k3": ks[3]}
    for tag, kk, nt in (("k1_sym", 1, "sym"), ("k2_sym", 2, "sym"), ("k4_sym", 4, "sym"), ("k3_rw", 3, "rw"), ("k3_none", 3, None)):
        out["cheb_" + tag] = cheb_m.chebynet(T(x), T(ei), T(w), kk, [T(a) for a in ks[:kk]], T(bias), tf.nn.relu, normalization_type=nt)
    ni, nw = cheb_m.chebynet_norm_edge(T(ei), n, T(w), "sym")
    out["norm_index"], out["norm_w"] = ni, nw
    save("chebynet", **out)

    # ---- RandomNeighborSampler: the deterministic branches, and the per-row COUNTS of the random ones ----------------------
    n = 40
    ei = graph(n, 260, 23, False)
    ei[0][ei[0] == 7] = 8                              # node 7 has no neighbours
    w = rs.rand(ei.shape[1]).astype(np.float32)
    sampler = gu.RandomNeighborSampler(ei, w)
    subset = np.array([9, 4, 30, 12, 8, 21, 3, 17, 5, 33], np.int32)
    rows_sub, cols_sub = np.array([8, 3, 11, 30, 25], np.int32), np.array([1, 2, 3, 4, 5, 6, 10, 20, 30], np.int32)
    out = {"n": n, "ei": ei, "w": w, "subset": subset, "rows_sub": rows_sub, "cols_sub": cols_sub}
    for tag, kw in (("all", {}), ("k_big", {"k": 1000}), ("subset_all", {"sampled_node_index": subset}),
                    ("pair_k_big", {"sampled_node_index": (rows_sub, cols_sub), "k": 1000})):
        si, sw = sampler.sample(**kw)
        out[tag + "_index"], out[tag + "_w"] = si, sw
    np.random.seed(0)
    for tag, kw in (("k3", {"k": 3}), ("k3_pad", {"k": 3, "padding": True}), ("k9_pad", {"k": 9, "padding": True}),
                    ("ratio", {"ratio": 0.4}), ("subset_k2", {"k": 2, "sampled_node_index": subset})):
        si, _ = sampler.sample(**kw)
        rows_out = int(si[0].max()) + 1
        out[tag + "_counts"] = np.bincount(si[0], minlength=rows_out)
    save("sampler", **out)

    # ---- pooling beyond the segment reductions: topk_pool, set2set (the LSTM is an ARGUMENT of the reference function) ---
    topk_m = importlib.import_module("tf_geometric.nn.pool.topk_pool")
    s2s_m = importlib.import_module("tf_geometric.nn.pool.set2set")
    from oracle import tfg_oracle as oracle_mod
    n, g, d = 180, 9, 6
    gi = rs.randint(0, g, n).astype(np.int32)
    gi[gi == 4] = 3                                            # graph 4 is empty
    gi[:3] = g - 1                                             # the last graph exists
    score = rs.randn(n).astype(np.float32)
    out = {"gi": gi, "score": score}
    for tag, kw in (("k1", {"k": 1}), ("k5", {"k": 5}), ("k1000", {"k": 1000}), ("r30", {"ratio": 0.3}), ("r100", {"ratio": 1.0})):
        out["topk_" + tag] = topk_m.topk_pool(T(gi), T(score), **kw)
    out["topk_col_r50"] = topk_m.topk_pool(T(gi), T(score.reshape(-1, 1)), ratio=0.5)
    x = rs.randn(n, d).astype(np.float32)
    gi_sorted = np.sort(gi)
    lstm_k, lstm_r, lstm_b = glorot(rs, 2 * d, 4 * d), glorot(rs, d, 4 * d), (rs.randn(4 * d) * 0.1).astype(np.float32)
    np_lstm = oracle_mod.numpy_lstm(lstm_k, lstm_r, lstm_b)

    def shim_lstm(inputs, initial_state=None, training=None):
        seq, h, c = np_lstm(np.asarray(inputs), [np.asarray(s) for s in initial_state], training)
        return T(seq), T(h), T(c)
    out.update(x=x, gi_sorted=gi_sorted, lstm_k=lstm_k, lstm_r=lstm_r, lstm_b=lstm_b)
    out["set2set_it3"] = s2s_m.set2set(T(x), T(gi_sorted), shim_lstm, 3)
    out["set2set_unsorted_it2"] = s2s_m.set2set(T(x), T(gi), shim_lstm, 2)
    save("pool2", **out)

    # ---- Graph / BatchGraph: induced subgraphs, batching, and the pooling functions built on them --------------------------
    import types as _types
    data_pkg = _types.ModuleType("tf_geometric.data")
    data_pkg.__path__ = [os.path.join(REFERENCE, "tf_geometric", "data")]
    sys.modules["tf_geometric.data"] = data_pkg
    graph_m = importlib.import_module("tf_geometric.data.graph")
    sag_m = importlib.import_module("tf_geometric.nn.pool.sag_pool")
    sort_m = importlib.import_module("tf_geometric.nn.pool.sort_pool")
    n, g = 90, 7
    ei = graph(n, 700, 31, False)
    w = rs.rand(ei.shape[1]).astype(np.float32)
    x = rs.randn(n, 5).astype(np.float32)
    y = rs.randint(0, 4, n).astype(np.int32)
    gi = np.sort(rs.randint(0, g, n)).astype(np.int32)
    gi[-1] = g - 1
    keep = rs.permutation(n)[:35].astype(np.int32)
    out = {"n": n, "ei": ei, "w": w, "x": x, "y": y, "gi": gi, "keep": keep}
    sub = graph_m.BatchGraph(T(x), T(ei), T(gi), None, y=T(y), edge_weight=T(w)).sample_new_graph_by_node_index(T(keep))
    out.update(sub_x=sub.x, sub_ei=sub.edge_index, sub_w=sub.edge_weight, sub_gi=sub.node_graph_index, sub_y=sub.y)
    sub_np = graph_m.Graph(x, ei, y=y, edge_weight=w).sample_new_graph_by_node_index(keep)        # numpy container path
    out.update(subnp_x=sub_np.x, subnp_ei=sub_np.edge_index, subnp_w=sub_np.edge_weight)
    score = rs.randn(n, 1).astype(np.float32)
    out["score"] = score
    for tag, kw in (("k4", {"k": 4}), ("r50", {"ratio": 0.5})):
        px, pei, pw, pgi = sag_m.sag_pool(T(x), T(ei), T(w), T(gi), lambda inputs, training=None: T(score),
                                          score_activation=lambda v: T(np.tanh(np.asarray(v))), **kw)
        out.update({"sag_%s_x" % tag: px, "sag_%s_ei" % tag: pei, "sag_%s_w" % tag: pw, "sag_%s_gi" % tag: pgi})
        px, pei, pw, pgi = sort_m.sort_pool(T(x), T(ei), T(w), T(gi), sort_index=1, **kw)
        out.update({"sort_%s_x" % tag: px, "sort_%s_ei" % tag: pei, "sort_%s_w" % tag: pw, "sort_%s_gi" % tag: pgi})
    parts = []
    for i, size in enumerate((4, 1, 6)):
        pe = graph(size, 3 * size, 40 + i, False) % size if size > 1 else np.zeros((2, 0), np.int32)
        parts.append((rs.randn(size, 3).astype(np.float32), pe.astype(np.int32), rs.rand(pe.shape[1]).astype(np.float32),
                      (np.arange(size) + 10 * i).astype(np.int32)))
    bg = graph_m.BatchGraph.from_graphs([graph_m.Graph(T(px_), T(pe_), y=T(py_), edge_weight=T(pw_)) for px_, pe_, pw_, py_ in parts])
    for i, (px_, pe_, pw_, py_) in enumerate(parts):
        out.update({"part%d_x" % i: px_, "part%d_ei" % i: pe_, "part%d_w" % i: pw_, "part%d_y" % i: py_})
    out.update(batch_x=bg.x, batch_ei=bg.edge_index, batch_w=bg.edge_weight, batch_y=bg.y, batch_gi=bg.node_graph_index,
               batch_egi=bg.edge_graph_index)
    save("graph", **out)

    # ---- link prediction: negative_sampling, edge_train_test_split, negative_sampling_with_start_node ------------------
    # tests/golden/link_exec.npz: the reference's full negative candidate list in its own order, the split sizes with the
    # merged upper edges and their max weights, and start-node samples (whose draws only allow property checks).
    # Own RandomState (and np.random seeds of its own), so adding this section leaves every fixture above unchanged.
    lrs = np.random.RandomState(2024)
    n = 30
    ei = graph(n, 150, 61, True)
    ei = np.concatenate([ei, np.array([[4, 9, 9], [4, 2, 2]], np.int32)], axis=1)     # a self loop and a duplicate
    w = lrs.rand(ei.shape[1]).astype(np.float32)
    up, _ = gu.convert_edge_to_upper(ei)
    num_cand = n * (n - 1) // 2 - int(len(set(zip(up[0][up[0] < up[1]].tolist(), up[1][up[0] < up[1]].tolist()))))
    # replace=False with num_samples = C draws a permutation of the candidate list with np.random.choice; replaying
    # the seeded choice recovers the list in the reference's own (row-major np.nonzero) order
    np.random.seed(11)
    neg = gu.negative_sampling(num_cand, n, ei, replace=False)
    np.random.seed(11)
    p = np.random.choice(list(range(num_cand)), num_cand, replace=False)
    cand = np.empty_like(neg)
    cand[:, p] = neg
    out = {"n": n, "ei": ei, "w": w, "candidates": cand}
    np.random.seed(12)
    tr_i, te_i, tr_w, te_w = gu.edge_train_test_split(ei, 0.2, edge_weight=w)
    out.update(split_train_index=tr_i, split_test_index=te_i, split_train_w=tr_w, split_test_w=te_w)
    np.random.seed(13)
    tr_i, te_i, _, _ = gu.edge_train_test_split(ei, 7)
    out.update(split7_train_index=tr_i, split7_test_index=te_i)
    start = lrs.randint(0, n, 40).astype(np.int32)
    np.random.seed(14)
    out.update(start=start, start_sample=gu.negative_sampling_with_start_node(start, n, ei))
    # named apart from ref_exec_*: those are replayed case by case through tests/golden_cases.py, while this one is read
    # by tests/test_link_host.py and tests/test_gpu_link.py
    np.savez_compressed(os.path.join(OUT, "link_exec.npz"), **{k: np.asarray(v) for k, v in out.items()})
    print("wrote link_exec.npz: {}".format(", ".join(sorted(out))))

    # ---- DiffPool / MinCutPool: nn/pool/{cluster_pool,diff_pool,min_cut_pool}.py and utils convert_dense_* -----------
    # tests/golden/cluster_pool_exec.npz (read by tests/test_cluster_pool_host.py and tests/test_gpu_cluster_pool.py).  The
    # sub-GNNs are arguments of the reference functions: simple deterministic callables, restated in
    # tests/cluster_pool_ref.py.  Own RandomState, so the fixtures above are unchanged.
    cluster_pool_fixture()

    # ---- convert_x_to_3d and lstm_graph_sage: utils/graph_utils.py:215-249, nn/conv/graph_sage.py:290-356 -----------
    # tests/golden/padded_exec.npz (read by tests/test_padded_host.py and tests/test_gpu_padded.py).  Own RandomState.
    padded_fixture()

    # ---- cluster_pool with a sparse assignment and ASAP: nn/pool/cluster_pool.py, nn/pool/asap.py ------------------------
    # tests/golden/asap_exec.npz (read by tests/test_asap_host.py and tests/test_gpu_asap.py).  Own RandomState.
    asap_fixture()


def asap_fixture():
    cp_m = importlib.import_module("tf_geometric.nn.pool.cluster_pool")
    sys.modules["tf_geometric.nn"].max_pool = pool_m.max_pool           # asap.py: from tf_geometric.nn import max_pool
    asap_m = importlib.import_module("tf_geometric.nn.pool.asap")
    ars = np.random.RandomState(321)
    out = {}
    # cluster_pool, assignment [node, cluster]: duplicates in S ((2, 1) twice) and in A ((2, 3) twice), node 6 in no
    # cluster, cluster 3 empty, a self loop (3, 3), and the zero-weight edge (3, 5) whose pooled entry (1, 2) is exactly 0
    ei = np.array([[0, 1, 2, 2, 3, 3, 4, 5, 1], [1, 2, 3, 3, 3, 5, 0, 4, 0]], np.int32)
    w = np.array([1.0, 0.5, 2.0, 2.0, 1.5, 0.0, 0.75, 1.25, -1.0], np.float32)
    aei = np.array([[0, 1, 2, 2, 3, 4, 5, 0], [0, 0, 1, 1, 1, 2, 2, 2]], np.int32)
    aw = ars.uniform(0.1, 2.0, aei.shape[1]).astype(np.float32)
    x = ars.randn(7, 3).astype(np.float32)
    out.update(cp_ei=ei, cp_w=w, cp_aei=aei, cp_aw=aw, cp_x=x)
    for tag, ew, aew in (("w", T(w), T(aw)), ("none", None, None)):
        px, pei, pw = cp_m.cluster_pool(T(x), T(ei), ew, T(aei), aew, 4)
        out.update({"cp_%s_%s" % (tag, k): v for k, v in zip(("x", "ei", "w"), (px, pei, pw))})

    # asap.py with its two call sites read the one way that runs (DESIGN.md section 5 (9)):
    #   adapter 1: gcn(x, edge_index, edge_weight, kernel, bias) (asap.py:54) is the edge-list GCN, as layers/conv/gcn.py
    #              reads [x, edge_index, edge_weight] inputs;
    #   adapter 2: the assignment stacked as [cluster, node] (asap.py:107-115) reaches cluster_pool as [node, cluster].
    asap_m.gcn = lambda x_, ei_, ew_, k_, b_=None, cache=None: gcn_m.gcn(
        x_, tfs.SparseMatrix(ei_, ew_, [np.shape(x_)[0]] * 2), k_, b_, cache=cache)

    def cluster_pool_node_cluster(x_, ei_, ew_, aei_, aew_, k_, num_nodes=None):
        return cp_m.cluster_pool(x_, ei_, ew_, T(np.asarray(aei_)[::-1].copy()), aew_, k_, num_nodes=num_nodes)
    asap_m.cluster_pool = cluster_pool_node_cluster

    # graphs of 7, 1 (edgeless), 9 and 5 nodes, relabelled so that node_graph_index is unsorted; duplicates, self loops
    sizes, f = [7, 1, 9, 5], 4
    rows, cols, base = [], [], 0
    for size in sizes:
        if size > 1:
            e = ars.randint(0, size, (2, 3 * size))
            rows += list(base + e[0]) + [base + e[0, 0]]
            cols += list(base + e[1]) + [base + e[1, 0]]
        base += size
    n = base
    perm = ars.permutation(n)
    inv = np.empty_like(perm)
    inv[perm] = np.arange(n)
    ei = inv[np.array([rows, cols])].astype(np.int32)
    gi = np.repeat(np.arange(len(sizes)), sizes)[perm].astype(np.int32)
    w = ars.uniform(0.5, 1.5, ei.shape[1]).astype(np.float32)
    x = ars.randn(n, f).astype(np.float32)
    names = ("attention_gcn_kernel", "attention_gcn_bias", "attention_query_kernel", "attention_query_bias",
             "attention_score_kernel", "attention_score_bias", "le_conv_self_kernel", "le_conv_self_bias",
             "le_conv_aggr_self_kernel", "le_conv_aggr_self_bias", "le_conv_aggr_neighbor_kernel")
    shapes = ((f, f), (f,), (f, f), (f,), (2 * f, 1), (1,), (f, 1), (1,), (f, 1), (1,), (f, 1))
    params = [glorot(ars, *s) if len(s) == 2 else (ars.randn(*s) * 0.1).astype(np.float32) for s in shapes]
    out.update(asap_ei=ei, asap_w=w, asap_x=x, asap_gi=gi, **{"asap_p_" + k: v for k, v in zip(names, params)})
    for tag, ew, kw in (("r50_w", T(w), {"ratio": 0.5}), ("r50_none", None, {"ratio": 0.5}), ("k2_w", T(w), {"k": 2}),
                        ("k3_none", None, {"k": 3})):
        res = asap_m.asap(T(x), T(ei), ew, T(gi), *[T(p) for p in params], None, training=False, **kw)
        out.update({"asap_%s_%s" % (tag, k): v for k, v in zip(("x", "ei", "w", "gi"), res)})
    np.savez_compressed(os.path.join(OUT, "asap_exec.npz"), **{k: np.asarray(v) for k, v in out.items()})
    print("wrote asap_exec.npz: {}".format(", ".join(sorted(out))))


def padded_fixture():
    prs = np.random.RandomState(99)
    out = {}
    # unsorted source ids with a gap (id 2 never appears): groups of sizes 3, 1, 0, 4, 2
    sid = prs.permutation(np.repeat(np.array([0, 1, 3, 4], np.int32), [3, 1, 4, 2])).astype(np.int32)
    x3 = prs.randn(sid.shape[0], 3).astype(np.float32)
    out.update(x3d_x=x3, x3d_sid=sid)
    for tag, kw in (("none", {}), ("k2", {"k": 2}), ("k6_pad", {"k": 6, "pad": True}), ("k6_nopad", {"k": 6, "pad": False})):
        out["x3d_" + tag] = gu.convert_x_to_3d(T(x3), T(sid), **kw)
    # a graph with an isolated node (0), a duplicate edge and a self loop; the LSTM is oracle.numpy_lstm behind the Keras
    # return_sequences=True convention with a zero initial state
    from oracle import tfg_oracle as oracle_mod
    n, f, u = 12, 5, 4
    ei = prs.randint(1, n, (2, 30)).astype(np.int32)
    ei = np.concatenate([ei, ei[:, :1], np.array([[5], [5]], np.int32)], axis=1)
    x = prs.randn(n, f).astype(np.float32)
    w = prs.rand(ei.shape[1]).astype(np.float32)
    lstm_k, lstm_r = glorot(prs, f, 4 * u), glorot(prs, u, 4 * u)
    lstm_b = (prs.randn(4 * u) * 0.1).astype(np.float32)
    np_lstm = oracle_mod.numpy_lstm(lstm_k, lstm_r, lstm_b)

    def keras_lstm(inputs, training=None):
        zeros = np.zeros((np.shape(inputs)[0], u), np.float32)
        return T(np_lstm(np.asarray(inputs), [zeros, zeros], training)[0])
    out.update(lstm_ei=ei, lstm_x=x, lstm_w=w, lstm_k=lstm_k, lstm_r=lstm_r, lstm_b=lstm_b)
    for concat in (True, False):
        ws, wn = glorot(prs, f, u), glorot(prs, u, u)
        bias = (prs.randn(2 * u if concat else u) * 0.1).astype(np.float32)
        tag = "concat" if concat else "sum"
        out.update({"lstm_%s_ws" % tag: ws, "lstm_%s_wn" % tag: wn, "lstm_%s_bias" % tag: bias})
        out["lstm_%s_relu" % tag] = sage_m.lstm_graph_sage(T(x), T(ei), keras_lstm, T(ws), T(wn), bias=T(bias),
                                                           activation=tf.nn.relu, concat=concat)
        out["lstm_%s_l2" % tag] = sage_m.lstm_graph_sage(T(x), T(ei), keras_lstm, T(ws), T(wn), bias=T(bias),
                                                         concat=concat, normalize=True)
    np.savez_compressed(os.path.join(OUT, "padded_exec.npz"), **{k: np.asarray(v) for k, v in out.items()})
    print("wrote padded_exec.npz: {}".format(", ".join(sorted(out))))


def golden_gnn(weight, mix):
    """[x, edge_index, edge_weight] -> x W + sum_{e: row_e = r} w_e (x M)[col_e], then tanh when it is a feature GNN."""
    def gnn(inputs, training=None, cache=None):
        x, ei, w = (np.asarray(a) for a in inputs)
        h, m = (x @ weight).astype(np.float32), (x @ mix).astype(np.float32)
        agg = np.zeros_like(m)
        for e in range(ei.shape[1]):
            agg[ei[0, e]] = agg[ei[0, e]] + w[e] * m[ei[1, e]]
        return T((h + agg).astype(np.float32))
    return gnn


def cluster_pool_fixture():
    diff_m = importlib.import_module("tf_geometric.nn.pool.diff_pool")
    mc_m = importlib.import_module("tf_geometric.nn.pool.min_cut_pool")
    crs = np.random.RandomState(77)
    sizes = [6, 3, 8, 5]                                       # graph 1 has no edge
    rows, cols, base = [], [], 0
    for g, size in enumerate(sizes):
        if g != 1:
            half = 2 * size
            u, v = crs.randint(0, size, half), crs.randint(0, size, half)
            keep = u != v
            rows += list(base + u[keep]) + list(base + v[keep])
            cols += list(base + v[keep]) + list(base + u[keep])
        base += size
    rows += [rows[0], 0, 10]                                   # a duplicate of edge 0 and two self loops
    cols += [cols[0], 0, 10]
    n = base
    gi_sorted = np.repeat(np.arange(len(sizes)), sizes).astype(np.int32)
    perm = crs.permutation(n)                                  # node p of the batch is sorted node perm[p]: unsorted gi
    inv = np.empty_like(perm)
    inv[perm] = np.arange(n)
    ei = inv[np.array([rows, cols])].astype(np.int32)
    gi = gi_sorted[perm].astype(np.int32)
    w = (crs.rand(ei.shape[1]) + 0.3).astype(np.float32)
    f_in, f_out = 4, 5
    x = crs.randn(n, f_in).astype(np.float32)
    out = {"x": x, "ei": ei, "w": w, "gi": gi}
    for c in (3, 1):
        wf, mf = glorot(crs, f_in, f_out), glorot(crs, f_in, f_out)
        wa, ma = glorot(crs, f_in, c), glorot(crs, f_in, c)
        bias = (crs.randn(f_out) * 0.1).astype(np.float32)
        out.update({"wf_c%d" % c: wf, "mf_c%d" % c: mf, "wa_c%d" % c: wa, "ma_c%d" % c: ma, "bias_c%d" % c: bias})
        feat, assign = golden_gnn(wf, mf), golden_gnn(wa, ma)
        relu = tf.nn.relu
        cases = {"diff": lambda ew: diff_m.diff_pool(T(x), T(ei), ew, T(gi), feat, assign, c, bias=T(bias), activation=relu)}
        for tag, ew in (("w", T(w)), ("none", None)):
            px, pei, pw, pgi = cases["diff"](ew)
            out.update({"diff_%s_c%d_%s" % (tag, c, k): v for k, v in zip(("x", "ei", "w", "gi"), (px, pei, pw, pgi))})
        for tag, normed in (("normed", True), ("raw", False)):
            (px, pei, pw, pgi), (cut, orth) = mc_m.min_cut_pool(T(x), T(ei), T(w), T(gi), feat, assign, c, bias=T(bias),
                                                                 activation=relu, gnn_use_normed_edge=normed,
                                                                 return_losses=True)
            out.update({"mincut_%s_c%d_%s" % (tag, c, k): v
                        for k, v in zip(("x", "ei", "w", "gi", "cut", "orth"), (px, pei, pw, pgi, cut, orth))})
    dense = crs.randn(5, 5).astype(np.float32)
    dense[dense < 0.2] = 0.0
    dense[1, 3] = np.nan
    out["dense_adj"] = dense
    out["dense_adj_ei"], out["dense_adj_w"] = gu.convert_dense_adj_to_edge(T(dense))
    assign = crs.rand(n, 3).astype(np.float32)
    out["dense_assign"] = assign
    out["dense_assign_ei"], out["dense_assign_w"] = gu.convert_dense_assign_to_edge(T(assign), T(gi))
    np.savez_compressed(os.path.join(OUT, "cluster_pool_exec.npz"), **{k: np.asarray(v) for k, v in out.items()})
    print("wrote cluster_pool_exec.npz: {}".format(", ".join(sorted(out))))


if __name__ == "__main__":
    main()
