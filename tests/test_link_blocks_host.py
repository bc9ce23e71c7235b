# coding=utf-8
"""Link prediction on blocks without a GPU: the declaration of the new entries and their argument checks; the pair
relabelling, the exclusion lists and the virtual-to-real position mapping of tests/link_blocks_fake_backend.py against
set-based restatements; batch assembly through the shared helper against sample_blocks (over the endpoint list, and over
the graph with the excluded entries deleted); the routing of LinkBlocks.predict_edge; the refusals."""
import numpy as np
import pytest
import torch

import link_blocks_fake_backend as fake_link
from test_blocks_host import _sampler_graph

ENTRIES = {"tfgk_block_pairs_workspace_bytes": 2, "tfgk_block_sample_begin_pairs": 12, "tfgk_link_tail_negatives_i32": 9,
           "tfgk_block_exclusion_workspace_bytes": 2, "tfgk_block_exclusion_count": 13, "tfgk_block_exclusion_fill": 11,
           "tfgk_block_exclusion_fill_mapped": 11, "tfgk_block_sample_count_excl": 15, "tfgk_block_sample_fill_excl": 27,
           "tfgk_block_sample_fill_mapped_excl": 27, "tfgk_block_gcn_values_excl_f32": 16}


@pytest.fixture
def fake(monkeypatch):
    calls = fake_link.install(monkeypatch)
    import tf_geometric_b200 as tfg
    monkeypatch.setattr(tfg.ops, "build_plan", lambda csr: None)
    return tfg, calls


def test_entries_are_declared_and_check_their_arguments():
    import tf_geometric_b200 as tfg
    from tf_geometric_b200 import _ffi
    assert "LinkBlocks" in dir(tfg.utils) and _ffi.ABI_VERSION == 7
    for name, arity in ENTRIES.items():
        assert len(_ffi.SIGNATURES[name]) == arity, name
    for name in ("tfgk_block_exclusion_count", "tfgk_block_sample_fill_excl", "tfgk_block_sample_fill_mapped_excl",
                 "tfgk_link_tail_negatives_i32"):
        assert name in _ffi.NOT_CAPTURABLE
    bad = [("tfgk_block_sample_begin_pairs", (None, None, -1, 5, None, None, None, 1, None, None, 0, None)),
           ("tfgk_block_sample_begin_pairs", (None, None, 3, 5, None, None, None, 1, None, None, 0, None)),
           ("tfgk_link_tail_negatives_i32", (None, 2, -1, 5, 0, 2, None, None, None)),
           ("tfgk_link_tail_negatives_i32", (None, 2, 3, 0, 0, 2, None, None, None)),          # no nodes to draw
           ("tfgk_block_exclusion_count", (None, 5, None, None, -1, None, None, 0, None, None, None, 0, None)),
           ("tfgk_block_sample_count_excl", (None, 5, None, None, 0, 1, 4, 3, 0, None, 4, None, None, 0, None)),
           ("tfgk_block_gcn_values_excl_f32", (None, None, None, 0, None, 2, None, None, 0, 1, 1.0, 1.0, None, 2, None,
                                               None))]
    for name, args in bad:
        with pytest.raises(_ffi.TfgkError) as err:
            _ffi.call(name, *args)
        assert err.value.code == _ffi.ERR_INVALID_ARGUMENT, name
    size = __import__("ctypes").c_size_t()
    _ffi.call("tfgk_block_pairs_workspace_bytes", 0, size)
    _ffi.call("tfgk_link_tail_negatives_i32", None, 0, 3, 0, 0, 2, None, None, None)         # nothing to draw


@pytest.mark.parametrize("pairs", [[[3, 3, 7, 0], [7, 3, 3, 9]], [[5], [5]], np.zeros((2, 0)),
                                   [[1, 20, 2], [-1, 2, 1]]], ids=["repeats", "self-loop", "empty", "bad id"])
def test_pair_relabelling_is_first_occurrence(pairs):
    pairs = np.asarray(pairs, np.int64).reshape(2, -1)
    seeds, local, n_bad = fake_link.pair_begin_np(pairs, 10)
    order = []
    for u, v in pairs.T:
        for x in (u, v):
            if 0 <= x < 10 and x not in order:
                order.append(int(x))
    assert seeds.tolist() == order and n_bad == int(((pairs < 0) | (pairs >= 10)).sum())
    for side in range(2):
        for i, v in enumerate(pairs[side]):
            assert local[side, i] == (order.index(v) if v in order else -1)


def _set_exclusion(rowptr, col, nodes, pairs_local_src, dst):
    """Row t's excluded positions: every p of its row whose column is among t's targets, in CSR order."""
    targets = {}
    for s, d in zip(pairs_local_src, dst):
        if s >= 0:
            targets.setdefault(int(s), set()).add(int(d))
    return {t: [p for p in range(rowptr[nodes[t]], rowptr[nodes[t] + 1]) if col[p] in ds]
            for t, ds in targets.items()}


def test_exclusion_lists_against_sets():
    # rows: 0 -> [4, 2, 4, 9] (a duplicate edge), 1 -> [0], 2 -> [], 3 -> [5, 6]
    rowptr = np.array([0, 4, 5, 5, 7], np.int64)
    col = np.array([4, 2, 4, 9, 0, 5, 6], np.int64)
    nodes = np.array([0, 3, 1, 2], np.int64)                 # list position -> node
    ts = np.array([0, 0, 0, 1, 1, 2, 3, -1], np.int64)       # repeated target, both of row 3's edges, a non-edge, bad
    td = np.array([4, 4, 9, 5, 6, 7, 1, 4], np.int64)
    off, pos = fake_link.exclusion_lists_np(rowptr, col, nodes, 6, ts, td)
    want = _set_exclusion(rowptr, col, nodes, ts, td)
    for t in range(6):
        assert pos[off[t]:off[t + 1]].tolist() == want.get(t, []), t
    assert off[-1] == 5 and np.diff(off).tolist() == [3, 2, 0, 0, 0, 0]      # row 3 emptied, a non-edge excludes nothing


@pytest.mark.parametrize("excluded", [[], [0], [3], [0, 1, 2], [1, 4, 5, 9], [0, 2, 4, 6, 8]])
def test_virtual_to_real_mapping(excluded):
    deg = 12
    kept = [p for p in range(deg) if p not in excluded]
    assert [fake_link.virtual_to_real_np(excluded, v) for v in range(len(kept))] == kept


def _pairs(ei):
    return np.concatenate([ei[:, [0, 1, 2, 60, 0]], [[7, 3], [7, 299]]], axis=1).astype(np.int32)   # a hub row (7)


@pytest.mark.parametrize("fanouts,padding", [([5, 3], False), ([2, 4], True), ([4], "head"), ([None, 2], False)])
def test_batches_match_sample_blocks(fake, fanouts, padding):
    tfg, calls = fake
    ei, w = _sampler_graph()
    s = tfg.utils.RandomNeighborSampler(ei, w)
    pos = _pairs(ei)
    b = s.sample_link_blocks(pos, fanouts, num_negatives=2, padding=padding, seed=3)
    N = s._neighborhood_structure()[3].numel()
    neg = fake_link.tail_negatives_np(pos[0], 2, N, 3)
    assert np.array_equal(b.node_index.numpy()[b.neg_index.numpy()], neg)
    seeds, _, _ = fake_link.pair_begin_np(np.concatenate([pos, neg], axis=1), N)
    want = s.sample_blocks(seeds, fanouts, padding=padding, seed=3)
    assert isinstance(b, tfg.utils.SampledBlocks) and b.hop_sizes == want.hop_sizes
    assert torch.equal(b.node_index, want.node_index)
    for x, y in zip(b.blocks, want.blocks):
        assert torch.equal(x.edge_index, y.edge_index) and torch.equal(x.edge_weight, y.edge_weight)
    for exclude in ("self", "reverse"):
        drop = {(int(u), int(v)) for u, v in pos.T}
        if exclude == "reverse":
            drop |= {(v, u) for u, v in drop}
        keep = np.array([(int(u), int(v)) not in drop for u, v in ei.T])
        deleted = tfg.utils.RandomNeighborSampler(ei[:, keep], w[keep])
        b = s.sample_link_blocks(pos, fanouts, num_negatives=2, exclude=exclude, padding=padding, seed=3)
        want = deleted.sample_blocks(seeds, fanouts, padding=padding, seed=3)
        assert torch.equal(b.node_index, want.node_index) and b.hop_sizes == want.hop_sizes
        for x, y in zip(b.blocks, want.blocks):
            assert torch.equal(x.edge_index, y.edge_index) and torch.equal(x.edge_weight, y.edge_weight)
            assert x.excluded is not None and y.excluded is None


def test_predict_edge_routing(fake):
    tfg, calls = fake
    ei, w = _sampler_graph()
    s = tfg.utils.RandomNeighborSampler(ei, w)
    b = s.sample_link_blocks(_pairs(ei), [3], num_negatives=1, seed=1)
    n = b.hop_sizes[0]
    h = torch.randn(n, 4)
    calls["csr_build_plan"].clear()
    pl, nl = b.predict_edge(h)
    assert calls["edge_dot"] == 1 and calls["csr_build_plan"] == []          # one K6 launch, no CSR without grad
    pairs = torch.cat([b.pos_index, b.neg_index], dim=1).long()
    want = (h[pairs[0]] * h[pairs[1]]).sum(1)
    assert torch.allclose(torch.cat([pl, nl]), want) and pl.shape == (7,) and nl.shape == (7,)
    hg = h.clone().requires_grad_(True)
    b.predict_edge(hg)
    assert calls["csr_build_plan"] == [(True, False)]                        # ids in range, no plan: no sync
    b.predict_edge(hg)
    assert len(calls["csr_build_plan"]) == 1                                 # kept on the batch
    with pytest.raises(ValueError):
        b.predict_edge(torch.randn(n + 1, 4))


def test_refusals(fake):
    tfg, calls = fake
    ei, w = _sampler_graph()
    s = tfg.utils.RandomNeighborSampler(ei, w)
    pos = _pairs(ei)
    node_map = s._neighborhood_structure()[3]
    cases = [((pos[0],), {}, ValueError), ((pos.astype(np.float32),), {}, TypeError),
             ((pos,), {"num_negatives": -1}, ValueError), ((pos,), {"num_negatives": 1.5}, ValueError),
             ((pos,), {"num_negatives": True}, ValueError), ((pos,), {"negative_edge_index": pos}, ValueError),
             ((pos,), {"exclude": "both"}, ValueError), ((np.array([[0], [10 ** 6]]),), {}, ValueError),
             ((pos,), {"padding": "head"}, ValueError)]
    for args, kwargs, err in cases:
        before = calls["link_block_sample"]
        with pytest.raises(err):
            s.sample_link_blocks(*args, [4] if kwargs.get("padding") != "head" else [None], **kwargs)
        assert bool((node_map == -1).all())
        if err is TypeError or kwargs.get("exclude") or "num_negatives" in kwargs:
            assert calls["link_block_sample"] == before                       # refused before any device work
