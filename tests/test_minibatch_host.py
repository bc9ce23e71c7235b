# coding=utf-8
"""The mini-batch sampler and the sampled-subgraph helpers without a GPU: RandomNeighborSampler.sample_neighborhood over
the CPU fake of K13 and the relabelling entries, against the dict-based restatement of tests/minibatch_ref.py; the
helpers' numpy and tensor paths against the reference restated with sets; the ABI declarations and argument checks."""
import numpy as np
import pytest
import torch

import minibatch_fake_backend as fake_mb
import minibatch_ref as ref
from conftest import random_graph
from oracle import c_oracle


@pytest.fixture
def fake(monkeypatch):
    fake_mb.install(monkeypatch)
    import tf_geometric_b200 as tfg
    return tfg


def test_ffi_declares_the_entries_and_refuses_capture():
    from tf_geometric_b200 import _ffi
    assert _ffi.ABI_VERSION == 7
    sizes = {"tfgk_neighbor_sample_rows_count": 12, "tfgk_neighbor_sample_rows_fill": 13, "tfgk_relabel_workspace_bytes": 2,
             "tfgk_reindex_i32": 11, "tfgk_frontier_i32": 12}
    for name, n in sizes.items():
        assert len(_ffi.SIGNATURES[name]) == n, name
    for name in ("tfgk_neighbor_sample_rows_count", "tfgk_neighbor_sample_rows_fill", "tfgk_reindex_i32",
                 "tfgk_frontier_i32"):
        assert name in _ffi.NOT_CAPTURABLE


def test_argument_validation_without_gpu():
    from tf_geometric_b200 import _ffi
    with pytest.raises(_ffi.TfgkError) as err:
        _ffi.call("tfgk_neighbor_sample_rows_count", None, 4, None, 3, 2, 0.5, 0, None, None, None, 0, None)
    assert err.value.code == _ffi.ERR_INVALID_ARGUMENT and "simultaneously" in str(err.value)
    with pytest.raises(_ffi.TfgkError) as err:
        _ffi.call("tfgk_neighbor_sample_rows_fill", None, 4, None, 3, 2, -1.0, 7, 0, 1, None, None, None, None)
    assert err.value.code == _ffi.ERR_INVALID_ARGUMENT and "padding" in str(err.value)
    with pytest.raises(_ffi.TfgkError) as err:
        _ffi.call("tfgk_frontier_i32", None, -1, 4, None, 0, None, None, None, None, None, 0, None)
    assert err.value.code == _ffi.ERR_INVALID_ARGUMENT
    import ctypes
    dup = ctypes.c_int32(7)
    with pytest.raises(_ffi.TfgkError) as err:
        _ffi.call("tfgk_reindex_i32", None, 3, None, 0, 8, None, None, ctypes.byref(dup), None, 0, None)
    assert err.value.code == _ffi.ERR_INVALID_ARGUMENT and dup.value == 0


def _sampler_graph():
    ei = random_graph(300, 2400, seed=5, isolated=20, hub=(7, 400))
    ei = np.concatenate([ei, ei[:, :50]], axis=1)                       # duplicate edges
    ei = np.concatenate([ei, [[3], [350]]], axis=1).astype(np.int32)    # a column id past the last source row
    w = np.random.RandomState(6).rand(ei.shape[1]).astype(np.float32)
    return ei, w


def _csr(ei, w):
    n_rows = int(ei[0].max()) + 1
    rowptr, col, perm = c_oracle.csr_build(ei[0], ei[1], n_rows)
    return rowptr, col, w[perm]


@pytest.mark.parametrize("fanouts,padding", [([5, 3], False), ([2, 4, 3], True), ([4], "head"), ([], False)])
def test_sample_neighborhood_matches_restatement(fake, fanouts, padding):
    ei, w = _sampler_graph()
    sampler = fake.utils.RandomNeighborSampler(ei, w)
    seeds = np.array([7, 0, 299, 350, 3, 150], np.int32)
    b = sampler.sample_neighborhood(seeds, fanouts, padding=padding, seed=11)
    rowptr, col, w_csr = _csr(ei, w)
    nodes, edges, weights, sizes = ref.neighborhood(rowptr, col, w_csr, seeds, fanouts, padding, 11)
    np.testing.assert_array_equal(b.node_index.numpy(), nodes)
    assert b.hop_sizes == sizes and len(b.edge_index_list) == len(fanouts) == len(b.edge_weight_list)
    for i, (got, want, gw, ww) in enumerate(zip(b.edge_index_list, edges, b.edge_weight_list, weights)):
        np.testing.assert_array_equal(got.numpy(), want)
        np.testing.assert_array_equal(gw.numpy(), ww)
        assert got.numpy()[0].max(initial=-1) < sizes[-2 - i]


def test_sample_neighborhood_layer_fanouts_and_keys(fake):
    ei, w = _sampler_graph()
    sampler = fake.utils.RandomNeighborSampler(ei, w)
    b = sampler.sample_neighborhood([7], [1, 6], seed=3)
    deg7 = int(np.sum(ei[0] == 7))
    assert b.edge_index_list[1].shape[1] == 6 and deg7 > 6             # the seeds' hop uses fanouts[-1]
    again = sampler.sample_neighborhood([7], [1, 6], seed=3)
    np.testing.assert_array_equal(b.node_index.numpy(), again.node_index.numpy())
    for x, y in zip(b.edge_index_list, again.edge_index_list):
        np.testing.assert_array_equal(x.numpy(), y.numpy())
    other = sampler.sample_neighborhood([7], [1, 6], seed=4)
    assert not np.array_equal(b.node_index.numpy()[:7], other.node_index.numpy()[:7])


def test_sample_neighborhood_rejects_bad_seeds(fake):
    ei, w = _sampler_graph()
    sampler = fake.utils.RandomNeighborSampler(ei, w)
    with pytest.raises(ValueError, match="duplicate"):
        sampler.sample_neighborhood([4, 9, 4], [3])
    with pytest.raises(ValueError, match="outside"):
        sampler.sample_neighborhood([4, 351], [3])
    with pytest.raises(ValueError, match="outside"):
        sampler.sample_neighborhood([-1], [3])


def _helper_inputs():
    rs = np.random.RandomState(8)
    ei = rs.randint(0, 40, (2, 300)).astype(np.int32)
    ei = np.concatenate([ei, ei[::-1, :30], ei[:, 5:25]], axis=1)       # reversed and repeated pairs
    w = rs.rand(ei.shape[1]).astype(np.float32)
    nodes = rs.permutation(45)[:25].astype(np.int32)                    # some ids no edge uses
    return ei, w, nodes


@pytest.mark.parametrize("container", ["numpy", "tensor"])
def test_parity_helpers_match_reference(fake, container):
    from tf_geometric_b200.utils import graph_utils as gu
    ei, w, nodes = _helper_inputs()
    box = (lambda a: a) if container == "numpy" else torch.from_numpy
    out = gu.reindex_sampled_edge_index(box(ei), box(nodes))
    assert isinstance(out, np.ndarray) == (container == "numpy")
    np.testing.assert_array_equal(np.asarray(out), ref.reindex_sampled_edge_index(ei, nodes))
    assert (np.asarray(out) == -1).any() and (np.asarray(out) >= 0).any()
    with pytest.raises(ValueError):
        gu.reindex_sampled_edge_index(box(ei), box(np.concatenate([nodes, nodes[3:4]])))
    mask = gu.compute_edge_mask_by_node_index(box(ei), box(nodes))
    np.testing.assert_array_equal(np.asarray(mask), ref.compute_edge_mask_by_node_index(ei, nodes))
    for mode in ("undirected", "directed"):
        got_i, got_w = gu.extract_unique_edge(box(ei), box(w), mode=mode)
        want_i, want_w = ref.extract_unique_edge(ei, w, mode)
        assert isinstance(got_i, np.ndarray) == (container == "numpy")
        np.testing.assert_array_equal(np.asarray(got_i), want_i)
        np.testing.assert_array_equal(np.asarray(got_w), want_w)
        got_i, none = gu.extract_unique_edge(box(ei), None, mode=mode)
        assert none is None and np.array_equal(np.asarray(got_i), want_i)


def test_demo_block_restated(fake):
    """demo/demo_sample_neighbors.py's first block against tfg, then its commented-out reindexing step."""
    edge_index = [
        [0, 0, 1, 1, 1, 2, 2, 2, 3, 3, 4, 4, 4, 4, 5, 5, 5, 5, 5, 5, 5],
        [1, 2, 3, 4, 5, 0, 4, 7, 1, 7, 2, 3, 6, 9, 0, 2, 3, 4, 7, 8, 10]
    ]
    sampler = fake.utils.graph_utils.RandomNeighborSampler(edge_index)
    ei, ew = sampler.sample(k=5, sampled_node_index=([4, 2], [2, 6, 7, 8, 9, 10]), padding=False)
    assert ei.numpy().tolist() == [[0, 0, 0, 1], [0, 1, 4, 2]] and ew.numpy().tolist() == [1.0] * 4
    global_ei = np.array([[4, 4, 4, 2, 2], [2, 6, 9, 0, 7]], np.int32)
    out = fake.utils.graph_utils.reindex_sampled_edge_index(global_ei, [4, 2, 6, 7, 9])
    assert out.tolist() == [[0, 0, 0, 1, 1], [1, 2, 4, -1, 3]]
