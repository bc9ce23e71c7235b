# coding=utf-8
"""Link prediction without a GPU: the oracle against the reference's own negative_sampling / edge_train_test_split /
negative_sampling_with_start_node (tests/golden/link_exec.npz), the public API over the CPU fake of the kernel
layer, and the float64 predict_edge reference under gradcheck."""
import math
import os

import numpy as np
import pytest
import torch

import link_oracle as lo
import link_fake_backend

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "link_exec.npz")


@pytest.fixture(scope="module")
def ref():
    return dict(np.load(GOLDEN))


def _pairs(ei):
    return set(zip(np.asarray(ei[0]).tolist(), np.asarray(ei[1]).tolist()))


def test_oracle_candidate_list_is_the_reference_order(ref):
    got = lo.negative_candidates(ref["ei"], int(ref["n"]))
    assert got.dtype == np.int32
    np.testing.assert_array_equal(got, ref["candidates"])


def test_oracle_decodes_every_candidate_index(ref):
    rowptr, col, offsets = lo.negative_structure(ref["ei"], int(ref["n"]))
    C = int(offsets[-1])
    k = np.array([0, C - 1, C // 2, 3, 3], np.int64)
    np.testing.assert_array_equal(lo.negative_decode(rowptr, col, offsets, k), ref["candidates"][:, k])


def test_oracle_split_matches_reference_sizes_and_merged_set(ref):
    n_up = len(_pairs(ref["split_train_index"])) + len(_pairs(ref["split_test_index"]))
    tr, te, tr_w, te_w = lo.edge_train_test_split(ref["ei"], 0.2, ref["w"], seed=5)
    assert te.shape[1] == ref["split_test_index"].shape[1] == math.ceil(0.2 * n_up)
    assert tr.shape[1] == ref["split_train_index"].shape[1]
    want = dict(zip(zip(*np.concatenate([ref["split_train_index"], ref["split_test_index"]], 1).tolist()),
                    np.concatenate([ref["split_train_w"], ref["split_test_w"]]).tolist()))
    got = dict(zip(zip(*np.concatenate([tr, te], 1).tolist()), np.concatenate([tr_w, te_w]).tolist()))
    assert got == want                                    # same merged upper edges, same (max) weights, bit for bit
    tr7, te7, _, _ = lo.edge_train_test_split(ref["ei"], 7, seed=5)
    assert te7.shape[1] == ref["split7_test_index"].shape[1] == 7
    assert tr7.shape[1] == ref["split7_train_index"].shape[1]


def test_oracle_start_node_sampling_has_the_reference_properties(ref):
    n, ei, start = int(ref["n"]), ref["ei"], ref["start"]
    edges = _pairs(ei)
    for sample in (ref["start_sample"], lo.negative_sampling_with_start_node(start, n, ei, seed=9)):
        assert sample.shape == (2, len(start))
        np.testing.assert_array_equal(sample[0], start)
        assert np.all(sample[0] != sample[1])
        assert not (_pairs(sample) & edges)


def test_oracle_samplers_properties(ref):
    n, ei = int(ref["n"]), ref["ei"]
    cand = _pairs(ref["candidates"])
    C = len(cand)
    for replace, S in ((True, 50), (False, 20), (False, C - 3), (False, C)):
        s = lo.negative_sampling(S, n, ei, replace=replace, seed=3)
        assert s.shape == (2, S) and _pairs(s) <= cand
        if not replace:
            assert len(_pairs(s)) == S
    assert _pairs(lo.negative_sampling(C, n, ei, replace=False, seed=4)) == cand
    with pytest.raises(ValueError):
        lo.negative_sampling(C + 1, n, ei, replace=False)


def test_predict_edge_reference_gradcheck():
    rs = np.random.RandomState(0)
    h = torch.tensor(rs.randn(7, 5), dtype=torch.float64, requires_grad=True)
    ei = torch.tensor([[0, 1, 3, 3, 6, 2], [4, 1, 2, 2, 0, 5]], dtype=torch.int64)       # a self loop and a duplicate
    assert torch.autograd.gradcheck(lambda x: lo.predict_edge_torch(x, ei), (h,))
    np.testing.assert_allclose(lo.predict_edge_torch(h, ei).detach().numpy(), lo.predict_edge(h.detach().numpy(), ei.numpy()))


# ---- the public API over the CPU fake of the kernel layer ------------------------------------------------------------

@pytest.fixture
def tfg(monkeypatch):
    link_fake_backend.install(monkeypatch)
    import tf_geometric_b200 as tfg
    return tfg


def test_negative_sampling_api_matches_oracle(tfg, ref):
    n, ei = int(ref["n"]), ref["ei"]
    C = ref["candidates"].shape[1]
    for replace, S in ((True, 40), (False, 25), (False, C - 2)):
        got = tfg.utils.negative_sampling(S, n, ei, replace=replace, seed=17)
        assert isinstance(got, np.ndarray)
        np.testing.assert_array_equal(got, lo.negative_sampling(S, n, ei, replace=replace, seed=17))
    got = tfg.utils.negative_sampling(10, n, torch.from_numpy(ei), replace=False, batch_size=3, seed=2)
    want = lo.negative_sampling(10, n, ei, replace=False, batch_size=3, seed=2)
    assert len(got) == 3 and all(torch.is_tensor(g) for g in got)
    for g, w in zip(got, want):
        np.testing.assert_array_equal(g.numpy(), w)
    assert not np.array_equal(want[0], want[1])
    np.testing.assert_array_equal(tfg.utils.negative_sampling(12, n, None, seed=8).numpy(),
                                  lo.negative_sampling(12, n, None, seed=8))


def test_negative_sampling_api_errors(tfg, ref):
    n, ei = int(ref["n"]), ref["ei"]
    C = ref["candidates"].shape[1]
    with pytest.raises(ValueError):
        tfg.utils.negative_sampling(C + 1, n, ei, replace=False)
    with pytest.raises(ValueError):
        tfg.utils.negative_sampling(5, n - 1, ei)                       # ids >= num_nodes
    full = np.array([[0, 0, 1], [1, 2, 2]], np.int32)
    with pytest.raises(ValueError):
        tfg.utils.negative_sampling(1, 3, full)                          # C == 0
    assert tfg.utils.negative_sampling(0, 3, full).shape == (2, 0)
    with pytest.raises(NotImplementedError):
        tfg.utils.negative_sampling(1, n, ei, mode="directed")


def test_start_node_and_split_api_match_oracle(tfg, ref):
    n, ei, w = int(ref["n"]), ref["ei"], ref["w"]
    start = ref["start"]
    got = tfg.utils.negative_sampling_with_start_node(start, n, ei, seed=6)
    np.testing.assert_array_equal(got, lo.negative_sampling_with_start_node(start, n, ei, seed=6))
    star = np.array([[0, 0, 0, 1], [1, 2, 3, 0]], np.int32)              # node 0 is adjacent to every other node
    with pytest.raises(ValueError):
        tfg.utils.negative_sampling_with_start_node(np.array([1, 0]), 4, star)
    got = tfg.utils.edge_train_test_split(ei, 0.2, edge_weight=w, seed=4)
    want = lo.edge_train_test_split(ei, 0.2, w, seed=4)
    for g, wt in zip(got, want):
        np.testing.assert_array_equal(g, wt)
    got = tfg.utils.edge_train_test_split(torch.from_numpy(ei), 7, seed=4)
    assert torch.is_tensor(got[0]) and got[2] is None and got[1].shape == (2, 7)
    with pytest.raises(NotImplementedError):
        tfg.utils.edge_train_test_split(ei, 0.2, mode="directed")


def test_predict_edge_api_forward_and_backward(tfg):
    rs = np.random.RandomState(1)
    h64 = torch.tensor(rs.randn(9, 6), dtype=torch.float64, requires_grad=True)
    ei = torch.tensor([[0, 1, 3, 3, 8, 2, 5], [4, 1, 2, 2, 0, 5, 5]], dtype=torch.int32)
    g = torch.tensor(rs.randn(7))
    lo.predict_edge_torch(h64, ei.long()).backward(g)
    h = h64.detach().to(torch.float32).requires_grad_(True)
    out = tfg.nn.predict_edge(h, ei)
    np.testing.assert_allclose(out.detach().numpy(), lo.predict_edge_torch(h64, ei.long()).detach().numpy(), rtol=1e-5, atol=1e-5)
    out.backward(g.to(torch.float32))
    np.testing.assert_allclose(h.grad.numpy(), h64.grad.numpy(), rtol=1e-5, atol=1e-5)
    with pytest.raises(ValueError):
        tfg.nn.predict_edge(h, torch.tensor([[0], [9]], dtype=torch.int32))


def test_api_reproduces_the_reference_execution(tfg, ref):
    """What does not depend on the generator: replace=False with num_samples = C returns every candidate once (the
    fixture holds them in the reference's order), and the split has the reference's sizes and covers the same merged
    upper edges with the same max weights."""
    n, cand = int(ref["n"]), ref["candidates"]
    got = tfg.utils.negative_sampling(cand.shape[1], n, torch.from_numpy(ref["ei"]), replace=False, seed=1).numpy()
    np.testing.assert_array_equal(got[:, np.lexsort((got[1], got[0]))], cand)
    for size, tag in ((0.2, "split"), (7, "split7")):
        tr, te, tr_w, te_w = tfg.utils.edge_train_test_split(ref["ei"], size, edge_weight=ref["w"], seed=1)
        assert tr.shape == ref[tag + "_train_index"].shape and te.shape == ref[tag + "_test_index"].shape
        union = np.concatenate([tr, te], axis=1)
        want = np.concatenate([ref[tag + "_train_index"], ref[tag + "_test_index"]], axis=1)
        assert _pairs(union) == _pairs(want) and union.shape == want.shape
        if tag == "split":
            got_w = dict(zip(zip(*union.tolist()), np.concatenate([tr_w, te_w]).tolist()))
            want_w = dict(zip(zip(*want.tolist()), np.concatenate([ref["split_train_w"], ref["split_test_w"]]).tolist()))
            assert got_w == want_w
