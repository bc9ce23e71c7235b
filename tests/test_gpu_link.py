# coding=utf-8
"""Link prediction on the H100: K6 edge scoring (tfgk_edge_dot_f32) and its half-edge backward against float64
autograd over link_oracle.predict_edge_torch, exact negative sampling / start-node sampling / the edge split
bit for bit against the oracle's restatement, and a graph autoencoder trained end to end with these pieces."""
import os

import numpy as np
import pytest
import torch

import tf_geometric_b200 as tfg
from tf_geometric_b200 import ops, autograd
from oracle import tfg_oracle as o
import link_oracle as lo
from conftest import assert_close

pytestmark = pytest.mark.gpu
DEV = torch.device("cuda", 0)
GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "link_exec.npz")


@pytest.fixture(scope="module")
def ref():
    return dict(np.load(GOLDEN))


def _pairs(ei):
    ei = ei.cpu().numpy() if torch.is_tensor(ei) else np.asarray(ei)
    return set(zip(ei[0].tolist(), ei[1].tolist()))


def _query_edges(n, e, seed):
    """Random pairs plus repeated pairs and self loops, int32 [2, E'] on the device."""
    rs = np.random.RandomState(seed)
    ei = rs.randint(0, n, (2, e))
    ei = np.concatenate([ei, ei[:, :e // 10], np.stack([np.arange(0, n, 7)] * 2)], axis=1)
    return torch.from_numpy(ei.astype(np.int32)).to(DEV)


def _ref_logits(h, ei):
    return lo.predict_edge_torch(h.detach().cpu().double(), ei.cpu().long()).numpy()


# ---- K6 forward ----------------------------------------------------------------------------------------------------

@pytest.mark.parametrize("D", [1, 3, 16, 64, 128, 256])
def test_edge_dot_matches_float64(D):
    n = 700
    h = torch.randn((n, D), generator=torch.Generator().manual_seed(D), dtype=torch.float32).to(DEV)
    ei = _query_edges(n, 5000, D)
    row, col = ei[0].contiguous(), ei[1].contiguous()
    out = ops.edge_dot(h, row, col)
    assert_close(out.cpu().numpy(), _ref_logits(h, ei), rtol=1e-4, atol_scale=1e-4, what="D=%d" % D)
    # an edge's bits depend on the edge and h only: split + concatenate, and reversed order, give the same bits
    cut = 1237
    parts = torch.cat([ops.edge_dot(h, row[:cut].contiguous(), col[:cut].contiguous()),
                       ops.edge_dot(h, row[cut:].contiguous(), col[cut:].contiguous())])
    assert torch.equal(parts, out)
    assert torch.equal(ops.edge_dot(h, row.flip(0).contiguous(), col.flip(0).contiguous()).flip(0), out)
    assert torch.equal(tfg.nn.predict_edge(h, ei), out)


@pytest.mark.parametrize("D", [5, 16, 64])
def test_edge_dot_column_slice_with_odd_leading_dimension(D):
    n = 300
    big = torch.randn((n, 2 * D + 3), generator=torch.Generator().manual_seed(7), dtype=torch.float32).to(DEV)
    h = big[:, 3:3 + D]                                         # odd ldh, unaligned base: the scalar path
    assert h.stride(0) % 2 == 1
    ei = _query_edges(n, 2000, 3)
    out = tfg.nn.predict_edge(h, ei)
    assert_close(out.cpu().numpy(), _ref_logits(h, ei), rtol=1e-4, atol_scale=1e-4)


def test_edge_dot_empty_and_out_of_range():
    h = torch.randn((10, 8), device=DEV)
    assert tfg.nn.predict_edge(h, torch.zeros((2, 0), dtype=torch.int32, device=DEV)).shape == (0,)
    with pytest.raises(ValueError):
        tfg.nn.predict_edge(h, torch.tensor([[0, 1], [2, 10]], dtype=torch.int32, device=DEV))
    # the kernel itself never reads an out-of-range row: such an edge scores NaN, the others are unaffected
    out = ops.edge_dot(h, torch.tensor([0, 10, 3], dtype=torch.int32, device=DEV),
                       torch.tensor([1, 2, -1], dtype=torch.int32, device=DEV)).cpu()
    assert torch.isnan(out[1]) and torch.isnan(out[2])
    assert torch.equal(out[0], ops.edge_dot(h, torch.tensor([0], dtype=torch.int32, device=DEV),
                                            torch.tensor([1], dtype=torch.int32, device=DEV)).cpu()[0])


# ---- gradients ---------------------------------------------------------------------------------------------------------

@pytest.mark.parametrize("D", [16, 64])
def test_gradients_match_float64_autograd(D):
    n, hub = 4000, 11
    rs = np.random.RandomState(D)
    base = _query_edges(n, 8000, D).cpu().numpy()
    hub_edges = np.stack([np.full(2600, hub), rs.randint(0, n, 2600)])     # node 11 is in > 2048 queried edges
    ei_np = np.concatenate([base, hub_edges[:, :1300], hub_edges[::-1, 1300:]], axis=1).astype(np.int32)
    ei = torch.from_numpy(ei_np).to(DEV)
    h0 = torch.randn((n, D), generator=torch.Generator().manual_seed(1), dtype=torch.float32)
    g = torch.randn((ei.shape[1],), generator=torch.Generator().manual_seed(2), dtype=torch.float32)

    h64 = h0.double().requires_grad_(True)
    lo.predict_edge_torch(h64, torch.from_numpy(ei_np).long()).backward(g.double())

    grads = []
    for _ in range(2):
        h = h0.to(DEV).requires_grad_(True)
        tfg.nn.predict_edge(h, ei).backward(g.to(DEV))
        grads.append(h.grad.clone())
    assert_close(grads[0].cpu().numpy(), h64.grad.numpy(), rtol=1e-4, atol_scale=1e-4, what="dh D=%d" % D)
    assert torch.equal(grads[0], grads[1])                                 # run-to-run identical
    csr = autograd._half_edge_csr(ei, n)
    assert csr.plan is not None and csr.plan.n_hubs > 0                    # the hub row went through the work plan


# ---- negative sampling ---------------------------------------------------------------------------------------------------

def _check_negatives(s, ei, n, distinct):
    s = s.cpu().numpy() if torch.is_tensor(s) else s
    assert s.dtype == np.int32 and np.all(s[0] < s[1]) and np.all(s >= 0) and np.all(s < n)
    up = np.asarray(ei)
    assert not (_pairs(s) & _pairs(np.stack([up.min(0), up.max(0)])))
    if distinct:
        assert len(_pairs(s)) == s.shape[1]


@pytest.mark.parametrize("replace,S,batch", [(True, 300, None), (False, 40, None), (False, 300, None), (True, 50, 3),
                                             (False, 100, 2)])
def test_negative_sampling_bit_exact(ref, replace, S, batch):
    n, ei = int(ref["n"]), ref["ei"]
    got = tfg.utils.negative_sampling(S, n, torch.from_numpy(ei).to(DEV), replace=replace, batch_size=batch, seed=99)
    want = lo.negative_sampling(S, n, ei, replace=replace, batch_size=batch, seed=99)
    got, want = ([got], [want]) if batch is None else (got, want)
    assert len(got) == len(want)
    for g, w in zip(got, want):
        assert g.is_cuda
        np.testing.assert_array_equal(g.cpu().numpy(), w)
        _check_negatives(g, ei, n, not replace)


def test_negative_sampling_full_candidate_set_and_numpy_container(ref):
    n, ei, cand = int(ref["n"]), ref["ei"], ref["candidates"]
    C = cand.shape[1]
    got = tfg.utils.negative_sampling(C, n, ei, replace=False, seed=5)
    assert isinstance(got, np.ndarray)
    assert _pairs(got) == _pairs(cand) and got.shape == (2, C)
    np.testing.assert_array_equal(got, lo.negative_sampling(C, n, ei, replace=False, seed=5))


def test_negative_sampling_without_edge_index_draws_64_bit_ids():
    """Both ends are random_below64 draws 2 s and 2 s + 1 of each batch's key (uniform on [0, N) to within N / 2^64)."""
    got = tfg.utils.negative_sampling(1000, 37, None, batch_size=2, seed=4)
    want = lo.negative_sampling(1000, 37, None, batch_size=2, seed=4)
    for g, w in zip(got, want):
        assert g.is_cuda
        np.testing.assert_array_equal(g.cpu().numpy(), w)


def test_negative_sampling_is_uniform():
    from scipy.stats import chisquare
    ei = np.array([[0, 1, 2, 5, 7, 3, 3], [1, 2, 9, 6, 0, 3, 4]], np.int32)
    n = 12
    cand = lo.negative_candidates(ei, n)
    C = cand.shape[1]
    S = 200 * C
    s = tfg.utils.negative_sampling(S, n, torch.from_numpy(ei).to(DEV), replace=True, seed=2024).cpu().numpy()
    index = {p: i for i, p in enumerate(zip(cand[0].tolist(), cand[1].tolist()))}
    counts = np.bincount([index[p] for p in zip(s[0].tolist(), s[1].tolist())], minlength=C)
    assert chisquare(counts).pvalue > 1e-3


def test_negative_sampling_errors(ref):
    n, ei = int(ref["n"]), torch.from_numpy(ref["ei"]).to(DEV)
    C = ref["candidates"].shape[1]
    with pytest.raises(ValueError):
        tfg.utils.negative_sampling(C + 1, n, ei, replace=False)
    with pytest.raises(ValueError):
        tfg.utils.negative_sampling(10, n - 1, ei)
    full = torch.tensor([[0, 0, 1, 2], [1, 2, 2, 2]], dtype=torch.int32, device=DEV)
    with pytest.raises(ValueError):
        tfg.utils.negative_sampling(1, 3, full)
    assert tfg.utils.negative_sampling(0, 3, full).shape == (2, 0)


def test_negative_sampling_on_a_graph_the_reference_cannot_hold():
    n = 100000                                               # the reference's dense N x N float64 matrix would be 80 GB
    gen = torch.Generator().manual_seed(3)
    ei_np = torch.randint(0, n, (2, 600000), generator=gen, dtype=torch.int32).numpy()
    ei = torch.from_numpy(ei_np).to(DEV)
    for replace in (True, False):
        got = tfg.utils.negative_sampling(20000, n, ei, replace=replace, seed=31)
        np.testing.assert_array_equal(got.cpu().numpy(), lo.negative_sampling(20000, n, ei_np, replace=replace, seed=31))
        s = got.cpu().numpy().astype(np.int64)
        assert np.all(s[0] < s[1])
        up = np.stack([ei_np.min(0), ei_np.max(0)]).astype(np.int64)
        assert not np.isin(s[0] * n + s[1], up[0] * n + up[1]).any()
        if not replace:
            assert len(np.unique(s[0] * n + s[1])) == s.shape[1]


# ---- start node ------------------------------------------------------------------------------------------------------------

def test_start_node_sampling_draws_64_bit_ids(ref):
    """Partners against the restatement, with edge_index (a candidate index per start node) and without (the
    random_below64 draw 2 s + 1 of the key)."""
    n, ei, start = int(ref["n"]), ref["ei"], ref["start"]
    got = tfg.utils.negative_sampling_with_start_node(torch.from_numpy(start).to(DEV), n, torch.from_numpy(ei).to(DEV),
                                                      seed=12)
    assert got.is_cuda
    g = got.cpu().numpy()
    np.testing.assert_array_equal(g, lo.negative_sampling_with_start_node(start, n, ei, seed=12))
    np.testing.assert_array_equal(g[0], start)
    assert np.all(g[0] != g[1]) and not (_pairs(g) & _pairs(ei))
    np.testing.assert_array_equal(tfg.utils.negative_sampling_with_start_node(start, n, None, seed=3),
                                  lo.negative_sampling_with_start_node(start, n, None, seed=3))
    star = torch.tensor([[0, 0, 0, 2], [1, 2, 3, 0]], dtype=torch.int32, device=DEV)     # 0 is adjacent to 1, 2, 3
    ok = tfg.utils.negative_sampling_with_start_node(torch.tensor([2, 1, 3], device=DEV), 4, star, seed=1).cpu().numpy()
    assert np.all(ok[0] != ok[1])
    with pytest.raises(ValueError):
        tfg.utils.negative_sampling_with_start_node(torch.tensor([1, 0], device=DEV), 4, star)


# ---- edge split ----------------------------------------------------------------------------------------------------------

@pytest.mark.parametrize("test_size", [0.2, 7])
def test_edge_train_test_split(ref, test_size):
    ei, w = ref["ei"], ref["w"]
    got = tfg.utils.edge_train_test_split(torch.from_numpy(ei).to(DEV), test_size, edge_weight=torch.from_numpy(w).to(DEV),
                                          seed=77)
    want = lo.edge_train_test_split(ei, test_size, w, seed=77)
    for g, wt in zip(got, want):
        assert g.is_cuda
        np.testing.assert_array_equal(g.cpu().numpy(), wt)
    tr, te = got[0].cpu().numpy(), got[1].cpu().numpy()
    up, (up_w,) = o.convert_edge_to_upper(ei, [w], ["max"])
    n_test = int(np.ceil(test_size * up.shape[1])) if isinstance(test_size, float) else test_size
    assert te.shape[1] == n_test and tr.shape[1] == up.shape[1] - n_test
    assert not (_pairs(tr) & _pairs(te)) and (_pairs(tr) | _pairs(te)) == _pairs(up)
    weight = dict(zip(zip(up[0].tolist(), up[1].tolist()), up_w.tolist()))
    got_w = np.concatenate([got[2].cpu().numpy(), got[3].cpu().numpy()])
    assert [weight[p] for p in zip(*np.concatenate([tr, te], 1).tolist())] == got_w.tolist()


# ---- end to end: a graph autoencoder (demo/demo_gae.py) on a planted-partition graph -----------------------------------

def _auc(pos, neg):
    scores = np.concatenate([pos, neg])
    ranks = np.empty(len(scores))
    ranks[np.argsort(scores, kind="stable")] = np.arange(1, len(scores) + 1)
    return (ranks[:len(pos)].sum() - len(pos) * (len(pos) + 1) / 2) / (len(pos) * len(neg))


# measured on an H100 (this seed, 300 steps): 0.806; chance is 0.5
GAE_AUC_THRESHOLD = 0.7


def test_gae_trains_to_a_held_out_auc_well_above_chance():
    rs = np.random.RandomState(0)
    n, k = 600, 6
    block = rs.randint(0, k, n)
    iu = np.triu_indices(n, 1)
    p = np.where(block[iu[0]] == block[iu[1]], 0.08, 0.002)
    keep = rs.rand(len(p)) < p
    und = np.stack([iu[0][keep], iu[1][keep]]).astype(np.int32)
    tfg.set_seed(0)
    train_und, test_und, _, _ = tfg.utils.edge_train_test_split(torch.from_numpy(und).to(DEV), 0.15, seed=1)
    test_neg = tfg.utils.negative_sampling(test_und.shape[1], n, torch.from_numpy(und).to(DEV), replace=False, seed=2)
    train_ei, _ = tfg.utils.convert_edge_to_directed(train_und)
    x = torch.from_numpy(rs.randn(n, 32).astype(np.float32)).to(DEV)
    graph = tfg.Graph(x, train_ei)
    gcn0 = tfg.layers.GCN(32, activation=tfg.nn.relu, seed=3, trainable=True)
    gcn1 = tfg.layers.GCN(16, seed=4, trainable=True)
    gcn0.build_cache_for_graph(graph)

    def encode():
        h = gcn0([graph.x, graph.edge_index, graph.edge_weight], cache=graph.cache, training=True)
        return gcn1([h, graph.edge_index, graph.edge_weight], cache=graph.cache, training=True)

    encode()
    params = list(gcn0.parameters()) + list(gcn1.parameters())
    opt = torch.optim.Adam(params, lr=1e-2)
    bce = torch.nn.functional.binary_cross_entropy_with_logits
    for step in range(300):
        opt.zero_grad()
        h = encode()
        neg = tfg.utils.negative_sampling(graph.edge_index.shape[1], n, None, seed=1000 + step)
        pos_logits, neg_logits = tfg.nn.predict_edge(h, graph.edge_index), tfg.nn.predict_edge(h, neg)
        loss = bce(pos_logits, torch.ones_like(pos_logits)) + bce(neg_logits, torch.zeros_like(neg_logits))
        loss.backward()
        opt.step()
    with torch.no_grad():
        h = encode()
        auc = _auc(torch.sigmoid(tfg.nn.predict_edge(h, test_und)).cpu().numpy(),
                   torch.sigmoid(tfg.nn.predict_edge(h, test_neg)).cpu().numpy())
    print("GAE held-out AUC %.4f" % auc)
    assert auc > GAE_AUC_THRESHOLD
