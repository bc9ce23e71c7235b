# coding=utf-8
"""Host-side logic of the reference-facing API, exercised on CPU through a test double of the kernel layer
(tests/fake_backend.py): argument plumbing, graph.cache, quirks, layer wiring, weight names, casting rules.
The SAME test bodies run against the real kernels in the test_gpu_*.py modules on the H100."""
import numpy as np
import pytest
import torch

import tf_geometric_b200 as tfg
import fake_backend
import test_gpu_index
import test_gpu_spmm
import test_gpu_gat
import test_gpu_models
import test_gpu_train
import test_gpu_pool2


@pytest.fixture
def fake(monkeypatch):
    fake_backend.install(monkeypatch)
    yield
    from tf_geometric_b200 import _structure
    _structure.clear()


def test_graph_casting_rules():
    """data/graph.py:58-91: list/ndarray edge_index -> int32, weights -> float32, float64 features -> float32."""
    g = tfg.Graph(np.random.randn(5, 3), [[0, 0, 1, 3], [1, 2, 2, 1]])
    assert g.x.dtype == np.float32 and g.edge_index.dtype == np.int32 and g.edge_weight.dtype == np.float32
    assert g.edge_weight.tolist() == [1, 1, 1, 1] and g.num_nodes == 5 and g.num_edges == 4 and g.num_features == 3
    assert g.cache == {} and "x => (5, 3)" in str(g)
    g = tfg.Graph(np.zeros((2, 1), np.float16), np.array([[0], [1]], np.int64), edge_weight=[2])
    assert g.x.dtype == np.float16 and g.edge_index.dtype == np.int32 and g.edge_weight.dtype == np.float32
    g = tfg.Graph(torch.zeros(3, 2, dtype=torch.float64), torch.tensor([[0, 1], [1, 2]]))
    assert g.x.dtype == torch.float32 and g.edge_index.dtype == torch.int32 and torch.is_tensor(g.edge_weight)
    assert tfg.Graph(np.zeros((3, 2)), np.zeros((2, 0))).num_edges == 0


def test_compute_num_or_size_splits():
    f = tfg.utils.compute_num_or_size_splits
    assert f(128, None) is None and f(128, 1) is None and f(128, 4) == 4
    assert f(10, 3) == [4, 4, 2] and f(10, 4) == [3, 3, 3, 1]
    with pytest.raises(Exception):
        f(5, 4)           # ceil(5/4) = 2 -> [2, 2, 1] has 3 parts, not 4


def test_cache_key_format():
    assert tfg.nn.compute_cache_key("both", True, True, True, False) == "gcn_normed_adj_both_True_True_True_False"


# ---- the GPU test bodies, replayed on the fake backend -------------------------------------------------------------

def test_index_paths(fake):
    test_gpu_index.test_add_self_loop_edge(1000, 20000)
    test_gpu_index.test_segment_count(6, 9)
    test_gpu_index.test_gcn_norm_derived_kat_and_cache()
    test_gpu_index.test_to_directed_and_merge_match_oracle()
    for args in (("both", True, True, True, False), ("both", True, True, False, False), ("both", True, False, True, True),
                 ("left", True, False, True, False), ("right", True, False, True, False)):
        test_gpu_index.test_gcn_norm_adj_index_bit_exact_values_close(*args)


def test_aggregate_paths(fake):
    test_gpu_spmm.test_aggregate_sum_bit_exact_all_widths(7, True)
    test_gpu_spmm.test_aggregate_sum_bit_exact_all_widths(16, False)
    test_gpu_spmm.test_aggregate_mean_max(7, "mean")
    test_gpu_spmm.test_aggregate_mean_max(16, "max")
    test_gpu_spmm.test_aggregate_defaults_sum_updater_and_empty_edge_index()
    test_gpu_spmm.test_generic_mapper_route_and_standalone_reducers()


def test_gat_paths(fake):
    test_gpu_gat.test_segment_softmax(None)
    test_gpu_gat.test_segment_softmax(3)
    test_gpu_gat.test_gat_forward_matches_oracle(24, 64, 64, 8, True)
    test_gpu_gat.test_gat_forward_matches_oracle(16, 48, 40, 4, False)
    test_gpu_gat.test_gat_layer_defaults_and_weight_names()


def test_model_paths(fake):
    test_gpu_models.test_gcn_functional("both", True, True, True, False, "relu")
    test_gpu_models.test_gcn_functional("right", False, False, True, False, "relu")
    test_gpu_models.test_gcn_two_layer_cora_shaped_model_with_cache()
    test_gpu_models.test_plain_graph_sage("mean", True, True)
    test_gpu_models.test_plain_graph_sage("sum", False, False)
    test_gpu_models.test_pool_and_gcn_graph_sage_and_layers()
    test_gpu_models.test_appnp(10, 0.1)
    test_gpu_models.test_appnp(0, 0.1)
    test_gpu_models.test_sparse_features_and_column_splits()
    test_gpu_models.test_training_with_sparse_features_matches_dense_features()
    test_gpu_models.test_graph_sage_forward_backward("mean", False, True)
    test_gpu_models.test_graph_sage_forward_backward("mean", True, False)
    test_gpu_models.test_graph_sage_forward_backward("sum", True, True)
    test_gpu_models.test_propagation_layers_sgc_ssgc_tagcn_gin_leconv()
    test_gpu_models.test_gcn_two_layer_forward_backward(True)
    test_gpu_models.test_gcn_two_layer_forward_backward(False)
    test_gpu_models.test_chebynet_layer_static_and_dynamic_lambda()
    test_gpu_models.test_degenerate_graphs_empty_edges_single_node()


def test_golden_fixtures_through_public_api(fake):
    """The committed reference-execution fixtures replayed through the product's host logic (fake kernels)."""
    import os
    import golden_cases
    golden = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")
    files = sorted(f for f in os.listdir(golden) if f.startswith("ref_exec_"))
    assert len(files) >= 6
    for f in files:
        golden_cases.replay(f, np.load(os.path.join(golden, f), allow_pickle=False), golden_cases.ProductApi())


def test_training_extras_and_samplers(fake):
    """dropout / GAT backward / drop_edge / samplers: host logic over the numpy restatements of the kernels."""
    test_gpu_train.test_dropout_mask_bit_exact(4099, 0.9)
    test_gpu_train.test_spmm_heads_bit_exact(3, 5, "split", True, 0.0)
    # the fake kernels bypass the C ABI, so there are no call counts to say which backward ran (path=None)
    test_gpu_train.test_gat_gradients_match_reference_autodiff(24, 64, 128, 8, True, True, 0.4, False, None)
    test_gpu_train.test_gat_gradients_match_reference_autodiff(10, 12, 20, 4, True, False, 0.0, False, None)
    test_gpu_train.test_gat_gradients_match_reference_autodiff(10, 12, 6, 3, False, True, 0.0, False, None)
    test_gpu_train.test_gat_gradients_match_reference_autodiff(10, 12, 6, 3, False, False, 0.3, False, None)
    test_gpu_train.test_gat_gradients_match_reference_autodiff(16, 32, 32, 4, True, True, 0.0, True, None)
    test_gpu_train.test_gcn_edge_dropout_forward_and_gradients()
    test_gpu_train.test_appnp_training_gradients_and_dense_dropout()
    test_gpu_train.test_drop_edge_matches_oracle(False)
    test_gpu_train.test_drop_edge_matches_oracle(True)
    test_gpu_train.test_uniform_neighbor_sampler_matches_oracle()
    test_gpu_train.test_random_neighbor_sampler_matches_oracle(5, None, False)
    test_gpu_train.test_random_neighbor_sampler_matches_oracle(40, None, True)
    test_gpu_train.test_random_neighbor_sampler_matches_oracle(None, 0.3, False)
    import golden_cases
    golden_cases.replay("ref_exec_sampler.npz", np.load(test_gpu_train.GOLDEN + "/ref_exec_sampler.npz"), golden_cases.ProductApi())


def test_gat_layer_trains_on_the_fake_backend(fake):
    test_gpu_train.test_gat_layer_learns()


def test_pooling_family_on_the_fake_backend(fake):
    import golden_cases
    test_gpu_pool2.test_sort_keys_and_stable_argsort()
    test_gpu_pool2.test_topk_pool_matches_oracle(7, None)
    test_gpu_pool2.test_topk_pool_matches_oracle(None, 0.25)
    test_gpu_pool2.test_set2set_matches_oracle(6, 9, 200)
    test_gpu_pool2.test_induced_subgraph_and_batch_graph()
    test_gpu_pool2.test_pools_over_few_large_graphs_use_edge_sized_tasks()
    test_gpu_pool2.test_sag_pool_matches_oracle(3, None)
    test_gpu_pool2.test_sag_pool_matches_oracle(None, 0.4)
    test_gpu_pool2.test_sort_pool_drop_edge_layer_and_map_reduce_layer()
    test_gpu_pool2.test_set2set_gradients_match_autodiff(6, 7, 150)
    golden_cases.replay("ref_exec_pool2.npz", np.load(test_gpu_train.GOLDEN + "/ref_exec_pool2.npz"), golden_cases.ProductApi())


def test_remaining_convs_train_on_the_fake_backend(fake):
    for name in ("sgc", "ssgc", "tagcn", "gin", "le_conv", "chebynet", "gcn_graph_sage", "mean_pool_graph_sage",
                 "max_pool_graph_sage"):
        test_gpu_train.test_conv_training_gradients_match_autodiff(name)
    test_gpu_train.test_every_trainable_layer_gets_gradients()


def test_pooling_passes_gradients_on_the_fake_backend(fake):
    test_gpu_train.test_every_pool_layer_passes_gradients()


def test_sparse_matrix_product_is_differentiable(fake):
    """`A @ h` in a user's own training loop (tf_sparse products sit under tf.GradientTape in the reference's demos): the
    gradient reaches h and the bias; epilogue forms without a backward raise instead of cutting the graph."""
    rs = np.random.RandomState(4)
    n, m, d = 40, 30, 6
    index = np.stack([rs.randint(0, n, 200), rs.randint(0, m, 200)]).astype(np.int32)
    value = rs.rand(200).astype(np.float32)
    a = tfg.SparseMatrix(index, value, [n, m])
    h = torch.from_numpy(rs.randn(m, d).astype(np.float32)).requires_grad_(True)
    g = torch.from_numpy(rs.randn(n, d).astype(np.float32))
    y = a @ h
    assert y.requires_grad
    (y * g).sum().backward()
    dense = torch.zeros(n, m, dtype=torch.float64)
    dense.index_put_((torch.from_numpy(index[0]).long(), torch.from_numpy(index[1]).long()), torch.from_numpy(value).double(),
                     accumulate=True)
    np.testing.assert_allclose(y.detach().numpy(), (dense @ h.detach().double()).numpy(), rtol=1e-5, atol=1e-5)
    np.testing.assert_allclose(h.grad.numpy(), (dense.t() @ g.double()).numpy(), rtol=1e-5, atol=1e-5)
    with pytest.raises(NotImplementedError):
        a.matmul(h, alpha=2.0)
    with torch.no_grad():
        assert not (a @ h).requires_grad
