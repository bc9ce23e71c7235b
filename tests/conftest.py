# coding=utf-8
import os
import sys

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs a CUDA device (run on the H100 with -m gpu)")


def pytest_collection_modifyitems(config, items):
    """`-m gpu` tests are skipped (not failed) when collected on a machine without a GPU and no marker filter."""
    try:
        import torch
        has_gpu = torch.cuda.is_available()
    except Exception:
        has_gpu = False
    if has_gpu:
        return
    skip = pytest.mark.skip(reason="no CUDA device")
    for item in items:
        if "gpu" in item.keywords:
            item.add_marker(skip)


# ---- shared helpers -------------------------------------------------------------------------------------------

def assert_close(actual, expected, rtol=1e-4, atol_scale=1e-4, what=""):
    """north_star tolerance for fp32 embeddings: allclose(rtol=1e-4, atol=1e-4 * max|ref|) (SURVEY.md section 7)."""
    actual = np.asarray(actual, dtype=np.float64)
    expected = np.asarray(expected, dtype=np.float64)
    assert actual.shape == expected.shape, "{} shape {} != {}".format(what, actual.shape, expected.shape)
    scale = float(np.max(np.abs(expected))) if expected.size else 0.0
    atol = atol_scale * max(scale, 1e-30)
    err = np.abs(actual - expected)
    bound = atol + rtol * np.abs(expected)
    if not np.all(err <= bound):
        i = int(np.argmax(err - bound))
        raise AssertionError("{}: mismatch at flat index {}: got {!r}, expected {!r} (max abs err {:.3e}, atol {:.3e})"
                             .format(what, i, actual.flat[i], expected.flat[i], err.max(), atol))


def random_graph(num_nodes, num_edges, seed, symmetric=False, isolated=0, hub=None):
    """Random COO edge list (int32 [2, E]); `isolated` leading nodes get no in-edges; `hub` = (node, degree)."""
    rs = np.random.RandomState(seed)
    lo = isolated
    if symmetric:
        half = num_edges // 2
        u = rs.randint(lo, num_nodes, half)
        v = rs.randint(lo, num_nodes, half)
        keep = u != v
        u, v = u[keep], v[keep]
        row = np.concatenate([u, v])
        col = np.concatenate([v, u])
    else:
        row = rs.randint(lo, num_nodes, num_edges)
        col = rs.randint(0, num_nodes, num_edges)
    if hub is not None:
        node, deg = hub
        row = np.concatenate([row, np.full(deg, node)])
        col = np.concatenate([col, rs.randint(0, num_nodes, deg)])
        p = rs.permutation(len(row))
        row, col = row[p], col[p]
    return np.stack([row, col]).astype(np.int32)


def glorot(rs, fan_in, fan_out):
    limit = np.sqrt(6.0 / (fan_in + fan_out))
    return rs.uniform(-limit, limit, size=(fan_in, fan_out)).astype(np.float32)
