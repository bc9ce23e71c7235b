# coding=utf-8
"""K11 on the H100: max aggregation with tie counts (tfgk_spmm_max_f32) against K1 MAX and numpy, its backward over the
transposed CSR (tfgk_spmm_max_bwd_f32) against the composition TakeRows + SegmentReduce("max") it replaces, and the
layers that train through it (MaxPoolGraphSage, ASAP's query, aggregate_neighbors with max_reducer)."""
import numpy as np
import pytest
import torch

import asap_ref
import max_agg_ref as ref
from conftest import random_graph

pytestmark = pytest.mark.gpu
DEV = "cuda"
LOWEST = np.finfo(np.float32).min


def _dev(a, grad=False):
    t = torch.tensor(a, device=DEV)
    return t.requires_grad_(grad) if grad else t


def _bits(t):
    return t.detach().contiguous().view(torch.int32)


def _same_bits(a, b, what):
    assert a.shape == b.shape, "{}: shape {} != {}".format(what, tuple(a.shape), tuple(b.shape))
    diff = (_bits(a) != _bits(b)).sum().item()
    assert diff == 0, "{}: {} entries differ in their bits".format(what, diff)


def _tied_table(rs, n, d):
    """Values on a coarse grid with ReLU zeros: many exact ties, signed zeros among them."""
    h = (rs.randint(-4, 5, (n, d)) * 0.5).astype(np.float32)
    h[:, ::3] = np.maximum(h[:, ::3], 0)
    h[rs.rand(n, d) < 0.05] = -0.0
    return h


def _k11a_both(ei, n, h, w=None):
    from tf_geometric_b200 import ops, _structure
    csr, _ = _structure.csr_for_edge_index(ei, n)
    w_csr = None if w is None else _structure.weights_in_csr_order(w, csr)
    out, cnt = ops.spmm_max(csr, w_csr, h)
    k1 = ops.spmm(csr, w_csr, h, reduce="max")
    return csr, w_csr, out, cnt, k1


def _check_counts(csr, w_csr, h, cnt, what):
    want_out, want_cnt = ref.k11a(csr.rowptr.cpu().numpy(), csr.col.cpu().numpy(),
                                  None if w_csr is None else w_csr.cpu().numpy(), h.cpu().numpy())
    got = cnt.cpu().numpy()
    assert np.array_equal(got, want_cnt), "{}: {} counts differ".format(what, int((got != want_cnt).sum()))


# ---- K11a ------------------------------------------------------------------------------------------------------

@pytest.mark.parametrize("weighted", [False, True])
@pytest.mark.parametrize("D", [1, 3, 16, 32, 47, 64, 100, 128, 256, 512, 600])
def test_k11a_is_k1_max_with_exact_tie_counts(D, weighted):
    rs = np.random.RandomState(D + 7 * weighted)
    n = 700
    ei = _dev(random_graph(n, 6000, seed=D, isolated=4))
    h = _dev(_tied_table(rs, n, D))
    w = _dev(rs.choice([0.5, 1.0, 2.0, -1.0], ei.shape[1]).astype(np.float32)) if weighted else None
    csr, w_csr, out, cnt, k1 = _k11a_both(ei, n, h, w)
    _same_bits(out, k1, "out vs K1 MAX")
    assert cnt.dtype == torch.int32 and (cnt[:4] == 0).all()
    _check_counts(csr, w_csr, h, cnt, "D={}".format(D))


@pytest.mark.parametrize("layout", ["dense", "odd_ld"])
@pytest.mark.parametrize("D", [47, 64, 128])
def test_k11a_awkward_inputs_and_a_hub_row_through_the_plan(D, layout):
    """Empty rows, duplicate edges, ReLU rows of zeros, +-0, NaN, +-inf and -FLT_MAX messages, and a destination of
    in-degree 60,000 (hub slices of the plan wherever K1 takes it); an odd leading dimension takes the scalar path."""
    rs = np.random.RandomState(D)
    n = 3000
    ei = random_graph(n, 30000, seed=D + 1, isolated=10, hub=(17, 60000))
    dup = ei[:, :500]
    ei = np.concatenate([ei, dup, dup], axis=1)
    h = _tied_table(rs, n, D)
    h[rs.rand(n, D) < 0.01] = np.nan
    h[rs.rand(n, D) < 0.01] = np.inf
    h[rs.rand(n, D) < 0.01] = -np.inf
    h[rs.rand(n, D) < 0.01] = LOWEST
    h[100:140] = 0.0                                          # ReLU rows of zeros
    h[140:150] = -np.inf
    ei[1, :2000] = rs.randint(100, 150, 2000)                 # many rows see them
    if layout == "odd_ld":
        wide = torch.empty((n, D + 3), dtype=torch.float32, device=DEV)
        wide[:, :D] = _dev(h)
        ht = wide[:, :D]
    else:
        ht = _dev(h)
    ei_t = _dev(ei)
    csr, w_csr, out, cnt, k1 = _k11a_both(ei_t, n, ht)
    assert csr.plan is not None and csr.plan.n_hubs >= 1
    _same_bits(out, k1, "out vs K1 MAX")
    _check_counts(csr, w_csr, ht, cnt, "awkward D={} {}".format(D, layout))
    assert int(cnt[17].max()) > 0


# ---- K11b ------------------------------------------------------------------------------------------------------

def _both_routes(h_np, ei_np, n, g_np, w_np=None):
    """(out, dh) of NeighborMax and of the composition TakeRows + SegmentReduce("max") it replaces."""
    from tf_geometric_b200 import autograd
    ei = _dev(ei_np)
    g = _dev(g_np)
    w = None if w_np is None else _dev(w_np)
    res = []
    for k11 in (True, False):
        h = _dev(h_np, grad=True)
        if k11:
            out = autograd.NeighborMax.apply(h, ei, w, n)
        else:
            msg = autograd.TakeRows.apply(h, ei[1].contiguous())
            if w is not None:
                msg = msg * w.unsqueeze(1)
            out = autograd.SegmentReduce.apply(msg, ei[0].contiguous(), n, "max")
        (dh,) = torch.autograd.grad(out, h, g)
        res.append((out.detach(), dh))
    return res


@pytest.mark.parametrize("weighted", [False, True])
@pytest.mark.parametrize("D", [1, 16, 47, 64, 128, 512, 600])
def test_k11b_is_bit_identical_to_the_composition(D, weighted):
    """Includes a NaN and an inf upstream entry (they reach every neighbour of their rows) and a source of out-degree
    60,000 (a hub row of the transposed CSR, summed through the plan where K1 would)."""
    rs = np.random.RandomState(3 * D + weighted)
    n = 2500
    ei = random_graph(n, 25000, seed=D, isolated=3)
    hub_src = np.stack([rs.randint(0, n, 60000), np.full(60000, 11)]).astype(np.int32)
    ei = np.concatenate([ei, hub_src], axis=1)[:, rs.permutation(ei.shape[1] + 60000)]
    h = _tied_table(rs, n, D)
    g = rs.randn(n, D).astype(np.float32)
    g[5, 0] = np.nan
    g[9, D - 1] = np.inf
    w = rs.choice([0.5, 1.0, 2.0, -1.5], ei.shape[1]).astype(np.float32) if weighted else None
    (out_k, dh_k), (out_c, dh_c) = _both_routes(h, ei, n, g, w)
    _same_bits(out_k, out_c, "forward")
    _same_bits(dh_k, dh_c, "dh")
    assert torch.isnan(dh_k).any()


def test_k11b_is_deterministic_and_agrees_with_float64():
    from tf_geometric_b200 import autograd
    rs = np.random.RandomState(4)
    n, D = 4000, 64
    ei_np = random_graph(n, 60000, seed=5, isolated=6, hub=(3, 9000))
    x_np = np.maximum(rs.randn(n, D), 0).astype(np.float32)          # ReLU: ties at 0 in fp32 and fp64 alike
    g_np = rs.randn(n, D).astype(np.float32)
    ei = _dev(ei_np)
    grads = []
    for _ in range(2):
        x = _dev(x_np, grad=True)
        (dx,) = torch.autograd.grad(autograd.NeighborMax.apply(x, ei, None, n), x, _dev(g_np))
        grads.append(dx)
    _same_bits(grads[0], grads[1], "run to run")
    x64 = torch.tensor(x_np, dtype=torch.float64, requires_grad=True)
    idx = torch.tensor(ei_np[0]).long().unsqueeze(1).expand(-1, D)
    want = torch.full((n, D), float(LOWEST), dtype=torch.float64).scatter_reduce(
        0, idx, x64[torch.tensor(ei_np[1]).long()], "amax", include_self=False)
    (want * torch.tensor(g_np, dtype=torch.float64)).sum().backward()
    np.testing.assert_allclose(grads[0].cpu().numpy(), x64.grad.numpy(), rtol=1e-5, atol=1e-5)


# ---- layers ----------------------------------------------------------------------------------------------------

def _composition(monkeypatch):
    """Device tensors take the composition TakeRows + SegmentReduce (the route host tensors take)."""
    from tf_geometric_b200 import autograd
    monkeypatch.setattr(autograd, "_is_device", lambda t: False)


def _max_sage_run(x_np, ei_np, seed):
    import tf_geometric_b200 as tfg
    layer = tfg.layers.MaxPoolGraphSage(64, activation=tfg.nn.relu, trainable=True, seed=seed)
    x = _dev(x_np, grad=True)
    ei = _dev(ei_np)
    out = layer([x, ei, torch.ones(ei.shape[1], device=DEV)])
    g = _dev(np.random.RandomState(9).randn(*out.shape).astype(np.float32))
    params = list(layer.parameters())
    grads = torch.autograd.grad(out, [x] + params, g)
    return [out.detach()] + list(grads)


def test_max_pool_graph_sage_forward_and_gradients_match_the_composition(monkeypatch):
    rs = np.random.RandomState(1)
    n = 3000
    ei = random_graph(n, 40000, seed=2, hub=(8, 5000))
    x = rs.randn(n, 40).astype(np.float32)
    new = _max_sage_run(x, ei, 3)
    _composition(monkeypatch)
    old = _max_sage_run(x, ei, 3)
    for i, (a, b) in enumerate(zip(new, old)):
        _same_bits(a, b, "output" if i == 0 else "gradient {}".format(i))


def _asap_run(x_np, ei_np, w_np, ngi_np, F):
    import tf_geometric_b200 as tfg
    p = {k: _dev(v, grad=True) for k, v in asap_ref.random_params(F, 4).items()}
    x = _dev(x_np, grad=True)
    px, _, _, _ = tfg.nn.asap(x, _dev(ei_np), _dev(w_np), _dev(ngi_np), *[p[k] for k in asap_ref.ORDER], None,
                              ratio=0.5)
    grads = torch.autograd.grad((px * px).sum(), [x] + [p[k] for k in asap_ref.ORDER], allow_unused=True)
    return [px.detach()] + [g if g is not None else torch.zeros(1, device=DEV) for g in grads]


def test_asap_forward_and_gradients_match_the_composition(monkeypatch):
    F = 16
    x, ei, w, ngi = asap_ref.batch([30, 25, 40, 2, 60], seed=9, F=F)
    new = _asap_run(x, ei, w, ngi, F)
    _composition(monkeypatch)
    old = _asap_run(x, ei, w, ngi, F)
    for i, (a, b) in enumerate(zip(new, old)):
        _same_bits(a, b, "pooled x" if i == 0 else "gradient {}".format(i))


@pytest.mark.parametrize("weighted", [False, True])
def test_aggregate_neighbors_max_against_float64(weighted):
    import tf_geometric_b200 as tfg
    from tf_geometric_b200.nn.kernel import map_reduce as mr
    rs = np.random.RandomState(6)
    n, D = 2000, 24
    ei = random_graph(n, 20000, seed=7, isolated=2)
    x_np = np.maximum(rs.randn(n, D), 0).astype(np.float32)
    w_np = (rs.rand(ei.shape[1]) + 0.5).astype(np.float32)
    g_np = rs.randn(n, D).astype(np.float32)
    x = _dev(x_np, grad=True)
    agg = tfg.nn.aggregate_neighbors(x, _dev(ei), _dev(w_np) if weighted else None,
                                     mr.gcn_mapper if weighted else mr.identity_mapper, mr.max_reducer, mr.sum_updater)
    (agg * _dev(g_np)).sum().backward()
    x64 = torch.tensor(x_np, dtype=torch.float64, requires_grad=True)
    msg = x64[torch.tensor(ei[1]).long()]
    if weighted:
        msg = msg * torch.tensor(w_np, dtype=torch.float64).unsqueeze(1)
    idx = torch.tensor(ei[0]).long().unsqueeze(1).expand(-1, D)
    want = x64 + torch.full((n, D), float(LOWEST), dtype=torch.float64).scatter_reduce(0, idx, msg, "amax",
                                                                                        include_self=False)
    (want * torch.tensor(g_np, dtype=torch.float64)).sum().backward()
    np.testing.assert_allclose(agg.detach().cpu().numpy(), want.detach().numpy(), rtol=1e-6)
    np.testing.assert_allclose(x.grad.cpu().numpy(), x64.grad.numpy(), rtol=1e-5, atol=1e-5)


def _planted(rs, n, k, p_in, p_out):
    labels = np.repeat(np.arange(k), n // k)
    same = labels[:, None] == labels[None, :]
    upper = np.triu(rs.rand(n, n) < np.where(same, p_in, p_out), 1)
    r, c = np.nonzero(upper)
    return np.stack([np.concatenate([r, c]), np.concatenate([c, r])]).astype(np.int32), labels


def test_two_layer_max_pool_graph_sage_learns_planted_partition():
    import tf_geometric_b200 as tfg
    rs = np.random.RandomState(0)
    n, c, f = 2000, 4, 16
    ei, labels = _planted(rs, n, c, 0.012, 0.0008)
    x = rs.randn(n, f).astype(np.float32)
    x[np.arange(n), labels] += 0.6
    x, y, ei = _dev(x), _dev(labels.astype(np.int64)), _dev(ei)
    w = torch.ones(ei.shape[1], device=DEV)
    perm = rs.permutation(n)
    train, test = _dev(perm[:n // 2].astype(np.int64)), _dev(perm[n // 2:].astype(np.int64))
    torch.manual_seed(0)
    sages = [tfg.layers.MaxPoolGraphSage(32, activation=tfg.nn.relu, trainable=True, seed=1),
             tfg.layers.MaxPoolGraphSage(32, activation=tfg.nn.relu, trainable=True, seed=2)]
    head = torch.nn.Linear(32, c, device=DEV)

    def forward():
        h = x
        for sage in sages:
            h = sage([h, ei, w])
        return head(h)

    forward()
    opt = torch.optim.Adam([p for s in sages for p in s.parameters()] + list(head.parameters()), lr=0.01)
    for _ in range(60):
        loss = torch.nn.functional.cross_entropy(forward()[train], y[train])
        opt.zero_grad()
        loss.backward()
        opt.step()
    with torch.no_grad():
        acc = float((forward()[test].argmax(1) == y[test]).float().mean())
    assert acc >= 0.8, "held-out accuracy {:.3f}".format(acc)


def test_max_pool_graph_sage_trains_at_the_products_shape():
    """One forward + backward of MaxPoolGraphSage(256) (a 512-wide neighbour MLP) at the ogbn-products shape used by
    bench.py: 2,449,029 nodes, 123,718,280 edges, 100 features.  The per-edge route needed 253 GB for each [E, 512] fp32
    tensor; the peak here stays below twelve [N, 512] fp32 tables plus 48 bytes per edge."""
    import tf_geometric_b200 as tfg
    n, e, f = 2449029, 123718280, 100
    gen = torch.Generator(device=DEV).manual_seed(0)
    ei = torch.randint(0, n, (2, e), dtype=torch.int32, device=DEV, generator=gen)
    x = torch.randn((n, f), device=DEV, generator=gen).requires_grad_()
    w = torch.ones(e, device=DEV)
    layer = tfg.layers.MaxPoolGraphSage(256, activation=tfg.nn.relu, trainable=True, seed=1)
    layer.build([(n, f)], device=x.device)
    layer.built = True
    torch.cuda.synchronize()
    torch.cuda.reset_peak_memory_stats()
    out = layer([x, ei, w])
    out.sum().backward()
    torch.cuda.synchronize()
    peak = torch.cuda.max_memory_allocated()
    bound = 12 * n * 512 * 4 + 48 * e
    print("products MaxPoolGraphSage(256) forward + backward: peak {:.2f} GB, bound {:.2f} GB".format(peak / 1e9,
                                                                                                    bound / 1e9))
    assert peak < bound
    assert torch.isfinite(x.grad).all() and all(torch.isfinite(p.grad).all() for p in layer.parameters())
