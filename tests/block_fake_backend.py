# coding=utf-8
"""TEST DOUBLE for the block sampler (ops.block_sample), the in-range CSR build and K11 (ops.spmm_max / spmm_max_bwd): the CPU fakes of
tests/minibatch_fake_backend.py plus a numpy restatement of the block sampler built on tests/minibatch_ref.py, so that
the host logic of RandomNeighborSampler.sample_blocks and of GraphSAGE over blocks runs without a GPU.  Injected with
monkeypatch; the product has no such path.  `calls` records the ids_in_range flag of every CSR build."""
import numpy as np

import minibatch_fake_backend
import minibatch_ref as ref
from fake_backend import _np, _t


def install(monkeypatch):
    minibatch_fake_backend.install(monkeypatch)
    from tf_geometric_b200 import ops
    fake_as_device = ops.as_device

    def as_device(x, dtype=None, device=None):           # the product's refusal of sampled inputs, then the fake
        ops.refuse_sampled(x)
        return fake_as_device(x, dtype, device)
    calls = {"csr_build": []}
    plain_csr_build = ops.csr_build

    def csr_build(row, col, n_rows, n_cols=None, ids_in_range=False):
        calls["csr_build"].append(bool(ids_in_range))
        return plain_csr_build(row, col, n_rows, n_cols)

    def block_sample(rowptr, col, w_csr, seeds, fanouts, keys, node_map, padding=False, rng_stream=1):
        assert np.all(_np(node_map) == -1), "the map must be clean between calls"
        if not isinstance(padding, bool) and padding == ops.SAMPLE_HEAD:
            padding = "head"
        rowptr, col, w_csr, N = _np(rowptr), _np(col), _np(w_csr), node_map.numel()
        nodes = [int(v) for v in _np(seeds)]
        n_bad = sum(1 for v in nodes if v < 0 or v >= N)
        n_dup = len(nodes) - len(set(nodes))
        if n_bad or n_dup:
            return _t(np.array(nodes, np.int32)), [len(nodes)] * (len(fanouts) + 1), [], n_bad, n_dup
        where = {v: i for i, v in enumerate(nodes)}
        sizes, hops = [len(nodes)], []
        for k, key in zip(fanouts, keys):
            t, pos, offsets = ref.sample_rows(rowptr, np.array(nodes, np.int64), k, None, padding, key, rng_stream)
            gcol = col[pos].astype(np.int32)
            for c in gcol.tolist():
                if c not in where:
                    where[c] = len(nodes)
                    nodes.append(c)
            local = np.array([where[c] for c in gcol.tolist()], np.int32)
            hops.append((_t(offsets), _t(t), _t(local), _t(gcol), _t(w_csr[pos].astype(np.float32))))
            sizes.append(len(nodes))
        return _t(np.array(nodes, np.int32)), sizes, hops, 0, 0

    def spmm_max(csr, w_csr, h):
        assert w_csr is None
        rp, c, hn = _np(csr.rowptr), _np(csr.col), _np(h)
        out = np.full((csr.n_rows, hn.shape[1]), np.finfo(np.float32).min, np.float32)
        cnt = np.zeros(out.shape, np.int32)
        for r in range(csr.n_rows):
            if rp[r + 1] > rp[r]:
                m = hn[c[rp[r]:rp[r + 1]]]
                out[r] = m.max(axis=0)
                cnt[r] = (m == out[r]).sum(axis=0)
        return _t(out), _t(cnt)

    def spmm_max_bwd(csr_t, w_t, h, out, cnt, g):
        assert w_t is None
        rp, r_of, hn, o, n, gn = (_np(t) for t in (csr_t.rowptr, csr_t.col, h, out, cnt, g))
        dh = np.zeros(hn.shape, np.float32)
        for src in range(csr_t.n_rows):
            for r in r_of[rp[src]:rp[src + 1]]:
                dh[src] += (gn[r] / np.maximum(n[r], 1)) * (hn[src] == o[r])
        return _t(dh)

    monkeypatch.setattr(ops, "as_device", as_device)
    monkeypatch.setattr(ops, "spmm_max", spmm_max)
    monkeypatch.setattr(ops, "spmm_max_bwd", spmm_max_bwd)
    monkeypatch.setattr(ops, "csr_build", csr_build)
    monkeypatch.setattr(ops, "block_sample", block_sample)
    return calls
