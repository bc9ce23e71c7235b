# coding=utf-8
"""TEST DOUBLE for the link-prediction wrappers of tf_geometric_b200.ops (K6 edge scoring, negative sampling): the
CPU fake kernel layer of tests/fake_backend.py plus these ops, restated by tests/link_oracle.py, so that the host logic
of predict_edge / negative_sampling / negative_sampling_with_start_node / edge_train_test_split runs without a GPU.
It lives under tests/ and is injected with monkeypatch; the product has no such path."""
import numpy as np

import fake_backend
import link_oracle as lo
from fake_backend import _np, _t


def install(monkeypatch):
    fake_backend.install(monkeypatch)
    from tf_geometric_b200 import ops

    def edge_dot(h, row, col, out=None):
        hn, r, c = _np(h), _np(row), _np(col)
        return _t((hn[r] * hn[c]).sum(-1, dtype=np.float32).astype(np.float32))

    def neg_offsets(csr, mode):
        rowptr, n = _np(csr.rowptr), csr.n_rows
        base = np.zeros(n, np.int64) if mode == ops.NEG_START else np.arange(1, n + 1, dtype=np.int64)
        counts = np.maximum((n - base) - np.diff(rowptr), 0)
        offsets = np.concatenate([[0], np.cumsum(counts)]).astype(np.int64)
        return _t(offsets), int(offsets[-1])

    def neg_draw(C, n, seed, round=0, index=None, out=None, device=None, rng_stream=ops.RNG_STREAM_LINK):
        idx = np.arange(n, dtype=np.uint64) if index is None else _np(index).astype(np.uint64)
        vals = lo.random_below64(seed, rng_stream, (np.uint64(round) << np.uint64(32)) | idx, C)
        k = np.zeros(n, np.int64) if out is None else _np(out).copy()
        k[idx.astype(np.int64)] = vals
        if out is not None:
            out.copy_(_t(k))
            return out
        return _t(k)

    def neg_dup_flags(k, order):
        kn, od = _np(k), _np(order)
        flag = np.zeros(len(kn), np.int32)
        flag[od[1:]] = kn[od[1:]] == kn[od[:-1]]
        return _t(flag)

    def neg_decode(csr, offsets, mode, k):
        return _t(lo.negative_decode(_np(csr.rowptr), _np(csr.col), _np(offsets), _np(k), start=mode == ops.NEG_START))

    def neg_sample_start(csr, start, seed, rng_stream=ops.RNG_STREAM_LINK):
        rowptr, col, n = _np(csr.rowptr), _np(csr.col), csr.n_rows
        out = np.empty(start.numel(), np.int32)
        for s, a in enumerate(_np(start)):
            cnt = n - int(rowptr[a + 1] - rowptr[a])
            r = int(lo.random_below64(seed, rng_stream, np.array([s], np.uint64), cnt)[0]) if cnt > 0 else -1
            out[s] = lo._decode_in_row(col[rowptr[a]:rowptr[a + 1]], 0, r) if cnt > 0 else -1
        return _t(out)

    def random_pairs(num_nodes, num_samples, seed, device, rng_stream=ops.RNG_STREAM_LINK):
        s2 = np.arange(num_samples, dtype=np.uint64) * np.uint64(2)
        return _t(np.stack([lo.random_below64(seed, rng_stream, s2, num_nodes),
                            lo.random_below64(seed, rng_stream, s2 + np.uint64(1), num_nodes)]).astype(np.int32))

    for name, fn in dict(edge_dot=edge_dot, neg_offsets=neg_offsets, neg_draw=neg_draw, neg_dup_flags=neg_dup_flags,
                         neg_decode=neg_decode, neg_sample_start=neg_sample_start, random_pairs=random_pairs).items():
        monkeypatch.setattr(ops, name, fn)
