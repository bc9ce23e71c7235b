# coding=utf-8
"""Op-for-op torch restatements of the reference's convert_x_to_3d (utils/graph_utils.py:215-249) and lstm_graph_sage
(nn/conv/graph_sage.py:290-356), in any dtype, for float64 autograd comparisons; and a Keras-convention LSTM callable
made of torch ops (gate order i, f, c, o; zero initial state; returns the sequence)."""
import numpy as np
import torch


def torch_lstm(kernel, recurrent_kernel, bias):
    """lstm(inputs [B, T, F], training=None) -> [B, T, U] in the dtype and on the device of the weights."""
    units = recurrent_kernel.shape[0]

    def lstm(inputs, training=None):
        inputs = inputs.to(kernel.dtype)
        h = inputs.new_zeros((inputs.shape[0], units))
        c = inputs.new_zeros((inputs.shape[0], units))
        seq = []
        for t in range(inputs.shape[1]):
            z = inputs[:, t] @ kernel + h @ recurrent_kernel + bias
            i, f, g, o = (z[:, j * units:(j + 1) * units] for j in range(4))
            c = torch.sigmoid(f) * c + torch.sigmoid(i) * torch.tanh(g)
            h = torch.sigmoid(o) * torch.tanh(c)
            seq.append(h)
        return torch.stack(seq, dim=1)
    return lstm


def neighbor_matrix(edge_index, num_nodes):
    """(matrix [N, K] with num_nodes for padding, K): graph_sage.py:316-331, argsort stable by row."""
    row, col = np.asarray(edge_index[0]), np.asarray(edge_index[1])
    order = np.argsort(row, kind="stable")
    row, col = row[order], col[order]
    degree = np.bincount(row, minlength=num_nodes)
    K = int(degree.max())
    before = np.concatenate([[0], np.cumsum(degree)[:-1]])
    j = np.arange(len(row)) - before[row]
    m = np.full((num_nodes, K), num_nodes, np.int64)
    m[row, j] = col
    return m, K


def lstm_graph_sage(x, edge_index, lstm, self_kernel, neighbor_kernel, bias=None, activation=None, concat=True,
                    normalize=False):
    m, _ = neighbor_matrix(edge_index, x.shape[0])
    padded_x = torch.cat([x, x.new_zeros((1, x.shape[1]))], dim=0)
    h = lstm(padded_x[torch.as_tensor(m, device=x.device)]).mean(dim=1)
    from_neighbor = h @ neighbor_kernel
    from_x = x @ self_kernel
    out = torch.cat([from_x, from_neighbor], dim=1) if concat else from_x + from_neighbor
    if bias is not None:
        out = out + bias
    if activation is not None:
        out = activation(out)
    if normalize:
        out = out / torch.sqrt(torch.clamp((out * out).sum(-1, keepdim=True), min=1e-12))
    return out


def convert_x_to_3d(x, source_index, k=None, pad=True):
    """numpy: stable grouping, zero-padded to k (graph_utils.py:215-249)."""
    x, sid = np.asarray(x), np.asarray(source_index)
    counts = np.bincount(sid)
    largest = int(counts.max())
    if k is None or (k > largest and not pad):
        k = largest
    out = np.zeros((len(counts), k, x.shape[1]), x.dtype)
    seen = np.zeros(len(counts), np.int64)
    for i in range(len(sid)):
        s = sid[i]
        if seen[s] < k:
            out[s, seen[s]] = x[i]
        seen[s] += 1
    return out
