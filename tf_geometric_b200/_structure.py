# coding=utf-8
"""Memoisation of destination-sorted CSR structures.

The reference rebuilds nothing per call because tf.gather/unsorted_segment_sum need no preprocessing; the CUDA path
needs a dst-sorted CSR, built once per edge list and reused by every forward ("warm cache", the same regime as
`graph.cache` in demo/demo_gcn.py:47,99-105).  Keys are tensor identities (weakref + in-place version counter), so a
stale hit is impossible; a user-supplied `cache` dict (the `graph.cache` convention) takes precedence.
"""
import collections
import weakref

import torch

from . import ops

_LRU_CAPACITY = 16
_lru = collections.OrderedDict()


def _lookup(tensor, tag):
    key = (id(tensor), tag)
    hit = _lru.get(key)
    if hit is None:
        return None
    ref, version, shape, value = hit
    if ref() is tensor and tensor._version == version and tuple(tensor.shape) == shape:
        _lru.move_to_end(key)
        return value
    del _lru[key]
    return None


def _store(tensor, tag, value):
    key = (id(tensor), tag)
    _lru[key] = (weakref.ref(tensor), tensor._version, tuple(tensor.shape), value)
    _lru.move_to_end(key)
    while len(_lru) > _LRU_CAPACITY:
        _lru.popitem(last=False)
    return value


def clear():
    _lru.clear()


def csr_for_edge_index(edge_index, num_nodes, add_self_loop=False, cache=None):
    """CSR (rows = edge_index[0]) of a device int32 [2, E] edge list, optionally with the self loops that
    utils/graph_utils.py:350-366 appends.  Returns (csr, edge_index_used)."""
    tag = ("csr", int(num_nodes), bool(add_self_loop))
    if cache is not None:
        ckey = "tfgk_csr_{}_{}".format(int(num_nodes), "loop" if add_self_loop else "plain")
        hit = cache.get(ckey)
        if hit is not None and hit[0] is edge_index and hit[1] == edge_index._version:
            return hit[2], hit[3]
    hit = _lookup(edge_index, tag)
    if hit is None:
        used = ops.self_loops(edge_index, num_nodes) if add_self_loop else edge_index
        csr = ops.csr_build(used[0].contiguous(), used[1].contiguous(), num_nodes, num_nodes)
        hit = _store(edge_index, tag, (csr, used))
    if cache is not None:
        cache[ckey] = (edge_index, edge_index._version, hit[0], hit[1])
    return hit


def csr_for_segment_ids(segment_ids, num_segments):
    """CSR over a plain id vector (reducers / segment_softmax): col is unused, perm gathers the data rows."""
    tag = ("seg", int(num_segments))
    hit = _lookup(segment_ids, tag)
    if hit is None:
        zeros = torch.zeros_like(segment_ids)
        hit = _store(segment_ids, tag, ops.csr_build(segment_ids, zeros, num_segments, 1))
    return hit


def weights_in_csr_order(edge_weight, csr):
    """edge_weight permuted into the order of `csr`, memoised per (weight tensor, CSR object); the CSR is held by weak
    reference so that a recycled id() can never alias another structure."""
    tag = ("wcsr", id(csr))
    hit = _lookup(edge_weight, tag)
    if hit is not None and hit[0]() is csr:
        return hit[1]
    value = ops.permute(edge_weight, csr.perm)
    _store(edge_weight, tag, (weakref.ref(csr), value))
    return value
