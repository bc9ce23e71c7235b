# coding=utf-8
"""Host side of CUDA-graph capture, without a GPU: the device-key entry points of libtfgk.so, the key sequence of _rng
outside and inside a (mocked) capture, and the refusal of every host-synchronising op before it launches anything."""
import ctypes
import os
import re

import numpy as np
import pytest
import torch

import tf_geometric_b200 as tfg
from tf_geometric_b200 import _ffi, _rng, ops

HEADER = open(os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "include", "tfgk.h")).read()

DEVKEY_ENTRIES = ["tfgk_dropout_devkey_f32", "tfgk_spmm_heads_devkey_f32", "tfgk_gat_softmax_bwd_devkey_f32",
                  "tfgk_rng_advance", "tfgk_capture_id"]


def _header_arity(name):
    m = re.search(r"\bint\s+" + name + r"\s*\(([^;]*)\)\s*;", HEADER)
    assert m, name
    return len([a for a in m.group(1).split(",") if a.strip()])


@pytest.mark.parametrize("name", DEVKEY_ENTRIES)
def test_devkey_entries_are_exported_with_the_header_arity(name):
    lib = _ffi.lib()
    assert hasattr(lib, name)
    assert len(_ffi.SIGNATURES[name]) == _header_arity(name)


def test_devkey_entries_replace_the_seed_by_base_and_slot():
    for name in ("tfgk_dropout", "tfgk_spmm_heads", "tfgk_gat_softmax_bwd"):
        plain, dev = _ffi.SIGNATURES[name + "_f32"], _ffi.SIGNATURES[name + "_devkey_f32"]
        i = plain.index(_ffi._u64)
        assert dev[:i] == plain[:i] and dev[i:i + 2] == [_ffi._ptr, _ffi._u64] and dev[i + 2:] == plain[i + 1:]


def _status(name, *args):
    lib = _ffi.lib()
    rc = getattr(lib, name)(*args)
    return rc, lib.tfgk_last_error().decode()


def test_devkey_entries_check_their_arguments():
    base = ctypes.c_uint64(0)
    out = ctypes.c_float(0)
    # null key_base
    rc, msg = _status("tfgk_dropout_devkey_f32", None, 1, 0.5, None, 0, 0, ctypes.byref(out), None)
    assert rc == _ffi.ERR_INVALID_ARGUMENT and "key_base" in msg
    rc, msg = _status("tfgk_spmm_heads_devkey_f32", None, None, None, None, None, 8, 1, 1, 8, 0, 0.5, None, 0, 0, 1.0,
                      None, 0, None, 8, None)
    assert rc == _ffi.ERR_INVALID_ARGUMENT and "key_base" in msg
    rc, msg = _status("tfgk_gat_softmax_bwd_devkey_f32", None, None, None, None, 8, None, 8, 1, 1, 8, 1, 0.5, None, 0, 0,
                      None, None)
    assert rc == _ffi.ERR_INVALID_ARGUMENT and "key_base" in msg
    rc, msg = _status("tfgk_rng_advance", None, None, None)
    assert rc == _ffi.ERR_INVALID_ARGUMENT and "key_base" in msg
    rc, msg = _status("tfgk_capture_id", None, None)
    assert rc == _ffi.ERR_INVALID_ARGUMENT
    # negative sizes and rates outside [0, 1), with a key_base given (checked before any launch)
    rc, msg = _status("tfgk_dropout_devkey_f32", None, -1, 0.5, ctypes.byref(base), 0, 0, ctypes.byref(out), None)
    assert rc == _ffi.ERR_INVALID_ARGUMENT and "negative" in msg
    rc, msg = _status("tfgk_dropout_devkey_f32", None, 1, 1.0, ctypes.byref(base), 0, 0, ctypes.byref(out), None)
    assert rc == _ffi.ERR_INVALID_ARGUMENT and "rate" in msg
    rc, msg = _status("tfgk_spmm_heads_devkey_f32", None, None, None, None, None, 8, -1, 1, 8, 0, 0.5, ctypes.byref(base),
                      0, 0, 1.0, None, 0, None, 8, None)
    assert rc == _ffi.ERR_INVALID_ARGUMENT and "bad size" in msg
    rc, msg = _status("tfgk_gat_softmax_bwd_devkey_f32", None, None, None, None, 8, None, 8, -1, 1, 8, 1, 0.5,
                      ctypes.byref(base), 0, 0, None, None)
    assert rc == _ffi.ERR_INVALID_ARGUMENT and "bad size" in msg
    # empty work with a valid key_base launches nothing
    rc, _ = _status("tfgk_dropout_devkey_f32", None, 0, 0.5, ctypes.byref(base), 0, 0, None, None)
    assert rc == _ffi.OK


# ---- the key sequence ------------------------------------------------------------------------------------------------

def _np_key(base, j):
    """The header's rule in numpy uint64 arithmetic (wrapping): splitmix64(base + golden * (j + 1))."""
    with np.errstate(over="ignore"):
        z = np.uint64(base) + np.uint64(_rng.GOLDEN) * np.uint64(j + 1)
        z = (z ^ (z >> np.uint64(30))) * np.uint64(0xBF58476D1CE4E5B9)
        z = (z ^ (z >> np.uint64(27))) * np.uint64(0x94D049BB133111EB)
        return int(z ^ (z >> np.uint64(31)))


@pytest.mark.parametrize("base", [0, 1, 0x5DEECE66D, (1 << 64) - 1, 0x8000000000000000])
def test_key_rule_restatement_equals_next_seed(base):
    tfg.set_seed(base)
    for j in range(1000):
        assert _rng.next_seed() == _np_key(base, j)


def test_resolve_outside_capture_is_the_host_sequence():
    # the sequence of earlier releases: splitmix64 of (base + golden * calls), explicit seeds reduced mod 2^64
    def legacy(seed, calls):
        m = (1 << 64) - 1
        z = (seed + 0x9E3779B97F4A7C15 * calls) & m
        z = ((z ^ (z >> 30)) * 0xBF58476D1CE4E5B9) & m
        z = ((z ^ (z >> 27)) * 0x94D049BB133111EB) & m
        return z ^ (z >> 31)
    tfg.set_seed(77)
    got = [_rng.resolve(None, torch.device("cpu")) for _ in range(20)]
    assert got == [legacy(77, c) for c in range(1, 21)]
    assert _rng.resolve(-1) == (1 << 64) - 1 and _rng.resolve(5) == 5
    assert _rng.resolve_host(None) == legacy(77, 21)


@pytest.fixture
def mocked_capture(monkeypatch):
    """Capture switched on, CPU tensors standing in for the device base and the epoch words, capture ids and advances
    (with the word each one writes) recorded."""
    state = {"id": 41, "advances": []}
    base = torch.zeros(1, dtype=torch.int64)
    words = torch.zeros(4, dtype=torch.int64)
    monkeypatch.setattr(_rng, "_device_index", lambda device: 0)
    monkeypatch.setattr(_rng, "_bases", {0: base})
    monkeypatch.setattr(_rng, "_epochs", {0: {"spare": [words[i:i + 1] for i in range(4)], "taken": []}})
    monkeypatch.setattr(_rng, "_capture", {"id": 0, "epoch": None, "draws": 0})
    monkeypatch.setattr(_rng, "_capture_id", lambda b: state["id"])

    def advance(b, epoch):
        assert b is base
        state["advances"].append(epoch)
    monkeypatch.setattr(_rng, "_advance", advance)
    tfg.set_seed(3)
    monkeypatch.setattr(_ffi, "capturing", lambda: True)
    return state, base


def test_resolve_under_capture_returns_consecutive_slots(mocked_capture):
    state, base = mocked_capture
    calls_before = _rng._state["calls"]
    keys = [_rng.resolve(None) for _ in range(5)]
    assert all(isinstance(k, _rng.DeviceKey) for k in keys)
    assert [k.slot for k in keys] == list(range(5))
    assert len(state["advances"]) == 1                     # once, at the first draw of the capture ...
    first = state["advances"][0]
    assert all(k.base is first for k in keys)              # ... which writes the word every key of the capture reads
    assert first is not base
    assert _rng._state["calls"] == calls_before            # the host sequence does not move
    assert _rng.resolve(1234) == 1234                      # an explicit seed stays a constant key
    state["id"] = 42                                       # a new capture: a new epoch in a word of its own
    again = [_rng.resolve(None) for _ in range(3)]
    assert [k.slot for k in again] == [0, 1, 2]
    assert len(state["advances"]) == 2 and state["advances"][1] is not first
    assert all(k.base is state["advances"][1] for k in again)
    assert _rng.capture_epochs() == state["advances"]


def test_each_capture_keeps_its_own_epoch_word(mocked_capture):
    # make_graphed_callables over two modules replays fwd1, fwd2, bwd2, bwd1: bwd1 must still read fwd1's epoch, so the
    # second capture's advance must not write the word the first capture's keys point at
    state, _ = mocked_capture
    k1 = _rng.resolve(None)
    state["id"] = 43
    k2 = _rng.resolve(None)
    assert k1.base.data_ptr() != k2.base.data_ptr()


def test_captures_beyond_the_spare_words_ask_for_an_eager_step(mocked_capture):
    state, _ = mocked_capture
    for cid in range(100, 104):
        state["id"] = cid
        _rng.resolve(None)
    state["id"] = 104
    with pytest.raises(RuntimeError, match="Run an eager step between captures"):
        _rng.resolve(None)


def test_a_draw_on_a_stream_that_is_not_capturing_is_refused(mocked_capture):
    state, _ = mocked_capture
    state["id"] = 0
    with pytest.raises(RuntimeError, match="must draw on its own device"):
        _rng.resolve(None)


def test_set_seed_is_refused_under_capture(mocked_capture):
    with pytest.raises(RuntimeError, match="set_seed cannot be captured"):
        tfg.set_seed(5)


def test_resolve_under_capture_without_a_base_asks_for_a_warm_up(mocked_capture, monkeypatch):
    monkeypatch.setattr(_rng, "_bases", {})
    with pytest.raises(RuntimeError, match="run one eager step before capturing"):
        _rng.resolve(None)


def test_ops_route_device_keys_to_the_devkey_entries(mocked_capture, monkeypatch):
    calls = []
    monkeypatch.setattr(_ffi, "call", lambda name, *args: calls.append((name, args)))
    monkeypatch.setattr(ops, "_check", lambda *a: None)
    monkeypatch.setattr(ops, "_stream", lambda t: None)
    key = _rng.resolve(None)
    x = torch.ones(8)
    ops.dropout(x, 0.5, key)
    ops.dropout(x, 0.5, 99)
    assert calls[0][0] == "tfgk_dropout_devkey_f32" and calls[0][1][3].value == _rng.capture_epochs()[0].data_ptr()
    assert calls[0][1][4] == key.slot
    assert calls[1][0] == "tfgk_dropout_f32" and calls[1][1][3] == 99


# ---- refusals --------------------------------------------------------------------------------------------------------

# entries that only compute sizes on the host: calling them launches nothing
HOST_QUERIES = re.compile(r"_workspace_bytes$|^tfgk_plan_capacity$|^tfgk_version$")


class _RecordingLib(object):
    def __init__(self):
        self.calls = []

    def __getattr__(self, name):
        def fn(*args):
            self.calls.append(name)
            return 0
        return fn


@pytest.fixture
def refusing(monkeypatch):
    rec = _RecordingLib()
    monkeypatch.setattr(_ffi, "lib", lambda: rec)
    monkeypatch.setattr(_ffi, "capturing", lambda: True)
    monkeypatch.setattr(ops, "_check", lambda *a: None)
    monkeypatch.setattr(ops, "_stream", lambda t: None)
    cpu = torch.device("cpu")
    monkeypatch.setattr(ops, "default_device", lambda: cpu)
    monkeypatch.setattr(ops, "as_device", lambda x, dtype=None, device=None: None if x is None else (
        torch.as_tensor(np.asarray(x) if not torch.is_tensor(x) else x).to(dtype or (x.dtype if torch.is_tensor(x)
                                                                                       else None)).contiguous()))
    return rec


def _i32(*a):
    return torch.tensor(a, dtype=torch.int32)


def _csr():
    return ops.CSR(torch.tensor([0, 1, 2], dtype=torch.int64), _i32(1, 0), _i32(0, 1), 2, 2)


REFUSED = {
    "csr_build": (lambda: ops.csr_build(_i32(0, 1), _i32(1, 0), 2), "CSR build"),
    "build_plan": (lambda: ops.build_plan(_csr()), "work-plan build"),
    "edge_unique": (lambda: ops.edge_unique(_i32(0, 1), _i32(1, 0), 2), "edge merge"),
    "select_flagged": (lambda: ops.select_flagged(_i32(1, 0, 1)), "select_flagged"),
    "drop_edge": (lambda: tfg.nn.drop_edge([_i32(0, 1, 1, 0).reshape(2, 2)], 0.5, training=True), "edge filtering"),
    "neighbor_sample": (lambda: ops.neighbor_sample(_csr(), k=1), "neighbour sampler"),
    "negative_sampling": (lambda: tfg.utils.negative_sampling(4, 3, edge_index=_i32(0, 1, 1, 0).reshape(2, 2)),
                          "edge filtering"),
    "random_pairs": (lambda: tfg.utils.negative_sampling(4, 3), "negative sampling"),
    "spgemm": (lambda: ops.spgemm(_csr().rowptr, _csr().col, torch.ones(2), _csr().rowptr, _csr().col, torch.ones(2), 2),
               "K10's plan"),
    "spgemm_rowptr": (lambda: ops._ffi.call("tfgk_spgemm_rowptr"), "K10's row pointers"),
    "spgemm_grad_plan": (lambda: ops._ffi.call("tfgk_spgemm_grad_plan"), "K12's plan"),
    "topk_pool": (lambda: tfg.nn.topk_pool(_i32(0, 0, 1), torch.ones(3), ratio=0.5), "topk_pool"),
    "lambda_max": (lambda: __import__("tf_geometric_b200.nn.conv.propagation", fromlist=["x"]).laplacian_max_eigenvalue(
        _i32(0, 1, 1, 0).reshape(2, 2), 2, None), "dynamic lambda_max"),
}


@pytest.mark.parametrize("op", sorted(REFUSED))
def test_host_synchronising_ops_refuse_capture_before_any_kernel(op, refusing):
    fn, what = REFUSED[op]
    with pytest.raises(RuntimeError, match=re.escape(what) + ".*cannot be captured in a CUDA graph"):
        fn()
    launched = [c for c in refusing.calls if not HOST_QUERIES.search(c)]
    assert launched == [], "{} launched {} before refusing".format(op, launched)


def test_every_refused_entry_is_exported():
    lib = _ffi.lib()
    for name in _ffi.NOT_CAPTURABLE:
        assert hasattr(lib, name), name
