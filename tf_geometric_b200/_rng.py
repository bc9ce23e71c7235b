# coding=utf-8
"""Seeds for the counter-based dropout / sampling kernels.

The reference relies on TensorFlow's and numpy's global generators (tf.nn.dropout in gcn.py:262 / gat.py:85,
tf.random.uniform and np.random.choice in utils/graph_utils.py:741-841).  Here every random operator call takes a
64-bit Philox key; callers may pass one explicitly (`seed=`) for reproducible runs, otherwise it is derived from a
process-wide base seed and a call counter, so consecutive calls draw independent masks.

Under CUDA-graph capture a key passed by value would be replayed unchanged, so `resolve(None)` then returns a
`DeviceKey` instead: the key is computed on the device, by the same rule as `next_seed` (include/tfgk.h, "device keys"),
from the draw's slot in the captured region and that region's epoch word.  The first draw of a capture enqueues
tfgk_rng_advance, which moves the device's base to a new epoch and copies it into the epoch word, so every replay draws new
masks, and a backward regenerates its forward's masks from the word its forward read, whatever other graphs replay in
between."""
import collections
import ctypes
import threading

from . import _ffi

_lock = threading.Lock()
_state = {"seed": 0x5DEECE66D, "calls": 0}
_MASK64 = (1 << 64) - 1
GOLDEN = 0x9E3779B97F4A7C15

_bases = {}                                   # device index -> int64 [1] tensor holding the base of the device keys
# device index -> {"spare": epoch words not yet given to a capture, "taken": the words captures took, in order}.  The
# words are int64 [1] views of chunks allocated by eager draws: memory allocated during a capture would come from that
# graph's private pool
_epochs = {}
EPOCH_CHUNK = 256                             # words per allocation
EPOCH_RESERVE = 64                            # an eager draw allocates a new chunk when fewer words than this are spare
# the capture sequence that drew last, its epoch word and how many keys it drew.  Captures are recorded one at a time:
# the process-wide counter assumes no two threads capture graphs that draw keys at once
_capture = {"id": 0, "epoch": None, "draws": 0}


class DeviceKey(collections.namedtuple("DeviceKey", "base slot")):
    """The key of draw `slot` of a captured region: splitmix64(base[0] + GOLDEN * (slot + 1)), computed by the kernel
    when the graph runs.  `base` is the region's epoch word (int64 [1]), which each replay sets to the device's advanced
    base before the region's first keyed launch."""


def splitmix64(z):
    """The output function of splitmix64 (no Weyl step), on Python ints."""
    z = ((z ^ (z >> 30)) * 0xBF58476D1CE4E5B9) & _MASK64
    z = ((z ^ (z >> 27)) * 0x94D049BB133111EB) & _MASK64
    return z ^ (z >> 31)


def _signed(v):
    return v - (1 << 64) if v >= (1 << 63) else v


def set_seed(seed):
    """Reset the process-wide base seed (the analogue of tf.random.set_seed / np.random.seed), and the base of the
    device keys on every device that has one.  Refused while the current stream records a CUDA graph: the graph would
    reset the base on every replay and so draw the same masks every time."""
    if _ffi.capturing():
        raise RuntimeError("set_seed cannot be captured in a CUDA graph: every replay would reset the device-key base and "
                           "draw the same masks. Call it outside the capture.")
    with _lock:
        _state["seed"] = int(seed) & _MASK64
        _state["calls"] = 0
        for base in _bases.values():
            base.fill_(_signed(_state["seed"]))


def next_seed():
    """A fresh 64-bit key: splitmix64 of (base seed + call counter)."""
    with _lock:
        _state["calls"] += 1
        z = (_state["seed"] + GOLDEN * _state["calls"]) & _MASK64
    return splitmix64(z)


def _device_index(device):
    import torch
    if device is None:
        return torch.cuda.current_device() if torch.cuda.is_available() else None
    device = torch.device(device)
    if device.type != "cuda":
        return None
    return torch.cuda.current_device() if device.index is None else device.index


def key_base(device=None):
    """The int64 [1] base tensor of the device keys on `device` (default: the current device), or None before the
    first eager draw there.  Read it as an unsigned 64-bit value with `int(t.item()) & (2**64 - 1)`."""
    return _bases.get(_device_index(device))


def capture_epochs(device=None):
    """The epoch words of the captures that drew keys on `device`, in capture order (int64 [1] tensors).  After a replay,
    word k holds the base that replay's k-th capture drew its keys from; tfg.set_seed(that value) before the same calls
    run eagerly reproduces its masks."""
    return list(_epochs.get(_device_index(device), {}).get("taken", ()))


def _ensure_base(device):
    idx = _device_index(device)
    if idx is None or (idx in _bases and len(_epochs[idx]["spare"]) >= EPOCH_RESERVE):
        return
    import torch
    dev = torch.device("cuda", idx)
    with _lock:
        if idx not in _bases:
            _bases[idx] = torch.tensor([_signed(_state["seed"])], dtype=torch.int64, device=dev)
            _epochs[idx] = {"spare": [], "taken": []}
        if len(_epochs[idx]["spare"]) < EPOCH_RESERVE:
            chunk = torch.zeros((EPOCH_CHUNK,), dtype=torch.int64, device=dev)
            _epochs[idx]["spare"].extend(chunk[i:i + 1] for i in range(EPOCH_CHUNK))


def _stream(base):
    import torch
    return ctypes.c_void_p(torch.cuda.current_stream(base.device).cuda_stream)


def _capture_id(base):
    cid = ctypes.c_uint64()
    _ffi.call("tfgk_capture_id", _stream(base), ctypes.byref(cid))
    return cid.value


def _advance(base, epoch):
    _ffi.call("tfgk_rng_advance", ctypes.c_void_p(base.data_ptr()), ctypes.c_void_p(epoch.data_ptr()), _stream(base))


def _capture_draw(device):
    idx = _device_index(device)
    base = _bases.get(idx)
    if base is None:
        raise RuntimeError("a random draw under CUDA-graph capture needs the device-key base of cuda:{}, which is created "
                           "by the first eager draw on that device: run one eager step before capturing".format(idx))
    cid = _capture_id(base)
    if cid == 0:
        raise RuntimeError("a random draw on cuda:{} while another device's stream records a CUDA graph: a captured "
                           "region must draw on its own device".format(idx))
    with _lock:
        if cid != _capture["id"]:
            # first draw of this capture: the graph starts by moving the base to the next epoch, into a word of its own
            spare = _epochs[idx]["spare"]
            if not spare:
                raise RuntimeError("no spare device-key epoch word on cuda:{}: graphs captured since the last eager draw "
                                   "there took every one (at least {}). Run an eager step between captures"
                                   .format(idx, EPOCH_RESERVE))
            epoch = spare.pop(0)
            _advance(base, epoch)
            _epochs[idx]["taken"].append(epoch)
            _capture["id"], _capture["epoch"], _capture["draws"] = cid, epoch, 0
        slot = _capture["draws"]
        _capture["draws"] += 1
        epoch = _capture["epoch"]
    return DeviceKey(epoch, slot)


def resolve(seed, device=None):
    """The key of one random operator call on `device` (default: the current CUDA device).

    Eagerly: `seed` itself, or the next host key when it is None (the first eager call on a device also creates that
    device's key base).  While the current stream records a CUDA graph and `seed` is None: a DeviceKey, whose key the
    kernel derives from the device's base when the graph runs, so every replay draws new masks.  An explicit `seed`
    stays a constant key under capture too: every replay then draws the same mask."""
    if seed is not None:
        return int(seed) & _MASK64
    if _ffi.capturing():
        return _capture_draw(device)
    _ensure_base(device)
    return next_seed()


def resolve_host(seed):
    """`seed`, or the next host key: for the samplers and negative sampling, whose kernels take only a host key.  Those
    ops synchronise with the host and refuse to run under CUDA-graph capture (see _ffi.NOT_CAPTURABLE)."""
    return next_seed() if seed is None else int(seed) & _MASK64
