#!/usr/bin/env python
# coding=utf-8
"""Peer-pull bandwidth over NVLink (run under torchrun with >= 2 ranks): every rank pulls a buffer from rank+1 with
tfgk_peer_pull at several CTA counts, and with a copy-engine transfer of the same bytes for comparison."""
import ctypes
import json
import os
import sys

import torch
import torch.distributed as dist

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from tf_geometric_b200 import peer, _ffi  # noqa: E402

rank, world, local = int(os.environ["RANK"]), int(os.environ["WORLD_SIZE"]), int(os.environ["LOCAL_RANK"])
torch.cuda.set_device(local)
dev = torch.device("cuda", local)
os.environ.setdefault("NCCL_DEBUG", "WARN")
dist.init_process_group("nccl", device_id=dev)
nbytes = int(float(os.environ.get("GB", "2")) * (1 << 30))
buf = peer.PeerBuffer(nbytes, dev)
buf.local.fill_(rank + 1)
dst = torch.empty(nbytes, dtype=torch.uint8, device=dev)
src_rank = (rank + 1) % world
stream = torch.cuda.current_stream(dev)
res = {}


def timed(fn, reps=5):
    fn()
    torch.cuda.synchronize(); dist.barrier(); torch.cuda.synchronize()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(reps):
        fn()
    b.record()
    torch.cuda.synchronize()
    t = torch.tensor([a.elapsed_time(b) / reps], device=dev)
    dist.all_reduce(t, op=dist.ReduceOp.MAX)
    return float(t)


sms = torch.cuda.get_device_properties(dev).multi_processor_count
for ctas in (32, 64, sms, 2 * sms, 4 * sms, 8 * sms):
    ms = timed(lambda: _ffi.call("tfgk_peer_pull", ctypes.c_void_p(buf.ptrs[src_rank]), ctypes.c_void_p(dst.data_ptr()), nbytes,
                                 ctas, ctypes.c_void_p(stream.cuda_stream)))
    res["pull_ctas_%d" % ctas] = {"ms": ms, "GBps": nbytes / ms / 1e6}
assert int(dst[12345]) == src_rank + 1
peer_view = torch.as_tensor(peer._Raw(buf.ptrs[src_rank], nbytes, buf), device=dev)
ms = timed(lambda: dst.copy_(peer_view, non_blocking=True))
res["copy_engine"] = {"ms": ms, "GBps": nbytes / ms / 1e6}
if world > 2:      # every rank pulls from all the others, one after the other (the all-gather pattern)
    def allgather():
        for k in range(1, world):
            r = (rank + k) % world
            _ffi.call("tfgk_peer_pull", ctypes.c_void_p(buf.ptrs[r]), ctypes.c_void_p(dst.data_ptr()), nbytes, 4 * sms,
                      ctypes.c_void_p(stream.cuda_stream))
    ms = timed(allgather, reps=2)
    res["pull_all_peers_ctas_%d" % (4 * sms)] = {"ms": ms, "GBps": (world - 1) * nbytes / ms / 1e6}
if rank == 0:
    print(json.dumps(res, indent=1))
dist.barrier()
buf.close()
dist.destroy_process_group()
