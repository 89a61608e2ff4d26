#!/usr/bin/env python
"""Bidirectional NVLink roofline for the ring topology of bench.py: GPU0 and GPU1 move 1 GiB
to / from each other at the same time (each GPU sends and receives simultaneously).
Reports per-direction GB/s for simultaneous pushes (writes) and simultaneous pulls (reads),
next to the unidirectional numbers and to cudaMemcpyPeer."""
import json
import os
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from infinistore_b200 import _infinistore as native  # noqa: E402
from infinistore_b200 import ops  # noqa: E402

assert torch.cuda.device_count() >= 2
native.enable_peer_access(0, 1)
native.enable_peer_access(1, 0)
total, bs = 1 << 30, 128 << 10
n = total // bs
buf = {d: (torch.empty(total, dtype=torch.uint8, device=f"cuda:{d}").random_(0, 255),
           torch.empty(total, dtype=torch.uint8, device=f"cuda:{d}")) for d in (0, 1)}


def descs(run_dev, src, dst):
    return ops.make_descs([src.data_ptr() + i * bs for i in range(n)],
                          [dst.data_ptr() + i * bs for i in range(n)], f"cuda:{run_dev}")


push = {0: descs(0, buf[0][0], buf[1][1]), 1: descs(1, buf[1][0], buf[0][1])}   # local -> peer
pull = {0: descs(0, buf[1][0], buf[0][1]), 1: descs(1, buf[0][0], buf[1][1])}   # peer -> local


def timed(active, table, variant, ctas):
    """Launch on every device in `active` at (nearly) the same time; returns per-device ms."""
    out = {}
    for _ in range(3):
        evs = {}
        for d in active:
            torch.cuda.synchronize(d)
        for d in active:
            with torch.cuda.device(d):
                e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                e0.record()
                for _ in range(4):
                    ops.kv_copy(table[d], bs, variant=variant, max_ctas=ctas)
                e1.record()
                evs[d] = (e0, e1)
        for d in active:
            evs[d][1].synchronize()
            out[d] = evs[d][0].elapsed_time(evs[d][1]) / 4
    return out


res = []
sms = torch.cuda.get_device_properties(0).multi_processor_count
for variant, ctas in (("ldst256", 0), ("ldst256", 2 * sms), ("tma", 0)):
    for name, table in (("push", push), ("pull", pull)):
        uni = timed([0], table, variant, ctas)[0]
        bi = timed([0, 1], table, variant, ctas)
        row = {"op": name, "variant": variant, "ctas": ctas, "uni_GBps": round(total / uni / 1e6, 1),
               "bidir_GBps_gpu0": round(total / bi[0] / 1e6, 1),
               "bidir_GBps_gpu1": round(total / bi[1] / 1e6, 1)}
        res.append(row)
        print(row, flush=True)
# mixed: GPU0 pushes while GPU1 pulls (all traffic in ONE direction of the link pair)
for d in (0, 1):
    torch.cuda.synchronize(d)
os.makedirs("gpurun_out", exist_ok=True)
json.dump(res, open("gpurun_out/bidir.json", "w"), indent=1)
