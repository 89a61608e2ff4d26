#!/usr/bin/env python
"""Where a flagship round loses time against the copy engine, one layer at a time.

The flagship shapes (bench.py --gpus 1): 4 GiB of 128 KB bf16 pages per phase, 32 calls of
1024 pages, pool in the same GPU's HBM.  Every variant moves the same bytes; variants are
interleaved, repeated --reps times and timed with CUDA events; each row gives the median and
the spread.  Subtracting one row from the next gives the cost of one layer:

  ce                cudaMemcpyAsync device to device (the copy engine)
  mover_one_launch  the TMA page mover (kernels.kv_copy), all pages in one launch, no commit,
                    no index: the mover's steady-state rate
  mover_32x4        the same bytes as 32 launches round-robin over 4 streams: the launch structure
  api_write         one write phase through InfinityConnection (fresh keys, in-band commit) + sync
  api_read          one read phase of those keys (device index resolver) + sync
  api_round         write -> sync -> read -> sync: adds the phase boundaries

`drains` is ClientStats::drains over --step-rounds flagship rounds: staging allocations that had
to block the host until an earlier launch completed.  One JSON line on stdout, with the card's
name and power limit read in the same run."""
from __future__ import annotations

import argparse
import json
import os
import statistics
import subprocess
import sys
import uuid

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import infinistore_b200 as ist  # noqa: E402
from infinistore_b200 import _infinistore as native  # noqa: E402
from infinistore_b200 import ops  # noqa: E402


def card(index: int) -> dict:
    q = "name,power.limit,clocks.max.sm"
    try:
        out = subprocess.run(["nvidia-smi", "-i", str(index), f"--query-gpu={q}",
                              "--format=csv,noheader,nounits"],
                             capture_output=True, text=True, timeout=30).stdout.strip()
        name, power, clock = [x.strip() for x in out.split(",")]
        return {"name": name, "power_limit_W": float(power), "max_sm_clock_MHz": float(clock)}
    except Exception as e:  # noqa: BLE001
        return {"name": torch.cuda.get_device_name(index), "power_limit_W": None,
                "nvidia_smi_error": repr(e)[:120]}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--size-mb", type=int, default=4096)
    ap.add_argument("--block-kb", type=int, default=128)
    ap.add_argument("--layers", type=int, default=32)
    ap.add_argument("--streams", type=int, default=4)
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--step-rounds", type=int, default=24)
    ap.add_argument("--port", type=int, default=24300)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("mover_gap.py needs a CUDA device")

    dev = torch.device("cuda", 0)
    torch.cuda.set_device(dev)
    bs = a.block_kb << 10
    size = a.size_mb << 20
    n = size // bs
    per = n // a.layers
    elems = bs // 2
    stream = torch.cuda.Stream(device=dev)

    scfg = native.ServerConfig()
    scfg.service_port = a.port
    scfg.host = "127.0.0.1"
    scfg.pool_backend = "hbm"
    scfg.pool_devices = [0]
    scfg.minimal_allocate_size = max(16, min(a.block_kb, 64))
    scfg.prealloc_bytes = 2 * size + (64 << 20)  # one write phase + one round, then a purge
    scfg.log_level = "warning"
    server = native.Server(scfg)
    server.start()
    conn = ist.InfinityConnection(ist.ClientConfig(
        host_addr="127.0.0.1", service_port=a.port, connection_type=ist.TYPE_RDMA,
        log_level="warning", device=0, device_lookup=True, copy_variant="auto",
        streams=a.streams))
    conn.connect()

    src = torch.randn(n * elems, device=dev, dtype=torch.float32).to(torch.bfloat16)
    dst = torch.zeros_like(src)
    conn.register_mr(src)
    conn.register_mr(dst)
    offsets = [i * elems for i in range(n)]
    descs = ops.make_descs([src.data_ptr() + i * bs for i in range(n)],
                           [dst.data_ptr() + i * bs for i in range(n)], dev)
    side = [torch.cuda.Stream(device=dev) for _ in range(a.streams)]

    def mover(d, s):
        native.kernels.kv_copy(d.data_ptr(), d.shape[0], bs, ops.VARIANTS["tma"], 0, s.cuda_stream,
                               0, 0, 0, 0, 0, 0, 0, True, 0, 0, 0, [])

    def fresh():
        tag = uuid.uuid4().hex
        keys = [f"{tag}-{i:07d}" for i in range(n)]
        return conn.allocate_rdma(keys, bs), list(zip(keys, offsets))

    def write(remote):
        for l in range(a.layers):
            conn.rdma_write_cache(src, offsets[l * per:(l + 1) * per], elems,
                                  remote[l * per:(l + 1) * per])
        conn.sync()

    def read(blocks):
        for l in range(a.layers):
            conn.read_cache(dst, blocks[l * per:(l + 1) * per], elems)
        conn.sync()

    def timed(fn):
        """Device time (ms) of fn() on `stream`, as bench.py times a round."""
        torch.cuda.synchronize()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        with torch.cuda.stream(stream):
            e0.record(stream)
            fn()
            e1.record(stream)
        e1.synchronize()
        return e0.elapsed_time(e1)

    def one_launch():
        mover(descs, stream)

    def launches_32x4():
        start = torch.cuda.Event()
        start.record(stream)
        for l in range(a.layers):
            s = side[l % len(side)]
            if l < len(side):
                s.wait_event(start)
            mover(descs[l * per:(l + 1) * per], s)
        for s in side:
            stream.wait_stream(s)

    times = {k: [] for k in ("ce", "mover_one_launch", "mover_32x4", "api_write", "api_read",
                             "api_round")}
    moved = {"api_round": 2 * size}
    for rep in range(a.reps + 1):  # repetition 0 warms every shape up and is not kept
        server.purge()
        w_remote, w_blocks = fresh()
        r_remote, r_blocks = fresh()
        row = {"ce": timed(lambda: dst.copy_(src, non_blocking=True)),
               "mover_one_launch": timed(one_launch),
               "mover_32x4": timed(launches_32x4),
               "api_write": timed(lambda: write(w_remote)),
               "api_read": timed(lambda: read(w_blocks)),
               "api_round": timed(lambda: (write(r_remote), read(r_blocks)))}
        assert torch.equal(src, dst), "read-back mismatch"
        if rep:
            for k, v in row.items():
                times[k].append(v)

    # a flagship step: --step-rounds rounds with fresh keys, the pool purged every two rounds
    drains0 = conn.stats().get("drains")
    for r in range(a.step_rounds):
        if r % 2 == 0:
            server.purge()
            prepared = [fresh(), fresh()]
        remote, blocks = prepared[r % 2]
        with torch.cuda.stream(stream):
            write(remote)
            read(blocks)
    torch.cuda.synchronize()
    drains = None if drains0 is None else conn.stats()["drains"] - drains0
    ok = bool(torch.equal(src, dst))
    conn.close()
    server.stop()

    rows = {}
    for k, ts in times.items():
        b = moved.get(k, size)
        rows[k] = {"ms_median": round(statistics.median(ts), 3),
                   "ms_min": round(min(ts), 3), "ms_max": round(max(ts), 3),
                   "GBps_median": round(b / statistics.median(ts) / 1e6, 1),
                   "GBps_min": round(b / max(ts) / 1e6, 1), "GBps_max": round(b / min(ts) / 1e6, 1),
                   "payload_bytes": b}
    print(json.dumps({"card": card(0), "reps": a.reps, "pages": n, "page_bytes": bs,
                      "calls_per_phase": a.layers, "streams": a.streams, "rows": rows,
                      "drains": drains, "drains_rounds": a.step_rounds, "verified": ok}))


if __name__ == "__main__":
    main()
