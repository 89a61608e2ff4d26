#!/usr/bin/env python
"""Layer-wise reads of all-layer KV pages under a toy decode step, Llama-3-8B in vLLM's layout.

The decode-side twin of layerwise_gather.py.  32 layers, 8 KV heads of 128, one
[2, pages, block_size, 8, 128] tensor per layer, pool in the same GPU's HBM, device lookup.
The pages are written once per configuration with the gathered write (one key per page).
A decode step runs one toy attention step per layer on the consumer (current) stream: bf16
matmuls sized by --layer-ms, then a read of a slice of the layer's pages.  Five arms fetch the
same pages, each in bf16 and in fp8:

  compute           the decode step alone (the pages are already there)
  oneshot           read_cache_scatter[_fp8] of every layer, sync(), then the step
  per_layer_sync    one read of layer l + 1 ahead, with a host sync() before layer l (the
                    pattern of example/demo_decode.py)
  per_layer_events  a streams=0 connection: one read per layer on a side stream, each followed
                    by an event the consumer stream waits on (no host sync per layer)
  layered           one read_cache_scatter_layered, ScatterRead.wait(l) before layer l

The window runs from the first read to the end of the step and sync(), ended by a device
synchronise.  Per arm: the median window over --reps rounds (the arms interleaved) with its
minimum and maximum, the overhead over compute, the client's host time per step
(ns_build + ns_launch) and the Python time spent in the read and wait calls, the kernel
launches per step (counted), and the key probes per step (derived, not counted: the number
of read calls times the pages, since each call resolves each of its keys once).  Every
round's pages are verified: bf16 bit-exact against the source, fp8 bit-identical to the
one-shot fp8 read.  Prints the card's name, power limit and SM clock from the same run, then
one JSON line.  No arm is expected to win: the numbers
are reported as measured."""
from __future__ import annotations

import argparse
import gc
import json
import os
import statistics
import sys
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "bench"))
import infinistore_b200 as ist  # noqa: E402
from infinistore_b200 import _infinistore as native  # noqa: E402
from layerwise_gather import card, host_ns, parts_of  # noqa: E402

LAYERS, HEADS, DIM = 32, 8, 128
ARMS = ("compute", "oneshot", "per_layer_sync", "per_layer_events", "layered")


class ToyAttention:
    """bf16 matmuls of about `ms` milliseconds, then a read of a slice of the layer's pages."""

    def __init__(self, dev, ms: float):
        self.a = torch.randn(4096, 4096, device=dev).to(torch.bfloat16)
        self.b = torch.randn(4096, 4096, device=dev).to(torch.bfloat16)
        self.out = torch.empty_like(self.a)
        self.sink = torch.empty(1 << 16, dtype=torch.bfloat16, device=dev)
        for _ in range(3):
            torch.mm(self.a, self.b, out=self.out)
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for _ in range(20):
            torch.mm(self.a, self.b, out=self.out)
        e1.record()
        torch.cuda.synchronize()
        self.reps = max(1, round(ms / (e0.elapsed_time(e1) / 20)))

    def __call__(self, kv: torch.Tensor):
        for _ in range(self.reps):
            torch.mm(self.a, self.b, out=self.out)
        self.sink.copy_(kv.view(-1)[-self.sink.numel():])


def connect(port, streams=None):
    cfg = dict(host_addr="127.0.0.1", service_port=port, connection_type=ist.TYPE_RDMA,
               device_lookup=True, log_level="warning")
    if streams is not None:
        cfg["streams"] = streams
    conn = ist.InfinityConnection(ist.ClientConfig(**cfg))
    conn.connect()
    return conn


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--pages", type=int, nargs="+", default=[256, 2048])
    ap.add_argument("--block-sizes", type=int, nargs="+", default=[16, 32])
    ap.add_argument("--layer-ms", type=float, default=0.5)
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--pool-gb", type=int, default=20)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("layerwise_read.py needs a CUDA device")
    dev = torch.device("cuda", 0)
    torch.cuda.set_device(dev)
    info = card(0)
    print(f"card: {info}", flush=True)

    scfg = native.ServerConfig()
    scfg.service_port = 0
    scfg.host = "127.0.0.1"
    scfg.pool_backend = "hbm"
    scfg.pool_devices = [0]
    scfg.minimal_allocate_size = 16
    scfg.prealloc_bytes = a.pool_gb << 30
    srv = native.Server(scfg)
    port = srv.start()
    results = []
    toy = ToyAttention(dev, a.layer_ms)
    try:
        conn = connect(port)
        conn0 = connect(port, streams=0)  # per_layer_events: launches on the caller's stream
        for n in a.pages:
            for bsz in a.block_sizes:
                page = bsz * HEADS * DIM  # elements of one layer's K (or V) page
                g = torch.Generator(device=dev).manual_seed(bsz + n)
                ref = [(torch.randn(2, n, bsz, HEADS, DIM, generator=g, device=dev) * 2)
                       .to(torch.bfloat16) for _ in range(LAYERS)]
                dst = [torch.zeros_like(t) for t in ref]
                for t in ref + dst:
                    conn.register_mr(t)
                    conn0.register_mr(t)
                offs = np.arange(n, dtype=np.int64) * page
                for fp8 in (False, True):
                    dt = "fp8" if fp8 else "bf16"
                    keys = [f"{dt}-{n}-{bsz}-{i}" for i in range(n)]
                    gblock = (conn.fp8_gather_block_bytes(2 * LAYERS, page) if fp8
                              else 2 * LAYERS * page * 2)
                    write = (conn.rdma_write_cache_gather_fp8 if fp8
                             else conn.rdma_write_cache_gather)
                    write(parts_of(ref, n, page), offs, page, conn.allocate_rdma(keys, gblock))
                    conn.sync()
                    rs = conn.read_cache_scatter_fp8 if fp8 else conn.read_cache_scatter
                    rs0 = conn0.read_cache_scatter_fp8 if fp8 else conn0.read_cache_scatter
                    expect = ref
                    if fp8:  # the one-shot fp8 read is the reference of every fp8 arm
                        expect = [torch.zeros_like(t) for t in ref]
                        rs(parts_of(expect, n, page), (keys, offs), page)
                        conn.sync()
                    times = {arm: {"ms": [], "host": [], "api": [], "launches": []}
                             for arm in ARMS}
                    reads = {"compute": 0, "oneshot": 1, "per_layer_sync": LAYERS,
                             "per_layer_events": LAYERS, "layered": 1}
                    side = torch.cuda.Stream()
                    for rep in range(a.reps + 1):  # round 0 warms every arm up
                        for arm in ARMS:
                            for t in dst:
                                t.zero_()
                            c = conn0 if arm == "per_layer_events" else conn
                            gc.collect()
                            torch.cuda.synchronize()
                            before = c.stats()
                            api = 0.0
                            t0 = time.perf_counter()
                            if arm == "compute":
                                for layer in range(LAYERS):
                                    toy(ref[layer])
                            elif arm == "oneshot":
                                rs(parts_of(dst, n, page), (keys, offs), page)
                                api += time.perf_counter() - t0
                                conn.sync()
                                for layer in range(LAYERS):
                                    toy(dst[layer])
                            elif arm == "per_layer_sync":
                                t1 = time.perf_counter()
                                rs(parts_of(dst[:1], n, page), (keys, offs), page, first_part=0)
                                api += time.perf_counter() - t1
                                for layer in range(LAYERS):
                                    conn.sync()
                                    if layer + 1 < LAYERS:
                                        t1 = time.perf_counter()
                                        rs(parts_of(dst[layer + 1:layer + 2], n, page),
                                           (keys, offs), page, first_part=2 * (layer + 1))
                                        api += time.perf_counter() - t1
                                    toy(dst[layer])
                            elif arm == "per_layer_events":
                                cur = torch.cuda.current_stream()
                                side.wait_stream(cur)
                                evs = []
                                t1 = time.perf_counter()
                                for layer in range(LAYERS):
                                    rs0(parts_of(dst[layer:layer + 1], n, page), (keys, offs),
                                        page, first_part=2 * layer, stream=side)
                                    ev = torch.cuda.Event()
                                    ev.record(side)
                                    evs.append(ev)
                                api += time.perf_counter() - t1
                                for layer in range(LAYERS):
                                    cur.wait_event(evs[layer])
                                    toy(dst[layer])
                            else:  # layered
                                t1 = time.perf_counter()
                                r = conn.read_cache_scatter_layered(
                                    parts_of(dst, n, page), (keys, offs), page, fp8=fp8)
                                api += time.perf_counter() - t1
                                for layer in range(LAYERS):
                                    t1 = time.perf_counter()
                                    r.wait(layer)
                                    api += time.perf_counter() - t1
                                    toy(dst[layer])
                            c.sync()
                            torch.cuda.synchronize()
                            dt_s = time.perf_counter() - t0
                            after = c.stats()
                            host = host_ns(c, before)
                            launches = after["kernel_launches"] - before["kernel_launches"]
                            if arm != "compute":
                                ok = all(torch.equal(e, d) for e, d in zip(expect, dst))
                                if not ok:
                                    raise SystemExit(f"{arm} {dt} pages {n} block_size {bsz} "
                                                     f"round {rep}: pages differ")
                            if rep:
                                times[arm]["ms"].append(dt_s * 1e3)
                                times[arm]["host"].append(host)
                                times[arm]["api"].append(api * 1e3)
                                times[arm]["launches"].append(launches)
                    base = statistics.median(times["compute"]["ms"])
                    for arm in ARMS:
                        ms = times[arm]["ms"]
                        med = statistics.median(ms)
                        row = {
                            "pages": n, "block_size": bsz, "dtype": dt, "arm": arm,
                            "layer_ms": a.layer_ms, "matmuls_per_layer": toy.reps,
                            "window_ms": round(med, 3), "window_ms_min": round(min(ms), 3),
                            "window_ms_max": round(max(ms), 3),
                            "window_ms_all": [round(x, 3) for x in ms],
                            "overhead_ms": round(med - base, 3),
                            "overhead_pct": round(100 * (med - base) / base, 2),
                            "host_ms_per_step": round(statistics.median(times[arm]["host"]) / 1e6,
                                                      3),
                            "api_ms_per_step": round(statistics.median(times[arm]["api"]), 3),
                            "launches_per_step": statistics.median(times[arm]["launches"]),
                            "key_probes_per_step_derived": reads[arm] * n,
                            "verified": arm != "compute",
                        }
                        results.append(row)
                        print(json.dumps(row), flush=True)
                    srv.purge()
                    conn.sync()
                del ref, dst
                torch.cuda.empty_cache()
        conn0.close()
        conn.close()
    finally:
        srv.stop()
    print(json.dumps({"bench": "layerwise_read", "card": card(0), "card_at_start": info,
                      "results": results}))


if __name__ == "__main__":
    main()
