#!/usr/bin/env python
"""Layer-wise writes of all-layer KV pages under a toy prefill, Llama-3-8B in vLLM's layout.

32 layers, 8 KV heads of 128, one [2, pages, block_size, 8, 128] bf16 tensor per layer, 2048
pages, pool in the same GPU's HBM.  A forward pass runs one toy compute step per layer (bf16
matmuls sized by --layer-ms, then a copy that writes the layer's pages).  Four arms store the
same pages, each in bf16 and in fp8:

  compute     the forward pass alone
  per_layer   one key per page and layer (rdma_write_cache[_fp8]) after each layer, 64 calls
  oneshot     one key per page, one rdma_write_cache_gather[_fp8] call after the last layer
  layerwise   one key per page, GatherWriter.write of each layer's K and V after that layer

The window runs from the forward's start to the end of sync(), ended by a device synchronise;
allocation is outside it.  Per arm: the median window over --reps rounds (the arms
interleaved), its overhead over compute only, and the client's host time per phase
(ns_build + ns_launch), with every round's window and staging drains.  The garbage of each
arm's setup is collected before its window.  Every round's pages are verified: bf16
bit-exact against the source, fp8 layer-wise and per-layer pages bit-identical to the
one-shot fp8 arm's.  Prints the card's name, power limit and SM clock from the same run,
then one JSON line."""
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
from gather_fp8 import card, host_ns, parts_of  # noqa: E402

LAYERS, HEADS, DIM = 32, 8, 128
ARMS = ("compute", "oneshot", "per_layer", "layerwise")  # oneshot's fp8 pages are the reference


class ToyLayer:
    """bf16 matmuls of about `ms` milliseconds, then the layer's pages are written."""

    def __init__(self, dev, ms: float):
        self.a = torch.randn(4096, 4096, device=dev).to(torch.bfloat16)
        self.b = torch.randn(4096, 4096, device=dev).to(torch.bfloat16)
        self.out = torch.empty_like(self.a)
        for _ in range(3):
            torch.mm(self.a, self.b, out=self.out)
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for _ in range(20):
            torch.mm(self.a, self.b, out=self.out)
        e1.record()
        torch.cuda.synchronize()
        self.reps = max(1, round(ms / (e0.elapsed_time(e1) / 20)))

    def __call__(self, kv: torch.Tensor, ref: torch.Tensor):
        for _ in range(self.reps):
            torch.mm(self.a, self.b, out=self.out)
        kv.copy_(ref)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--pages", type=int, default=2048)
    ap.add_argument("--block-sizes", type=int, nargs="+", default=[16, 32])
    ap.add_argument("--layer-ms", type=float, default=1.0)
    ap.add_argument("--reps", type=int, default=7)
    ap.add_argument("--pool-gb", type=int, default=20)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("layerwise_gather.py needs a CUDA device")
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
    toy = ToyLayer(dev, a.layer_ms)
    try:
        conn = ist.InfinityConnection(ist.ClientConfig(
            host_addr="127.0.0.1", service_port=port, connection_type=ist.TYPE_RDMA,
            device_lookup=True, log_level="warning"))
        conn.connect()
        n = a.pages
        for bsz in a.block_sizes:
            page = bsz * HEADS * DIM  # elements of one layer's K (or V) page
            g = torch.Generator(device=dev).manual_seed(bsz)
            ref = [(torch.randn(2, n, bsz, HEADS, DIM, generator=g, device=dev) * 2)
                   .to(torch.bfloat16) for _ in range(LAYERS)]
            kv = [torch.zeros_like(t) for t in ref]
            dst = [torch.zeros_like(t) for t in ref]
            for t in kv + dst:
                conn.register_mr(t)
            offs = np.arange(n, dtype=np.int64) * page
            for fp8 in (False, True):
                dt = "fp8" if fp8 else "bf16"
                gblock = (conn.fp8_gather_block_bytes(2 * LAYERS, page) if fp8
                          else 2 * LAYERS * page * 2)
                lblock = conn.fp8_page_bytes(page) if fp8 else page * 2
                times = {arm: {"ms": [], "host": [], "drains": []} for arm in ARMS}
                oneshot_pages = [torch.empty_like(t) for t in ref] if fp8 else None
                for rep in range(a.reps + 1):  # round 0 warms every arm up
                    for arm in ARMS:
                        for t in kv:
                            t.zero_()
                        tag = f"{arm}-{dt}-{bsz}-{rep}"
                        keys = [f"{tag}-{i}" for i in range(n)]
                        after_layer, after_all = None, None
                        if arm == "per_layer":
                            lkeys = [[[f"{tag}-{l}-{k}-{i}" for i in range(n)] for k in (0, 1)]
                                     for l in range(LAYERS)]
                            lblocks = [[conn.allocate_rdma(lkeys[l][k], lblock) for k in (0, 1)]
                                       for l in range(LAYERS)]
                            wl = conn.rdma_write_cache_fp8 if fp8 else conn.rdma_write_cache

                            def after_layer(layer):
                                for k in (0, 1):
                                    wl(kv[layer], offs + k * n * page, page, lblocks[layer][k])
                        elif arm == "oneshot":
                            blocks = conn.allocate_rdma(keys, gblock)
                            wg = (conn.rdma_write_cache_gather_fp8 if fp8
                                  else conn.rdma_write_cache_gather)

                            def after_all():
                                wg(parts_of(kv, n, page), offs, page, blocks)
                        elif arm == "layerwise":
                            writer = conn.gather_writer(conn.allocate_rdma(keys, gblock), offs,
                                                        2 * LAYERS, page, fp8=fp8)

                            def after_layer(layer):
                                writer.write(parts_of([kv[layer]], n, page), 2 * layer)
                        # the arms' setup leaves hundreds of thousands of Python objects (keys,
                        # block arrays); collect them here, not inside some later window
                        gc.collect()
                        torch.cuda.synchronize()
                        before = conn.stats()
                        t0 = time.perf_counter()
                        for layer in range(LAYERS):
                            toy(kv[layer], ref[layer])
                            if after_layer:
                                after_layer(layer)
                        if after_all:
                            after_all()
                        conn.sync()
                        torch.cuda.synchronize()
                        dt_s = time.perf_counter() - t0
                        host = host_ns(conn, before)
                        drains = conn.stats()["drains"] - before["drains"]
                        # verify the round's pages
                        if arm != "compute":
                            for t in dst:
                                t.zero_()
                            if arm == "per_layer":
                                rl = conn.read_cache_fp8 if fp8 else conn.read_cache
                                for layer in range(LAYERS):
                                    for k in (0, 1):
                                        rl(dst[layer], list(zip(lkeys[layer][k],
                                                                (offs + k * n * page).tolist())),
                                           page)
                            else:
                                rs = conn.read_cache_scatter_fp8 if fp8 else conn.read_cache_scatter
                                rs(parts_of(dst, n, page), (keys, offs), page)
                            conn.sync()
                            if not fp8:
                                ok = all(torch.equal(s, d) for s, d in zip(ref, dst))
                            elif arm == "oneshot":
                                for t, d in zip(oneshot_pages, dst):
                                    t.copy_(d)
                                ok = True
                            else:  # the same quantiser: bit-identical to the one-shot arm
                                ok = all(torch.equal(t, d) for t, d in zip(oneshot_pages, dst))
                            if not ok:
                                raise SystemExit(f"{arm} {dt} block_size {bsz} round {rep}: "
                                                 "pages differ")
                            srv.purge()
                            conn.sync()
                        if rep:
                            times[arm]["ms"].append(dt_s * 1e3)
                            times[arm]["host"].append(host)
                            times[arm]["drains"].append(drains)
                base = statistics.median(times["compute"]["ms"])
                for arm in ARMS:
                    med = statistics.median(times[arm]["ms"])
                    host_ms = statistics.median(times[arm]["host"]) / 1e6
                    row = {
                        "block_size": bsz, "dtype": dt, "arm": arm, "pages": n,
                        "layer_ms": a.layer_ms, "matmuls_per_layer": toy.reps,
                        "window_ms": round(med, 3),
                        "window_ms_all": [round(x, 3) for x in times[arm]["ms"]],
                        "window_ms_max": round(max(times[arm]["ms"]), 3),
                        "staging_drains": times[arm]["drains"],
                        "host_ms_all": [round(x / 1e6, 3) for x in times[arm]["host"]],
                        "overhead_ms": round(med - base, 3),
                        "overhead_pct": round(100 * (med - base) / base, 2),
                        "host_ms_per_phase": round(host_ms, 3),
                        "host_ms_per_layer_call": (round(host_ms / LAYERS, 4)
                                                   if arm == "layerwise" else None),
                        "verified": arm != "compute",
                    }
                    results.append(row)
                    print(json.dumps(row), flush=True)
            del ref, kv, dst
            torch.cuda.empty_cache()
        conn.close()
    finally:
        srv.stop()
    print(json.dumps({"bench": "layerwise_gather", "card": card(0), "card_at_start": info,
                      "results": results}))


if __name__ == "__main__":
    main()
