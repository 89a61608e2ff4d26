#!/usr/bin/env python
"""Gathered fp8 KV blocks against gathered bf16 and per-layer fp8, Llama-3-8B in vLLM's layout.

32 layers, 8 KV heads of 128, one [2, pages, block_size, 8, 128] bf16 tensor per layer, 2048
pages, pool in the same GPU's HBM, reads through the device index.  Three arms move the same
pages:

  gather_bf16     rdma_write_cache_gather / read_cache_scatter: one call, 2048 keys per phase
  gather_fp8      rdma_write_cache_gather_fp8 / read_cache_scatter_fp8: the same, e4m3 in the pool
  per_layer_fp8   rdma_write_cache_fp8 / read_cache_fp8: 64 calls, 131072 keys per phase

A phase is the calls plus sync(), timed on the host clock after a device synchronise, so it
ends in one.  Allocation is outside the window.  For each arm and block size: the median
phase time over --reps rounds (the arms interleaved) in GB/s of bf16-equivalent bytes and
of pool bytes, pool bytes per page from the server's used_bytes, and the client's host time
per phase (ns_build + ns_launch).  Every round's pages are verified: bf16 bit-exact against
the source, the two fp8 arms bit-identical to each other and within one bf16 ulp of the
largest value of the fp32 reference.  Prints the card's name, power limit and SM clock from
the same run, then one JSON line."""
from __future__ import annotations

import argparse
import json
import os
import statistics
import subprocess
import sys
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import infinistore_b200 as ist  # noqa: E402
from infinistore_b200 import _infinistore as native  # noqa: E402
from infinistore_b200 import ops  # noqa: E402

LAYERS, HEADS, DIM = 32, 8, 128


def card(index: int) -> dict:
    q = "name,power.limit,clocks.sm,clocks.max.sm"
    try:
        out = subprocess.run(["nvidia-smi", "-i", str(index), f"--query-gpu={q}",
                              "--format=csv,noheader,nounits"],
                             capture_output=True, text=True, timeout=30).stdout.strip()
        name, power, clock, max_clock = [x.strip() for x in out.split(",")]
        return {"name": name, "power_limit_W": float(power), "sm_clock_MHz": float(clock),
                "max_sm_clock_MHz": float(max_clock)}
    except Exception as e:  # noqa: BLE001
        return {"name": torch.cuda.get_device_name(index), "power_limit_W": None,
                "nvidia_smi_error": repr(e)[:120]}


def parts_of(kv, pages, page):
    return [p for t in kv for p in ((t, 0), (t, pages * page))]


def host_ns(conn, before):
    st = conn.stats()
    return (st["ns_build"] + st["ns_launch"]) - (before["ns_build"] + before["ns_launch"])


def phase(conn, fn):
    """(seconds, host ns) of fn() + sync()."""
    torch.cuda.synchronize()
    before = conn.stats()
    t0 = time.perf_counter()
    fn()
    conn.sync()
    torch.cuda.synchronize()
    return time.perf_counter() - t0, host_ns(conn, before)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--pages", type=int, default=2048)
    ap.add_argument("--block-sizes", type=int, nargs="+", default=[16, 32])
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--pool-gb", type=int, default=12)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("gather_fp8.py needs a CUDA device")
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
    try:
        conn = ist.InfinityConnection(ist.ClientConfig(
            host_addr="127.0.0.1", service_port=port, connection_type=ist.TYPE_RDMA,
            device_lookup=True, log_level="warning"))
        conn.connect()
        n = a.pages
        for bsz in a.block_sizes:
            page = bsz * HEADS * DIM  # elements of one layer's K (or V) page
            g = torch.Generator(device=dev).manual_seed(bsz)
            src = [(torch.randn(2, n, bsz, HEADS, DIM, generator=g, device=dev) * 2)
                   .to(torch.bfloat16) for _ in range(LAYERS)]
            dst = [torch.zeros_like(t) for t in src]
            for t in src + dst:
                conn.register_mr(t)
            offs = np.arange(n, dtype=np.int64) * page
            bf16_bytes = n * 2 * LAYERS * page * 2
            pool_block = {"gather_bf16": 2 * LAYERS * page * 2,
                          "gather_fp8": conn.fp8_gather_block_bytes(2 * LAYERS, page),
                          "per_layer_fp8": 2 * LAYERS * conn.fp8_page_bytes(page)}
            times = {k: {"write": [], "read": [], "host_write": [], "host_read": [],
                         "used": []} for k in pool_block}
            ref8 = [torch.empty_like(t) for t in src]
            for rep in range(a.reps):
                for arm in pool_block:
                    for t in dst:
                        t.zero_()
                    tag = f"{arm}-{bsz}-{rep}"
                    used0 = srv.stats()["used_bytes"]
                    if arm == "per_layer_fp8":
                        lreads, lblocks = [], []
                        for layer in range(LAYERS):
                            for kv in (0, 1):
                                ks = [f"{tag}-{layer}-{kv}-{i}" for i in range(n)]
                                lreads.append(list(zip(ks, (offs + kv * n * page).tolist())))
                                lblocks.append(conn.allocate_rdma(ks, conn.fp8_page_bytes(page)))

                        def write():
                            for j, blocks in enumerate(lblocks):
                                layer, kv = divmod(j, 2)
                                conn.rdma_write_cache_fp8(src[layer], offs + kv * n * page, page,
                                                          blocks)

                        def read():
                            for j, blocks in enumerate(lreads):
                                conn.read_cache_fp8(dst[j // 2], blocks, page)
                    else:
                        fp8 = arm == "gather_fp8"
                        keys = [f"{tag}-{i}" for i in range(n)]
                        blocks = conn.allocate_rdma(keys, pool_block[arm])
                        w = conn.rdma_write_cache_gather_fp8 if fp8 else conn.rdma_write_cache_gather
                        r = conn.read_cache_scatter_fp8 if fp8 else conn.read_cache_scatter

                        def write():
                            w(parts_of(src, n, page), offs, page, blocks)

                        def read():
                            r(parts_of(dst, n, page), (keys, offs), page)
                    tw, hw = phase(conn, write)
                    times[arm]["used"].append(srv.stats()["used_bytes"] - used0)
                    tr, hr = phase(conn, read)
                    times[arm]["write"].append(tw)
                    times[arm]["read"].append(tr)
                    times[arm]["host_write"].append(hw)
                    times[arm]["host_read"].append(hr)
                    # verify every round's pages
                    if arm == "gather_bf16":
                        ok = all(torch.equal(s, d) for s, d in zip(src, dst))
                    elif arm == "gather_fp8":
                        for t, d in zip(ref8, dst):
                            t.copy_(d)
                        ok = True
                        for s, d in zip(src, dst):
                            dq, _, _ = ops.fp8_reference(s)
                            err = (d.float() - dq.to(torch.bfloat16).float()).abs().max().item()
                            ok = ok and err <= float(s.float().abs().max()) * 2 ** -7
                    else:  # per-layer fp8 reads back the gathered fp8 arm's pages bit for bit
                        ok = all(torch.equal(t, d) for t, d in zip(ref8, dst))
                    if not ok:
                        raise SystemExit(f"{arm} block_size {bsz} round {rep}: pages differ")
                    srv.purge()
                    conn.sync()
            for arm, t in times.items():
                wmed, rmed = statistics.median(t["write"]), statistics.median(t["read"])
                pool_bytes = n * pool_block[arm]
                row = {
                    "block_size": bsz, "arm": arm, "pages": n,
                    "write_GBps_bf16": round(bf16_bytes / wmed / 1e9, 1),
                    "read_GBps_bf16": round(bf16_bytes / rmed / 1e9, 1),
                    "write_GBps_pool": round(pool_bytes / wmed / 1e9, 1),
                    "read_GBps_pool": round(pool_bytes / rmed / 1e9, 1),
                    "write_ms": [round(x * 1e3, 2) for x in t["write"]],
                    "read_ms": [round(x * 1e3, 2) for x in t["read"]],
                    "pool_bytes_per_page": int(statistics.median(t["used"]) // n),
                    "host_ms_write": round(statistics.median(t["host_write"]) / 1e6, 2),
                    "host_ms_read": round(statistics.median(t["host_read"]) / 1e6, 2),
                    "verified": True,
                }
                results.append(row)
                print(json.dumps(row), flush=True)
            del src, dst, ref8
            torch.cuda.empty_cache()
        conn.close()
    finally:
        srv.stop()
    print(json.dumps({"bench": "gather_fp8", "card": card(0), "card_at_start": info,
                      "results": results}))


if __name__ == "__main__":
    main()
