#!/usr/bin/env python
"""Position-free KV segments (write_segment / read_segment) against the all-layer page calls of
the same bytes, in two geometries:

  llama    Llama-3-70B: 80 layers of 16-token pages of 8 KV heads x 128, neox pairs over the
           full head (only the K parts turn); 5 MiB per all-layer page
  mla      DeepSeek-V3 MLA: 61 layers of 64-token pages of 512 latent + 64 RoPE elements,
           interleaved pairs over the trailing 64; 4.3 MiB per all-layer page

A pool in the GPU's own HBM, device lookup, a streams=0 connection, about --gib GiB of bf16
per phase.  Arms:

  segment write   write_segment at position p0 (the keys' RoPE turned by -p0 in the write)
  segment read    read_segment at position p1 (turned by +p1 in the read)
  page write      write_pages of the same pages (plain gathered write)
  page read       read_pages of them (plain scattered read)
  memcpy          cudaMemcpyAsync device-to-device of the stored bytes

Each phase is timed on the device, events around the call and the sync() that follows it,
under fresh keys each round, with --warmup rounds first; the store is purged after every round.
Reported: the median over --reps rounds and GB/s.  The last round's segment read is checked on
two sampled pages against the numpy model of tests/rope_model.py.  Prints the card's name,
power limit and SM clock from the same run, then one JSON line."""
from __future__ import annotations

import argparse
import json
import os
import statistics
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "bench"))
sys.path.insert(0, os.path.join(ROOT, "tests"))
import infinistore_b200 as ist  # noqa: E402
from infinistore_b200 import RotaryConfig, rope_inv_freq  # noqa: E402
from infinistore_b200 import _infinistore as native  # noqa: E402
from infinistore_b200.models import MLA_LAYOUTS, MLAKVCache, PagedKVCache, get_layout  # noqa: E402
from gather_fp8 import card  # noqa: E402
from mla_pages import device_ms, memcpy_ms  # noqa: E402
import rope_model as rm  # noqa: E402


def bits(t):
    return t.contiguous().view(torch.int16).cpu().numpy().view(np.uint16)


def geometry(kind):
    """(layout, rotary config, cache class) of a geometry."""
    if kind == "llama":
        return (get_layout("llama-3-70b", page_tokens=16),
                RotaryConfig(128, rope_inv_freq(128, 500000.0), interleaved=False), PagedKVCache)
    return (MLA_LAYOUTS["deepseek-v3"], RotaryConfig(64, rope_inv_freq(64, 10000.0), True),
            MLAKVCache)


def page_parts(c, p):
    d = c.data
    if c._per_layer == 2:
        return [bits(d[layer, kv, p]) for layer in range(c.layout.layers) for kv in (0, 1)]
    return [bits(d[layer, p]) for layer in range(c.layout.layers)]


def check(kind, src, dst, pages, rpages, p0, p1):
    head, off, even = src._segment_geometry()
    for j in (0, len(pages) - 1):
        stored = rm.shift_parts(page_parts(src, pages[j]), src.rotary, -p0, head, off, even)
        want = rm.shift_parts(stored, src.rotary, p1, head, off, even)
        for x, y in zip(page_parts(dst, rpages[j]), want):
            if not rm.same_bits(x, y):
                raise SystemExit(f"{kind}: segment read differs from the model")


def run(kind, a, srv, port, dev, out):
    lay_pages, rot, cls = geometry(kind)
    per = 2 if kind == "llama" else 1
    block = per * lay_pages.layers * lay_pages.page_bytes
    pages = max(1, int(a.gib * 2**30) // block)
    src, dst, dstp = (cls(lay_pages, pages, dev, rotary=rot) for _ in range(3))
    g = torch.Generator(device=dev).manual_seed(0)
    src.data.copy_(torch.randn(src.data.shape, generator=g, device=dev))
    nbytes = pages * block
    conn = ist.InfinityConnection(ist.ClientConfig(
        host_addr="127.0.0.1", service_port=port, connection_type=ist.TYPE_RDMA,
        device_lookup=True, streams=0, log_level="warning"))
    conn.connect()
    B = lay_pages.page_tokens
    p0, p1 = 7 * B, 4096 * B
    plist = list(range(pages))
    rpages = np.random.default_rng(1).permutation(pages).tolist()
    arms = {k: [] for k in ("segment write", "segment read", "page write", "page read")}
    mc = memcpy_ms(nbytes, a.reps, dev)
    for rep in range(a.warmup + a.reps):
        hs = [f"{kind}-seg-{rep}-{i}" for i in range(pages)]
        hp = [f"{kind}-page-{rep}-{i}" for i in range(pages)]

        def timed(fn):
            return device_ms(lambda: (fn(), conn.sync()))

        t = {"segment write": timed(lambda: src.write_segment(conn, plist, hs, p0)),
             "segment read": timed(lambda: dst.read_segment(conn, rpages, hs, p1)),
             "page write": timed(lambda: src.write_pages(conn, plist, hp)),
             "page read": timed(lambda: dstp.read_pages(conn, rpages, hp))}
        if rep >= a.warmup:
            for k, v in t.items():
                arms[k].append(v)
        if rep == a.warmup + a.reps - 1:
            check(kind, src, dst, plist, rpages, p0, p1)
        srv.purge()
    conn.close()
    res = {"pages": pages, "page_tokens": B, "layers": lay_pages.layers, "bytes": nbytes,
           "memcpy_ms": round(mc, 3), "arms": {}}
    print(f"{kind}: {pages} pages, {nbytes / 2**30:.2f} GiB per phase; cudaMemcpyAsync D2D "
          f"{mc:8.3f} ms {nbytes / (mc * 1e-3) / 1e9:7.1f} GB/s", flush=True)
    for k, v in arms.items():
        ms = statistics.median(v)
        res["arms"][k] = {"ms": round(ms, 3), "GBps": round(nbytes / (ms * 1e-3) / 1e9, 1),
                          "vs_memcpy": round(mc / ms, 3)}
        print(f"  {k:14s} {ms:8.3f} ms {nbytes / (ms * 1e-3) / 1e9:7.1f} GB/s "
              f"({mc / ms:.2f} of memcpy)", flush=True)
    out["geometries"][kind] = res
    del src, dst, dstp
    torch.cuda.empty_cache()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--gib", type=float, default=2.0, help="bf16 bytes per phase")
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--pool-gb", type=int, default=8)
    ap.add_argument("--geometries", default="llama,mla")
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("rope_segments.py needs a CUDA device")
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
    out = {"card": info, "reps": a.reps, "geometries": {}}
    try:
        for kind in a.geometries.split(","):
            run(kind, a, srv, port, dev, out)
        print("verified: the last round's segment reads against the numpy model, on two pages")
    finally:
        srv.stop()
    print(json.dumps(out))


if __name__ == "__main__":
    main()
