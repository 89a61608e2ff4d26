#!/usr/bin/env python
"""e4m3 KV caches (PagedKVCache(kv_scales=)) against the bf16 cache's fp8 pages, in Llama-3-70B
geometry: 80 layers of 16-token pages of 8 KV heads x 128, 5 MiB per all-layer page in bf16,
2.6 MiB stored as fp8 pages.

A pool in the GPU's own HBM, device lookup, a streams=0 connection.  --pages pages (about
2 GiB of bf16 payload per phase by default).  Arms:

  e4m3 write        an e4m3 cache's write_pages(fp8=True): bytes kept, group scales stored
  e4m3 read same    read_pages(fp8=True) into an e4m3 cache at the writer's scales (verbatim)
  e4m3 read other   the same into an e4m3 cache at other scales (every group requantised)
  bf16 fp8 write    the bf16 cache's write_pages(fp8=True) of the same pages (quantising)
  bf16 fp8 read     its read_pages(fp8=True) (dequantising)

Each phase is timed on the device, events around the call and the sync() that follows it,
under fresh keys each round, with --warmup rounds first; the store is purged after every round.
Reported: the median over --reps rounds, GB/s of bf16 payload and of stored bytes, and next to
them cudaMemcpyAsync device-to-device of the stored bytes measured in the same run.  Every read
is checked on two sampled pages against the numpy model of tests/e4m3_cache.py (the e4m3
reads) and the exact e4m3 reference of tests/fp8_exact.py (the bf16 read).  Prints the card's
name, power limit and SM clock from the same run, then one JSON line."""
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
from infinistore_b200 import _infinistore as native  # noqa: E402
from infinistore_b200.models import PagedKVCache, get_layout  # noqa: E402
from gather_fp8 import card  # noqa: E402
from mla_pages import device_ms, memcpy_ms  # noqa: E402
import e4m3_cache as ec  # noqa: E402
import fp8_exact as fx  # noqa: E402

ROW = 128


def u8(t):
    return t.contiguous().view(torch.uint8).cpu().numpy()


def check(label, src_e, src_b, dst_same, dst_other, dst_b, pages, rpages):
    """Two sampled pages of every read against the models."""
    lay = src_e.layout
    for j in (0, len(pages) - 1):
        p, d = pages[j], rpages[j]
        q = u8(src_e.data[:, :, p])  # (layers, 2, elems)
        if not np.array_equal(u8(dst_same.data[:, :, d]), q):
            raise SystemExit(f"{label}: e4m3 read at the same scales is not the written bytes")
        got = u8(dst_other.data[:, :, d])
        for layer in range(lay.layers):
            for kv in (0, 1):
                g = q[layer, kv].reshape(-1, ROW)
                want = ec.requant(g, np.full(len(g), src_e.kv_scales[layer, kv], np.float32),
                                  dst_other.kv_scales[layer, kv]).reshape(-1)
                if not np.array_equal(got[layer, kv], want):
                    raise SystemExit(f"{label}: e4m3 read at other scales differs from the model")
        x = src_b.data[:, :, p].contiguous().view(torch.int16).cpu().numpy().view(np.uint16)
        pq, ps = fx.quantise(x.reshape(-1, ROW))
        want_b = fx.dequantise(pq, ps).reshape(x.shape)
        got_b = dst_b.data[:, :, d].contiguous().view(torch.int16).cpu().numpy().view(np.uint16)
        if not np.array_equal(got_b, want_b):
            raise SystemExit(f"{label}: bf16 fp8 read differs from the exact reference")


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--pages", type=int, default=409, help="409 pages: 2.0 GiB of bf16")
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--pool-gb", type=int, default=8)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("e4m3_pages.py needs a CUDA device")
    dev = torch.device("cuda", 0)
    torch.cuda.set_device(dev)
    info = card(0)
    print(f"card: {info}", flush=True)
    lay_b = get_layout("llama-3-70b", page_tokens=16)
    lay_e = get_layout("llama-3-70b", page_tokens=16, dtype=torch.float8_e4m3fn)
    L, elems = lay_b.layers, lay_b.page_elems
    bf16_bytes = a.pages * 2 * L * lay_b.page_bytes
    stored = a.pages * ist.InfinityConnection.fp8_gather_block_bytes(2 * L, elems)
    rng = np.random.default_rng(0)
    s1 = (rng.uniform(0.5, 2, (L, 2)) * 2.0 ** -6).astype(np.float32)
    s2 = (rng.uniform(0.5, 2, (L, 2)) * 2.0 ** -5).astype(np.float32)
    scfg = native.ServerConfig()
    scfg.service_port = 0
    scfg.host = "127.0.0.1"
    scfg.pool_backend = "hbm"
    scfg.pool_devices = [0]
    scfg.minimal_allocate_size = 16
    scfg.prealloc_bytes = a.pool_gb << 30
    srv = native.Server(scfg)
    port = srv.start()
    out = {"card": info, "model": lay_b.name, "pages": a.pages, "page_tokens": lay_b.page_tokens,
           "bf16_payload_bytes": bf16_bytes, "stored_bytes": stored, "reps": a.reps, "arms": {}}
    try:
        mc = memcpy_ms(stored, a.reps, dev)
        out["memcpy_d2d_stored_ms"] = round(mc, 3)
        print(f"cudaMemcpyAsync D2D of the stored bytes ({stored / 2**30:.2f} GiB): {mc:8.3f} ms "
              f"{stored / (mc * 1e-3) / 1e9:7.1f} GB/s", flush=True)
        conn = ist.InfinityConnection(ist.ClientConfig(
            host_addr="127.0.0.1", service_port=port, connection_type=ist.TYPE_RDMA,
            device_lookup=True, streams=0, log_level="warning"))
        conn.connect()
        g = torch.Generator(device=dev).manual_seed(0)
        src_b = PagedKVCache(lay_b, a.pages, dev)
        src_b.data.copy_(torch.randn(src_b.data.shape, generator=g, device=dev))
        src_e = PagedKVCache(lay_e, a.pages, dev, kv_scales=s1)
        # an engine's e4m3 cache of the same values: e4m3(x / s) per layer's K and V
        sc = torch.from_numpy(s1).to(dev)[:, :, None, None]
        src_e.data.copy_((src_b.data.float() / sc).clamp(-448, 448).to(torch.float8_e4m3fn))
        dst_same = PagedKVCache(lay_e, a.pages, dev, kv_scales=s1)
        dst_other = PagedKVCache(lay_e, a.pages, dev, kv_scales=s2)
        dst_b = PagedKVCache(lay_b, a.pages, dev)
        pages = list(range(a.pages))
        rpages = np.random.default_rng(1).permutation(a.pages).tolist()
        arms = {k: [] for k in ("e4m3 write", "e4m3 read same", "e4m3 read other",
                                "bf16 fp8 write", "bf16 fp8 read")}
        for rep in range(a.warmup + a.reps):
            he = [f"e4m3-{rep}-{i}" for i in range(a.pages)]
            hb = [f"bf16-{rep}-{i}" for i in range(a.pages)]

            def timed(fn):
                return device_ms(lambda: (fn(), conn.sync()))

            t = {"e4m3 write": timed(lambda: src_e.write_pages(conn, pages, he, fp8=True))}
            for d in (dst_same, dst_other, dst_b):
                d.data.view(torch.uint8).zero_()
            t["e4m3 read same"] = timed(lambda: dst_same.read_pages(conn, rpages, he, fp8=True))
            t["e4m3 read other"] = timed(lambda: dst_other.read_pages(conn, rpages, he, fp8=True))
            t["bf16 fp8 write"] = timed(lambda: src_b.write_pages(conn, pages, hb, fp8=True))
            t["bf16 fp8 read"] = timed(lambda: dst_b.read_pages(conn, rpages, hb, fp8=True))
            if rep >= a.warmup:
                for k, v in t.items():
                    arms[k].append(v)
            if rep == a.warmup + a.reps - 1:
                check("last round", src_e, src_b, dst_same, dst_other, dst_b, pages, rpages)
            srv.purge()
        for k, v in arms.items():
            ms = statistics.median(v)
            res = {"ms": round(ms, 3),
                   "GBps_bf16_payload": round(bf16_bytes / (ms * 1e-3) / 1e9, 1),
                   "GBps_stored": round(stored / (ms * 1e-3) / 1e9, 1),
                   "vs_memcpy_of_stored": round(mc / ms, 3)}
            out["arms"][k] = res
            print(f"{k:16s} {res['ms']:8.3f} ms {res['GBps_bf16_payload']:7.1f} GB/s bf16 "
                  f"{res['GBps_stored']:7.1f} GB/s stored ({res['vs_memcpy_of_stored']:.2f} of "
                  f"memcpy)", flush=True)
        print("verified: e4m3 reads against the numpy model, the bf16 read against the exact "
              "e4m3 reference, on two pages")
        conn.close()
    finally:
        srv.stop()
    print(json.dumps(out))


if __name__ == "__main__":
    main()
