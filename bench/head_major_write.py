#!/usr/bin/env python
"""Writes of all-layer KV pages from a head-major cache (HeadMajorKVCache), Llama-3-8B layout.

32 layers, 8 KV heads of 128, 256 pages of 16 tokens, pool in the writer GPU's HBM, device
lookup, a streams=0 connection (every launch on the caller's stream, so device events around a
call bracket all of its kernels).  TP rank 0 of a writer at TP 1 (8 heads per page, 8 slices
per stored row) and at TP 4 (2 heads, 2 slices), in bf16 and fp8.  Two sections.

Store calls.  Arms, each writing the same pages under fresh keys, in an order rotated by one
arm every round (round k starts with arm k mod 5), so that no arm always follows the refill of
the pages or the purge of the store:

  head_major   HeadMajorKVCache.write_pages: the gathering write kernel fills each stored
               token-major part from the [head][token][dim] page (row-sliced write)
  staging      today's workaround: a torch permute-copy into a token-major staging cache
               (allocated once, outside the timed window), then PagedKVCache.write_pages
  token_major  PagedKVCache.write_pages of the same bytes from a token-major cache: the
               ceiling (no transposition).  On a pool in the writer's own HBM the connection
               runs the fp8 ld/st kernels for fp8 parts, as it does for the head-major write
  layered_hm / layered_tm
               page_writer(...).write_layers one layer per call, head-major against
               token-major

Each window runs from an event before the first call to an event after the last launch, then
the device is synchronised; it includes the calls' host work (allocation round trip, key
staging, launches).  Every round reads each arm's pages back with PagedKVCache.read_pages and
checks them bit for bit against the token-major arm's, then purges the store.

Kernels alone.  The page movers the store calls launch, on pre-allocated pool blocks with no
allocation, lookup or publish: ops.kv_gather / ops.kv_gather_fp8 with rows= from the head-major
pages (kv_gather_ldst<VEC, kRows>, kv_write_fp8_gather<SlicedRows>) against the same call
without rows from the token-major pages (kv_gather_ldst<VEC, kWhole>; fp8: the ld/st kernel
and the TMA pipeline), and the staging arm's torch permute-copy alone.  Events around
--launches back-to-back launches per window, arms rotated every round as above; the pool
bytes of the two writes are checked equal.

Reported per arm: the median window over --reps rounds (per launch for kernels) with its
minimum and maximum, and GB/s of stored bytes at the median.  Prints the card's name, power
limit and SM clock from the same run, then one JSON line.  A pool behind NVLink and several
GPUs are not measured here."""
from __future__ import annotations

import argparse
import json
import os
import statistics
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "bench"))
import infinistore_b200 as ist  # noqa: E402
from infinistore_b200 import _infinistore as native  # noqa: E402
from infinistore_b200 import ops  # noqa: E402
from infinistore_b200.models.kv_layout import KVLayout  # noqa: E402
from infinistore_b200.models.paged_kv import HeadMajorKVCache, PagedKVCache  # noqa: E402
from gather_fp8 import card  # noqa: E402

LAYERS, HEADS, DIM, TOKENS = 32, 8, 128, 16
ARMS = ("head_major", "staging", "token_major", "layered_hm", "layered_tm")


def tm_view(cache):
    lay = cache.layout
    return cache.data.view(lay.layers, 2, cache.num_pages, lay.page_tokens, lay.heads_per_rank,
                           lay.head_dim)


def same_bits(a, b):
    return torch.equal(a.contiguous().view(torch.int16), b.contiguous().view(torch.int16))


def timed(fn):
    """Device milliseconds of fn() on the current stream."""
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    torch.cuda.synchronize()
    e0.record()
    fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1)


def rotated(arms, rep):
    """The arms in round `rep`'s order: rotated by one arm per round."""
    k = rep % len(arms)
    return arms[k:] + arms[:k]


def stats(ms, stored):
    med = statistics.median(ms)
    return {"ms_median": round(med, 4), "ms_min": round(min(ms), 4), "ms_max": round(max(ms), 4),
            "GBps": round(stored / (med * 1e-3) / 1e9, 1)}


def kernels(lay, n, fp8, dev, a):
    """Per-launch device ms of the write kernels alone (see the module docstring)."""
    hm = HeadMajorKVCache(lay, n, dev)
    hm.data.copy_(torch.randn(hm.data.shape, generator=torch.Generator(device=dev).manual_seed(7),
                              device=dev))
    tm = PagedKVCache(lay, n, dev)
    tm_view(tm).copy_(hm.data.transpose(3, 4))
    staging = PagedKVCache(lay, n, dev)
    elems = lay.page_elems
    nparts = 2 * LAYERS
    bb = ops.fp8_gather_bytes(nparts, elems) if fp8 else nparts * elems * 2
    pitch = (bb + 4095) // 4096 * 4096
    pools = [torch.zeros(n * pitch, dtype=torch.uint8, device=dev) for _ in range(2)]
    offs = [p * elems * 2 for p in range(n)]
    descs = [ops.make_descs(offs, [p.data_ptr() + i * pitch for i in range(n)], dev)
             for p in pools]

    def bases(cache):
        return [cache.data.data_ptr() + cache.page_offset(layer, kv, 0) * 2
                for layer in range(LAYERS) for kv in (0, 1)]

    rows = hm._write_rows().native(2)
    hb, tb = bases(hm), bases(tm)

    def write(d, b, r, variant="ldst"):
        if fp8:
            ops.kv_gather_fp8(d, b, elems, write=True, variant=variant, rows=r)
        else:
            ops.kv_gather(d, b, elems * 2, write=True, rows=r)

    arms = {"head_major": lambda: write(descs[0], hb, rows),
            "token_major": lambda: write(descs[1], tb, None),
            "permute": lambda: tm_view(staging).copy_(hm.data.transpose(3, 4))}
    if fp8:
        arms["token_major_tma"] = lambda: write(descs[1], tb, None, "auto")
    names = list(arms)
    ms = {k: [] for k in names}
    for rep in range(a.warmup + a.reps):
        for k in rotated(names, rep):
            def run(fn=arms[k]):
                for _ in range(a.launches):
                    fn()
            t = timed(run) / a.launches
            if rep >= a.warmup:
                ms[k].append(t)
    torch.cuda.synchronize()
    assert torch.equal(pools[0], pools[1]), "kernels: row write differs from the whole-part write"
    res = {k: stats(ms[k], n * bb) for k in names}
    del hm, tm, staging, pools
    torch.cuda.empty_cache()
    return res


def layered(cache, conn, pages, hashes, fp8):
    pw = cache.page_writer(conn, pages, hashes, fp8=fp8)
    for layer in range(LAYERS):
        pw.write_layers(range(layer, layer + 1))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--pages", type=int, default=256)
    ap.add_argument("--reps", type=int, default=9)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--pool-gb", type=int, default=6)
    ap.add_argument("--tp", type=int, nargs="*", default=[1, 4])
    ap.add_argument("--dtypes", nargs="*", default=["bf16", "fp8"])
    ap.add_argument("--launches", type=int, default=20, help="kernel launches per window")
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("head_major_write.py needs a CUDA device")
    dev = torch.device("cuda", 0)
    torch.cuda.set_device(dev)
    info = card(0)
    print(f"card: {info}", flush=True)
    base = KVLayout("llama-3-8b", LAYERS, HEADS, DIM, TOKENS)
    n = a.pages
    pages = list(range(n))

    scfg = native.ServerConfig()
    scfg.service_port = 0
    scfg.host = "127.0.0.1"
    scfg.pool_backend = "hbm"
    scfg.pool_devices = [0]
    scfg.minimal_allocate_size = 16
    scfg.prealloc_bytes = a.pool_gb << 30
    srv = native.Server(scfg)
    port = srv.start()
    out = {"card": info, "layout": "llama-3-8b", "pages": n, "page_tokens": TOKENS,
           "reps": a.reps, "cases": {}}
    try:
        conn = ist.InfinityConnection(ist.ClientConfig(
            host_addr="127.0.0.1", service_port=port, connection_type=ist.TYPE_RDMA,
            device_lookup=True, streams=0, log_level="warning"))
        conn.connect()
        for tp in a.tp:
            lay = base.with_tp(tp)
            hm = HeadMajorKVCache(lay, n, dev)
            tm = PagedKVCache(lay, n, dev)
            staging = PagedKVCache(lay, n, dev)
            check = PagedKVCache(lay, n, dev)
            want = PagedKVCache(lay, n, dev)
            for dtype in a.dtypes:
                fp8 = dtype == "fp8"
                nbytes = (conn.fp8_gather_block_bytes(2 * LAYERS, lay.page_elems) if fp8
                          else 2 * LAYERS * lay.page_bytes)
                stored = n * nbytes
                ms = {k: [] for k in ARMS}
                for rep in range(a.warmup + a.reps):
                    g = torch.Generator(device=dev).manual_seed(rep)
                    hm.data.copy_(torch.randn(hm.data.shape, generator=g, device=dev))  # fresh
                    tm_view(tm).copy_(hm.data.transpose(3, 4))
                    keys = {k: [f"{tp}-{dtype}-{rep}-{k}-{i}" for i in range(n)] for k in ARMS}

                    def stage():
                        tm_view(staging).copy_(hm.data.transpose(3, 4))
                        staging.write_pages(conn, pages, keys["staging"], fp8=fp8)

                    arms = {
                        "head_major": lambda: hm.write_pages(conn, pages, keys["head_major"],
                                                             fp8=fp8),
                        "staging": stage,
                        "token_major": lambda: tm.write_pages(conn, pages, keys["token_major"],
                                                              fp8=fp8),
                        "layered_hm": lambda: layered(hm, conn, pages, keys["layered_hm"], fp8),
                        "layered_tm": lambda: layered(tm, conn, pages, keys["layered_tm"], fp8),
                    }
                    for k in rotated(list(ARMS), rep):
                        t = timed(arms[k])
                        conn.sync()
                        if rep >= a.warmup:
                            ms[k].append(t)
                    want.read_pages(conn, pages, keys["token_major"], fp8=fp8)
                    conn.sync()
                    if not fp8:
                        assert same_bits(want.data, tm.data), f"tp {tp}: token-major pages"
                    for k in ARMS:
                        check.data.zero_()
                        check.read_pages(conn, pages, keys[k], fp8=fp8)
                        conn.sync()
                        assert same_bits(check.data, want.data), f"tp {tp} {dtype} {k}: pages"
                    srv.purge()
                res = {"tp": tp, "slices": lay.heads_per_rank, "fp8": fp8,
                       "stored_bytes": stored, "staging_bytes": staging.data.numel() * 2}
                for k in ARMS:
                    res[k] = stats(ms[k], stored)
                hmed = statistics.median(ms["head_major"])
                res["staging_over_head_major"] = round(statistics.median(ms["staging"]) / hmed, 3)
                res["head_major_of_token_major"] = round(
                    statistics.median(ms["token_major"]) / hmed, 3)
                res["layered_hm_of_layered_tm"] = round(
                    statistics.median(ms["layered_tm"]) / statistics.median(ms["layered_hm"]), 3)
                print(f"TP {tp} {dtype}: " + ", ".join(
                    f"{k} {res[k]['ms_median']:.3f} ms [{res[k]['ms_min']:.3f}-"
                    f"{res[k]['ms_max']:.3f}] ({res[k]['GBps']} GB/s)" for k in ARMS), flush=True)
                kt = kernels(lay, n, fp8, dev, a)
                res["kernels"] = kt
                print(f"TP {tp} {dtype} kernels alone (per launch): " + ", ".join(
                    f"{k} {v['ms_median']:.3f} ms [{v['ms_min']:.3f}-{v['ms_max']:.3f}] "
                    f"({v['GBps']} GB/s)" for k, v in kt.items()), flush=True)
                out["cases"][f"tp{tp}-{dtype}"] = res
            del hm, tm, staging, check, want
            torch.cuda.empty_cache()
        conn.close()
    finally:
        srv.stop()
    out["card_after"] = card(0)
    print(json.dumps(out))


if __name__ == "__main__":
    main()
