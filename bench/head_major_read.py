#!/usr/bin/env python
"""Reads of all-layer KV pages into a head-major cache (HeadMajorKVCache), Llama-3-8B layout.

32 layers, 8 KV heads of 128, 16-token bf16 pages, pool in the reader GPU's HBM, device lookup,
a streams=0 connection (every launch on the caller's stream, so device events around a call
bracket all of its kernels).  The pages are written token-major with PagedKVCache.write_pages
at TP 1, 2 and 8 (one key per page and rank).  Three directions, each read into TP rank 0 of
the reader:

  1 -> 1   same TP: 8 heads of one source per page
  8 -> 2   a TP 2 decode rank reads pages a TP 8 prefill wrote: 4 sources of 1 head per page
  2 -> 8   a TP 8 decode rank reads pages a TP 2 prefill wrote: 1 head of 1 source per page

Four arms, alternated within each round:

  head_major       HeadMajorKVCache.read_pages(source_tp=W): one call; the sliced scatter
                   kernel lands each source's heads as [head][token][dim]
  per_head_blocks  the workaround with single-slice row geometry (PartRows without slices):
                   one block per (page, source, head).  A row geometry is per call, and each
                   head of a source sits at its own column, so this is one call per head
                   position, each with one block per (page, source)
  staging          the workaround through a token-major staging cache: PagedKVCache.read_pages
                   into it (allocated once, outside the timed window), then a torch
                   permute-copy into the head-major cache
  token_major      PagedKVCache.read_pages(source_tp=W) of the same bytes into a token-major
                   cache: the ceiling (no transposition)

Each window runs from an event before the first call to an event after the last kernel, on the
caller's stream.  Reported per arm: the median window over --reps rounds with its minimum and
maximum, and GB/s of destination bytes (pages x layers x 2 x the reader's page bytes) at the
median.  The layered flavour (read_pages_layered) is timed to the release of layer 0 and of
the last layer, as seen by a consumer stream that waits for them.  Every round's pages are
checked bit for bit.  Prints the card's name, power limit and SM clock from the same run, then
one JSON line.  A pool behind NVLink and several GPUs are not measured here.

--fp8: the pages are written as fp8 and every arm reads with fp8=True; every round is checked
against a staging read taken before the timed rounds."""
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
import infinistore_b200 as ist  # noqa: E402
from infinistore_b200 import _infinistore as native  # noqa: E402
from infinistore_b200.lib import PartRows  # noqa: E402
from infinistore_b200.models.kv_layout import ALL_LAYERS, KVLayout, page_key, tp_sources  # noqa: E402
from infinistore_b200.models.paged_kv import HeadMajorKVCache, PagedKVCache  # noqa: E402
from gather_fp8 import card  # noqa: E402

LAYERS, HEADS, DIM, TOKENS = 32, 8, 128, 16
DIRECTIONS = ((1, 1), (8, 2), (2, 8))
ARMS = ("head_major", "per_head_blocks", "staging", "token_major")


def heads_of(tp, rank):
    per = max(HEADS // tp, 1)
    return list(range(rank * per, rank * per + per)) if tp <= HEADS else [rank * HEADS // tp]


def tm_view(cache):
    lay = cache.layout
    return cache.data.view(lay.layers, 2, cache.num_pages, lay.page_tokens, lay.heads_per_rank,
                           lay.head_dim)


def same_bits(a, b):
    """Equal bf16 bits (NaN included)."""
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


def per_head_calls(hm, wl, srcs, pages, hashes):
    """The single-slice workaround: for head position h of every source, one row-sliced read
    of that head's column into its head-major rows; returns [(keys, offsets, PartRows)]."""
    lay = hm.layout
    calls = []
    for h in range(srcs[0][3]):
        keys = [page_key(lay.name, ALL_LAYERS, "KV", w, p) for p in hashes for w, *_ in srcs]
        offs = (np.asarray(pages, dtype=np.int64)[:, None] * lay.page_elems
                + np.asarray([(d + h) * TOKENS * DIM for _, _, d, _ in srcs],
                             dtype=np.int64)[None, :]).reshape(-1)
        rows = PartRows(TOKENS, DIM, wl.heads_per_rank * DIM, (srcs[0][1] + h) * DIM,
                        dst_pitch=DIM)
        calls.append((keys, offs, rows))
    return calls


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--pages", type=int, default=256)
    ap.add_argument("--reps", type=int, default=9)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--pool-gb", type=int, default=4)
    ap.add_argument("--fp8", action="store_true", help="fp8 pages (write_pages(fp8=True))")
    a = ap.parse_args()
    fp8 = a.fp8
    if not torch.cuda.is_available():
        raise SystemExit("head_major_read.py needs a CUDA device")
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
           "reps": a.reps, "fp8": fp8, "directions": {}}
    try:
        conn = ist.InfinityConnection(ist.ClientConfig(
            host_addr="127.0.0.1", service_port=port, connection_type=ist.TYPE_RDMA,
            device_lookup=True, streams=0, log_level="warning"))
        conn.connect()
        g = torch.Generator(device=dev).manual_seed(0)
        full = torch.randn(LAYERS, 2, n, TOKENS, HEADS, DIM, generator=g,
                           device=dev).to(torch.bfloat16)
        tps = sorted({wt for wt, _ in DIRECTIONS})
        hashes = {tp: [f"tp{tp}-{i}" for i in range(n)] for tp in tps}
        for tp in tps:  # every rank writes its heads, token-major
            for w in range(tp):
                c = PagedKVCache(base.with_tp(tp), n, dev, tp_rank=w)
                tm_view(c).copy_(full[:, :, :, :, heads_of(tp, w), :])
                c.write_pages(conn, pages, hashes[tp], fp8=fp8)
                conn.sync()
                del c
        torch.cuda.empty_cache()

        for wt, rt in DIRECTIONS:
            rl, wl = base.with_tp(rt), base.with_tp(wt)
            srcs = tp_sources(rl, rt, 0, wt)
            hm = HeadMajorKVCache(rl, n, dev, tp_rank=0)
            tm = PagedKVCache(rl, n, dev, tp_rank=0)
            staging = PagedKVCache(rl, n, dev, tp_rank=0)
            src = None if wt == rt else wt
            # the pages each arm must produce: a token-major read, outside the timed rounds
            staging.read_pages(conn, pages, hashes[wt], source_tp=src, fp8=fp8)
            conn.sync()
            want_tm = tm_view(staging).clone()
            want_hm = want_tm.transpose(3, 4).contiguous()
            if not fp8:
                assert same_bits(want_tm, full[:, :, :, :, heads_of(rt, 0), :])
            ncalls = srcs[0][3]
            dst_bytes = n * LAYERS * 2 * rl.page_bytes

            def head_major():
                hm.read_pages(conn, pages, hashes[wt], source_tp=src, fp8=fp8)

            def per_head():  # builds its blocks per call, as read_pages does
                read = conn.read_cache_scatter_fp8 if fp8 else conn.read_cache_scatter
                parts = hm._parts(range(LAYERS))
                for keys, offs, rows in per_head_calls(hm, wl, srcs, pages, hashes[wt]):
                    read(parts, (keys, offs), wl.page_elems, rows=rows)

            def stage():
                staging.read_pages(conn, pages, hashes[wt], source_tp=src, fp8=fp8)
                hm.data.copy_(tm_view(staging).transpose(3, 4))

            def token_major():
                tm.read_pages(conn, pages, hashes[wt], source_tp=src, fp8=fp8)

            arms = {"head_major": head_major, "per_head_blocks": per_head, "staging": stage,
                    "token_major": token_major}
            ms = {k: [] for k in ARMS}
            for rep in range(a.warmup + a.reps):
                for k in ARMS:
                    dst = tm if k == "token_major" else hm
                    dst.data.zero_()
                    t = timed(arms[k])
                    conn.sync()
                    ok = (same_bits(tm_view(tm), want_tm) if k == "token_major"
                          else same_bits(hm.data, want_hm))
                    assert ok, f"{wt}->{rt} {k}: wrong pages"
                    if rep >= a.warmup:
                        ms[k].append(t)
            res = {"writer_tp": wt, "reader_tp": rt, "sources_per_page": len(srcs),
                   "heads_per_source": srcs[0][3], "blocks": n * len(srcs),
                   "per_head_calls": ncalls, "per_head_blocks": n * len(srcs) * ncalls,
                   "dst_bytes": dst_bytes, "staging_bytes": staging.data.numel() * 2}
            for k in ARMS:
                med = statistics.median(ms[k])
                res[k] = {"ms_median": round(med, 4), "ms_min": round(min(ms[k]), 4),
                          "ms_max": round(max(ms[k]), 4),
                          "GBps": round(dst_bytes / (med * 1e-3) / 1e9, 1)}
            hmed = statistics.median(ms["head_major"])
            res["staging_over_head_major"] = round(statistics.median(ms["staging"]) / hmed, 3)
            res["per_head_over_head_major"] = round(
                statistics.median(ms["per_head_blocks"]) / hmed, 3)
            res["head_major_of_token_major"] = round(statistics.median(ms["token_major"]) / hmed, 3)
            # layered: time to layer 0's release and to the last layer's, on a consumer stream
            cons = torch.cuda.Stream()
            first, last = [], []
            for rep in range(a.warmup + a.reps):
                hm.data.zero_()
                torch.cuda.synchronize()
                e0, e1, e2 = (torch.cuda.Event(enable_timing=True) for _ in range(3))
                e0.record()
                read = hm.read_pages_layered(conn, pages, hashes[wt], source_tp=src, fp8=fp8)
                read.wait_layer(0, stream=cons)
                e1.record(cons)
                read.wait_layer(LAYERS - 1, stream=cons)
                e2.record(cons)
                torch.cuda.synchronize()
                conn.sync()
                assert same_bits(hm.data, want_hm), f"{wt}->{rt} layered: wrong pages"
                if rep >= a.warmup:
                    first.append(e0.elapsed_time(e1))
                    last.append(e0.elapsed_time(e2))
            res["layered"] = {"first_layer_ms_median": round(statistics.median(first), 4),
                              "last_layer_ms_median": round(statistics.median(last), 4),
                              "first_layer_ms_min": round(min(first), 4),
                              "last_layer_ms_min": round(min(last), 4)}
            print(f"{wt} -> {rt}: " + ", ".join(
                f"{k} {res[k]['ms_median']:.3f} ms ({res[k]['GBps']} GB/s)" for k in ARMS)
                + f", layered first/last layer {res['layered']['first_layer_ms_median']:.3f}"
                f"/{res['layered']['last_layer_ms_median']:.3f} ms", flush=True)
            out["directions"][f"{wt}->{rt}"] = res
            del hm, tm, staging
            torch.cuda.empty_cache()
        conn.close()
    finally:
        srv.stop()
    print(json.dumps(out))


if __name__ == "__main__":
    main()
