#!/usr/bin/env python
"""Reads of all-layer KV pages written at another tensor-parallel degree, Llama-3-70B layout.

80 layers, 8 KV heads of 128, 16-token bf16 pages, pool in the reader GPU's HBM, device lookup,
a streams=0 connection (every launch on the caller's stream, so device events around a call
bracket all of its kernels).  The pages are written once at TP 8 and once at TP 2 (one key
per page and rank, write_pages).  Two directions, each read into TP rank 0 of the reader:

  8 -> 2   a TP 2 decode rank reads pages a TP 8 prefill wrote: 4 sources per page
  2 -> 8   a TP 8 decode rank reads pages a TP 2 prefill wrote: 1 head of 1 source per page

Three arms fetch the same destination bytes, alternated within each round:

  rows      PagedKVCache.read_pages(source_tp=W): one call, the row-sliced scatter kernel
  staging   the workaround: read_pages of each source rank into a staging PagedKVCache at
            the writer's TP (allocated once, outside the timed window), then a torch copy of
            its head slice into the reader's cache
  same_tp   read_pages of pages written at the reader's own TP: the ceiling

Each window runs from an event before the first call to an event after the last kernel, on
the caller's stream.  Reported per arm: the median window over --reps rounds with its minimum
and maximum, and GB/s of destination bytes (pages x layers x 2 x the reader's page bytes) at
the median.  The layered flavour (read_pages_layered(source_tp=W)) is timed to the release of
layer 0 and of the last layer, as seen by a consumer stream that waits for them.  Every
round's pages are checked bit for bit against the full-head source.  Prints the card's name,
power limit and SM clock from the same run, then one JSON line.  Over NVLink (a pool on
another GPU) the numbers may differ; that is not measured here."""
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
from infinistore_b200.models.kv_layout import KVLayout, tp_sources  # noqa: E402
from infinistore_b200.models.paged_kv import PagedKVCache  # noqa: E402
from gather_fp8 import card  # noqa: E402

LAYERS, HEADS, DIM, TOKENS = 80, 8, 128, 16
DIRECTIONS = ((8, 2), (2, 8))
ARMS = ("rows", "staging", "same_tp")


def heads_of(tp, rank):
    per = max(HEADS // tp, 1)
    return list(range(rank * per, rank * per + per)) if tp <= HEADS else [rank * HEADS // tp]


def view(cache):
    lay = cache.layout
    return cache.data.view(lay.layers, 2, cache.num_pages, lay.page_tokens, lay.heads_per_rank,
                           lay.head_dim)


def timed(fn):
    """Device milliseconds of fn() on the current stream."""
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    torch.cuda.synchronize()
    e0.record()
    fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--pages", type=int, default=256)
    ap.add_argument("--reps", type=int, default=9)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--pool-gb", type=int, default=8)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("tp_regroup_read.py needs a CUDA device")
    dev = torch.device("cuda", 0)
    torch.cuda.set_device(dev)
    info = card(0)
    print(f"card: {info}", flush=True)
    base = KVLayout("llama-3-70b", LAYERS, HEADS, DIM, TOKENS)
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
    out = {"card": info, "layout": "llama-3-70b", "pages": n, "page_tokens": TOKENS,
           "reps": a.reps, "directions": {}}
    try:
        conn = ist.InfinityConnection(ist.ClientConfig(
            host_addr="127.0.0.1", service_port=port, connection_type=ist.TYPE_RDMA,
            device_lookup=True, streams=0, log_level="warning"))
        conn.connect()
        g = torch.Generator(device=dev).manual_seed(0)
        full = torch.randn(LAYERS, 2, n, TOKENS, HEADS, DIM, generator=g,
                           device=dev).to(torch.bfloat16)
        hashes = {tp: [f"tp{tp}-{i}" for i in range(n)] for tp in (2, 8)}
        for tp in (2, 8):  # every rank of both degrees writes its heads
            for w in range(tp):
                c = PagedKVCache(base.with_tp(tp), n, dev, tp_rank=w)
                view(c).copy_(full[:, :, :, :, heads_of(tp, w), :])
                c.write_pages(conn, pages, hashes[tp])
                conn.sync()
                del c
        torch.cuda.empty_cache()

        for wt, rt in DIRECTIONS:
            rl, wl = base.with_tp(rt), base.with_tp(wt)
            srcs = tp_sources(rl, rt, 0, wt)
            want = full[:, :, :, :, heads_of(rt, 0), :]
            reader = PagedKVCache(rl, n, dev, tp_rank=0)
            staging = [PagedKVCache(wl, n, dev, tp_rank=w) for w, *_ in srcs]
            dst_bytes = n * LAYERS * 2 * rl.page_bytes

            def rows():
                reader.read_pages(conn, pages, hashes[wt], source_tp=wt)

            def stage():
                v = view(reader)
                for st, (w, sh, dh, k) in zip(staging, srcs):
                    st.read_pages(conn, pages, hashes[wt])
                    v[:, :, :, :, dh:dh + k].copy_(view(st)[:, :, :, :, sh:sh + k])

            def same():
                reader.read_pages(conn, pages, hashes[rt])

            arms = {"rows": rows, "staging": stage, "same_tp": same}
            ms = {k: [] for k in ARMS}
            for rep in range(a.warmup + a.reps):
                for k in ARMS:
                    reader.data.zero_()
                    t = timed(arms[k])
                    conn.sync()
                    assert torch.equal(view(reader), want), f"{wt}->{rt} {k}: wrong pages"
                    if rep >= a.warmup:
                        ms[k].append(t)
            res = {"writer_tp": wt, "reader_tp": rt, "sources_per_page": len(srcs),
                   "blocks": n * len(srcs), "dst_bytes": dst_bytes,
                   "staging_bytes": sum(s.data.numel() * 2 for s in staging)}
            for k in ARMS:
                med = statistics.median(ms[k])
                res[k] = {"ms_median": round(med, 4), "ms_min": round(min(ms[k]), 4),
                          "ms_max": round(max(ms[k]), 4),
                          "GBps": round(dst_bytes / (med * 1e-3) / 1e9, 1)}
            res["rows_over_staging"] = round(statistics.median(ms["staging"])
                                             / statistics.median(ms["rows"]), 3)
            res["rows_of_same_tp"] = round(statistics.median(ms["same_tp"])
                                           / statistics.median(ms["rows"]), 3)
            # layered: time to layer 0's release and to the last layer's, on a consumer stream
            cons = torch.cuda.Stream()
            first, last = [], []
            for rep in range(a.warmup + a.reps):
                reader.data.zero_()
                torch.cuda.synchronize()
                e0, e1, e2 = (torch.cuda.Event(enable_timing=True) for _ in range(3))
                e0.record()
                read = reader.read_pages_layered(conn, pages, hashes[wt], source_tp=wt)
                read.wait_layer(0, stream=cons)
                e1.record(cons)
                read.wait_layer(LAYERS - 1, stream=cons)
                e2.record(cons)
                torch.cuda.synchronize()
                conn.sync()
                assert torch.equal(view(reader), want), f"{wt}->{rt} layered: wrong pages"
                if rep >= a.warmup:
                    first.append(e0.elapsed_time(e1))
                    last.append(e0.elapsed_time(e2))
            res["layered"] = {"first_layer_ms_median": round(statistics.median(first), 4),
                              "last_layer_ms_median": round(statistics.median(last), 4),
                              "first_layer_ms_min": round(min(first), 4)}
            print(f"{wt} -> {rt}: " + ", ".join(
                f"{k} {res[k]['ms_median']:.3f} ms ({res[k]['GBps']} GB/s)" for k in ARMS)
                + f", layered first layer {res['layered']['first_layer_ms_median']:.3f} ms",
                flush=True)
            out["directions"][f"{wt}->{rt}"] = res
            del reader, staging
            torch.cuda.empty_cache()
        conn.close()
    finally:
        srv.stop()
    print(json.dumps(out))


if __name__ == "__main__":
    main()
