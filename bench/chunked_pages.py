#!/usr/bin/env python
"""All-layer chunks against all-layer pages at an engine's 16-token page size.

The same tokens in every arm: --pages pages of 16 tokens of a token-major PagedKVCache, pool
in the GPU's own HBM, device lookup, a streams=0 connection (every launch on the caller's
stream, so device events around a call bracket all of its kernels).  Arms:

  pages   write_pages / read_pages: one key per 16-token page (today's unit)
  chunks  write_chunks / read_chunks: one key per chunk of --chunk-pages pages (256 tokens by
          default), landed through a shuffled block table into the same 16-token cache

Configurations: Llama-3-70B at TP 8 (one KV head per rank: 4 KB bf16 parts per page) and
Llama-3-8B at TP 1, each in bf16 and fp8, and one cross-TP read (pages and chunks written by
the 8 ranks of TP 8, read by rank 0 of TP 2, Llama-3-70B).  Each round writes under fresh
keys, reads the pages back into a zeroed cache and checks them bit for bit against the pages
arm, then purges the store; the arms alternate which goes first.

Reported per arm and phase: the median device-timed window over --reps rounds and the GB/s of
bf16-equivalent bytes (the cache bytes the phase moves), keys per phase, and host time per
phase (wall clock from the first call to the return of the last, without the synchronise).
Prints the card's name, power limit and SM clock from the same run, then one JSON line."""
from __future__ import annotations

import argparse
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
from infinistore_b200.models.kv_layout import get_layout  # noqa: E402
from infinistore_b200.models.paged_kv import PagedKVCache  # noqa: E402
from gather_fp8 import card  # noqa: E402

B = 16


def bits(t):
    return t.contiguous().view(torch.int16)


def window(fn):
    """(device ms, host ms) of fn(): events around it, host time up to its return."""
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    torch.cuda.synchronize()
    e0.record()
    t0 = time.perf_counter()
    fn()
    host = (time.perf_counter() - t0) * 1e3
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1), host


def run_case(conn, srv, name, writer_tp, reader_tp, fp8, a, dev):
    lay = get_layout(name, page_tokens=B, tp=writer_tp)
    rl = lay.with_tp(reader_tp)
    n, k = a.pages, a.chunk_pages
    nchunks = n // k
    pages = list(range(n))
    perm = np.random.default_rng(1).permutation(n)
    table = perm[:nchunks * k].reshape(nchunks, k)  # chunk b's pages, token order
    rtable = np.random.default_rng(2).permutation(n)[:nchunks * k].reshape(nchunks, k)
    writers = [PagedKVCache(lay, n, dev, tp_rank=w) for w in range(writer_tp)]
    reader = PagedKVCache(rl, n, dev, tp_rank=0)
    source_tp = None if writer_tp == reader_tp else writer_tp
    # bf16-equivalent bytes: the cache bytes each phase moves
    wbytes = writer_tp * n * 2 * lay.layers * lay.page_bytes
    rbytes = n * 2 * rl.layers * rl.page_bytes
    ms = {arm: {"write": [], "read": [], "write_host": [], "read_host": []}
          for arm in ("pages", "chunks")}
    for rep in range(a.warmup + a.reps):
        g = torch.Generator(device=dev).manual_seed(rep)
        for w in writers:
            w.data.copy_(torch.randn(w.data.shape, generator=g, device=dev))
        order = ["pages", "chunks"] if rep % 2 == 0 else ["chunks", "pages"]
        got = {}
        for arm in order:
            hashes = [f"{name}-{writer_tp}-{reader_tp}-{fp8}-{rep}-{arm}-{i}"
                      for i in range(n if arm == "pages" else nchunks)]

            def write():
                for w in writers:
                    if arm == "pages":
                        w.write_pages(conn, pages, hashes, fp8=fp8)
                    else:
                        w.write_chunks(conn, table, hashes, fp8=fp8)

            def read():
                if arm == "pages":  # the pages arm lands where the chunk table puts them
                    reader.read_pages(conn, rtable.reshape(-1).tolist(),
                                      [hashes[int(p)] for p in table.reshape(-1)],
                                      fp8=fp8, source_tp=source_tp)
                else:
                    reader.read_chunks(conn, rtable, hashes, fp8=fp8, source_tp=source_tp)

            wd, wh = window(write)
            conn.sync()
            reader.data.zero_()
            rd, rh = window(read)
            conn.sync()
            got[arm] = reader.data.clone()
            if rep >= a.warmup:
                ms[arm]["write"].append(wd)
                ms[arm]["read"].append(rd)
                ms[arm]["write_host"].append(wh)
                ms[arm]["read_host"].append(rh)
        if not torch.equal(bits(got["pages"]), bits(got["chunks"])) or not got["pages"].any():
            raise SystemExit(f"{name} {writer_tp}->{reader_tp} fp8={fp8}: chunks differ from pages")
        srv.purge()
    out = {}
    for arm, d in ms.items():
        keys_w = writer_tp * (n if arm == "pages" else nchunks)
        keys_r = len(reader.source_page_keys([0], source_tp)) if source_tp else 1
        keys_r *= n if arm == "pages" else nchunks
        res = {"keys_write": keys_w, "keys_read": keys_r}
        for ph, nbytes in (("write", wbytes), ("read", rbytes)):
            med = statistics.median(d[ph])
            res[ph] = {"ms_median": round(med, 3), "ms_min": round(min(d[ph]), 3),
                       "ms_max": round(max(d[ph]), 3),
                       "GBps": round(nbytes / (med * 1e-3) / 1e9, 1),
                       "host_ms_median": round(statistics.median(d[ph + "_host"]), 3)}
        out[arm] = res
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--pages", type=int, default=1024)
    ap.add_argument("--chunk-pages", type=int, default=16)
    ap.add_argument("--reps", type=int, default=7)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--pool-gb", type=int, default=24)
    ap.add_argument("--fp8", action="store_true", help="only the fp8 arms")
    ap.add_argument("--bf16", action="store_true", help="only the bf16 arms")
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("chunked_pages.py needs a CUDA device")
    if a.pages % a.chunk_pages:
        raise SystemExit("--pages must be a multiple of --chunk-pages")
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
    dtypes = [True] if a.fp8 else [False] if a.bf16 else [False, True]
    cases = [("llama-3-70b", 8, 8), ("llama-3-8b", 1, 1)]
    out = {"card": info, "pages": a.pages, "page_tokens": B,
           "chunk_tokens": a.chunk_pages * B, "reps": a.reps, "cases": {}}
    try:
        conn = ist.InfinityConnection(ist.ClientConfig(
            host_addr="127.0.0.1", service_port=port, connection_type=ist.TYPE_RDMA,
            device_lookup=True, streams=0, log_level="warning"))
        conn.connect()
        for fp8 in dtypes:
            for name, wtp, rtp in cases + ([("llama-3-70b", 8, 2)] if not fp8 else []):
                label = f"{name} tp{wtp}->{rtp} {'fp8' if fp8 else 'bf16'}"
                res = run_case(conn, srv, name, wtp, rtp, fp8, a, dev)
                out["cases"][label] = res
                for arm, r in res.items():
                    print(f"{label:28s} {arm:6s} keys w/r {r['keys_write']:6d}/{r['keys_read']:6d}"
                          f"  write {r['write']['ms_median']:8.3f} ms {r['write']['GBps']:7.1f} GB/s"
                          f" host {r['write']['host_ms_median']:7.2f} ms"
                          f"  read {r['read']['ms_median']:8.3f} ms {r['read']['GBps']:7.1f} GB/s"
                          f" host {r['read']['host_ms_median']:7.2f} ms", flush=True)
        conn.close()
    finally:
        srv.stop()
    print(json.dumps(out))


if __name__ == "__main__":
    main()
