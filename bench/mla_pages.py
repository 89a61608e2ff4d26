#!/usr/bin/env python
"""All-layer MLA pages (MLAKVCache) in DeepSeek-V3 geometry: 61 layers of 64-token pages of
512 latent + 64 RoPE dimensions, 4.5 MB per page in bf16 and 2.56 MB as fp8 token records.

A pool in the GPU's own HBM, device lookup, a streams=0 connection.  --pages pages (about
2 GiB of bf16 payload per phase by default).  Arms, each in bf16 and fp8:

  plain    write_pages, then read_pages
  layered  page_writer().write_layers(range(l, l + 1)) for every layer, then
           read_pages_layered with wait_layer(l) on the current stream for every layer

Each phase is timed on the device, events around the calls and the sync() that follows them
(write phase, sync(), read phase, sync()), under fresh keys each round, with --warmup rounds
first; the store is purged after every round.  Reported: the median over --reps rounds, GB/s of
bf16 payload and of stored bytes, and next to them cudaMemcpyAsync device-to-device of the
same bytes measured in the same run.  Every read is checked: bf16 bit for bit against the
written pages; fp8 plain and layered reads bit for bit against each other, and two pages
against the numpy codec of tests/fp8_records.py.  Prints the card's name, power limit and SM
clock from the same run, then one JSON line."""
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
from infinistore_b200.models import MLA_LAYOUTS, MLAKVCache  # noqa: E402
from gather_fp8 import card  # noqa: E402
import fp8_records as fr  # noqa: E402


def device_ms(fn):
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    torch.cuda.synchronize()
    e0.record()
    fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1)


def memcpy_ms(nbytes, reps, dev):
    """Median device time of one cudaMemcpyAsync device-to-device of nbytes."""
    a = torch.empty(nbytes, dtype=torch.uint8, device=dev)
    b = torch.empty_like(a)
    a.fill_(1)
    for _ in range(2):
        b.copy_(a)
    t = [device_ms(lambda: b.copy_(a)) for _ in range(reps)]
    del a, b
    return statistics.median(t)


def bits(t):
    return t.contiguous().view(torch.int16)


def run(conn, srv, src, dst, fp8, layered, a, tag):
    lay = src.layout
    pages = list(range(a.pages))
    rpages = np.random.default_rng(1).permutation(a.pages).tolist()
    wms, rms = [], []
    got = None
    for rep in range(a.warmup + a.reps):
        hashes = [f"{tag}-{rep}-{i}" for i in range(a.pages)]

        def write():
            if layered:
                pw = src.page_writer(conn, pages, hashes, fp8=fp8)
                for layer in range(lay.layers):
                    pw.write_layers(range(layer, layer + 1))
            else:
                src.write_pages(conn, pages, hashes, fp8=fp8)
            conn.sync()

        def read():
            if layered:
                r = dst.read_pages_layered(conn, rpages, hashes, fp8=fp8)
                for layer in range(lay.layers):
                    r.wait_layer(layer)
            else:
                dst.read_pages(conn, rpages, hashes, fp8=fp8)
            conn.sync()

        wd = device_ms(write)
        dst.data.zero_()
        rd = device_ms(read)
        if rep >= a.warmup:
            wms.append(wd)
            rms.append(rd)
        if rep == a.warmup + a.reps - 1:
            got = dst.data[:, rpages].clone()
        srv.purge()
    return statistics.median(wms), statistics.median(rms), got


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--pages", type=int, default=476, help="476 pages: 2.0 GiB of bf16")
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--pool-gb", type=int, default=8)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("mla_pages.py needs a CUDA device")
    dev = torch.device("cuda", 0)
    torch.cuda.set_device(dev)
    info = card(0)
    print(f"card: {info}", flush=True)
    lay = MLA_LAYOUTS["deepseek-v3"]
    rec = ist.FP8Records(lay.latent_dim, lay.rope_dim)
    bf16_bytes = a.pages * lay.layers * lay.page_bytes
    fp8_bytes = a.pages * ist.InfinityConnection.fp8_gather_block_bytes(
        lay.layers, lay.page_elems, records=rec)
    scfg = native.ServerConfig()
    scfg.service_port = 0
    scfg.host = "127.0.0.1"
    scfg.pool_backend = "hbm"
    scfg.pool_devices = [0]
    scfg.minimal_allocate_size = 16
    scfg.prealloc_bytes = a.pool_gb << 30
    srv = native.Server(scfg)
    port = srv.start()
    out = {"card": info, "model": lay.name, "pages": a.pages, "page_tokens": lay.page_tokens,
           "bf16_payload_bytes": bf16_bytes, "fp8_stored_bytes": fp8_bytes, "reps": a.reps,
           "arms": {}}
    try:
        memcpy = {"bf16": memcpy_ms(bf16_bytes, a.reps, dev),
                  "fp8": memcpy_ms(fp8_bytes, a.reps, dev)}
        for k, v in memcpy.items():
            nb = bf16_bytes if k == "bf16" else fp8_bytes
            out[f"memcpy_d2d_{k}_ms"] = round(v, 3)
            print(f"cudaMemcpyAsync D2D of the {k} bytes ({nb / 2**30:.2f} GiB): {v:8.3f} ms "
                  f"{nb / (v * 1e-3) / 1e9:7.1f} GB/s", flush=True)
        conn = ist.InfinityConnection(ist.ClientConfig(
            host_addr="127.0.0.1", service_port=port, connection_type=ist.TYPE_RDMA,
            device_lookup=True, streams=0, log_level="warning"))
        conn.connect()
        src, dst = MLAKVCache(lay, a.pages, dev), MLAKVCache(lay, a.pages, dev)
        src.data.copy_(torch.randn(src.data.shape, generator=torch.Generator(device=dev)
                                   .manual_seed(0), device=dev))
        want = src.data.clone()
        fp8_reads = {}
        for fp8 in (False, True):
            stored = fp8_bytes if fp8 else bf16_bytes
            for layered in (False, True):
                label = f"{'fp8' if fp8 else 'bf16'} {'layered' if layered else 'plain'}"
                w, r, got = run(conn, srv, src, dst, fp8, layered, a, label.replace(" ", "-"))
                # page i of the source landed in page rpages[i]: got[:, i] is page i
                if not fp8 and not torch.equal(bits(got), bits(want)):
                    raise SystemExit(f"{label}: read differs from the written pages")
                if fp8:
                    fp8_reads[layered] = got
                res = {}
                for ph, ms in (("write", w), ("read", r)):
                    res[ph] = {"ms": round(ms, 3),
                               "GBps_bf16_payload": round(bf16_bytes / (ms * 1e-3) / 1e9, 1),
                               "GBps_stored": round(stored / (ms * 1e-3) / 1e9, 1),
                               "vs_memcpy_of_stored": round(
                                   memcpy["fp8" if fp8 else "bf16"] / ms, 3)}
                out["arms"][label] = res
                print(f"{label:14s}" + "".join(
                    f"  {ph} {res[ph]['ms']:8.3f} ms {res[ph]['GBps_bf16_payload']:7.1f} GB/s bf16 "
                    f"{res[ph]['GBps_stored']:7.1f} GB/s stored "
                    f"({res[ph]['vs_memcpy_of_stored']:.2f} of memcpy)"
                    for ph in ("write", "read")), flush=True)
        if not torch.equal(bits(fp8_reads[False]), bits(fp8_reads[True])):
            raise SystemExit("fp8: the layered read differs from the plain one")
        for j in (0, a.pages - 1):  # two pages against the numpy codec
            tok = bits(want[:, j]).cpu().numpy().view(np.uint16).reshape(-1, lay.token_dim)
            ref = fr.decode(fr.encode(tok, lay.latent_dim, lay.rope_dim), lay.latent_dim,
                            lay.rope_dim)
            g = bits(fp8_reads[False][:, j]).cpu().numpy().view(np.uint16).reshape(ref.shape)
            if not np.array_equal(g, ref):
                raise SystemExit("fp8: a page differs from the codec")
        print("verified: bf16 reads bit for bit, fp8 plain == layered, two pages == codec")
        conn.close()
    finally:
        srv.stop()
    print(json.dumps(out))


if __name__ == "__main__":
    main()
