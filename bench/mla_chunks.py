#!/usr/bin/env python
"""All-layer MLA chunks (MLAKVCache.write_chunks / read_chunks) in DeepSeek-V3 geometry: 61
layers of 512 latent + 64 RoPE dimensions, 16-token engine pages (vLLM's Triton MLA default)
stored as chunks of k pages under one key, against 64-token pages of the same tokens.

A pool in the GPU's own HBM, device lookup, a streams=0 connection.  --tokens tokens (about
2 GiB of bf16 payload per phase by default).  Arms, each in bf16 and fp8 (token records), plain
and layered:

  16x4     16-token pages as chunks of k = 4 (64 tokens per key)
  16x16    16-token pages as chunks of k = 16 (256 tokens per key)
  64       64-token pages through write_pages / read_pages: the same bytes per phase, the
           reference a chunk arm is compared with

plain: one write call, then one read call; layered: a writer's write_layers(range(l, l + 1))
for every layer, then a layered read with wait_layer(l) on the current stream for every layer.
Chunks are written from the pages in token order and read through a shuffled block table.
Each phase is timed on the device, events around the calls and the sync() that follows them,
under fresh keys each round, with --warmup rounds first; the store is purged after every round.
Reported: the median over --reps rounds, GB/s of bf16 payload and of stored bytes, and
cudaMemcpyAsync device-to-device of the same bytes measured in the same run.  Every read is
checked: bf16 bit for bit against the written pages; every fp8 read bit for bit against the
64-token plain fp8 read (the stored records are the same), and two pages of that against the
numpy codec of tests/fp8_records.py.  Prints the card's name, power limit and SM clock from the
same run, then one JSON line."""
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
from infinistore_b200.models import MLA_LAYOUTS, MLAKVCache, MLALayout  # noqa: E402
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


def run(conn, srv, src, dst, k, fp8, layered, a, tag):
    """k > 0: chunks of k pages of src's page size; k == 0: pages.  Returns the median write
    and read times and the last read, as [layer, token, dim] in the written order."""
    lay = src.layout
    n = src.num_pages // max(k, 1)
    rng = np.random.default_rng(1)
    wt = np.arange(src.num_pages).reshape(n, k) if k else np.arange(n)
    rt = rng.permutation(src.num_pages).reshape(n, k) if k else rng.permutation(n)
    wms, rms = [], []
    got = None
    for rep in range(a.warmup + a.reps):
        hashes = [f"{tag}-{rep}-{i}" for i in range(n)]

        def write():
            if layered:
                w = (src.chunk_writer(conn, wt, hashes, fp8=fp8) if k
                     else src.page_writer(conn, wt.tolist(), hashes, fp8=fp8))
                for layer in range(lay.layers):
                    w.write_layers(range(layer, layer + 1))
            elif k:
                src.write_chunks(conn, wt, hashes, fp8=fp8)
            else:
                src.write_pages(conn, wt.tolist(), hashes, fp8=fp8)
            conn.sync()

        def read():
            if layered:
                r = (dst.read_chunks_layered(conn, rt, hashes, fp8=fp8) if k
                     else dst.read_pages_layered(conn, rt.tolist(), hashes, fp8=fp8))
                for layer in range(lay.layers):
                    r.wait_layer(layer)
            elif k:
                dst.read_chunks(conn, rt, hashes, fp8=fp8)
            else:
                dst.read_pages(conn, rt.tolist(), hashes, fp8=fp8)
            conn.sync()

        wd = device_ms(write)
        dst.data.zero_()
        rd = device_ms(read)
        if rep >= a.warmup:
            wms.append(wd)
            rms.append(rd)
        if rep == a.warmup + a.reps - 1:
            got = dst.data[:, rt.reshape(-1)].reshape(lay.layers, -1, lay.token_dim).clone()
        srv.purge()
    return statistics.median(wms), statistics.median(rms), got


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--tokens", type=int, default=476 * 64, help="30464 tokens: 2.0 GiB of bf16")
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--pool-gb", type=int, default=8)
    a = ap.parse_args()
    if a.tokens % 256:
        raise SystemExit("--tokens must be a multiple of 256 (whole chunks of 16 x 16 tokens)")
    if not torch.cuda.is_available():
        raise SystemExit("mla_chunks.py needs a CUDA device")
    dev = torch.device("cuda", 0)
    torch.cuda.set_device(dev)
    info = card(0)
    print(f"card: {info}", flush=True)
    v3 = MLA_LAYOUTS["deepseek-v3"]
    lay16 = MLALayout(v3.name, v3.layers, v3.latent_dim, v3.rope_dim, 16)
    rec = ist.FP8Records(v3.latent_dim, v3.rope_dim)
    bf16_bytes = a.tokens * v3.layers * v3.token_dim * 2
    fp8_bytes = a.tokens * v3.layers * rec.record_bytes
    scfg = native.ServerConfig()
    scfg.service_port = 0
    scfg.host = "127.0.0.1"
    scfg.pool_backend = "hbm"
    scfg.pool_devices = [0]
    scfg.minimal_allocate_size = 16
    scfg.prealloc_bytes = a.pool_gb << 30
    srv = native.Server(scfg)
    port = srv.start()
    out = {"card": info, "model": v3.name, "tokens": a.tokens, "bf16_payload_bytes": bf16_bytes,
           "fp8_stored_bytes": fp8_bytes, "reps": a.reps, "arms": {}}
    try:
        memcpy = {"bf16": memcpy_ms(bf16_bytes, a.reps, dev),
                  "fp8": memcpy_ms(fp8_bytes, a.reps, dev)}
        for f, v in memcpy.items():
            nb = bf16_bytes if f == "bf16" else fp8_bytes
            out[f"memcpy_d2d_{f}_ms"] = round(v, 3)
            print(f"cudaMemcpyAsync D2D of the {f} bytes ({nb / 2**30:.2f} GiB): {v:8.3f} ms "
                  f"{nb / (v * 1e-3) / 1e9:7.1f} GB/s", flush=True)
        conn = ist.InfinityConnection(ist.ClientConfig(
            host_addr="127.0.0.1", service_port=port, connection_type=ist.TYPE_RDMA,
            device_lookup=True, streams=0, log_level="warning"))
        conn.connect()
        caches = {64: (MLAKVCache(v3, a.tokens // 64, dev), MLAKVCache(v3, a.tokens // 64, dev)),
                  16: (MLAKVCache(lay16, a.tokens // 16, dev),
                       MLAKVCache(lay16, a.tokens // 16, dev))}
        caches[64][0].data.copy_(torch.randn(caches[64][0].data.shape, generator=torch.Generator(
            device=dev).manual_seed(0), device=dev))
        caches[16][0].data.copy_(caches[64][0].data.view(caches[16][0].data.shape))
        want = caches[64][0].data.view(v3.layers, -1, v3.token_dim)
        fp8_ref = None
        arms = [("64", 64, 0), ("16x4", 16, 4), ("16x16", 16, 16)]
        for fp8 in (False, True):
            stored = fp8_bytes if fp8 else bf16_bytes
            for layered in (False, True):
                for name, pt, k in arms:
                    label = f"{'fp8' if fp8 else 'bf16'} {'layered' if layered else 'plain'} {name}"
                    src, dst = caches[pt]
                    w, r, got = run(conn, srv, src, dst, k, fp8, layered, a,
                                    label.replace(" ", "-"))
                    if not fp8 and not torch.equal(bits(got), bits(want)):
                        raise SystemExit(f"{label}: read differs from the written pages")
                    if fp8 and fp8_ref is None:
                        fp8_ref = got  # the 64-token plain fp8 read
                    elif fp8 and not torch.equal(bits(got), bits(fp8_ref)):
                        raise SystemExit(f"{label}: read differs from the 64-token fp8 read")
                    res = {}
                    for ph, ms in (("write", w), ("read", r)):
                        res[ph] = {"ms": round(ms, 3),
                                   "GBps_bf16_payload": round(bf16_bytes / (ms * 1e-3) / 1e9, 1),
                                   "GBps_stored": round(stored / (ms * 1e-3) / 1e9, 1),
                                   "vs_memcpy_of_stored": round(
                                       memcpy["fp8" if fp8 else "bf16"] / ms, 3)}
                    out["arms"][label] = res
                    print(f"{label:20s}" + "".join(
                        f"  {ph} {res[ph]['ms']:8.3f} ms {res[ph]['GBps_bf16_payload']:7.1f} GB/s "
                        f"bf16 {res[ph]['GBps_stored']:7.1f} GB/s stored "
                        f"({res[ph]['vs_memcpy_of_stored']:.2f} of memcpy)"
                        for ph in ("write", "read")), flush=True)
        for j in (0, a.tokens // 64 - 1):  # two 64-token pages against the numpy codec
            tok = bits(want[:, 64 * j:64 * (j + 1)]).cpu().numpy().view(np.uint16).reshape(
                -1, v3.token_dim)
            ref = fr.decode(fr.encode(tok, v3.latent_dim, v3.rope_dim), v3.latent_dim,
                            v3.rope_dim)
            g = bits(fp8_ref[:, 64 * j:64 * (j + 1)]).cpu().numpy().view(np.uint16)
            if not np.array_equal(g.reshape(ref.shape), ref):
                raise SystemExit("fp8: a page differs from the codec")
        print("verified: bf16 reads bit for bit, every fp8 read == the 64-token plain fp8 read, "
              "two pages == codec")
        conn.close()
    finally:
        srv.stop()
    print(json.dumps(out))


if __name__ == "__main__":
    main()
