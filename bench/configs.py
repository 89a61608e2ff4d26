#!/usr/bin/env python
"""The configurations of BASELINE.json beyond the flagship (bench.py = config 2), single-block
latency percentiles and the emulated baselines - as functions bench.py calls inside its own
run (so they land in the driver-visible JSON line under `extra` / `baselines`) and as a CLI:

    torchrun --nproc-per-node N bench/configs.py {fanin,fp8,bcast,latency,baselines}

  fanin   (config 3)  N-1 client GPUs -> 1 pool GPU, Llama-3-8B KV pages (256 KiB per K or V
                      page per layer), layer-wise writes then reads.
  bcast   (config 4)  1 writer -> every GPU through the store's NVLS-replicated region
                      (multimem.st, 1 MB blocks), readers on every rank read their local
                      replica; plus get_match_last_index on the device vs the server op.
  fp8     (config 5)  fp8 KV path: write fused with the bf16->e4m3 cast, read fused with the
                      dequantising gather, 64 KB (fp8) blocks, ring over N GPUs.
  gather              Llama-3-8B in vLLM's layout, 2048 pages: per-layer keys against one
                      gathered key per page (all layers' K and V), 32 KB and 64 KB parts.

Timing: CUDA events recorded on the rank's current stream around (issue + sync()); the
stream is otherwise idle, so the pair brackets the transfer on the device clock; every number
is the max over ranks.
"""
from __future__ import annotations

import argparse
import json
import os
import sys
import time
import uuid
from dataclasses import dataclass
from typing import Any, Callable

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)
import infinistore_b200 as ist  # noqa: E402
from infinistore_b200 import _infinistore as native  # noqa: E402
from infinistore_b200.models import get_layout  # noqa: E402
from infinistore_b200.parallel import nvls_available, start_shard_server  # noqa: E402


@dataclass
class Ctx:
    dist: Any
    rank: int
    world: int
    local: int
    dev: torch.device
    base_port: int
    barrier: Callable[[], None]
    allmax: Callable[[float], float]
    allsum: Callable[[float], float]
    allmin: Callable[[float], float]


class DevTimer:
    """Accumulates device time (ms) between start() and stop() with CUDA events."""

    def __init__(self):
        self.ms = 0.0

    def start(self):
        self.e0 = torch.cuda.Event(enable_timing=True)
        self.e1 = torch.cuda.Event(enable_timing=True)
        self.e0.record()

    def stop(self):
        self.e1.record()
        self.e1.synchronize()
        self.ms += self.e0.elapsed_time(self.e1)


def _client(ctx: Ctx, port: int, **kw):
    conn = ist.InfinityConnection(ist.ClientConfig(
        host_addr="127.0.0.1", service_port=port, connection_type=ist.TYPE_RDMA,
        device=ctx.local, device_lookup=True, log_level="warning", **kw))
    conn.connect()
    return conn


# --------------------------------------------------------------------------- latency
def latency(ctx: Ctx, port: int, sizes_kb=(4, 128, 1024), samples=200):
    """One block written (or read) + sync(): p50 / p99 in microseconds per block size, against
    the store on `port` (the ring peer: NVLink for N >= 2, local HBM at N = 1).  Host clock
    around the call pair - this IS a host-visible latency - max over ranks of each
    percentile.  Two sync() flavours: "strict" (default: control-plane round trip, every
    client sees the write when sync() returns) and "posted" (ClientConfig(posted_commit=True):
    one-way commit like the reference's COMMIT SEND; device-path readers see the write at
    once through the in-band commit); "posted_in_stream" adds streams=0; "doorbell" /
    "posted_doorbell" hand single blocks to the persistent worker."""
    out = {"path": "NVLink (ring peer)" if ctx.world > 1 else "local HBM"}
    q = lambda v, p: v[min(len(v) - 1, int(p * len(v)))]  # noqa: E731
    modes = {"strict": {}, "posted": {"posted_commit": True},
             # launches in the caller's stream: no event record / wait between the caller's
             # stream and an internal one
             "posted_in_stream": {"posted_commit": True, "streams": 0},
             # latency mode: a persistent worker CTA polls a request ring in pinned host memory
             # (kernels/kv_doorbell.cu; blocks <= 256 KB, larger ones take the ordinary path)
             "doorbell": {"doorbell": True},
             "posted_doorbell": {"posted_commit": True, "doorbell": True}}
    for mode, kw in modes.items():
        conn = _client(ctx, port, **kw)
        res = {}
        for kb in sizes_kb:
            elems = kb * 1024 // 2
            src = torch.randn(elems, device=ctx.dev).to(torch.bfloat16)
            dst = torch.zeros_like(src)
            conn.register_mr(src)
            conn.register_mr(dst)
            keys = [f"lat-{mode}-{kb}-{ctx.rank}-{uuid.uuid4().hex[:8]}-{i}"
                    for i in range(samples + 20)]
            remote = conn.allocate_rdma(keys, kb * 1024)
            tw, tr = [], []
            for i, k in enumerate(keys):
                t0 = time.perf_counter()
                conn.rdma_write_cache(src, [0], elems, remote[i:i + 1])
                conn.sync()
                t1 = time.perf_counter()
                conn.read_cache(dst, [(k, 0)], elems)
                conn.sync()
                t2 = time.perf_counter()
                if i >= 20:
                    tw.append((t1 - t0) * 1e6)
                    tr.append((t2 - t1) * 1e6)
            tw.sort()
            tr.sort()
            assert torch.equal(src, dst)
            res[f"{kb}KB"] = {"write_sync_p50": round(ctx.allmax(q(tw, 0.5)), 1),
                              "write_sync_p99": round(ctx.allmax(q(tw, 0.99)), 1),
                              "read_sync_p50": round(ctx.allmax(q(tr, 0.5)), 1),
                              "read_sync_p99": round(ctx.allmax(q(tr, 0.99)), 1)}
        out[mode] = res
        conn.close()
    return out


# --------------------------------------------------------------------------- baselines
def baselines(ctx: Ctx, block_bytes: int, size_bytes: int = 1 << 30, layers: int = 32):
    """EMULATIONS, built from library calls only (none of this repo's kernels): the
    reference cannot be built offline, so its data-movement patterns are re-created.
      reference_localgpu_pattern : reference LOCAL_GPU path (src/infinistore.cpp:570-804):
          per block one cudaMemcpyAsync GPU -> pinned host pool (write) and back (read), a
          fresh stream + event per request.  All ranks run it at once.
      nccl_sendrecv_ring : "only calls NCCL": each request's pages as one contiguous tensor
          to the ring peer and back (N >= 2)."""
    out = {}
    nblocks = size_bytes // block_bytes
    per = nblocks // layers
    src = torch.empty(size_bytes, dtype=torch.uint8, device=ctx.dev).random_(0, 255)
    dst = torch.zeros_like(src)
    pool = torch.empty(size_bytes, dtype=torch.uint8).pin_memory()
    sp = [src.data_ptr() + i * block_bytes for i in range(nblocks)]
    pp = [pool.data_ptr() + i * block_bytes for i in range(nblocks)]
    dp = [dst.data_ptr() + i * block_bytes for i in range(nblocks)]
    tm = DevTimer()
    for it in range(2):
        torch.cuda.synchronize()
        ctx.barrier()
        if it:
            tm.start()
        for l in range(layers):
            native.baseline.memcpy_blocks(pp[l * per:(l + 1) * per], sp[l * per:(l + 1) * per],
                                          block_bytes, True, ctx.local)
        for l in range(layers):
            native.baseline.memcpy_blocks(dp[l * per:(l + 1) * per], pp[l * per:(l + 1) * per],
                                          block_bytes, True, ctx.local)
        torch.cuda.synchronize()
        if it:
            tm.stop()
    ok = bool(torch.equal(src, dst))
    ms = ctx.allmax(tm.ms)
    out["reference_localgpu_pattern"] = {
        "kind": "EMULATION of the reference's LOCAL_GPU path with per-block cudaMemcpyAsync to a "
                "pinned host pool, fresh stream+event per request (src/infinistore.cpp:570-804)",
        "aggregate_GBps": round(ctx.world * 2 * size_bytes / ms / 1e6, 2),
        "per_gpu_GBps": round(2 * size_bytes / ms / 1e6, 2), "block_kb": block_bytes >> 10,
        "verified": ok}
    del pool
    if ctx.world > 1:
        dist = ctx.dist
        nxt, prv = (ctx.rank + 1) % ctx.world, (ctx.rank - 1) % ctx.world
        rbuf = torch.empty_like(src)
        seg = size_bytes // layers
        tm = DevTimer()
        for it in range(2):
            torch.cuda.synchronize()
            ctx.barrier()
            if it:
                tm.start()
            for phase in range(2):  # "write" to the next rank's pool, "read" it back
                for l in range(layers):
                    s = slice(l * seg, (l + 1) * seg)
                    a, b = (src, rbuf) if phase == 0 else (rbuf, dst)
                    to, frm = (nxt, prv) if phase == 0 else (prv, nxt)
                    ops = [dist.P2POp(dist.isend, a[s], to), dist.P2POp(dist.irecv, b[s], frm)]
                    for r in dist.batch_isend_irecv(ops):
                        r.wait()
            torch.cuda.synchronize()
            if it:
                tm.stop()
        ms = ctx.allmax(tm.ms)
        out["nccl_sendrecv_ring"] = {
            "kind": "library baseline: NCCL send/recv of each request's pages as one tensor to "
                    "the ring peer and back",
            "aggregate_GBps": round(ctx.world * 2 * size_bytes / ms / 1e6, 1),
            "per_gpu_GBps": round(2 * size_bytes / ms / 1e6, 1)}
    return out


# --------------------------------------------------------------------------- config 3
def fanin(ctx: Ctx, pages: int = 64, iters: int = 2):
    layout = get_layout("llama-3-8b")           # 256 KiB pages
    layers, elems = layout.layers, layout.page_elems
    nblk = pages * 2 * layers                    # K and V pages of every layer
    per_client = nblk * layout.page_bytes
    port = ctx.base_port + 50
    server = None
    if ctx.rank == 0:
        server = start_shard_server(ctx.local, port,
                                    (ctx.world - 1) * per_client * (iters + 2) + (256 << 20),
                                    granule_kb=64)
    ctx.barrier()
    tw, tr = DevTimer(), DevTimer()
    ok = True
    conn = None
    if ctx.rank > 0:
        conn = _client(ctx, port)
        src = torch.randn(nblk * elems, device=ctx.dev).to(torch.bfloat16)
        dst = torch.zeros_like(src)
        conn.register_mr(src)
        conn.register_mr(dst)
        per_layer = pages * 2
        offs = np.arange(nblk, dtype=np.int64) * elems
    for it in range(iters + 1):
        if ctx.rank > 0:
            tag = uuid.uuid4().hex[:12]
            keys = [f"r{ctx.rank}/{tag}/{i}" for i in range(nblk)]
            remote = conn.allocate_rdma(keys, layout.page_bytes)
            blocks = list(zip(keys, offs.tolist()))
        torch.cuda.synchronize()
        ctx.barrier()
        if it:
            tw.start()
        if ctx.rank > 0:
            for l in range(layers):
                s = slice(l * per_layer, (l + 1) * per_layer)
                conn.rdma_write_cache(src, offs[s], elems, remote[s])
            conn.sync()
        if it:
            tw.stop()
        ctx.barrier()
        if it:
            tr.start()
        if ctx.rank > 0:
            for l in range(layers):
                s = slice(l * per_layer, (l + 1) * per_layer)
                conn.read_cache(dst, blocks[s], elems)
            conn.sync()
        if it:
            tr.stop()
        ctx.barrier()
    if ctx.rank > 0:
        ok = bool(torch.equal(src, dst))
        conn.close()
    w, r = ctx.allmax(tw.ms), ctx.allmax(tr.ms)
    okall = ctx.allsum(0.0 if ok else 1.0) == 0.0
    ctx.barrier()
    if server is not None:
        server.stop()
    total = (ctx.world - 1) * per_client * iters
    return {"what": f"{ctx.world - 1} client GPUs -> 1 pool GPU, Llama-3-8B KV pages",
            "page_kib": layout.page_bytes >> 10, "bytes_per_client_per_iter": per_client,
            "write_GBps_aggregate": round(total / w / 1e6, 1),
            "read_GBps_aggregate": round(total / r / 1e6, 1),
            "roofline": "pool GPU ingress / egress: 450 GB/s nominal (H100 SXM, NVLink 4)",
            "fraction_of_450": [round(total / w / 1e6 / 450, 3), round(total / r / 1e6 / 450, 3)],
            "verified": okall, "timing": "CUDA events around issue+sync, max over ranks"}


# --------------------------------------------------------------------------- config 5
def fp8_ring(ctx: Ctx, size_mb: int = 2048, iters: int = 2, layers: int = 32, **client_kw):
    elems = 65536                                  # 128 KB bf16 page -> 64 KB e4m3 (+ scales)
    nblk = (size_mb << 20) // (elems * 2)
    port = ctx.base_port + 60
    server = start_shard_server(ctx.local, port + ctx.rank,
                                (iters + 2) * nblk * 80 * 1024 + (256 << 20), granule_kb=16)
    ctx.barrier()
    conn = _client(ctx, port + (ctx.rank + 1) % ctx.world, **client_kw)
    src = (torch.randn(nblk * elems, device=ctx.dev) * 2).to(torch.bfloat16)
    dst = torch.zeros_like(src)
    conn.register_mr(src)
    conn.register_mr(dst)
    per = nblk // layers
    offs = np.arange(nblk, dtype=np.int64) * elems
    nbytes = conn.fp8_page_bytes(elems)
    tw, tr = DevTimer(), DevTimer()
    for it in range(iters + 1):
        tag = uuid.uuid4().hex[:12]
        keys = [f"{tag}-{i}" for i in range(nblk)]
        remote = conn.allocate_rdma(keys, nbytes)
        blocks = list(zip(keys, offs.tolist()))
        torch.cuda.synchronize()
        ctx.barrier()
        if it:
            tw.start()
        for l in range(layers):
            s = slice(l * per, (l + 1) * per)
            conn.rdma_write_cache_fp8(src, offs[s], elems, remote[s])
        conn.sync()
        if it:
            tw.stop()
            tr.start()
        for l in range(layers):
            s = slice(l * per, (l + 1) * per)
            conn.read_cache_fp8(dst, blocks[s], elems)
        conn.sync()
        if it:
            tr.stop()
        ctx.barrier()
    err = (dst.float() - src.float()).abs().max().item() / src.float().abs().max().item()
    w, r, err = ctx.allmax(tw.ms), ctx.allmax(tr.ms), ctx.allmax(err)
    conn.close()
    ctx.barrier()
    server.stop()
    fp8_bytes = ctx.world * nblk * nbytes * iters
    bf16_bytes = ctx.world * nblk * elems * 2 * iters
    return {"what": "fp8 KV path, ring over N GPUs: cast fused into the write, dequantising "
                    "gather fused into the read", "fp8_block_kb": nbytes / 1024,
            "pages_per_call": per, "calls_per_phase": layers,
            "write_GBps_fp8_bytes": round(fp8_bytes / w / 1e6, 1),
            "read_GBps_fp8_bytes": round(fp8_bytes / r / 1e6, 1),
            "write_GBps_bf16_equiv": round(bf16_bytes / w / 1e6, 1),
            "read_GBps_bf16_equiv": round(bf16_bytes / r / 1e6, 1),
            "fraction_of_450_on_fp8_bytes": [round(fp8_bytes / w / 1e6 / ctx.world / 450, 3),
                                             round(fp8_bytes / r / 1e6 / ctx.world / 450, 3)],
            "max_rel_err_vs_bf16": round(err, 4),
            "timing": "CUDA events around issue+sync, max over ranks"}


# --------------------------------------------------------------------------- gathered blocks
def gather(ctx: Ctx, pages: int = 2048, layers: int = 32, iters: int = 2):
    """Llama-3-8B KV in vLLM's flash layout, one [2, pages, block_size, 8, 128] bf16 tensor per
    layer.  (a) per-layer keys: one rdma_write_cache / read_cache per layer and K|V, i.e.
    2 * layers calls and keys per page; (b) one key per page holding every layer's K and V:
    one rdma_write_cache_gather and one read_cache_scatter.  block_size 16 makes 32 KB parts
    (the ld/st kernels), 32 makes 64 KB parts (the TMA pipeline): one workload on each side of
    kPipeMinBytes.  Pages are written from one permutation of the page ids and read into
    another.  The pool sits on the ring peer (local HBM with one process), as in fp8_ring."""
    port = ctx.base_port + 80
    heads, dim = 8, 128
    out = {"model": "llama-3-8b", "layers": layers, "pages": pages,
           "pool": "NVLink (ring peer)" if ctx.world > 1 else "local HBM",
           "timing": "CUDA events around issue+sync, max over ranks; host_us = stats() "
                     "ns_build + ns_launch per phase"}
    for block_size in (16, 32):
        page = block_size * heads * dim                  # elements of one K (or V) page
        part_bytes = page * 2
        block_bytes = 2 * layers * part_bytes
        server = start_shard_server(ctx.local, port + ctx.rank, pages * block_bytes + (512 << 20),
                                    granule_kb=16)
        ctx.barrier()
        conn = _client(ctx, port + (ctx.rank + 1) % ctx.world)
        src = [torch.randn(2, pages, block_size, heads, dim, device=ctx.dev).to(torch.bfloat16)
               for _ in range(layers)]
        dst = [torch.empty_like(t) for t in src]
        for t in src + dst:
            conn.register_mr(t)
        g = torch.Generator().manual_seed(block_size)
        wp = torch.randperm(pages, generator=g).numpy().astype(np.int64)
        rp = torch.randperm(pages, generator=g).numpy().astype(np.int64)
        wpt, rpt = torch.from_numpy(wp).to(ctx.dev), torch.from_numpy(rp).to(ctx.dev)
        res = {"part_kb": part_bytes >> 10,
               "path": "TMA pipeline" if part_bytes >= 64 << 10 else "ld/st"}
        for arm in ("per_layer", "gathered"):
            tw, tr = DevTimer(), DevTimer()
            host_ns = [0, 0]
            launches = [0, 0]
            ok = True
            for it in range(iters + 1):
                tag = uuid.uuid4().hex[:12]
                for t in dst:
                    t.zero_()
                if arm == "per_layer":
                    keys = [[f"{tag}/L{l}/{'KV'[kv]}/{p}" for p in range(pages)]
                            for l in range(layers) for kv in (0, 1)]
                    remote = [conn.allocate_rdma(k, part_bytes) for k in keys]
                else:
                    keys = [f"{tag}/all/{p}" for p in range(pages)]
                    remote = conn.allocate_rdma(keys, block_bytes)
                    sparts = [(t, b) for t in src for b in (0, pages * page)]
                    dparts = [(t, b) for t in dst for b in (0, pages * page)]
                torch.cuda.synchronize()
                ctx.barrier()
                for phase, timer in ((0, tw), (1, tr)):
                    s0 = conn.stats()
                    timer.start()
                    if arm == "per_layer":
                        for i in range(2 * layers):
                            l, kv = divmod(i, 2)
                            if phase == 0:
                                conn.rdma_write_cache(src[l], kv * pages * page + wp * page, page,
                                                      remote[i])
                            else:
                                conn.read_cache(dst[l], (keys[i], kv * pages * page + rp * page),
                                                page)
                    elif phase == 0:
                        conn.rdma_write_cache_gather(sparts, wp * page, page, remote)
                    else:
                        conn.read_cache_scatter(dparts, (keys, rp * page), page)
                    conn.sync()
                    if it:
                        timer.stop()
                        s1 = conn.stats()
                        host_ns[phase] += (s1["ns_build"] - s0["ns_build"]
                                           + s1["ns_launch"] - s0["ns_launch"])
                        launches[phase] += s1["kernel_launches"] - s0["kernel_launches"]
                    else:
                        timer.ms = 0.0
                ctx.barrier()
                ok = ok and all(torch.equal(d[:, rpt], s[:, wpt]) for s, d in zip(src, dst))
                server.purge()  # the next iteration's keys take the space
                ctx.barrier()
            w, r = ctx.allmax(tw.ms), ctx.allmax(tr.ms)
            nbytes = ctx.world * pages * block_bytes * iters
            res[arm] = {"keys_per_phase": pages * (2 * layers if arm == "per_layer" else 1),
                        "calls_per_phase": 2 * layers if arm == "per_layer" else 1,
                        "kernel_launches_write": launches[0] // iters,
                        "kernel_launches_read": launches[1] // iters,
                        "write_read_GBps": round(2 * nbytes / (w + r) / 1e6, 1),
                        "write_GBps": round(nbytes / w / 1e6, 1),
                        "read_GBps": round(nbytes / r / 1e6, 1),
                        "host_us_write": round(host_ns[0] / iters / 1e3, 1),
                        "host_us_read": round(host_ns[1] / iters / 1e3, 1),
                        "pages_match": bool(ctx.allmin(float(ok)))}
        out[f"block_size_{block_size}"] = res
        conn.close()
        del src, dst
        ctx.barrier()
        server.stop()
    return out


# --------------------------------------------------------------------------- config 4
def nvls_bcast(ctx: Ctx, blocks_n: int = 512, iters: int = 3, match_keys: int = 4096):
    """1 writer -> N replicas through the STORE API: rank 0 hosts a server with an
    NVLS-replicated region on every GPU; rank 0's client allocates replicated blocks and
    writes them once (multimem.st through the multicast mapping, in-band commit); every
    rank's client - separate processes, handles over the fd side channel - then reads its
    LOCAL replica.  Also: get_match_last_index on the device index vs the server 'M' op."""
    bs = 1 << 20
    out = {"what": "prefix broadcast 1 writer -> all GPUs, NVLS multicast, 1 MB blocks, store API"}
    if not nvls_available(ctx.local):
        out["unavailable"] = "NVLS multicast not supported on this box"
        return out
    port = ctx.base_port + 70
    server = None
    if ctx.rank == 0:
        cfg = native.ServerConfig()
        cfg.service_port = port
        cfg.host = "127.0.0.1"
        cfg.pool_backend = "hbm"
        cfg.pool_devices = [ctx.local]
        cfg.prealloc_bytes = 512 << 20
        cfg.minimal_allocate_size = 64
        cfg.replica_bytes = (iters + 2) * blocks_n * bs + (64 << 20)
        cfg.replica_devices = list(range(ctx.world))
        cfg.log_level = "warning"
        server = native.Server(cfg)
        server.start()
    ctx.barrier()
    conn = _client(ctx, port)
    elems = bs // 2
    src = torch.randn(blocks_n * elems, device=ctx.dev).to(torch.bfloat16) if ctx.rank == 0 else None
    dst = torch.zeros(blocks_n * elems, device=ctx.dev, dtype=torch.bfloat16)
    conn.register_mr(dst)
    offs = np.arange(blocks_n, dtype=np.int64) * elems
    tw, tr = DevTimer(), DevTimer()
    ok = True
    for it in range(iters + 1):
        tag = [uuid.uuid4().hex[:12]]
        if ctx.dist is not None:
            ctx.dist.broadcast_object_list(tag, src=0)
        keys = [f"{tag[0]}-{i}" for i in range(blocks_n)]
        blocks = list(zip(keys, offs.tolist()))
        torch.cuda.synchronize()
        ctx.barrier()
        if ctx.rank == 0:
            remote = conn.allocate_rdma(keys, bs, replicated=True)
            if it:
                tw.start()
            conn.rdma_write_cache(src, offs, elems, remote)
            conn.sync()
            if it:
                tw.stop()
        ctx.barrier()
        if it:
            tr.start()
        conn.read_cache(dst, blocks, elems)
        conn.sync()
        if it:
            tr.stop()
        ctx.barrier()
    # verify: every rank's dst equals rank 0's pages
    chk = dst.float().sum().item()
    ref = [src.float().sum().item() if ctx.rank == 0 else 0.0]
    if ctx.dist is not None:
        ctx.dist.broadcast_object_list(ref, src=0)
    ok = abs(chk - ref[0]) <= 1e-3 * max(1.0, abs(ref[0]))
    w = ctx.allmax(tw.ms)          # only rank 0 wrote
    r = ctx.allmax(tr.ms)
    total = blocks_n * bs * iters
    out.update({
        "writer_egress_GBps": round(total / w / 1e6, 1),
        "delivered_GBps": round((ctx.world - 1) * total / w / 1e6, 1),
        "fraction_of_450_egress": round(total / w / 1e6 / 450, 3),
        "readers_local_replica_GBps_aggregate": round(ctx.world * total / r / 1e6, 1),
        "verified": ctx.allsum(0.0 if ok else 1.0) == 0.0})
    # get_match_last_index: device kernel vs server op, same keys (half present)
    if ctx.rank == 0:
        present = [f"{tag[0]}-{i}" for i in range(min(blocks_n, match_keys // 2))]
        probe = present + [f"absent-{i}" for i in range(match_keys - len(present))]
        host_conn = ist.InfinityConnection(ist.ClientConfig(
            host_addr="127.0.0.1", service_port=port, connection_type=ist.TYPE_RDMA,
            device=ctx.local, device_lookup=False, log_level="warning"))
        host_conn.connect()
        res = {}
        for name, c in (("device_kernel", conn), ("server_op", host_conn)):
            ts = []
            for _ in range(30):
                t0 = time.perf_counter()
                m = c.get_match_last_index(probe)
                ts.append((time.perf_counter() - t0) * 1e6)
            ts.sort()
            res[name] = {"result": m, "p50_us": round(ts[len(ts) // 2], 1), "p99_us": round(ts[-1], 1)}
        res["keys"] = len(probe)
        res["expected"] = len(present) - 1
        out["get_match_last_index"] = res
        host_conn.close()
    conn.close()
    ctx.barrier()
    if server is not None:
        server.stop()
    return out


# --------------------------------------------------------------------------- CLI
def _standalone_ctx():
    rank, world = int(os.environ.get("RANK", "0")), int(os.environ.get("WORLD_SIZE", "1"))
    local = int(os.environ.get("LOCAL_RANK", "0"))
    torch.cuda.set_device(local)
    dev = torch.device("cuda", local)
    dist = None
    if world > 1:
        import torch.distributed as dist

        dist.init_process_group("nccl", device_id=dev)

    def red(x, op):
        if dist is None:
            return x
        t = torch.tensor([x], dtype=torch.float64, device=dev)
        dist.all_reduce(t, op=getattr(dist.ReduceOp, op))
        return float(t.item())

    def barrier():
        if dist is not None:
            dist.barrier()
        torch.cuda.synchronize()

    return Ctx(dist, rank, world, local, dev,
               25000 + int(os.environ.get("MASTER_PORT", "0")) % 2000, barrier,
               lambda x: red(x, "MAX"), lambda x: red(x, "SUM"), lambda x: red(x, "MIN"))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("config", choices=["fanin", "bcast", "fp8", "gather", "latency", "baselines"])
    ap.add_argument("--max-ctas", type=int, default=0, help="fp8: grid cap of the client's kernels")
    ap.add_argument("--layers", type=int, default=32,
                    help="fp8: calls per phase (pages per call = 16384 / layers)")
    a = ap.parse_args()
    ctx = _standalone_ctx()
    if a.config == "fanin":
        res = fanin(ctx)
    elif a.config == "fp8":
        res = fp8_ring(ctx, layers=a.layers, **({"max_ctas": a.max_ctas} if a.max_ctas else {}))
    elif a.config == "bcast":
        res = nvls_bcast(ctx)
    elif a.config == "gather":
        res = gather(ctx)
    elif a.config == "baselines":
        res = baselines(ctx, 128 << 10)
    else:
        srv = start_shard_server(ctx.local, ctx.base_port + ctx.rank, 4 << 30, granule_kb=16)
        ctx.barrier()
        res = latency(ctx, ctx.base_port + (ctx.rank + 1) % ctx.world)
        ctx.barrier()
        srv.stop()
    if ctx.rank == 0:
        print(json.dumps({a.config: res}))
        os.makedirs("gpurun_out", exist_ok=True)
        with open(f"gpurun_out/config_{a.config}_n{ctx.world}.json", "w") as f:
            json.dump(res, f, indent=1)
    if ctx.dist is not None:
        ctx.dist.destroy_process_group()


if __name__ == "__main__":
    main()
