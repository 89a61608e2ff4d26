#!/usr/bin/env python
"""Round-2 kernel lab (1 or 2 GPUs, device-timed with CUDA events, 1 GiB working sets):

  ce      : copy-engine rooflines - cudaMemcpyPeerAsync GPU0->GPU1 alone and both directions
            at once (the independent NVLink roofline bench.py quotes), local cudaMemcpy
  geom    : TMA pipeline (kv_pipe) ring geometry x grid at 128 KB blocks, local / push / pull
  sizes   : block-size sweep, TMA pipeline vs ld/st, local / push / pull
  bidir   : both GPUs pushing / pulling at once with the kernels (ring topology of bench.py)
  mcast   : cluster multicast read (1 fetch, K destinations) vs K separate copies

    python bench/r2_lab.py [--only ce,geom,...] [--out gpurun_out/r2_lab.json]
"""
import argparse
import json
import os
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from infinistore_b200 import _infinistore as native  # noqa: E402
from infinistore_b200 import ops  # noqa: E402

TOTAL = 1 << 30


def ev_time(fn, dev, iters=5, warm=2):
    with torch.cuda.device(dev):
        for _ in range(warm):
            fn()
        torch.cuda.synchronize(dev)
        ts = []
        for _ in range(iters):
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            fn()
            e1.record()
            e1.synchronize()
            ts.append(e0.elapsed_time(e1))
    ts.sort()
    return ts[len(ts) // 2]


def gbps(ms, nbytes=TOTAL):
    return round(nbytes / ms / 1e6, 1)


def buffers(dev):
    src = torch.empty(TOTAL, dtype=torch.uint8, device=dev).random_(0, 255)
    dst = torch.empty(TOTAL, dtype=torch.uint8, device=dev)
    return src, dst


def descs_for(src, dst, bs, run_dev, shuffle=True):
    n = TOTAL // bs
    perm = torch.randperm(n).tolist() if shuffle else list(range(n))
    return ops.make_descs([src.data_ptr() + i * bs for i in range(n)],
                          [dst.data_ptr() + perm[i] * bs for i in range(n)], run_dev)


def lab_ce(out, two):
    s0, d0 = buffers("cuda:0")
    out["ce_local_GBps"] = gbps(ev_time(lambda: d0.copy_(s0, non_blocking=True), 0))
    if not two:
        return
    s1, d1 = buffers("cuda:1")
    out["ce_push_uni_GBps"] = gbps(ev_time(lambda: d1.copy_(s0, non_blocking=True), 0))
    # a copy issued from the destination device's stream (pull semantics for the CE)
    out["ce_pull_uni_GBps"] = gbps(ev_time(lambda: d0.copy_(s1, non_blocking=True), 0))
    # both directions at once: GPU0 -> GPU1 on a GPU0 stream, GPU1 -> GPU0 on a GPU1 stream
    st0 = torch.cuda.Stream(device=0)
    st1 = torch.cuda.Stream(device=1)
    best = {0: [], 1: []}
    for it in range(6):
        torch.cuda.synchronize(0)
        torch.cuda.synchronize(1)
        evs = {}
        for d, st, (a, b) in ((0, st0, (d1, s0)), (1, st1, (d0, s1))):
            with torch.cuda.device(d), torch.cuda.stream(st):
                e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                e0.record()
                for _ in range(4):
                    a.copy_(b, non_blocking=True)
                e1.record()
                evs[d] = (e0, e1)
        for d in (0, 1):
            evs[d][1].synchronize()
            if it >= 2:
                best[d].append(evs[d][0].elapsed_time(evs[d][1]) / 4)
    out["ce_bidir_GBps"] = {d: gbps(sorted(best[d])[len(best[d]) // 2]) for d in (0, 1)}
    print("ce", {k: v for k, v in out.items() if k.startswith("ce_")}, flush=True)


def paths(two):
    s0, d0 = buffers("cuda:0")
    p = {"local": (s0, d0)}
    if two:
        s1, d1 = buffers("cuda:1")
        p["push"] = (s0, d1)   # local -> peer (write_cache)
        p["pull"] = (s1, d0)   # peer -> local (read_cache)
    return p


def lab_geom(out, two):
    rows = []
    bs = 128 << 10
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    for name, (src, dst) in paths(two).items():
        descs = descs_for(src, dst, bs, "cuda:0")
        for stage_kb, ring_kb in ((8, 64), (16, 64), (16, 128), (32, 128), (16, 192), (32, 192)):
            for ctas in ((16, 32, sms // 2, sms) if name != "local" else (sms, 2 * sms)):
                if ring_kb > 110 and ctas > sms:
                    continue
                ms = ev_time(lambda: ops.kv_copy(descs, bs, variant="tma", max_ctas=ctas,
                                                 stage_bytes=stage_kb << 10,
                                                 ring_bytes=ring_kb << 10), 0)
                rows.append({"path": name, "stage_kb": stage_kb, "ring_kb": ring_kb, "ctas": ctas,
                             "GBps": gbps(ms)})
                print("geom", rows[-1], flush=True)
        ms = ev_time(lambda: ops.kv_copy(descs, bs, variant="ldst256"), 0)
        rows.append({"path": name, "variant": "ldst256", "GBps": gbps(ms)})
        print("geom", rows[-1], flush=True)
    out["geom"] = rows


def lab_sizes(out, two):
    rows = []
    for name, (src, dst) in paths(two).items():
        for bs in (4096, 8192, 16384, 65536, 131072, 1 << 20, 16 << 20):
            descs = descs_for(src, dst, bs, "cuda:0")
            row = {"path": name, "block_kb": bs >> 10}
            for v in ("tma", "ldst256"):
                row[v] = gbps(ev_time(lambda: ops.kv_copy(descs, bs, variant=v), 0))
            rows.append(row)
            print("sizes", row, flush=True)
    out["sizes"] = rows


def lab_bidir(out, two):
    if not two:
        return
    native.enable_peer_access(0, 1)
    native.enable_peer_access(1, 0)
    bs = 128 << 10
    buf = {d: buffers(f"cuda:{d}") for d in (0, 1)}
    push = {d: descs_for(buf[d][0], buf[1 - d][1], bs, f"cuda:{d}", shuffle=False) for d in (0, 1)}
    pull = {d: descs_for(buf[1 - d][0], buf[d][1], bs, f"cuda:{d}", shuffle=False) for d in (0, 1)}
    rows = []
    for variant in ("tma", "ldst256"):
        for name, table in (("push", push), ("pull", pull)):
            res = {}
            for it in range(5):
                for d in (0, 1):
                    torch.cuda.synchronize(d)
                evs = {}
                for d in (0, 1):
                    with torch.cuda.device(d):
                        e0 = torch.cuda.Event(enable_timing=True)
                        e1 = torch.cuda.Event(enable_timing=True)
                        e0.record()
                        for _ in range(4):
                            ops.kv_copy(table[d], bs, variant=variant)
                        e1.record()
                        evs[d] = (e0, e1)
                for d in (0, 1):
                    evs[d][1].synchronize()
                    res.setdefault(d, []).append(evs[d][0].elapsed_time(evs[d][1]) / 4)
            row = {"op": name, "variant": variant,
                   **{f"gpu{d}_GBps": gbps(sorted(res[d][1:])[len(res[d][1:]) // 2]) for d in (0, 1)}}
            rows.append(row)
            print("bidir", row, flush=True)
    out["bidir"] = rows


def lab_mcast(out, two):
    rows = []
    bs = 128 << 10
    n = (256 << 20) // bs  # 256 MiB of source pages
    src_dev = "cuda:1" if two else "cuda:0"
    src = torch.empty(n * bs, dtype=torch.uint8, device=src_dev).random_(0, 255)
    for K in (2, 4):
        dsts = [torch.zeros(n * bs, dtype=torch.uint8, device="cuda:0") for _ in range(K)]
        descs = ops.make_descs([src.data_ptr() + i * bs for i in range(n)],
                               [dsts[0].data_ptr() + i * bs for i in range(n)], "cuda:0")
        per = [ops.make_descs([src.data_ptr() + i * bs for i in range(n)],
                              [d.data_ptr() + i * bs for i in range(n)], "cuda:0") for d in dsts]
        deltas = [d.data_ptr() - dsts[0].data_ptr() for d in dsts]
        if two:  # multicast bulk loads from a peer-mapped source once wedged a GPU: never again
            ms_c = float("nan")
            ops.kv_copy(descs, bs, variant="tma", fan_deltas=deltas)
        else:
            ms_c = ev_time(lambda: ops.kv_copy_multicast(descs, bs, deltas), 0)
        torch.cuda.synchronize()
        ok = all(torch.equal(d, src.to("cuda:0")) for d in dsts)

        def separate():
            for p in per:
                ops.kv_copy(p, bs, variant="tma")
        ms_s = ev_time(separate, 0)
        ms_f = ev_time(lambda: ops.kv_copy(descs, bs, variant="tma", fan_deltas=deltas), 0)
        delivered = K * n * bs
        rows.append({"K": K, "source": "peer (NVLink)" if two else "local HBM", "verified": ok,
                     "cluster_ms": round(ms_c, 4), "separate_ms": round(ms_s, 4),
                     "fanout_ms": round(ms_f, 4),
                     "cluster_delivered_GBps": gbps(ms_c, delivered),
                     "fanout_delivered_GBps": gbps(ms_f, delivered),
                     "separate_delivered_GBps": gbps(ms_s, delivered),
                     "cluster_speedup": round(ms_s / ms_c, 2),
                     "fanout_speedup": round(ms_s / ms_f, 2)})
        print("mcast", rows[-1], flush=True)
    out["mcast"] = rows


def lab_fp8(out, two):
    """fp8 KV path kernels: GB/s of fp8 payload bytes (the bytes that cross the fabric)."""
    rows = []
    elems, pages = 65536, 2048  # 128 KB bf16 pages -> 64 KB e4m3 + 2 KB scales
    bb = ops.fp8_block_bytes(elems)
    stride = (bb + 255) // 256 * 256
    x = (torch.randn(pages, elems, device="cuda:0") * 3).to(torch.bfloat16)
    out_t = torch.zeros_like(x)
    for name, pool_dev in (("local", "cuda:0"),) + ((("nvlink", "cuda:1"),) if two else ()):
        pool = torch.zeros(pages, stride, dtype=torch.uint8, device=pool_dev)
        wd = ops.make_descs([x[i].data_ptr() for i in range(pages)],
                            [pool[i].data_ptr() for i in range(pages)], "cuda:0")
        rd = ops.make_descs([pool[i].data_ptr() for i in range(pages)],
                            [out_t[i].data_ptr() for i in range(pages)], "cuda:0")
        row = {"path": name}
        for v in ("auto", "pipe4", "ldst"):
            row["write_" + v] = gbps(ev_time(lambda: ops.kv_write_fp8(wd, elems, variant=v), 0), pages * bb)
            row["read_" + v] = gbps(ev_time(lambda: ops.kv_read_fp8(rd, elems, variant=v), 0), pages * bb)
        rows.append(row)
        print("fp8", row, flush=True)
    out["fp8"] = rows


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--only", default="ce,geom,sizes,bidir,mcast,fp8")
    ap.add_argument("--out", default="gpurun_out/r2_lab.json")
    a = ap.parse_args()
    two = torch.cuda.device_count() >= 2
    if two:
        assert native.enable_peer_access(0, 1) and native.enable_peer_access(1, 0)
    out = {"gpu": torch.cuda.get_device_name(0), "gpus": torch.cuda.device_count()}
    for name in a.only.split(","):
        globals()["lab_" + name](out, two)
        torch.cuda.empty_cache()
        os.makedirs(os.path.dirname(a.out) or ".", exist_ok=True)
        with open(a.out, "w") as f:
            json.dump(out, f, indent=1)


if __name__ == "__main__":
    main()
