#!/usr/bin/env python
"""Device-timed sweep of the kv_copy kernel: variant x block size x grid, local and peer.

CUDA events on the launching stream, >= 3 warm-up launches, working set per launch larger
than L2 (default 1 GiB src + 1 GiB dst), GB/s = payload bytes / time (each payload byte is
read once and written once).  Writes one JSON document to gpurun_out/ and prints a table.

    python bench/sweep_copy.py [--peer] [--out gpurun_out/sweep_copy.json]
"""
import argparse
import json
import os
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from infinistore_b200 import _infinistore as native  # noqa: E402
from infinistore_b200 import ops  # noqa: E402


def time_kernel(fn, dev, iters=10, warm=3):
    for _ in range(warm):
        fn()
    torch.cuda.synchronize(dev)
    ts = []
    for _ in range(iters):
        e0 = torch.cuda.Event(enable_timing=True)
        e1 = torch.cuda.Event(enable_timing=True)
        e0.record(torch.cuda.current_stream(dev))
        fn()
        e1.record(torch.cuda.current_stream(dev))
        e1.synchronize()
        ts.append(e0.elapsed_time(e1))
    ts.sort()
    return ts[len(ts) // 2], ts[0]


def sweep(src_dev, dst_dev, run_dev, total_bytes, sizes, variants, grids, label):
    rows = []
    src = torch.empty(total_bytes, dtype=torch.uint8, device=src_dev)
    dst = torch.empty(total_bytes, dtype=torch.uint8, device=dst_dev)
    src.random_(0, 255)
    for bs in sizes:
        n = total_bytes // bs
        # shuffled page order on the destination side: a paged KV cache is not contiguous
        perm = torch.randperm(n).tolist()
        descs = ops.make_descs([src.data_ptr() + i * bs for i in range(n)],
                               [dst.data_ptr() + perm[i] * bs for i in range(n)], run_dev)
        for v in variants:
            for g in grids:
                with torch.cuda.device(run_dev):
                    med, best = time_kernel(lambda: ops.kv_copy(descs, bs, variant=v, max_ctas=g),
                                            run_dev)
                rows.append({"path": label, "block": bs, "variant": v, "ctas": g,
                             "ms_median": round(med, 4), "ms_best": round(best, 4),
                             "gbps": round(total_bytes / med / 1e6, 1)})
                print(f"{label:22s} {bs >> 10:6d} KB {v:8s} ctas={g:5d} {med:8.3f} ms "
                      f"{total_bytes / med / 1e6:8.1f} GB/s", flush=True)
        # correctness spot check
        torch.cuda.synchronize()
        i = n // 2
        assert torch.equal(src[i * bs:(i + 1) * bs].cpu(), dst[perm[i] * bs:(perm[i] + 1) * bs].cpu())
    # library baseline: one cudaMemcpyAsync for the whole buffer
    with torch.cuda.device(run_dev):
        med, _ = time_kernel(lambda: dst.copy_(src, non_blocking=True), run_dev)
    rows.append({"path": label, "block": total_bytes, "variant": "cudaMemcpy", "ctas": 0,
                 "ms_median": round(med, 4), "gbps": round(total_bytes / med / 1e6, 1)})
    print(f"{label:22s} whole    cudaMemcpy            {med:8.3f} ms {total_bytes / med / 1e6:8.1f} GB/s")
    return rows


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--peer", action="store_true", help="also sweep GPU0 <-> GPU1 over NVLink")
    ap.add_argument("--total-mb", type=int, default=1024)
    ap.add_argument("--quick", action="store_true")
    ap.add_argument("--out", default="gpurun_out/sweep_copy.json")
    a = ap.parse_args()
    total = a.total_mb << 20
    sizes = [4096, 16384, 65536, 131072, 262144, 1 << 20, 16 << 20]
    variants = ["ldst", "ldst256", "tma"]
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    grids = [0, sms, 2 * sms, 4 * sms]
    if a.quick:
        sizes, grids = [4096, 131072, 1 << 20], [0, sms]
    rows = sweep("cuda:0", "cuda:0", "cuda:0", total, sizes, variants, grids, "local hbm->hbm")
    if a.peer and torch.cuda.device_count() >= 2:
        assert native.enable_peer_access(0, 1) and native.enable_peer_access(1, 0)
        rows += sweep("cuda:0", "cuda:1", "cuda:0", total, sizes, variants, grids,
                      "write push gpu0->gpu1")
        rows += sweep("cuda:1", "cuda:0", "cuda:0", total, sizes, variants, grids,
                      "read pull gpu1->gpu0")
    os.makedirs(os.path.dirname(a.out), exist_ok=True)
    with open(a.out, "w") as f:
        json.dump({"gpu": torch.cuda.get_device_name(0), "total_bytes": total, "rows": rows}, f,
                  indent=1)


if __name__ == "__main__":
    main()
