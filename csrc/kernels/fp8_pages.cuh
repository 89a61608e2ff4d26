// Which fp8 page a work item of the fp8 kernels (kv_fp8.cu, kv_fp8_pipe.cu) moves.  Both walk
// pages: page v of a launch is {bf16 page, fp8 page} for a write, {fp8 page or 0 = miss, bf16
// page} for a read, and its chunks are the work items.
//   OnePage       page v is descs[v] (launch_kv_write_fp8 / launch_kv_read_fp8).
//   BlockParts    page v is part s = v % nparts of gathered block v / nparts
//                 (launch_kv_gather_fp8), numbered as GatherLaunch numbers them:
//                   write  part_base[s] + local offset  ->  block + (first_part + s) * stride
//                   read   block + (first_part + s) * stride  ->  part_base[s] + local offset
//                 stride = fp8_gather_bytes(1, elems).
// head(v) is true on the first page of a block: a read counts a missing block there, once.
// `nparts` pages make a block, which is what the in-band commit counts; commit() runs the
// write's control warp (publish.cuh), layered when a gathered write carries a writer's state.
#pragma once

#include "kernels.h"
#include "publish.cuh"

namespace istore::kernels {

struct OnePage {
    static constexpr uint32_t nparts = 1;
    __device__ __forceinline__ CopyDesc at(const CopyDesc* __restrict__ descs, uint32_t v) const {
        return descs[v];
    }
    __device__ __forceinline__ bool head(uint32_t) const { return true; }
    __device__ __forceinline__ void commit(const Publish& pub, uint32_t lane, uint32_t first,
                                           uint32_t count, uint32_t stride, uint32_t cpb,
                                           uint32_t threads) const {
        control_warp(pub, lane, first, count, stride, cpb, threads);
    }
};

template <bool WRITE>
struct BlockParts {
    const GatherParts* parts;  // the kernel's __grid_constant__ parameter
    uint32_t nparts;
    uint32_t first_part;
    uint64_t stride;
    LayerCommit layer = {};  // writes
    __device__ __forceinline__ CopyDesc at(const CopyDesc* __restrict__ descs, uint32_t v) const {
        const uint32_t s = v % nparts;
        const CopyDesc b = descs[v / nparts];
        if constexpr (WRITE) return CopyDesc{parts->base[s] + b.src, b.dst + (first_part + s) * stride};
        return CopyDesc{b.src ? b.src + (first_part + s) * stride : 0, parts->base[s] + b.dst};
    }
    __device__ __forceinline__ bool head(uint32_t v) const { return v % nparts == 0; }
    __device__ __forceinline__ void commit(const Publish& pub, uint32_t lane, uint32_t first,
                                           uint32_t count, uint32_t stride_, uint32_t cpb,
                                           uint32_t threads) const {
        gather_control_warp(pub, layer, lane, first, count, stride_, cpb, nparts, threads);
    }
};

}  // namespace istore::kernels
