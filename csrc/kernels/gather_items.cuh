// The item walks of the gathered ld/st movers (GatherLaunch): which item of which block a CTA
// moves next, and everything around the copy that does not depend on the part's shape -
// descriptor prefetch, miss counting, group release and the write's control warp.  Each
// kernel passes the copy of one item as a body (kv_copy.cu: kv_scatter_ldst_kernel,
// kv_gather_ldst_kernel; kv_fp8.cu: kv_read_fp8_scatter_kernel).  The fp8 writes walk their
// pages in kv_fp8.cu's write_fp8, which every fp8 write shape shares through its load policy.
#pragma once

#include <cstring>
#include <type_traits>

#include "common.cuh"
#include "copy_span.cuh"
#include "kernels.h"
#include "launch_plan.h"
#include "publish.cuh"

namespace istore::kernels {

// How a gathered launch lays out each part (GatherLaunch::rows: PartRows).
enum class PartShape { kWhole, kRows, kSlices, kPieces };

// Calls go with the launch's shape as a compile-time constant.  Writes have no sliced body:
// their row body takes any number of slices.
template <bool WRITE, typename Go>
cudaError_t with_shape(const GatherLaunch& a, Go&& go) {
    using S = PartShape;
    if (!a.rows.rows) return go(std::integral_constant<S, S::kWhole>{});
    if (a.rows.pieces > 1) return go(std::integral_constant<S, S::kPieces>{});
    if constexpr (!WRITE)
        if (a.rows.slices > 1) return go(std::integral_constant<S, S::kSlices>{});
    return go(std::integral_constant<S, S::kRows>{});
}

// Calls go with the plan's ld/st vector width (1, 16 or 32) as a compile-time constant.
template <typename Go>
cudaError_t with_vec(Kernel k, Go&& go) {
    switch (k) {
        case Kernel::kLdSt1:
            return go(std::integral_constant<int, 1>{});
        case Kernel::kLdSt32:
            return go(std::integral_constant<int, 32>{});
        default:
            return go(std::integral_constant<int, 16>{});
    }
}

inline GatherParts parts_of(const GatherLaunch& a) {
    GatherParts parts;
    std::memcpy(parts.base, a.part_base, size_t(a.nparts) * sizeof(uint64_t));
    return parts;
}

inline GroupRelease release_of(const GatherLaunch& a) {
    return GroupRelease{a.group_flags, a.group_counters, a.group_seq, a.group_parts};
}

// The read walk.  Item = chunk c of part s of block b, numbered (b * nparts + s) * cpp + c, or,
// LAYERED, group-major with rel.gp parts per group (launch_plan.h: layered_item), group g
// released by leave_group (publish.cuh) when this CTA's stream leaves it.  The next item's
// descriptor is loaded before this item is copied: descriptors may sit in host memory.  A
// missing block (src == 0) counts once in status[kStatMiss], on its first item (group 0, part
// 0, chunk 0), and its parts are left untouched; its items still count as arrivals.
// body(desc, item) copies every item of a found block on the CTA's kLdStThreads threads.
template <bool LAYERED, typename Body>
__device__ __forceinline__ void scatter_items(const CopyDesc* __restrict__ descs, uint32_t n,
                                              uint32_t nparts, uint32_t cpp, uint32_t* status,
                                              const GroupRelease& rel, Body&& body) {
    const uint32_t cpb = nparts * cpp;
    const uint32_t group_items = n * rel.gp * cpp;
    const uint32_t total = n * cpb;
    const auto item_at = [&](uint32_t item) {
        if constexpr (LAYERED) {
            return layered_item(item, n, rel.gp, cpp);
        } else {
            const uint32_t in_block = item % cpb;
            return LayeredItem{0, item / cpb, in_block / cpp, in_block % cpp};
        }
    };
    const auto block_of = [&](uint32_t item) {
        if constexpr (LAYERED)
            return layered_item(item, n, rel.gp, cpp).block;
        else
            return item / cpb;
    };
    uint32_t item = blockIdx.x;
    CopyDesc next = item < total ? descs[block_of(item)] : CopyDesc{0, 0};
    for (; item < total; item += gridDim.x) {
        const CopyDesc d = next;
        const uint32_t nxt = item + gridDim.x;
        if (nxt < total) next = descs[block_of(nxt)];
        const LayeredItem it = item_at(item);
        if (d.src != 0)
            body(d, it);
        else if (threadIdx.x == 0 && it.part == 0 && it.chunk == 0 && status)
            atomicAdd(status + kStatMiss, 1u);
        if constexpr (LAYERED) {
            if (nxt >= total || nxt / group_items != it.group) {
                const uint32_t lo = it.group * group_items;
                leave_group(rel, it.group, cta_items(lo, lo + group_items, blockIdx.x, gridDim.x),
                            group_items, kLdStThreads);
            }
        }
    }
}

// The bf16 write walk.  Item = chunk c of part s of block b, numbered (b * nparts + s) * cpp + c
// (GatherLaunch), each storing bytes [off, off + len) of stored part s; the next item's
// descriptor is prefetched.  Threads [0, kLdStThreads) call body(desc, block, s, off, len);
// warp 8 is the control warp (in-band commit, or a layered writer's LayerCommit), which counts
// nparts * cpp arrivals per block.
template <typename Body>
__device__ __forceinline__ void gather_items(const CopyDesc* __restrict__ descs, uint32_t n,
                                             uint32_t nparts, uint32_t part_bytes, uint32_t chunk,
                                             uint32_t cpp, const Publish& pub,
                                             const LayerCommit& lc, Body&& body) {
    const uint32_t cpb = nparts * cpp;  // items per block: what the commit counter counts
    const uint32_t total = n * cpb;
    if (threadIdx.x >= kLdStThreads) {
        if (!pub.recs) return;
        const uint32_t count = blockIdx.x < total ? (total - blockIdx.x + gridDim.x - 1) / gridDim.x : 0;
        gather_control_warp(pub, lc, threadIdx.x - kLdStThreads, blockIdx.x, count, gridDim.x,
                            cpb, nparts, kLdStThreads + 32);
        return;
    }
    uint32_t item = blockIdx.x;
    CopyDesc next = item < total ? descs[item / cpb] : CopyDesc{0, 0};
    for (; item < total; item += gridDim.x) {
        const CopyDesc d = next;
        const uint32_t nxt = item + gridDim.x;
        if (nxt < total) next = descs[nxt / cpb];
        const uint32_t in_block = item % cpb;
        const uint32_t off = (in_block % cpp) * chunk;
        body(d, item / cpb, in_block / cpp, off, min(chunk, part_bytes - off));
    }
    if (pub.recs) ctrl_barrier_arrive(kLdStThreads + 32);
}

}  // namespace istore::kernels
