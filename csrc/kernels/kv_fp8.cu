// fp8 KV path: the quantisation is fused into the page mover.  This file holds the ld/st
// flavour (any page size that is a multiple of 128 elements); pages of a multiple of 512
// elements - every real KV layout - take the TMA-pipelined flavour in kv_fp8_pipe.cu.
//
//   kv_write_fp8 : bf16 page in the client's paged KV cache -> e4m3 payload + one fp32 scale
//                  per 128-element row (head_dim) written straight into the (peer) pool
//                  block, then the in-band commit.  Half the NVLink bytes of a bf16 write and
//                  no separate cast kernel / staging buffer.
//   kv_read_fp8  : pool block -> dequantised bf16 scattered into the destination pages.
//   kv_write_fp8_gather / kv_read_fp8_scatter : the same for gathered blocks, whose parts are
//                  fp8 pages end to end (launch_kv_gather_fp8, fp8_pages.cuh).
// The reference moves raw bytes only (dtype-agnostic, infinistore/lib.py:377-379); this is
// the "write fused with fp8 cast / read fused with gather" item of the north star.
//
// Pool block layout: [elems x e4m3][elems/128 x fp32 scale].
// A half-warp owns one 128-element row per step (lane l: elements 8l..8l+7, one 16-byte
// load), reduces |x| max with shuffles inside the half, and emits 8 bytes per lane (one
// coalesced 128-byte store per row).  Eight rows are in flight per warp to cover the
// NVLink / HBM latency.
// The row maths (amax, scale, cvt, dequant8) are fp8_row.cuh's, shared with kv_fp8_pipe.cu.
#include <cuda_bf16.h>
#include <cuda_fp16.h>

#include <cstring>

#include "common.cuh"
#include "fp8_pages.cuh"
#include "fp8_row.cuh"
#include "kernels.h"
#include "launch_plan.h"
#include "publish.cuh"

namespace istore::kernels {

namespace {

using namespace fp8row;

constexpr int kThreads = 256;
constexpr int kWarps = kThreads / 32;
constexpr uint32_t kRow = 128;                 // elements sharing a scale

__device__ __forceinline__ uint2 ld_u2(const void* p) {
    uint2 r;
    asm volatile("ld.global.L1::no_allocate.v2.u32 {%0,%1}, [%2];" : "=r"(r.x), "=r"(r.y) : "l"(p));
    return r;
}
__device__ __forceinline__ uint32_t ld_u1(const void* p) {
    uint32_t r;
    asm volatile("ld.global.L1::no_allocate.u32 %0, [%1];" : "=r"(r) : "l"(p));
    return r;
}
// A half-warp owns one 128-element row per step (lane l of the half: elements 8l..8l+7, one
// 16-byte load), so a warp instruction covers two rows; kRowPairs such steps are in flight.
constexpr int kRowPairs = 4;  // 8 rows = 2 KB of bf16 in flight per warp

__device__ __forceinline__ uint4 ld_u4(const void* p) {
    uint4 r;
    asm volatile("ld.global.L1::no_allocate.v4.u32 {%0,%1,%2,%3}, [%4];"
                 : "=r"(r.x), "=r"(r.y), "=r"(r.z), "=r"(r.w)
                 : "l"(p));
    return r;
}

// Threads [0, 256) quantise + store; warp 8 is the control warp (in-band commit).  Work item
// k is chunk k % cpp of page k / cpp (`pages`, fp8_pages.cuh); n blocks of pages.nparts pages.
template <typename Pages>
__device__ __forceinline__ void write_fp8(const CopyDesc* __restrict__ descs, uint32_t n,
                                          uint32_t elems, uint32_t chunk, uint32_t cpp,
                                          const Publish& pub, const Pages& pages) {
    const uint32_t cpb = cpp * pages.nparts;  // items per block: what the commit counts
    const uint32_t total = n * cpb;
    if (threadIdx.x >= kThreads) {
        if (!pub.recs) return;
        const uint32_t count = blockIdx.x < total ? (total - blockIdx.x + gridDim.x - 1) / gridDim.x : 0;
        pages.commit(pub, threadIdx.x - kThreads, blockIdx.x, count, gridDim.x, cpb, kThreads + 32);
        return;
    }
    const uint32_t warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const uint32_t half = lane >> 4, hl = lane & 15;
    constexpr uint32_t kStep = 2 * kRowPairs;  // rows per warp iteration
    for (uint32_t item = blockIdx.x; item < total; item += gridDim.x) {
        const CopyDesc d = pages.at(descs, item / cpp);
        const uint32_t e0 = (item % cpp) * chunk;
        const uint32_t rows = min(chunk, elems - e0) / kRow;
        const uint32_t row0 = e0 / kRow;
        const uint8_t* src = reinterpret_cast<const uint8_t*>(d.src);  // bf16 page
        uint8_t* q = reinterpret_cast<uint8_t*>(d.dst);                // e4m3 payload
        float* scales = reinterpret_cast<float*>(q + elems);
        for (uint32_t r0 = warp * kStep; r0 < rows; r0 += kWarps * kStep) {
            uint4 v[kRowPairs];
#pragma unroll
            for (int u = 0; u < kRowPairs; ++u) {
                const uint32_t r = r0 + 2 * u + half;
                if (r < rows) v[u] = ld_u4(src + (size_t(row0 + r) * kRow + hl * 8) * 2);
            }
#pragma unroll
            for (int u = 0; u < kRowPairs; ++u) {
                const uint32_t r = r0 + 2 * u + half;
                const bool live = r < rows;
                float2 f[4];
                float amax = load8(v[u], f);
                if (!live) amax = 0.f;
#pragma unroll
                for (int o = 8; o > 0; o >>= 1)  // reduce within the half-warp that owns the row
                    amax = fmaxf(amax, __shfl_xor_sync(0xffffffffu, amax, o));
                if (__any_sync(0xffffffffu, has_inf(amax))) {  // rare: a row holds +-inf
                    amax = has_inf(amax) ? drop_inf8(f) : amax;
#pragma unroll
                    for (int o = 8; o > 0; o >>= 1)
                        amax = fmaxf(amax, __shfl_xor_sync(0xffffffffu, amax, o));
                }
                if (!live) continue;
                const float scale = row_scale(amax);
                *reinterpret_cast<uint2*>(q + size_t(row0 + r) * kRow + hl * 8) =
                    quant8(f, 1.f / scale);
                if (hl == 0) scales[row0 + r] = scale;
            }
        }
    }
    if (pub.recs) ctrl_barrier_arrive(kThreads + 32);
}

__global__ void __launch_bounds__(kThreads + 32)
    kv_write_fp8_kernel(const CopyDesc* __restrict__ descs, uint32_t n, uint32_t elems,
                        uint32_t chunk, uint32_t cpb, Publish pub) {
    write_fp8(descs, n, elems, chunk, cpb, pub, OnePage{});
}

// A missing block (src == 0) counts once in status[kStatMiss]; its page is not written.
__global__ void __launch_bounds__(kThreads)
    kv_read_fp8_kernel(const CopyDesc* __restrict__ descs, uint32_t n, uint32_t elems,
                       uint32_t chunk, uint32_t cpb, uint32_t* status) {
    const uint32_t total = n * cpb;
    const uint32_t warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const uint32_t half = lane >> 4, hl = lane & 15;
    constexpr uint32_t kStep = 2 * kRowPairs;
    for (uint32_t item = blockIdx.x; item < total; item += gridDim.x) {
        const CopyDesc d = descs[item / cpb];
        if (d.src == 0) {
            if (threadIdx.x == 0 && item % cpb == 0 && status) atomicAdd(status + kStatMiss, 1u);
            continue;
        }
        const uint32_t e0 = (item % cpb) * chunk;
        const uint32_t rows = min(chunk, elems - e0) / kRow;
        const uint32_t row0 = e0 / kRow;
        const uint8_t* q = reinterpret_cast<const uint8_t*>(d.src);
        const float* scales = reinterpret_cast<const float*>(q + elems);
        uint8_t* dst = reinterpret_cast<uint8_t*>(d.dst);
        for (uint32_t r0 = warp * kStep; r0 < rows; r0 += kWarps * kStep) {
            uint2 v[kRowPairs];
            float sc[kRowPairs];
#pragma unroll
            for (int u = 0; u < kRowPairs; ++u) {
                const uint32_t r = r0 + 2 * u + half;
                if (r < rows) {
                    v[u] = ld_u2(q + size_t(row0 + r) * kRow + hl * 8);
                    sc[u] = __uint_as_float(ld_u1(scales + row0 + r));
                }
            }
#pragma unroll
            for (int u = 0; u < kRowPairs; ++u) {
                const uint32_t r = r0 + 2 * u + half;
                if (r >= rows) continue;
                *reinterpret_cast<uint4*>(dst + (size_t(row0 + r) * kRow + hl * 8) * 2) =
                    dequant8(v[u], sc[u]);
            }
        }
    }
}

// Gathered blocks (launch_kv_gather_fp8): n blocks of nparts parts, cpp items per part; the
// part bases travel in the kernel parameters, as for kv_gather_ldst.
__global__ void __launch_bounds__(kThreads + 32)
    kv_write_fp8_gather_kernel(const CopyDesc* __restrict__ descs,
                               const __grid_constant__ GatherParts parts, uint32_t n,
                               uint32_t nparts, uint32_t elems, uint32_t chunk, uint32_t cpp,
                               uint32_t first_part, uint64_t stride, Publish pub,
                               LayerCommit lc) {
    write_fp8(descs, n, elems, chunk, cpp, pub,
              BlockParts<true>{&parts, nparts, first_part, stride, lc});
}

// The layered read (GatherLaunch::group_flags): kv_gather_ldst's gather_read_layered
// (kv_copy.cu) over fp8 pages.  Item order, miss counting and the group release are the same;
// the rows of an item are dequantised as in kv_read_fp8_scatter_kernel.
__device__ __forceinline__ void read_fp8_layered(const CopyDesc* __restrict__ descs,
                                                 const BlockParts<false>& pages, uint32_t n,
                                                 uint32_t elems, uint32_t chunk, uint32_t cpp,
                                                 uint32_t* status, const GroupRelease& rel) {
    const uint32_t group_items = n * rel.gp * cpp;
    const uint32_t total = n * pages.nparts * cpp;
    const uint32_t warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const uint32_t half = lane >> 4, hl = lane & 15;
    constexpr uint32_t kStep = 2 * kRowPairs;
    for (uint32_t item = blockIdx.x; item < total; item += gridDim.x) {
        const LayeredItem it = layered_item(item, n, rel.gp, cpp);
        const CopyDesc d = pages.at(descs, it.block * pages.nparts + it.part);
        if (d.src != 0) {
            const uint32_t e0 = it.chunk * chunk;
            const uint32_t rows = min(chunk, elems - e0) / kRow;
            const uint32_t row0 = e0 / kRow;
            const uint8_t* q = reinterpret_cast<const uint8_t*>(d.src);
            const float* scales = reinterpret_cast<const float*>(q + elems);
            uint8_t* dst = reinterpret_cast<uint8_t*>(d.dst);
            for (uint32_t r0 = warp * kStep; r0 < rows; r0 += kWarps * kStep) {
                uint2 v[kRowPairs];
                float sc[kRowPairs];
#pragma unroll
                for (int u = 0; u < kRowPairs; ++u) {
                    const uint32_t r = r0 + 2 * u + half;
                    if (r < rows) {
                        v[u] = ld_u2(q + size_t(row0 + r) * kRow + hl * 8);
                        sc[u] = __uint_as_float(ld_u1(scales + row0 + r));
                    }
                }
#pragma unroll
                for (int u = 0; u < kRowPairs; ++u) {
                    const uint32_t r = r0 + 2 * u + half;
                    if (r >= rows) continue;
                    *reinterpret_cast<uint4*>(dst + (size_t(row0 + r) * kRow + hl * 8) * 2) =
                        dequant8(v[u], sc[u]);
                }
            }
        } else if (threadIdx.x == 0 && item < group_items && item % (rel.gp * cpp) == 0 && status) {
            atomicAdd(status + kStatMiss, 1u);
        }
        const uint32_t nxt = item + gridDim.x;
        if (nxt >= total || nxt / group_items != it.group) {
            const uint32_t lo = it.group * group_items;
            leave_group(rel, it.group, cta_items(lo, lo + group_items, blockIdx.x, gridDim.x),
                        group_items, kThreads);
        }
    }
}

// The same loop as kv_read_fp8_kernel over the parts of gathered blocks.  A missing block
// counts once, on its first part's first item; none of its parts is written.  (The two kernels
// share the row maths, not the loop: inlining one loop body into both changed how the
// compiler schedules kv_read_fp8_kernel.)  LAYERED: a layered read (read_fp8_layered above).
template <bool LAYERED = false>
__global__ void __launch_bounds__(kThreads)
    kv_read_fp8_scatter_kernel(const CopyDesc* __restrict__ descs,
                               const __grid_constant__ GatherParts parts, uint32_t n,
                               uint32_t nparts, uint32_t first_part, uint32_t elems,
                               uint32_t chunk, uint32_t cpp, uint64_t stride, uint32_t* status,
                               GroupRelease rel) {
    const BlockParts<false> pages{&parts, nparts, first_part, stride};
    if constexpr (LAYERED) {
        read_fp8_layered(descs, pages, n, elems, chunk, cpp, status, rel);
        return;
    }
    const uint32_t total = n * nparts * cpp;
    const uint32_t warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const uint32_t half = lane >> 4, hl = lane & 15;
    constexpr uint32_t kStep = 2 * kRowPairs;
    for (uint32_t item = blockIdx.x; item < total; item += gridDim.x) {
        const CopyDesc d = pages.at(descs, item / cpp);
        if (d.src == 0) {
            if (threadIdx.x == 0 && pages.head(item / cpp) && item % cpp == 0 && status) atomicAdd(status + kStatMiss, 1u);
            continue;
        }
        const uint32_t e0 = (item % cpp) * chunk;
        const uint32_t rows = min(chunk, elems - e0) / kRow;
        const uint32_t row0 = e0 / kRow;
        const uint8_t* q = reinterpret_cast<const uint8_t*>(d.src);
        const float* scales = reinterpret_cast<const float*>(q + elems);
        uint8_t* dst = reinterpret_cast<uint8_t*>(d.dst);
        for (uint32_t r0 = warp * kStep; r0 < rows; r0 += kWarps * kStep) {
            uint2 v[kRowPairs];
            float sc[kRowPairs];
#pragma unroll
            for (int u = 0; u < kRowPairs; ++u) {
                const uint32_t r = r0 + 2 * u + half;
                if (r < rows) {
                    v[u] = ld_u2(q + size_t(row0 + r) * kRow + hl * 8);
                    sc[u] = __uint_as_float(ld_u1(scales + row0 + r));
                }
            }
#pragma unroll
            for (int u = 0; u < kRowPairs; ++u) {
                const uint32_t r = r0 + 2 * u + half;
                if (r >= rows) continue;
                *reinterpret_cast<uint4*>(dst + (size_t(row0 + r) * kRow + hl * 8) * 2) =
                    dequant8(v[u], sc[u]);
            }
        }
    }
}

}  // namespace

cudaError_t launch_kv_write_fp8(const Fp8Launch& a, cudaStream_t stream) {
    if (a.n == 0 || a.elems == 0) return cudaSuccess;
    if (a.group != kRow || a.elems % kRow != 0) return cudaErrorInvalidValue;
    const LaunchPlan p = plan_fp8(a, sm_count());
    if (!p.valid) return cudaErrorInvalidValue;  // pages that are not 16-byte aligned
    if (p.kernel != Kernel::kLdStFp8) return launch_kv_fp8_pipe(a, true, stream);
    kv_write_fp8_kernel<<<p.ctas, kThreads + 32, 0, stream>>>(a.descs, a.n, a.elems, p.chunk, p.cpb,
                                                             publish_of(a, true));
    return cudaGetLastError();
}

cudaError_t launch_kv_read_fp8(const Fp8Launch& a, cudaStream_t stream) {
    if (a.n == 0 || a.elems == 0) return cudaSuccess;
    if (a.group != kRow || a.elems % kRow != 0) return cudaErrorInvalidValue;
    const LaunchPlan p = plan_fp8(a, sm_count());
    if (!p.valid) return cudaErrorInvalidValue;  // pages that are not 16-byte aligned
    if (p.kernel != Kernel::kLdStFp8) return launch_kv_fp8_pipe(a, false, stream);
    kv_read_fp8_kernel<<<p.ctas, kThreads, 0, stream>>>(a.descs, a.n, a.elems, p.chunk, p.cpb,
                                                        a.status);
    return cudaGetLastError();
}

cudaError_t launch_kv_gather_fp8(const GatherLaunch& a, uint32_t elems, int variant,
                                 cudaStream_t stream) {
    if (a.n == 0) return cudaSuccess;
    if (!a.part_base || a.rows) return cudaErrorInvalidValue;  // no row-sliced fp8 reads
    // a layered read takes the ld/st kernel whatever the variant (no layered pipeline)
    const bool layered = a.group_flags != nullptr;
    if (layered && (a.write || !a.group_counters || !a.group_parts || a.nparts % a.group_parts))
        return cudaErrorInvalidValue;
    const LaunchPlan p = plan_gather_fp8(a, elems, layered ? int(kFp8LdSt) : variant, sm_count());
    if (!p.valid) return cudaErrorInvalidValue;  // the caller splits the batch
    if (p.kernel != Kernel::kLdStFp8) return launch_kv_fp8_pipe_gather(a, elems, stream);
    GatherParts parts;
    std::memcpy(parts.base, a.part_base, size_t(a.nparts) * sizeof(uint64_t));
    const uint64_t stride = fp8_gather_bytes(1, elems);
    const GroupRelease rel{a.group_flags, a.group_counters, a.group_seq, a.group_parts};
    if (a.write)
        kv_write_fp8_gather_kernel<<<p.ctas, kThreads + 32, 0, stream>>>(
            a.descs, parts, a.n, a.nparts, elems, p.chunk, p.cpb, a.first_part, stride,
            publish_of(a, true), layer_of(a));
    else if (layered)
        kv_read_fp8_scatter_kernel<true><<<p.ctas, kThreads, 0, stream>>>(
            a.descs, parts, a.n, a.nparts, a.first_part, elems, p.chunk, p.cpb, stride, a.status,
            rel);
    else
        kv_read_fp8_scatter_kernel<<<p.ctas, kThreads, 0, stream>>>(
            a.descs, parts, a.n, a.nparts, a.first_part, elems, p.chunk, p.cpb, stride, a.status,
            rel);
    return cudaGetLastError();
}

}  // namespace istore::kernels
