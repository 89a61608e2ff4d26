// fp8 KV path: the quantisation is fused into the page mover.  This file holds the ld/st
// flavour (any page size that is a multiple of 128 elements); pages of a multiple of 512
// elements - every real KV layout - take the TMA-pipelined flavour in kv_fp8_pipe.cu.
//
//   kv_write_fp8 : bf16 page in the client's paged KV cache -> e4m3 payload + one fp32 scale
//                  per 128-element row (head_dim) written straight into the (peer) pool
//                  block, then the in-band commit.  Half the NVLink bytes of a bf16 write and
//                  no separate cast kernel / staging buffer.
//   kv_read_fp8  : pool block -> dequantised bf16 scattered into the destination pages.
// The reference moves raw bytes only (dtype-agnostic, infinistore/lib.py:377-379); this is
// the "write fused with fp8 cast / read fused with gather" item of the north star.
//
// Pool block layout: [elems x e4m3][elems/128 x fp32 scale].
// A half-warp owns one 128-element row per step (lane l: elements 8l..8l+7, one 16-byte
// load), reduces |x| max with shuffles inside the half, and emits 8 bytes per lane (one
// coalesced 128-byte store per row).  Eight rows are in flight per warp to cover the
// NVLink / HBM latency.
// There is no direct bf16<->e4m3 cvt on sm_90a: quantise via f32, dequantise via f16x2.
#include <cuda_bf16.h>
#include <cuda_fp16.h>

#include <algorithm>

#include "common.cuh"
#include "kernels.h"
#include "publish.cuh"

namespace istore::kernels {

namespace {

constexpr int kThreads = 256;
constexpr int kWarps = kThreads / 32;
constexpr uint32_t kRow = 128;                 // elements sharing a scale
constexpr uint32_t kChunkElems = 8192;         // CTA work item: 64 rows
constexpr float kE4m3Max = 448.f;

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
__device__ __forceinline__ uint16_t cvt_e4m3x2(float hi, float lo) {  // F2FP.SATFINITE.E4M3.F32
    uint16_t r;
    asm("cvt.rn.satfinite.e4m3x2.f32 %0, %1, %2;" : "=h"(r) : "f"(hi), "f"(lo));
    return r;
}
__device__ __forceinline__ uint32_t cvt_f16x2_e4m3x2(uint16_t v) {  // F2FP.F16.E4M3.UNPACK_B
    uint32_t r;
    asm("cvt.rn.f16x2.e4m3x2 %0, %1;" : "=r"(r) : "h"(v));
    return r;
}
__device__ __forceinline__ float2 bf16x2_to_f2(uint32_t v) {
    return make_float2(__uint_as_float(v << 16), __uint_as_float(v & 0xffff0000u));
}
__device__ __forceinline__ uint32_t f2_to_bf16x2(float lo, float hi) {
    const __nv_bfloat162 b = __floats2bfloat162_rn(lo, hi);
    return *reinterpret_cast<const uint32_t*>(&b);
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

// Threads [0, 256) quantise + store; warp 8 is the control warp (in-band commit).
__global__ void __launch_bounds__(kThreads + 32)
    kv_write_fp8_kernel(const CopyDesc* __restrict__ descs, uint32_t n, uint32_t elems,
                        uint32_t chunk, uint32_t cpb, Publish pub) {
    const uint32_t total = n * cpb;
    if (threadIdx.x >= kThreads) {
        if (!pub.recs) return;
        const uint32_t count = blockIdx.x < total ? (total - blockIdx.x + gridDim.x - 1) / gridDim.x : 0;
        control_warp(pub, threadIdx.x - kThreads, blockIdx.x, count, gridDim.x, cpb, kThreads + 32);
        return;
    }
    const uint32_t warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const uint32_t half = lane >> 4, hl = lane & 15;
    constexpr uint32_t kStep = 2 * kRowPairs;  // rows per warp iteration
    for (uint32_t item = blockIdx.x; item < total; item += gridDim.x) {
        const CopyDesc d = descs[item / cpb];
        const uint32_t e0 = (item % cpb) * chunk;
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
                f[0] = bf16x2_to_f2(v[u].x);
                f[1] = bf16x2_to_f2(v[u].y);
                f[2] = bf16x2_to_f2(v[u].z);
                f[3] = bf16x2_to_f2(v[u].w);
                float amax = 0.f;
                if (live) {
#pragma unroll
                    for (int j = 0; j < 4; ++j) amax = fmaxf(amax, fmaxf(fabsf(f[j].x), fabsf(f[j].y)));
                }
#pragma unroll
                for (int o = 8; o > 0; o >>= 1)  // reduce within the half-warp that owns the row
                    amax = fmaxf(amax, __shfl_xor_sync(0xffffffffu, amax, o));
                if (!live) continue;
                const float scale = amax > 0.f ? amax * (1.f / kE4m3Max) : 1.f;
                const float inv = 1.f / scale;
                uint2 out;
                out.x = uint32_t(cvt_e4m3x2(f[0].y * inv, f[0].x * inv)) |
                        (uint32_t(cvt_e4m3x2(f[1].y * inv, f[1].x * inv)) << 16);
                out.y = uint32_t(cvt_e4m3x2(f[2].y * inv, f[2].x * inv)) |
                        (uint32_t(cvt_e4m3x2(f[3].y * inv, f[3].x * inv)) << 16);
                *reinterpret_cast<uint2*>(q + size_t(row0 + r) * kRow + hl * 8) = out;
                if (hl == 0) scales[row0 + r] = scale;
            }
        }
    }
    if (pub.recs) ctrl_barrier_arrive(kThreads + 32);
}

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
                const uint32_t w[2] = {v[u].x, v[u].y};
                uint32_t o[4];
#pragma unroll
                for (int j = 0; j < 2; ++j) {
                    const uint32_t h01 = cvt_f16x2_e4m3x2(uint16_t(w[j] & 0xffffu));
                    const uint32_t h23 = cvt_f16x2_e4m3x2(uint16_t(w[j] >> 16));
                    const float2 f01 = __half22float2(*reinterpret_cast<const __half2*>(&h01));
                    const float2 f23 = __half22float2(*reinterpret_cast<const __half2*>(&h23));
                    o[2 * j] = f2_to_bf16x2(f01.x * sc[u], f01.y * sc[u]);
                    o[2 * j + 1] = f2_to_bf16x2(f23.x * sc[u], f23.y * sc[u]);
                }
                *reinterpret_cast<uint4*>(dst + (size_t(row0 + r) * kRow + hl * 8) * 2) =
                    make_uint4(o[0], o[1], o[2], o[3]);
            }
        }
    }
}

}  // namespace

cudaError_t launch_kv_write_fp8(const Fp8Launch& a, cudaStream_t stream) {
    if (a.n == 0 || a.elems == 0) return cudaSuccess;
    if (a.group != kRow || a.elems % kRow != 0) return cudaErrorInvalidValue;
    if (a.variant != 1 && fp8_pipe_supported(a)) return launch_kv_fp8_pipe(a, true, stream);
    Publish pub{a.recs, a.table, a.table_mask, a.done, a.status, a.n, nullptr, !a.all_local, 0,
                a.shards};
    if (!a.table || !a.done) pub.recs = nullptr;
    // whole pages per CTA when there are enough of them (single-CTA commit, see kv_copy.cu)
    uint32_t chunk = kChunkElems;
    if (a.n >= uint32_t(sm_count()) && a.elems <= (1u << 19)) chunk = a.elems;
    const uint32_t cpb = (a.elems + chunk - 1) / chunk;
    const uint64_t total = uint64_t(a.n) * cpb;
    int ctas = a.max_ctas > 0 ? a.max_ctas : 6 * sm_count();
    ctas = int(std::min<uint64_t>(uint64_t(ctas), total));
    kv_write_fp8_kernel<<<ctas, kThreads + 32, 0, stream>>>(a.descs, a.n, a.elems, chunk, cpb, pub);
    return cudaGetLastError();
}

cudaError_t launch_kv_read_fp8(const Fp8Launch& a, cudaStream_t stream) {
    if (a.n == 0 || a.elems == 0) return cudaSuccess;
    if (a.group != kRow || a.elems % kRow != 0) return cudaErrorInvalidValue;
    if (a.variant != 1 && fp8_pipe_supported(a)) return launch_kv_fp8_pipe(a, false, stream);
    uint32_t chunk = kChunkElems;
    if (a.n >= uint32_t(sm_count()) && a.elems <= (1u << 19)) chunk = a.elems;
    const uint32_t cpb = (a.elems + chunk - 1) / chunk;
    const uint64_t total = uint64_t(a.n) * cpb;
    int ctas = a.max_ctas > 0 ? a.max_ctas : 6 * sm_count();
    ctas = int(std::min<uint64_t>(uint64_t(ctas), total));
    kv_read_fp8_kernel<<<ctas, kThreads, 0, stream>>>(a.descs, a.n, a.elems, chunk, cpb, a.status);
    return cudaGetLastError();
}

}  // namespace istore::kernels
