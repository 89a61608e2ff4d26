// The vector copy loop shared by the page movers: 256 threads stream one contiguous span
// with 128-bit accesses (LDG.E.128 / STG.E.128).  VEC = 16: four vectors in flight per
// thread, loads hinted L1::no_allocate.  VEC = 32 (the ldst256 variant, 32-byte aligned
// spans): Hopper has no 256-bit global load/store, so the same 128 bytes per thread that four
// 32-byte vectors held are kept in flight as eight 16-byte vectors, warp-contiguous.
#pragma once

#include <algorithm>

#include "common.cuh"
#include "launch_plan.h"

namespace istore::kernels {

using namespace dev;

constexpr int kLdStThreads = 256;

// CTAs per SM the 16- and 32-byte flavours of an ld/st kernel keep resident, for launches of
// `threads` threads.  The callers keep the answer for the life of the process.
template <typename K16, typename K32>
LdStResident ldst_resident(K16* k16, K32* k32, int threads) {
    LdStResident r;
    cudaOccupancyMaxActiveBlocksPerMultiprocessor(&r.r16, k16, threads, 0);
    cudaOccupancyMaxActiveBlocksPerMultiprocessor(&r.r32, k32, threads, 0);
    r.r16 = std::max(r.r16, 1);
    r.r32 = std::max(r.r32, 1);
    return r;
}

// NVLS: one 16-byte store to a multicast address lands in every replica  (multimem.st)
__device__ __forceinline__ void st_multicast_v4(void* mc, const uint4& v) {
    asm volatile("multimem.st.relaxed.sys.global.v4.f32 [%0], {%1,%2,%3,%4};" ::"l"(mc),
                 "f"(__uint_as_float(v.x)), "f"(__uint_as_float(v.y)), "f"(__uint_as_float(v.z)),
                 "f"(__uint_as_float(v.w))
                 : "memory");
}

// MC = true: `dst` is a multicast address (VEC must be 16).
template <int VEC, bool MC = false>
__device__ __forceinline__ void copy_span(uint8_t* dst, const uint8_t* src, uint32_t len) {
    static_assert(VEC == 16 || VEC == 32, "vector width");
    constexpr int U = VEC / 4;
    const uint32_t nvec = len / 16;
    const uint32_t tid = threadIdx.x;
    uint32_t i = tid;
    for (; i + (U - 1) * kLdStThreads < nvec; i += U * kLdStThreads) {
        uint4 v[U];
#pragma unroll
        for (int u = 0; u < U; ++u) {
            const uint8_t* s = src + size_t(i + u * kLdStThreads) * 16;
            v[u] = VEC == 16 ? ld_stream_v4(s) : ld_v4(s);
        }
#pragma unroll
        for (int u = 0; u < U; ++u) {
            if constexpr (MC)
                st_multicast_v4(dst + size_t(i + u * kLdStThreads) * 16, v[u]);
            else
                st_v4(dst + size_t(i + u * kLdStThreads) * 16, v[u]);
        }
    }
    for (; i < nvec; i += kLdStThreads) {
        if constexpr (MC)
            st_multicast_v4(dst + size_t(i) * 16, ld_stream_v4(src + size_t(i) * 16));
        else
            st_v4(dst + size_t(i) * 16, ld_stream_v4(src + size_t(i) * 16));
    }
    for (uint32_t b = nvec * 16 + tid; b < len; b += kLdStThreads) dst[b] = src[b];
}

// `nrows` rows of row_bytes, row r from src + r * src_pitch to dst + r * dst_pitch.  The 256
// threads walk the (row, vector) pairs flattened together, so rows much narrower than a CTA's
// 4 KB per pass (one KV head of 128 bf16 is 256 bytes) still keep every thread busy.  VEC = 16
// / 32 as for copy_span (row_bytes, both pitches and both bases aligned to VEC); VEC = 1: bytes.
template <int VEC>
__device__ __forceinline__ void copy_rows(uint8_t* dst, const uint8_t* src, uint32_t nrows,
                                          uint32_t row_bytes, uint32_t src_pitch,
                                          uint32_t dst_pitch) {
    const uint32_t tid = threadIdx.x;
    if constexpr (VEC == 1) {
        const uint32_t len = nrows * row_bytes;
        for (uint32_t b = tid; b < len; b += kLdStThreads) {
            const uint32_t r = b / row_bytes, c = b - r * row_bytes;
            dst[size_t(r) * dst_pitch + c] = src[size_t(r) * src_pitch + c];
        }
    } else {
        static_assert(VEC == 16 || VEC == 32, "vector width");
        constexpr int U = VEC / 4;
        const uint32_t vpr = row_bytes / 16;  // vectors per row
        const uint32_t nvec = nrows * vpr;
        const auto at = [vpr](uint32_t v, uint32_t pitch) {
            const uint32_t r = v / vpr;
            return size_t(r) * pitch + size_t(v - r * vpr) * 16;
        };
        uint32_t i = tid;
        for (; i + (U - 1) * kLdStThreads < nvec; i += U * kLdStThreads) {
            uint4 v[U];
#pragma unroll
            for (int u = 0; u < U; ++u) {
                const uint8_t* s = src + at(i + u * kLdStThreads, src_pitch);
                v[u] = VEC == 16 ? ld_stream_v4(s) : ld_v4(s);
            }
#pragma unroll
            for (int u = 0; u < U; ++u) st_v4(dst + at(i + u * kLdStThreads, dst_pitch), v[u]);
        }
        for (; i < nvec; i += kLdStThreads)
            st_v4(dst + at(i, dst_pitch), ld_stream_v4(src + at(i, src_pitch)));
    }
}

}  // namespace istore::kernels
