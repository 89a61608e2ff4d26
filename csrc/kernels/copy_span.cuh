// The vector copy loop shared by the page movers: 256 threads stream one contiguous span
// with 128-bit accesses (LDG.E.128 / STG.E.128).  VEC = 16: four vectors in flight per
// thread, loads hinted L1::no_allocate.  VEC = 32 (the ldst256 variant, 32-byte aligned
// spans): Hopper has no 256-bit global load/store, so the same 128 bytes per thread that four
// 32-byte vectors held are kept in flight as eight 16-byte vectors, warp-contiguous.
#pragma once

#include "common.cuh"

namespace istore::kernels {

using namespace dev;

constexpr int kLdStThreads = 256;

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

}  // namespace istore::kernels
