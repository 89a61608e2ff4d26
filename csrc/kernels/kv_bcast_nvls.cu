// kv_bcast_nvls: one writer -> every reader replication of KV blocks through an NVLS
// multicast mapping.
//
// The reference serves a shared prefix with N independent unicast reads, one RDMA_WRITE
// chain per client (src/infinistore.cpp:424-533).  On an NVSwitch box the writer instead
// stores each 16-byte vector ONCE to a multicast address (multimem.st) and the switch
// replicates it into the replica region of every bound GPU: writer egress stays at one
// copy while N copies are delivered.  Readers then consume their local replica at HBM
// speed.  Descriptors: src = local page, dst = address inside the multicast mapping.
#include <algorithm>

#include "common.cuh"
#include "kernels.h"
#include "launch_plan.h"

namespace istore::kernels {

namespace {

using namespace dev;

constexpr int kThreads = 256;
constexpr uint32_t kChunk = 32u << 10;

__device__ __forceinline__ void multimem_st_u4(void* mc, const uint4& v) {
    asm volatile("multimem.st.relaxed.sys.global.v4.f32 [%0], {%1,%2,%3,%4};" ::"l"(mc),
                 "f"(__uint_as_float(v.x)), "f"(__uint_as_float(v.y)), "f"(__uint_as_float(v.z)),
                 "f"(__uint_as_float(v.w))
                 : "memory");
}

// In-band readiness.  With `flags_mc` (a u32 per block inside the multicast mapping) the CTA
// that finishes a chunk adds 1 to the block's flag in EVERY replica with one
// multimem.red.release.sys: the release orders the CTA's data stores (bar.sync makes them
// cumulative) before the flag.  A reader on any GPU spins on its LOCAL copy of the flag with
// ld.acquire.sys (kv_read_when_ready below) - no host synchronisation, no traffic over the
// fabric while it waits; a block is complete when its flag reaches flag_base + cpb.
__device__ __forceinline__ void multimem_red_release_add(uint32_t* mc, uint32_t v) {
    asm volatile("multimem.red.release.sys.global.add.u32 [%0], %1;" ::"l"(mc), "r"(v) : "memory");
}

__global__ void __launch_bounds__(kThreads)
    kv_bcast_nvls_kernel(const CopyDesc* __restrict__ descs, uint32_t n, uint32_t bytes,
                         uint32_t chunk, uint32_t cpb, uint32_t* flags_mc) {
    constexpr int U = 4;
    const uint32_t total = n * cpb;
    for (uint32_t item = blockIdx.x; item < total; item += gridDim.x) {
        const CopyDesc d = descs[item / cpb];
        const uint32_t off = (item % cpb) * chunk;
        const uint32_t len = min(chunk, bytes - off);
        const uint8_t* src = reinterpret_cast<const uint8_t*>(d.src) + off;
        uint8_t* dst = reinterpret_cast<uint8_t*>(d.dst) + off;
        const uint32_t nvec = len / 16;
        uint32_t i = threadIdx.x;
        for (; i + (U - 1) * kThreads < nvec; i += U * kThreads) {
            uint4 v[U];
#pragma unroll
            for (int u = 0; u < U; ++u) v[u] = ld_stream_v4(src + size_t(i + u * kThreads) * 16);
#pragma unroll
            for (int u = 0; u < U; ++u) multimem_st_u4(dst + size_t(i + u * kThreads) * 16, v[u]);
        }
        for (; i < nvec; i += kThreads) multimem_st_u4(dst + size_t(i) * 16, ld_stream_v4(src + size_t(i) * 16));
        if (flags_mc) {
            __syncthreads();  // every thread's stores of this chunk are ordered before ...
            if (threadIdx.x == 0) multimem_red_release_add(flags_mc + item / cpb, 1u);  // ... the flag
        }
    }
    // without flags: make the replicated stores visible to every reader before the kernel's
    // completion is signalled (readers then synchronise on a stream event)
    if (!flags_mc) fence_sys();
}

// Reader side: copy blocks out of the LOCAL replica as soon as the writer has marked them
// ready - launched before, or concurrently with, the writer's broadcast.
__global__ void __launch_bounds__(kThreads)
    kv_read_when_ready_kernel(const CopyDesc* __restrict__ descs, uint32_t n, uint32_t bytes,
                              const uint32_t* __restrict__ flags_local, uint32_t ready_value,
                              uint32_t* status) {
    __shared__ uint32_t ok;
    for (uint32_t item = blockIdx.x; item < n; item += gridDim.x) {
        if (threadIdx.x == 0) {
            uint32_t v = 0;
            long long start = clock64();
            for (uint32_t spins = 0;; ++spins) {
                v = ld_acquire_sys(flags_local + item);
                if (v >= ready_value) break;
                if ((spins & 255) == 255) {
                    __nanosleep(200);
                    if (clock64() - start > 6000000000ll) break;  // ~3 s: the writer never came
                }
            }
            ok = v >= ready_value;
            if (!ok && status) atomicAdd(status + kStatMiss, 1u);
        }
        __syncthreads();  // the acquire of thread 0 + bar.sync orders the block's data for all
        if (ok) {
            const CopyDesc d = descs[item];
            const uint8_t* src = reinterpret_cast<const uint8_t*>(d.src);
            uint8_t* dst = reinterpret_cast<uint8_t*>(d.dst);
            for (uint32_t i = threadIdx.x; i < bytes / 16; i += kThreads)
                st_v4(dst + size_t(i) * 16, ld_stream_v4(src + size_t(i) * 16));
        }
        __syncthreads();
    }
}

}  // namespace

cudaError_t launch_kv_bcast_nvls(const BcastLaunch& a, cudaStream_t stream) {
    if (a.n == 0 || a.bytes == 0) return cudaSuccess;
    if (a.bytes % 16) return cudaErrorInvalidValue;
    const uint32_t chunk = std::min(a.bytes, kChunk);
    const uint32_t cpb = (a.bytes + chunk - 1) / chunk;
    const uint64_t total = uint64_t(a.n) * cpb;
    const int ctas = clamp_grid(a.max_ctas > 0 ? a.max_ctas : 4 * sm_count(), total);
    kv_bcast_nvls_kernel<<<ctas, kThreads, 0, stream>>>(a.descs, a.n, a.bytes, chunk, cpb, a.flags_mc);
    return cudaGetLastError();
}

uint32_t bcast_chunks_per_block(uint32_t bytes) {
    const uint32_t chunk = std::min(bytes, kChunk);
    return (bytes + chunk - 1) / chunk;
}

cudaError_t launch_kv_read_when_ready(const ReadyLaunch& a, cudaStream_t stream) {
    if (a.n == 0 || a.bytes == 0) return cudaSuccess;
    if (a.bytes % 16 || !a.flags_local) return cudaErrorInvalidValue;
    const int ctas = clamp_grid(a.max_ctas > 0 ? a.max_ctas : 2 * sm_count(), a.n);
    kv_read_when_ready_kernel<<<ctas, kThreads, 0, stream>>>(a.descs, a.n, a.bytes, a.flags_local,
                                                            a.ready_value, a.status);
    return cudaGetLastError();
}

}  // namespace istore::kernels
