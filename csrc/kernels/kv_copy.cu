// kv_copy: the batched page mover behind write_cache (client GPU -> pool HBM) and
// read_cache (pool HBM -> client GPU).
//
// One launch moves a whole batch of pages (a layer's worth) described by a descriptor
// array; either side of every descriptor may be a peer-mapped address, so the bytes cross
// NVLink / NVSwitch from inside the kernel.  This replaces, for one batch,
//   * N cudaMemcpyAsync calls on a fresh stream + event (reference local path,
//     src/infinistore.cpp:623-624,747-748),
//   * N RDMA_WRITE work requests chained 32 at a time (src/libinfinistore.cpp:905-970,
//     src/infinistore.cpp:456-530), and
//   * the COMMIT message round (src/libinfinistore.cpp:362-395 -> src/infinistore.cpp:
//     255-271): the kernel publishes each block in the HBM-resident index itself, with
//     release semantics at system scope, once the block's bytes have landed.
//
// Data paths, selected per launch (bench/sweep_copy.py compares them):
//   kCopyTma  : the default - the warp-specialised TMA pipeline of kv_pipe.cu (loader /
//               storer / control warps around an mbarrier-guarded SMEM ring);
//   kCopyLdSt / kCopyLdSt256 : this file - every thread streams 128-bit vectors, 4 (or,
//               for 32-byte aligned blocks, 8) in flight per thread; used for small or
//               unaligned blocks and for NVLS multicast stores (multimem.st has no bulk form).
#include <algorithm>
#include <cstring>
#include <mutex>

#include "common.cuh"
#include "kernels.h"
#include "copy_span.cuh"
#include "publish.cuh"

namespace istore::kernels {

namespace {

using namespace dev;

constexpr uint32_t kLdStChunk = 32u << 10;  // work item of the ld/st path

// ---------------------------------------------------------------- ld/st path (copy_span.cuh)
// Descriptors of small batches travel in the kernel parameters (constant bank): reading
// them from the pinned host ring costs a PCIe round trip at the start of every launch.
constexpr int kParamDescs = 256;
template <int N>
struct DescParam {
    CopyDesc d[N];
};

// VEC = 16 / 32: vector width; VEC = 1: byte fallback for unaligned tensors.
// Threads [0, 256) copy; warp 8 is the control warp (in-band commit, publish.cuh).
template <int VEC, bool PARAM, bool MC = false>
__global__ void __launch_bounds__(kLdStThreads + 32)
    kv_copy_ldst_kernel(const CopyDesc* __restrict__ descs,
                        const __grid_constant__ DescParam<PARAM ? kParamDescs : 1> pd, uint32_t n,
                        uint32_t bytes, uint32_t chunk, uint32_t cpb, Publish pub) {
    const uint32_t total = n * cpb;
    if (threadIdx.x >= kLdStThreads) {
        if (!pub.recs) return;
        const uint32_t count = blockIdx.x < total ? (total - blockIdx.x + gridDim.x - 1) / gridDim.x : 0;
        control_warp(pub, threadIdx.x - kLdStThreads, blockIdx.x, count, gridDim.x, cpb,
                     kLdStThreads + 32);
        return;
    }
    auto desc_at = [&](uint32_t block) -> CopyDesc {
        if constexpr (PARAM)
            return pd.d[block];
        else
            return descs[block];
    };
    uint32_t item = blockIdx.x;
    CopyDesc next = item < total ? desc_at(item / cpb) : CopyDesc{0, 0};
    for (; item < total; item += gridDim.x) {
        const CopyDesc d = next;
        const uint32_t nxt = item + gridDim.x;
        if (nxt < total) next = desc_at(nxt / cpb);  // prefetch: descriptors may sit in host memory
        if (d.src == 0) {  // key not found by the device lookup
            if (threadIdx.x == 0 && item % cpb == 0 && pub.status)
                atomicAdd(pub.status + kStatMiss, 1u);
            continue;
        }
        const uint32_t off = (item % cpb) * chunk;
        const uint32_t len = min(chunk, bytes - off);
        uint8_t* dst = reinterpret_cast<uint8_t*>(d.dst) + off;
        const uint8_t* src = reinterpret_cast<const uint8_t*>(d.src) + off;
        if constexpr (VEC == 1) {
            for (uint32_t b = threadIdx.x; b < len; b += kLdStThreads) dst[b] = src[b];
        } else {
            copy_span<VEC, MC>(dst, src, len);
        }
    }
    if (pub.recs) ctrl_barrier_arrive(kLdStThreads + 32);
}

}  // namespace

int sm_count() {
    static int cached[64] = {0};
    int dev = 0;
    if (cudaGetDevice(&dev) != cudaSuccess || dev < 0 || dev >= 64) return 132;
    if (!cached[dev]) {
        int n = 0;
        if (cudaDeviceGetAttribute(&n, cudaDevAttrMultiProcessorCount, dev) != cudaSuccess || n <= 0)
            n = 132;
        cached[dev] = n;
    }
    return cached[dev];
}

cudaError_t launch_kv_copy(const CopyLaunch& a, cudaStream_t stream) {
    if (a.n == 0 || a.bytes == 0) return cudaSuccess;
    Publish pub{a.recs, a.table, a.table_mask, a.done, a.status, a.n, a.trace, !a.all_local, a.debug,
                a.shards};
    if (!a.table || !a.done) pub.recs = nullptr;
    const int sms = sm_count();

    int variant = a.variant;
    // Alignment: bulk copies need 16-byte aligned addresses and sizes (the caller ORs every
    // local address into align_or; pool blocks are granule aligned).
    const bool aligned16 = (a.bytes % 16) == 0 && (a.align_or & 15) == 0;
    const bool aligned32 = (a.bytes % 32) == 0 && (a.align_or & 31) == 0;
    if (a.multicast) {
        if (!aligned16) return cudaErrorInvalidValue;  // multimem.st moves 16-byte vectors
        variant = kCopyLdSt;
    }
    // auto: the TMA pipeline from kPipeMinBytes up (3 warps per CTA); small blocks are bound
    // by per-block issue cost, where 256 threads win
    if (variant == kCopyAuto)
        variant = (aligned16 && a.bytes >= kPipeMinBytes) ? kCopyTma
                                                          : (aligned32 ? kCopyLdSt256 : kCopyLdSt);
    if (!aligned16 && (variant == kCopyTma || variant == kCopyLdSt256)) variant = kCopyLdSt;
    if (variant == kCopyLdSt256 && !aligned32) variant = kCopyLdSt;

    // small batches: descriptors ride in the kernel parameters
    const bool param = a.descs_host != nullptr && a.n <= uint32_t(kParamDescs) && aligned16;
    DescParam<kParamDescs> pd;
    if (param) std::memcpy(pd.d, a.descs_host, size_t(a.n) * sizeof(CopyDesc));
    const DescParam<1> none{};

    if (variant == kCopyTma) return launch_kv_pipe_copy(a, stream);

    // Work item = one 32 KB chunk, or - when there are at least as many blocks as SMs - one
    // whole block: then a block is moved by a single CTA, its commit needs no cross-CTA
    // counter (claim, one fence, one store) and a reader resolves every key exactly once.
    uint32_t chunk = std::min(a.bytes, kLdStChunk);
    if (a.n >= uint32_t(sms) && a.bytes <= (1u << 20)) chunk = a.bytes;
    const uint32_t cpb = (a.bytes + chunk - 1) / chunk;
    const uint64_t total = uint64_t(a.n) * cpb;
    constexpr int T = kLdStThreads + 32;
    // One wave: every CTA is resident and loops over its items, so the commit epilogue
    // (fence + release) runs once per CTA instead of once per item and per wave.
    static int resident16 = 0, resident32 = 0;
    if (!resident16) {
        int b16 = 0, b32 = 0;
        cudaOccupancyMaxActiveBlocksPerMultiprocessor(&b16, kv_copy_ldst_kernel<16, false>, T, 0);
        cudaOccupancyMaxActiveBlocksPerMultiprocessor(&b32, kv_copy_ldst_kernel<32, false>, T, 0);
        resident16 = std::max(b16, 1);
        resident32 = std::max(b32, 1);
    }
    const int per_sm = (variant == kCopyLdSt256) ? resident32 : resident16;
    int ctas = a.max_ctas > 0 ? a.max_ctas : per_sm * sms;
    ctas = int(std::min<uint64_t>(uint64_t(ctas), total));
    if (a.multicast && param)
        kv_copy_ldst_kernel<16, true, true><<<ctas, T, 0, stream>>>(a.descs, pd, a.n, a.bytes, chunk, cpb, pub);
    else if (a.multicast)
        kv_copy_ldst_kernel<16, false, true><<<ctas, T, 0, stream>>>(a.descs, none, a.n, a.bytes, chunk, cpb, pub);
    else if (!aligned16)
        kv_copy_ldst_kernel<1, false><<<ctas, T, 0, stream>>>(a.descs, none, a.n, a.bytes, chunk, cpb, pub);
    else if (variant == kCopyLdSt256 && param)
        kv_copy_ldst_kernel<32, true><<<ctas, T, 0, stream>>>(a.descs, pd, a.n, a.bytes, chunk, cpb, pub);
    else if (variant == kCopyLdSt256)
        kv_copy_ldst_kernel<32, false><<<ctas, T, 0, stream>>>(a.descs, none, a.n, a.bytes, chunk, cpb, pub);
    else if (param)
        kv_copy_ldst_kernel<16, true><<<ctas, T, 0, stream>>>(a.descs, pd, a.n, a.bytes, chunk, cpb, pub);
    else
        kv_copy_ldst_kernel<16, false><<<ctas, T, 0, stream>>>(a.descs, none, a.n, a.bytes, chunk, cpb, pub);
    return cudaGetLastError();
}

}  // namespace istore::kernels
