// e4m3 KV caches (GatherLaunch::part_scale): the gathered fp8 movers of an engine that keeps
// its KV cache itself in float8_e4m3fn, with one fp32 scale per part (a layer's K or V).
//
//   kv_write_e4m3_gather : e4m3 part -> fp8 page of the pool block, payload byte i = cache byte
//                          i (NaN codes included) and every 128-element group's scale = the
//                          part's scale, then the in-band commit (gather_items' control warp:
//                          one-shot or a layered writer's LayerCommit).
//   kv_read_e4m3_scatter : fp8 page -> e4m3 part, each group requantised from its stored scale
//                          to the part's scale (fp8_row.cuh: requant16), or copied verbatim
//                          when the two are the same float; plain or layered (scatter_items).
//
// The stored block is exactly the gathered fp8 block of launch_kv_gather_fp8 (part s at
// fp8_gather_bytes(first_part + s, elems)), so every fp8 reader reads what these write and
// these read what every fp8 writer stores.  Whole parts only: elems a multiple of 512, part
// bases and local offsets 16-byte aligned (plan_gather_e4m3).  ld/st only, local and peer pools
// alike.
#include <cuda_fp16.h>

#include "common.cuh"
#include "copy_span.cuh"
#include "fp8_row.cuh"
#include "gather_items.cuh"
#include "kernels.h"
#include "launch_plan.h"
#include "publish.cuh"

namespace istore::kernels {

namespace {

using namespace fp8row;

constexpr int kThreads = kLdStThreads;
constexpr uint32_t kGroup = 128;  // e4m3 bytes sharing a stored scale
constexpr int kVecs = 4;          // 16-byte vectors in flight per thread in the read

// The per-part scales of a launch (GatherLaunch::part_scale), a parameter of these kernels
// only: GatherParts, which every gathered kernel takes, stays as it is.
struct PartScales {
    float s[kGatherMaxParts];
};

__device__ __forceinline__ uint32_t ld_u1(const void* p) {
    uint32_t r;
    asm volatile("ld.global.L1::no_allocate.u32 %0, [%1];" : "=r"(r) : "l"(p));
    return r;
}

// Writes: gather_items' walk over (block, part, run of `chunk` bytes); run [off, off + len) of
// part s is copied from parts.base[s] + desc.src + off into stored part first_part + s, and
// one thread per 128-byte group of the run stores the part's scale.
__global__ void __launch_bounds__(kThreads + 32)
    kv_write_e4m3_gather_kernel(const CopyDesc* __restrict__ descs,
                                const __grid_constant__ GatherParts parts,
                                const __grid_constant__ PartScales sc, uint32_t n, uint32_t nparts,
                                uint32_t elems, uint32_t chunk, uint32_t cpp, uint32_t first_part,
                                uint64_t stride, Publish pub, LayerCommit lc) {
    gather_items(descs, n, nparts, elems, chunk, cpp, pub, lc,
                 [&](const CopyDesc& d, uint32_t, uint32_t s, uint32_t off, uint32_t len) {
                     uint8_t* q = reinterpret_cast<uint8_t*>(d.dst + (first_part + s) * stride);
                     copy_span<16>(q + off,
                                   reinterpret_cast<const uint8_t*>(parts.base[s] + d.src) + off,
                                   len);
                     float* scales = reinterpret_cast<float*>(q + elems) + off / kGroup;
                     for (uint32_t g = threadIdx.x; g < len / kGroup; g += kThreads)
                         scales[g] = sc.s[s];
                 });
}

// Reads: scatter_items' walk (misses counted once per block, parts left untouched; LAYERED:
// group-major items and group releases).  Thread i of a run takes 16 bytes of one group, so the
// 8 threads of a group take the same branch: verbatim when the stored scale is the part's,
// else requant16 at r = min(s_g / s_c, FLT_MAX) (IEEE division, not a reciprocal).
template <bool LAYERED>
__global__ void __launch_bounds__(kThreads)
    kv_read_e4m3_scatter_kernel(const CopyDesc* __restrict__ descs,
                                const __grid_constant__ GatherParts parts,
                                const __grid_constant__ PartScales sc, uint32_t n, uint32_t nparts,
                                uint32_t elems, uint32_t chunk, uint32_t cpp, uint32_t first_part,
                                uint64_t stride, uint32_t* status, GroupRelease rel) {
    scatter_items<LAYERED>(descs, n, nparts, cpp, status, rel, [&](const CopyDesc& d,
                                                                  const LayeredItem& it) {
        const uint32_t e0 = it.chunk * chunk;
        const uint32_t nvec = min(chunk, elems - e0) / 16;
        const uint8_t* q =
            reinterpret_cast<const uint8_t*>(d.src + uint64_t(first_part + it.part) * stride);
        const uint8_t* src = q + e0;
        const float* scales = reinterpret_cast<const float*>(q + elems) + e0 / kGroup;
        uint8_t* dst = reinterpret_cast<uint8_t*>(parts.base[it.part] + d.dst) + e0;
        const float s_c = sc.s[it.part];
        for (uint32_t i = threadIdx.x; i < nvec; i += kVecs * kThreads) {
            uint4 v[kVecs];
            float s_g[kVecs];
#pragma unroll
            for (int u = 0; u < kVecs; ++u) {
                const uint32_t k = i + u * kThreads;
                if (k >= nvec) continue;
                v[u] = ld_stream_v4(src + size_t(k) * 16);
                s_g[u] = __uint_as_float(ld_u1(scales + k / (kGroup / 16)));
            }
#pragma unroll
            for (int u = 0; u < kVecs; ++u) {
                const uint32_t k = i + u * kThreads;
                if (k >= nvec) continue;
                const uint4 out =
                    __float_as_uint(s_g[u]) == __float_as_uint(s_c)
                        ? v[u]
                        : requant16(v[u], fminf(__fdiv_rn(s_g[u], s_c), 3.40282347e38f));
                st_v4(dst + size_t(k) * 16, out);
            }
        }
    });
}

PartScales scales_of(const GatherLaunch& a) {
    PartScales sc;
    std::memcpy(sc.s, a.part_scale, size_t(a.nparts) * sizeof(float));
    return sc;
}

template <bool WRITE, bool LAYERED>
cudaError_t launch_e4m3(const GatherLaunch& a, uint32_t elems, cudaStream_t stream) {
    const LaunchPlan p =
        WRITE ? plan_gather_e4m3(a, elems, sm_count(),
                                 cached_resident<kv_write_e4m3_gather_kernel,
                                                 kv_write_e4m3_gather_kernel, kThreads + 32>())
              : plan_gather_e4m3(a, elems, sm_count(),
                                 cached_resident<kv_read_e4m3_scatter_kernel<LAYERED>,
                                                 kv_read_e4m3_scatter_kernel<LAYERED>, kThreads>());
    if (!p.valid) return cudaErrorInvalidValue;
    const GatherParts parts = parts_of(a);
    const PartScales sc = scales_of(a);
    const uint64_t stride = fp8_gather_bytes(1, elems);
    if constexpr (WRITE)
        kv_write_e4m3_gather_kernel<<<p.ctas, kThreads + 32, 0, stream>>>(
            a.descs, parts, sc, a.n, a.nparts, elems, p.chunk, p.cpb, a.first_part, stride,
            publish_of(a, true), layer_of(a));
    else
        kv_read_e4m3_scatter_kernel<LAYERED><<<p.ctas, kThreads, 0, stream>>>(
            a.descs, parts, sc, a.n, a.nparts, elems, p.chunk, p.cpb, a.first_part, stride,
            a.status, release_of(a));
    return cudaGetLastError();
}

}  // namespace

cudaError_t launch_kv_gather_e4m3(const GatherLaunch& a, uint32_t elems, cudaStream_t stream) {
    if (a.n == 0) return cudaSuccess;
    if (!a.part_base || !a.part_scale) return cudaErrorInvalidValue;
    const bool layered = a.group_flags != nullptr;
    if (layered && !a.group_counters) return cudaErrorInvalidValue;
    if (a.write) return launch_e4m3<true, false>(a, elems, stream);
    return layered ? launch_e4m3<false, true>(a, elems, stream)
                   : launch_e4m3<false, false>(a, elems, stream);
}

}  // namespace istore::kernels
