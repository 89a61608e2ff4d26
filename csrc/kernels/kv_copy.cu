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
#include <cuda.h>

#include <cstring>
#include <mutex>

#include "common.cuh"
#include "kernels.h"
#include "copy_span.cuh"
#include "gather_items.cuh"
#include "launch_plan.h"
#include "publish.cuh"

namespace istore::kernels {

namespace {

using namespace dev;

// ---------------------------------------------------------------- ld/st path (copy_span.cuh)
// Small batches: descriptors in the kernel parameters (launch_plan.h).
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

// ---------------------------------------------------------------- gathered blocks (ld/st)
// The launch's part geometry, every shape's fields in one kernel parameter (GatherLaunch):
// each body reads the fields of its own shape.
struct PartGeometry {
    uint32_t part_bytes;
    PartRows rows;
    const uint64_t* piece_off;
};

// Reads: gather_items.cuh's scatter_items walk, one body per part shape.  Item chunk c of part s
// of block b copies, from pool desc.src + (first_part + s) * part_bytes to local
// parts.base[s] + desc.dst:
//   kWhole   bytes [c * chunk, +chunk) of the part (copy_span);
//   kRows    rows [c * chunk, +chunk) (GatherLaunch::rows): row r from r * src_pitch + src_col
//            (row_bytes) to r * dst_pitch (copy_rows);
//   kSlices  (slice, row) pairs [c * chunk, +chunk) of the part (rows.slices > 1), numbered
//            slice-major, each placed by PartRows::pair (copy_rows<VEC, true>);
//   kPieces  the same pairs (rows.pieces > 1, any slices), cut where q / piece_rows changes;
//            each cut, one slice's rows inside one piece, is copied as plain rows to desc.dst +
//            piece_off[block * pieces + t] + the place PartRows::pair gives its first pair - one
//            piece-offset load per cut.
// No control warp: reads publish nothing.  The minimum of 3 CTAs per SM holds every flavour to
// 80 registers, which the 32-byte row reads use.
template <int VEC, bool LAYERED, PartShape S>
__global__ void __launch_bounds__(kLdStThreads, 3)
    kv_scatter_ldst_kernel(const CopyDesc* __restrict__ descs,
                           const __grid_constant__ GatherParts parts, uint32_t n, uint32_t nparts,
                           uint32_t first_part, uint32_t chunk, uint32_t cpp, PartGeometry g,
                           uint32_t* status, GroupRelease rel) {
    scatter_items<LAYERED>(descs, n, nparts, cpp, status, rel, [&](const CopyDesc& d,
                                                                  const LayeredItem& it) {
        const uint64_t src = d.src + uint64_t(first_part + it.part) * g.part_bytes;
        const uint64_t dst = parts.base[it.part] + d.dst;
        const auto at = [](uint64_t a) { return reinterpret_cast<uint8_t*>(a); };
        if constexpr (S == PartShape::kWhole) {
            const uint32_t off = it.chunk * chunk;
            const uint32_t len = min(chunk, g.part_bytes - off);
            if constexpr (VEC == 1) {
                for (uint32_t b = threadIdx.x; b < len; b += kLdStThreads)
                    at(dst + off)[b] = at(src + off)[b];
            } else {
                copy_span<VEC>(at(dst + off), at(src + off), len);
            }
        } else if constexpr (S == PartShape::kRows) {
            const uint32_t r0 = it.chunk * chunk;
            copy_rows<VEC>(at(dst + uint64_t(r0) * g.rows.dst_pitch),
                           at(src + uint64_t(r0) * g.rows.src_pitch + g.rows.src_col),
                           min(chunk, g.rows.rows - r0), g.rows);
        } else if constexpr (S == PartShape::kSlices) {
            const uint32_t q0 = it.chunk * chunk;
            copy_rows<VEC, true>(at(dst), at(src), min(chunk, g.rows.rows * g.rows.slices - q0),
                                 g.rows, q0);
        } else {
            const uint32_t piece_rows = g.rows.rows / g.rows.pieces;
            const uint32_t q0 = it.chunk * chunk, q1 = min(q0 + chunk, g.rows.rows * g.rows.slices);
            const uint64_t* off = g.piece_off + uint64_t(it.block) * g.rows.pieces;
            for (uint32_t q = q0; q < q1;) {
                const uint32_t e = min(q1, (q / piece_rows + 1) * piece_rows);
                const PairOffsets o = g.rows.pair(q, piece_rows);
                copy_rows<VEC>(at(dst + off[o.piece] + o.dst), at(src + o.src), e - q, g.rows);
                q = e;
            }
        }
    });
}

// bf16 writes: gather_items.cuh's gather_items walk.  Item chunk c of part s of block b stores
// bytes [off, off + len) of pool part first_part + s of desc.dst, each loaded from local
// parts.base[s] + desc.src:
//   kWhole   at the same offset (copy_span);
//   kRows    at PartRows::write_offset of its stored offset (GatherLaunch::rows with write, any
//            slices: copy_span_rows), so every item still stores one contiguous run of pool
//            bytes and the commit counts arrivals as for whole parts;
//   kPieces  the same, with the item's stored bytes cut at piece boundaries (piece_rows *
//            src_pitch bytes) and each cut loaded from desc.src + piece_off[block * pieces + t]
//            - one piece-offset load per cut.
// The minimum of 3 CTAs per SM lets the 32-byte flavour keep 64 registers; without it ptxas
// held it to 56 and spilled.
template <int VEC, PartShape S>
__global__ void __launch_bounds__(kLdStThreads + 32, 3)
    kv_gather_ldst_kernel(const CopyDesc* __restrict__ descs,
                          const __grid_constant__ GatherParts parts, uint32_t n, uint32_t nparts,
                          uint32_t first_part, uint32_t chunk, uint32_t cpp, PartGeometry g,
                          Publish pub, LayerCommit lc) {
    gather_items(descs, n, nparts, g.part_bytes, chunk, cpp, pub, lc, [&](const CopyDesc& d,
                                                                        uint32_t block,
                                                                        uint32_t s, uint32_t off,
                                                                        uint32_t len) {
        uint8_t* dst =
            reinterpret_cast<uint8_t*>(d.dst + uint64_t(first_part + s) * g.part_bytes + off);
        const uint64_t src = parts.base[s] + d.src;
        const auto at = [](uint64_t a) { return reinterpret_cast<const uint8_t*>(a); };
        if constexpr (S == PartShape::kWhole) {
            if constexpr (VEC == 1) {
                for (uint32_t b = threadIdx.x; b < len; b += kLdStThreads)
                    dst[b] = at(src + off)[b];
            } else {
                copy_span<VEC>(dst, at(src + off), len);
            }
        } else if constexpr (S == PartShape::kRows) {
            copy_span_rows<VEC>(dst, at(src), off, len, g.rows);
        } else {
            const uint32_t piece_bytes = g.part_bytes / g.rows.pieces;
            const uint64_t* poff = g.piece_off + uint64_t(block) * g.rows.pieces;
            for (uint32_t o = off; o < off + len;) {
                const uint32_t t = o / piece_bytes;
                const uint32_t e = min(off + len, (t + 1) * piece_bytes);
                copy_span_rows<VEC>(dst + (o - off), at(src + poff[t]), o - t * piece_bytes,
                                    e - o, g.rows);
                o = e;
            }
        }
    });
}

// One launch of a gathered ld/st kernel: the plan for its shape and direction, then the plan's
// vector width.  The residency is the launched kernel's own; whole parts take the TMA
// pipeline where plan_gather says so.
template <bool WRITE, bool LAYERED, PartShape S>
cudaError_t launch_ldst_gather(const GatherLaunch& a, const GatherParts& parts,
                               const PartGeometry& g, cudaStream_t stream) {
    constexpr int T = WRITE ? kLdStThreads + 32 : kLdStThreads;
    const LdStResident* res;
    if constexpr (WRITE)
        res = &cached_resident<kv_gather_ldst_kernel<16, S>, kv_gather_ldst_kernel<32, S>, T>();
    else
        res = &cached_resident<kv_scatter_ldst_kernel<16, LAYERED, S>,
                               kv_scatter_ldst_kernel<32, LAYERED, S>, T>();
    const LaunchPlan p = S == PartShape::kWhole ? plan_gather(a, sm_count(), *res)
                         : WRITE                ? plan_gather_rows_write(a, sm_count(), *res)
                                                : plan_gather_rows(a, sm_count(), *res);
    if (!p.valid) return cudaErrorInvalidValue;  // the caller checks the geometry and splits
    if (p.kernel == Kernel::kTma) return launch_kv_pipe_gather(a, stream);
    return with_vec(p.kernel, [&](auto vec) {
        constexpr int V = decltype(vec)::value;
        if constexpr (WRITE)
            kv_gather_ldst_kernel<V, S><<<p.ctas, T, 0, stream>>>(
                a.descs, parts, a.n, a.nparts, a.first_part, p.chunk, p.cpb, g,
                publish_of(a, true), layer_of(a));
        else
            kv_scatter_ldst_kernel<V, LAYERED, S><<<p.ctas, T, 0, stream>>>(
                a.descs, parts, a.n, a.nparts, a.first_part, p.chunk, p.cpb, g, a.status,
                release_of(a));
        return cudaGetLastError();
    });
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

cudaError_t set_smem_limits_once(bool (&done)[64], std::initializer_list<SmemLimit> limits) {
    static std::mutex mu;
    int dev = 0;
    cudaGetDevice(&dev);
    std::lock_guard<std::mutex> lk(mu);
    if (dev < 0 || dev >= 64 || done[dev]) return cudaSuccess;
    for (const SmemLimit& l : limits) {
        const cudaError_t e =
            cudaFuncSetAttribute(l.kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, l.bytes);
        if (e != cudaSuccess) return e;
    }
    done[dev] = true;
    return cudaSuccess;
}

cudaError_t launch_kv_copy(const CopyLaunch& a, cudaStream_t stream) {
    if (a.n == 0 || a.bytes == 0) return cudaSuccess;
    constexpr int T = kLdStThreads + 32;
    static const LdStResident res =
        ldst_resident(kv_copy_ldst_kernel<16, false>, kv_copy_ldst_kernel<32, false>, T);
    const LaunchPlan p = plan_copy(a, sm_count(), res);
    if (!p.valid) return cudaErrorInvalidValue;
    if (p.kernel == Kernel::kTma) return launch_kv_pipe_copy(a, stream);
    const Publish pub = publish_of(a, true, a.trace, a.debug);
    DescParam<kParamDescs> pd;
    if (p.param) std::memcpy(pd.d, a.descs_host, size_t(a.n) * sizeof(CopyDesc));
    const DescParam<1> none{};
    const auto go = [&](auto* kernel, const auto& descs_param) {
        kernel<<<p.ctas, T, 0, stream>>>(a.descs, descs_param, a.n, a.bytes, p.chunk, p.cpb, pub);
        return cudaGetLastError();
    };
    switch (p.kernel) {
        case Kernel::kLdSt16Mc:
            return p.param ? go(kv_copy_ldst_kernel<16, true, true>, pd)
                           : go(kv_copy_ldst_kernel<16, false, true>, none);
        case Kernel::kLdSt1:
            return go(kv_copy_ldst_kernel<1, false>, none);
        case Kernel::kLdSt32:
            return p.param ? go(kv_copy_ldst_kernel<32, true>, pd)
                           : go(kv_copy_ldst_kernel<32, false>, none);
        default:
            return p.param ? go(kv_copy_ldst_kernel<16, true>, pd)
                           : go(kv_copy_ldst_kernel<16, false>, none);
    }
}

cudaError_t launch_kv_gather(const GatherLaunch& a, cudaStream_t stream) {
    if (a.n == 0 || a.part_bytes == 0) return cudaSuccess;
    if (a.nparts == 0 || a.nparts > kGatherMaxParts || !a.part_base) return cudaErrorInvalidValue;
    if (uint64_t(a.nparts) * a.part_bytes > 0xffffffffull) return cudaErrorInvalidValue;
    const bool layered = a.group_flags != nullptr;
    if (layered && !a.group_counters) return cudaErrorInvalidValue;
    // RoPE shifts: the geometry is checked even when the table turns nothing, which the plain
    // movers below then copy verbatim
    if (a.rope) {
        if (!plan_gather_rope(a, 1, {}).valid || !a.rope->finite()) return cudaErrorInvalidValue;
        if (!a.rope->identity()) return launch_kv_gather_rope(a, stream);
    }
    // pieces split rows, at the offsets of the piece table
    if (a.rows.pieces != 1 && (!a.rows.rows || !a.piece_off)) return cudaErrorInvalidValue;
    const GatherParts parts = parts_of(a);
    const PartGeometry g{a.part_bytes, a.rows, a.piece_off};
    if (a.write)
        return with_shape<true>(a, [&](auto s) {
            return launch_ldst_gather<true, false, decltype(s)::value>(a, parts, g, stream);
        });
    return with_shape<false>(a, [&](auto s) {
        return layered ? launch_ldst_gather<false, true, decltype(s)::value>(a, parts, g, stream)
                       : launch_ldst_gather<false, false, decltype(s)::value>(a, parts, g, stream);
    });
}

// Resolved once per process, as fabric/nvls.cpp resolves its driver entry points.
cudaError_t stream_wait_geq(const uint32_t* addr, uint32_t value, cudaStream_t stream) {
    using WaitFn = CUresult (*)(CUstream, CUdeviceptr, cuuint32_t, unsigned int);
    static const WaitFn fn = [] {
        void* p = nullptr;
        cudaDriverEntryPointQueryResult q{};
        if (cudaGetDriverEntryPoint("cuStreamWaitValue32", &p, cudaEnableDefault, &q) !=
                cudaSuccess ||
            q != cudaDriverEntryPointSuccess)
            p = nullptr;
        (void)cudaGetLastError();
        return reinterpret_cast<WaitFn>(p);
    }();
    if (!fn) return cudaErrorNotSupported;
    const CUresult r = fn(stream, reinterpret_cast<CUdeviceptr>(addr), value,
                          CU_STREAM_WAIT_VALUE_GEQ);
    return r == CUDA_SUCCESS ? cudaSuccess : cudaErrorNotSupported;
}

}  // namespace istore::kernels
