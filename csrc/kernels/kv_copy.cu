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
// The layered read (GatherLaunch::group_flags): items numbered group-major
// (launch_plan.h: layered_item), group g released by leave_group (publish.cuh) when this
// CTA's stream leaves it.  A missing block counts once, on its first item (group 0, part 0,
// chunk 0), and its parts are left untouched; its items still count as arrivals.
template <int VEC>
__device__ __forceinline__ void gather_read_layered(const CopyDesc* __restrict__ descs,
                                                    const GatherParts& parts, uint32_t n,
                                                    uint32_t nparts, uint32_t part_bytes,
                                                    uint32_t first_part, uint32_t chunk,
                                                    uint32_t cpp, uint32_t* status,
                                                    const GroupRelease& rel) {
    const uint32_t group_items = n * rel.gp * cpp;
    const uint32_t total = n * nparts * cpp;
    uint32_t item = blockIdx.x;
    CopyDesc next = item < total ? descs[layered_item(item, n, rel.gp, cpp).block] : CopyDesc{0, 0};
    for (; item < total; item += gridDim.x) {
        const CopyDesc d = next;
        const LayeredItem it = layered_item(item, n, rel.gp, cpp);
        const uint32_t nxt = item + gridDim.x;
        if (nxt < total) next = descs[layered_item(nxt, n, rel.gp, cpp).block];
        if (d.src != 0) {
            const uint32_t off = it.chunk * chunk;
            const uint32_t len = min(chunk, part_bytes - off);
            uint8_t* dst = reinterpret_cast<uint8_t*>(parts.base[it.part] + d.dst + off);
            const uint8_t* src = reinterpret_cast<const uint8_t*>(
                d.src + uint64_t(first_part + it.part) * part_bytes + off);
            if constexpr (VEC == 1) {
                for (uint32_t b = threadIdx.x; b < len; b += kLdStThreads) dst[b] = src[b];
            } else {
                copy_span<VEC>(dst, src, len);
            }
        } else if (threadIdx.x == 0 && item < group_items && item % (rel.gp * cpp) == 0 && status) {
            atomicAdd(status + kStatMiss, 1u);
        }
        if (nxt >= total || nxt / group_items != it.group) {
            const uint32_t lo = it.group * group_items;
            leave_group(rel, it.group, cta_items(lo, lo + group_items, blockIdx.x, gridDim.x),
                        group_items, kLdStThreads);
        }
    }
}

// Item = chunk c of part s of block b, numbered (b * nparts + s) * cpp + c (GatherLaunch).
// write: local parts.base[s] + desc.src -> pool desc.dst + (first_part + s) * part_bytes;
// read:  pool desc.src + (first_part + s) * part_bytes -> local parts.base[s] + desc.dst.
// LAYERED: a layered read (gather_read_layered above); no publish.
// The minimum of 3 CTAs per SM lets the 32-byte flavour keep 64 registers; without it ptxas
// held it to 56 and spilled.
template <int VEC, bool LAYERED = false>
__global__ void __launch_bounds__(kLdStThreads + 32, 3)
    kv_gather_ldst_kernel(const CopyDesc* __restrict__ descs,
                          const __grid_constant__ GatherParts parts, uint32_t n, uint32_t nparts,
                          uint32_t part_bytes, uint32_t first_part, uint32_t chunk, uint32_t cpp,
                          bool write, Publish pub, LayerCommit lc, GroupRelease rel) {
    if constexpr (LAYERED) {
        if (threadIdx.x >= kLdStThreads) return;
        gather_read_layered<VEC>(descs, parts, n, nparts, part_bytes, first_part, chunk, cpp,
                                 pub.status, rel);
        return;
    }
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
        if (nxt < total) next = descs[nxt / cpb];  // prefetch: descriptors may sit in host memory
        const uint32_t in_block = item % cpb;
        if (!write && d.src == 0) {  // key not found: one miss per block, parts left untouched
            if (threadIdx.x == 0 && in_block == 0 && pub.status) atomicAdd(pub.status + kStatMiss, 1u);
            continue;
        }
        const uint32_t s = in_block / cpp;
        const uint32_t off = (in_block % cpp) * chunk;
        const uint32_t len = min(chunk, part_bytes - off);
        const uint64_t local = parts.base[s] + (write ? d.src : d.dst) + off;
        const uint64_t pool = (write ? d.dst : d.src) + uint64_t(first_part + s) * part_bytes + off;
        uint8_t* dst = reinterpret_cast<uint8_t*>(write ? pool : local);
        const uint8_t* src = reinterpret_cast<const uint8_t*>(write ? local : pool);
        if constexpr (VEC == 1) {
            for (uint32_t b = threadIdx.x; b < len; b += kLdStThreads) dst[b] = src[b];
        } else {
            copy_span<VEC>(dst, src, len);
        }
    }
    if (pub.recs) ctrl_barrier_arrive(kLdStThreads + 32);
}

// ---------------------------------------------------------------- row-sliced reads (ld/st)
struct RowGeometry {
    uint32_t rows, row_bytes, src_pitch, src_col, dst_pitch, part_bytes;
};

// GatherLaunch::rows.  Item = run c (`run` rows) of part s of block b, numbered
// (b * nparts + s) * cpp + c - which is layered_item's numbering with one group of all nparts
// parts - or, LAYERED, group-major with rel.gp parts per group, each group released by
// leave_group as in gather_read_layered.  Row r of the run:
//   pool desc.src + (first_part + s) * part_bytes + r * src_pitch + src_col   (row_bytes)
//     -> parts.base[s] + desc.dst + r * dst_pitch.
// A missing block counts once, on its first item, and its parts are left untouched; its items
// still count as arrivals.  No control warp: reads publish nothing.
// SLICED (kv_scatter_slices_kernel, GatherLaunch::slices > 1): a run is `run` (slice, row)
// pairs of the part, numbered slice-major, each placed by slice_pair (launch_plan.h).
// PIECES (kv_scatter_pieces_kernel, GatherLaunch::pieces > 1, any slices): the same items; the
// run's pairs are cut where q / piece_rows changes, and each cut, one slice's rows inside one
// piece, is copied as plain rows to desc.dst + piece_off[block * pieces + t] + the place
// piece_pair gives its first pair - one piece-offset load per cut.
template <int VEC, bool LAYERED, bool SLICED, bool PIECES = false>
__device__ __forceinline__ void scatter_rows(const CopyDesc* __restrict__ descs,
                                             const GatherParts& parts, uint32_t n,
                                             uint32_t nparts, uint32_t first_part,
                                             const RowGeometry& geo, uint32_t slices,
                                             uint32_t slice_pitch, uint32_t run, uint32_t cpp,
                                             uint32_t* status, const GroupRelease& rel,
                                             const uint64_t* piece_off = nullptr,
                                             uint32_t pieces = 1) {
    const uint32_t gp = LAYERED ? rel.gp : nparts;
    const uint32_t group_items = n * gp * cpp;
    const uint32_t total = n * nparts * cpp;
    uint32_t item = blockIdx.x;
    CopyDesc next = item < total ? descs[layered_item(item, n, gp, cpp).block] : CopyDesc{0, 0};
    for (; item < total; item += gridDim.x) {
        const CopyDesc d = next;
        const LayeredItem it = layered_item(item, n, gp, cpp);
        const uint32_t nxt = item + gridDim.x;
        if (nxt < total) next = descs[layered_item(nxt, n, gp, cpp).block];
        if (d.src != 0 && PIECES) {
            const uint32_t piece_rows = geo.rows / pieces;
            const uint32_t q0 = it.chunk * run, q1 = min(q0 + run, geo.rows * slices);
            const uint8_t* src = reinterpret_cast<const uint8_t*>(
                d.src + uint64_t(first_part + it.part) * geo.part_bytes);
            const uint64_t* off = piece_off + uint64_t(it.block) * pieces;
            for (uint32_t q = q0; q < q1;) {
                const uint32_t e = min(q1, (q / piece_rows + 1) * piece_rows);
                const PieceOffsets o = piece_pair(q, geo.rows, geo.row_bytes, geo.src_pitch,
                                                  geo.src_col, geo.dst_pitch, slice_pitch,
                                                  piece_rows);
                copy_rows<VEC>(
                    reinterpret_cast<uint8_t*>(parts.base[it.part] + d.dst + off[o.piece] + o.dst),
                    src + o.src, e - q, geo.row_bytes, geo.src_pitch, geo.dst_pitch);
                q = e;
            }
        } else if (d.src != 0 && SLICED) {
            const uint32_t q0 = it.chunk * run;
            const uint8_t* src = reinterpret_cast<const uint8_t*>(
                d.src + uint64_t(first_part + it.part) * geo.part_bytes);
            uint8_t* dst = reinterpret_cast<uint8_t*>(parts.base[it.part] + d.dst);
            copy_rows<VEC, true>(dst, src, min(run, geo.rows * slices - q0), geo.row_bytes,
                                 geo.src_pitch, geo.dst_pitch,
                                 RowSlices{q0, geo.rows, geo.src_col, slice_pitch});
        } else if (d.src != 0) {
            const uint32_t r0 = it.chunk * run;
            const uint8_t* src = reinterpret_cast<const uint8_t*>(
                d.src + uint64_t(first_part + it.part) * geo.part_bytes +
                uint64_t(r0) * geo.src_pitch + geo.src_col);
            uint8_t* dst = reinterpret_cast<uint8_t*>(parts.base[it.part] + d.dst +
                                                      uint64_t(r0) * geo.dst_pitch);
            copy_rows<VEC>(dst, src, min(run, geo.rows - r0), geo.row_bytes, geo.src_pitch,
                           geo.dst_pitch);
        } else if (threadIdx.x == 0 && item < group_items && item % (gp * cpp) == 0 && status) {
            atomicAdd(status + kStatMiss, 1u);
        }
        if constexpr (LAYERED) {
            if (nxt >= total || nxt / group_items != it.group) {
                const uint32_t lo = it.group * group_items;
                leave_group(rel, it.group, cta_items(lo, lo + group_items, blockIdx.x, gridDim.x),
                            group_items, kLdStThreads);
            }
        }
    }
}

template <int VEC, bool LAYERED>
__global__ void __launch_bounds__(kLdStThreads, 3)
    kv_scatter_rows_kernel(const CopyDesc* __restrict__ descs,
                           const __grid_constant__ GatherParts parts, uint32_t n, uint32_t nparts,
                           uint32_t first_part, RowGeometry geo, uint32_t run, uint32_t cpp,
                           uint32_t* status, GroupRelease rel) {
    scatter_rows<VEC, LAYERED, false>(descs, parts, n, nparts, first_part, geo, 1, 0, run, cpp,
                                      status, rel);
}

// GatherLaunch::slices > 1: runs of (slice, row) pairs (scatter_rows above).
template <int VEC, bool LAYERED>
__global__ void __launch_bounds__(kLdStThreads, 3)
    kv_scatter_slices_kernel(const CopyDesc* __restrict__ descs,
                             const __grid_constant__ GatherParts parts, uint32_t n,
                             uint32_t nparts, uint32_t first_part, RowGeometry geo,
                             uint32_t slices, uint32_t slice_pitch, uint32_t run, uint32_t cpp,
                             uint32_t* status, GroupRelease rel) {
    scatter_rows<VEC, LAYERED, true>(descs, parts, n, nparts, first_part, geo, slices,
                                     slice_pitch, run, cpp, status, rel);
}

// GatherLaunch::pieces > 1, one or more slices: runs cut at piece boundaries (scatter_rows).
template <int VEC, bool LAYERED>
__global__ void __launch_bounds__(kLdStThreads, 3)
    kv_scatter_pieces_kernel(const CopyDesc* __restrict__ descs,
                             const __grid_constant__ GatherParts parts, uint32_t n,
                             uint32_t nparts, uint32_t first_part, RowGeometry geo,
                             uint32_t slices, uint32_t slice_pitch, uint32_t run, uint32_t cpp,
                             uint32_t* status, GroupRelease rel, const uint64_t* piece_off,
                             uint32_t pieces) {
    scatter_rows<VEC, LAYERED, false, true>(descs, parts, n, nparts, first_part, geo, slices,
                                            slice_pitch, run, cpp, status, rel, piece_off,
                                            pieces);
}

cudaError_t launch_kv_scatter_pieces(const GatherLaunch& a, const LaunchPlan& p,
                                     const GatherParts& parts, const RowGeometry& geo,
                                     const GroupRelease& rel, cudaStream_t stream) {
    const bool layered = a.group_flags != nullptr;
    const auto go = [&](auto* kernel) {
        kernel<<<p.ctas, kLdStThreads, 0, stream>>>(a.descs, parts, a.n, a.nparts, a.first_part,
                                                    geo, a.slices, a.dst_slice_pitch, p.chunk,
                                                    p.cpb, a.status, rel, a.piece_off, a.pieces);
        return cudaGetLastError();
    };
    switch (p.kernel) {
        case Kernel::kLdSt1:
            return layered ? go(kv_scatter_pieces_kernel<1, true>)
                           : go(kv_scatter_pieces_kernel<1, false>);
        case Kernel::kLdSt32:
            return layered ? go(kv_scatter_pieces_kernel<32, true>)
                           : go(kv_scatter_pieces_kernel<32, false>);
        default:
            return layered ? go(kv_scatter_pieces_kernel<16, true>)
                           : go(kv_scatter_pieces_kernel<16, false>);
    }
}

cudaError_t launch_kv_scatter_slices(const GatherLaunch& a, const LaunchPlan& p,
                                     const GatherParts& parts, const RowGeometry& geo,
                                     const GroupRelease& rel, cudaStream_t stream) {
    const bool layered = a.group_flags != nullptr;
    const auto go = [&](auto* kernel) {
        kernel<<<p.ctas, kLdStThreads, 0, stream>>>(a.descs, parts, a.n, a.nparts, a.first_part,
                                                    geo, a.slices, a.dst_slice_pitch, p.chunk,
                                                    p.cpb, a.status, rel);
        return cudaGetLastError();
    };
    switch (p.kernel) {
        case Kernel::kLdSt1:
            return layered ? go(kv_scatter_slices_kernel<1, true>)
                           : go(kv_scatter_slices_kernel<1, false>);
        case Kernel::kLdSt32:
            return layered ? go(kv_scatter_slices_kernel<32, true>)
                           : go(kv_scatter_slices_kernel<32, false>);
        default:
            return layered ? go(kv_scatter_slices_kernel<16, true>)
                           : go(kv_scatter_slices_kernel<16, false>);
    }
}

cudaError_t launch_kv_scatter_rows(const GatherLaunch& a, cudaStream_t stream) {
    static const LdStResident res = ldst_resident(kv_scatter_rows_kernel<16, false>,
                                                  kv_scatter_rows_kernel<32, false>, kLdStThreads);
    static const LdStResident res_layered = ldst_resident(
        kv_scatter_rows_kernel<16, true>, kv_scatter_rows_kernel<32, true>, kLdStThreads);
    static const LdStResident res_sliced = ldst_resident(
        kv_scatter_slices_kernel<16, false>, kv_scatter_slices_kernel<32, false>, kLdStThreads);
    static const LdStResident res_sliced_layered = ldst_resident(
        kv_scatter_slices_kernel<16, true>, kv_scatter_slices_kernel<32, true>, kLdStThreads);
    static const LdStResident res_pieces = ldst_resident(
        kv_scatter_pieces_kernel<16, false>, kv_scatter_pieces_kernel<32, false>, kLdStThreads);
    static const LdStResident res_pieces_layered = ldst_resident(
        kv_scatter_pieces_kernel<16, true>, kv_scatter_pieces_kernel<32, true>, kLdStThreads);
    const bool layered = a.group_flags != nullptr;
    const bool sliced = a.slices > 1;
    const bool pieced = a.pieces > 1;
    if (pieced && !a.piece_off) return cudaErrorInvalidValue;
    const LaunchPlan p = plan_gather_rows(a, sm_count(),
                                          pieced   ? (layered ? res_pieces_layered : res_pieces)
                                          : sliced ? (layered ? res_sliced_layered : res_sliced)
                                          : layered ? res_layered
                                                    : res);
    if (!p.valid) return cudaErrorInvalidValue;  // the caller checks the geometry and splits
    GatherParts parts;
    std::memcpy(parts.base, a.part_base, size_t(a.nparts) * sizeof(uint64_t));
    const RowGeometry geo{a.rows, a.row_bytes, a.src_pitch, a.src_col, a.dst_pitch, a.part_bytes};
    const GroupRelease rel{a.group_flags, a.group_counters, a.group_seq, a.group_parts};
    if (pieced) return launch_kv_scatter_pieces(a, p, parts, geo, rel, stream);
    if (sliced) return launch_kv_scatter_slices(a, p, parts, geo, rel, stream);
    const auto go = [&](auto* kernel) {
        kernel<<<p.ctas, kLdStThreads, 0, stream>>>(a.descs, parts, a.n, a.nparts, a.first_part,
                                                    geo, p.chunk, p.cpb, a.status, rel);
        return cudaGetLastError();
    };
    switch (p.kernel) {
        case Kernel::kLdSt1:
            return layered ? go(kv_scatter_rows_kernel<1, true>) : go(kv_scatter_rows_kernel<1, false>);
        case Kernel::kLdSt32:
            return layered ? go(kv_scatter_rows_kernel<32, true>)
                           : go(kv_scatter_rows_kernel<32, false>);
        default:
            return layered ? go(kv_scatter_rows_kernel<16, true>)
                           : go(kv_scatter_rows_kernel<16, false>);
    }
}

// ---------------------------------------------------------------- row-sliced writes (ld/st)
// GatherLaunch::rows with write: kv_gather_ldst_kernel's items, (block, part, chunk of the
// stored part) numbered (b * nparts + s) * cpp + c, each storing one contiguous run of pool
// bytes, so the control warp (publish, or a layered writer's LayerCommit) counts arrivals
// exactly as for kv_gather_ldst.  Only the local load address differs: stored byte o of part
// s comes from parts.base[s] + desc.src + row_write_offset(o) (copy_span_rows).
// PIECES (kv_gather_pieces_write_kernel, GatherLaunch::pieces > 1): the item's stored bytes are
// cut at piece boundaries (piece_rows * src_pitch bytes), and each cut is loaded from
// parts.base[s] + desc.src + piece_off[block * pieces + t] (piece_write_offset's geometry) -
// one piece-offset load per cut.
template <int VEC, bool PIECES>
__device__ __forceinline__ void gather_rows_write(const CopyDesc* __restrict__ descs,
                                                  const GatherParts& parts, uint32_t n,
                                                  uint32_t nparts, uint32_t part_bytes,
                                                  uint32_t first_part, uint32_t chunk, uint32_t cpp,
                                                  const RowWrite& geo, const Publish& pub,
                                                  const LayerCommit& lc,
                                                  const uint64_t* piece_off = nullptr,
                                                  uint32_t pieces = 1) {
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
        if (nxt < total) next = descs[nxt / cpb];  // prefetch: descriptors may sit in host memory
        const uint32_t in_block = item % cpb;
        const uint32_t s = in_block / cpp;
        const uint32_t off = (in_block % cpp) * chunk;
        const uint32_t len = min(chunk, part_bytes - off);
        if constexpr (!PIECES) {
            const uint8_t* src = reinterpret_cast<const uint8_t*>(parts.base[s] + d.src);
            uint8_t* dst =
                reinterpret_cast<uint8_t*>(d.dst + uint64_t(first_part + s) * part_bytes + off);
            copy_span_rows<VEC>(dst, src, off, len, geo);
        } else {
            uint8_t* dst =
                reinterpret_cast<uint8_t*>(d.dst + uint64_t(first_part + s) * part_bytes + off);
            const uint32_t piece_bytes = part_bytes / pieces;
            const uint64_t* poff = piece_off + uint64_t(item / cpb) * pieces;
            for (uint32_t o = off; o < off + len;) {
                const uint32_t t = o / piece_bytes;
                const uint32_t e = min(off + len, (t + 1) * piece_bytes);
                copy_span_rows<VEC>(
                    dst + (o - off), reinterpret_cast<const uint8_t*>(parts.base[s] + d.src + poff[t]),
                    o - t * piece_bytes, e - o, geo);
                o = e;
            }
        }
    }
    if (pub.recs) ctrl_barrier_arrive(kLdStThreads + 32);
}

template <int VEC>
__global__ void __launch_bounds__(kLdStThreads + 32, 3)
    kv_gather_rows_write_kernel(const CopyDesc* __restrict__ descs,
                                const __grid_constant__ GatherParts parts, uint32_t n,
                                uint32_t nparts, uint32_t part_bytes, uint32_t first_part,
                                uint32_t chunk, uint32_t cpp, RowWrite geo, Publish pub,
                                LayerCommit lc) {
    gather_rows_write<VEC, false>(descs, parts, n, nparts, part_bytes, first_part, chunk, cpp,
                                  geo, pub, lc);
}

template <int VEC>
__global__ void __launch_bounds__(kLdStThreads + 32, 3)
    kv_gather_pieces_write_kernel(const CopyDesc* __restrict__ descs,
                                  const __grid_constant__ GatherParts parts, uint32_t n,
                                  uint32_t nparts, uint32_t part_bytes, uint32_t first_part,
                                  uint32_t chunk, uint32_t cpp, RowWrite geo, Publish pub,
                                  LayerCommit lc, const uint64_t* piece_off, uint32_t pieces) {
    gather_rows_write<VEC, true>(descs, parts, n, nparts, part_bytes, first_part, chunk, cpp, geo,
                                 pub, lc, piece_off, pieces);
}

cudaError_t launch_kv_gather_rows_write(const GatherLaunch& a, cudaStream_t stream) {
    constexpr int T = kLdStThreads + 32;
    static const LdStResident res =
        ldst_resident(kv_gather_rows_write_kernel<16>, kv_gather_rows_write_kernel<32>, T);
    static const LdStResident res_pieces =
        ldst_resident(kv_gather_pieces_write_kernel<16>, kv_gather_pieces_write_kernel<32>, T);
    const bool pieced = a.pieces > 1;
    if (pieced && !a.piece_off) return cudaErrorInvalidValue;
    const LaunchPlan p = plan_gather_rows_write(a, sm_count(), pieced ? res_pieces : res);
    if (!p.valid) return cudaErrorInvalidValue;  // the caller checks the geometry and splits
    GatherParts parts;
    std::memcpy(parts.base, a.part_base, size_t(a.nparts) * sizeof(uint64_t));
    const RowWrite geo{a.row_bytes, a.src_pitch, a.dst_pitch, a.dst_slice_pitch};
    if (pieced) {
        const auto go = [&](auto* kernel) {
            kernel<<<p.ctas, T, 0, stream>>>(a.descs, parts, a.n, a.nparts, a.part_bytes,
                                             a.first_part, p.chunk, p.cpb, geo, publish_of(a, true),
                                             layer_of(a), a.piece_off, a.pieces);
            return cudaGetLastError();
        };
        return p.kernel == Kernel::kLdSt1    ? go(kv_gather_pieces_write_kernel<1>)
               : p.kernel == Kernel::kLdSt32 ? go(kv_gather_pieces_write_kernel<32>)
                                             : go(kv_gather_pieces_write_kernel<16>);
    }
    const auto go = [&](auto* kernel) {
        kernel<<<p.ctas, T, 0, stream>>>(a.descs, parts, a.n, a.nparts, a.part_bytes, a.first_part,
                                         p.chunk, p.cpb, geo, publish_of(a, true), layer_of(a));
        return cudaGetLastError();
    };
    switch (p.kernel) {
        case Kernel::kLdSt1:
            return go(kv_gather_rows_write_kernel<1>);
        case Kernel::kLdSt32:
            return go(kv_gather_rows_write_kernel<32>);
        default:
            return go(kv_gather_rows_write_kernel<16>);
    }
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
    if (a.rows)
        return a.write ? launch_kv_gather_rows_write(a, stream) : launch_kv_scatter_rows(a, stream);
    if (a.pieces != 1) return cudaErrorInvalidValue;  // pieces split rows
    constexpr int T = kLdStThreads + 32;
    static const LdStResident res =
        ldst_resident(kv_gather_ldst_kernel<16>, kv_gather_ldst_kernel<32>, T);
    static const LdStResident res_layered =
        ldst_resident(kv_gather_ldst_kernel<16, true>, kv_gather_ldst_kernel<32, true>, T);
    const LaunchPlan p = layered ? plan_gather_layered(a, sm_count(), res_layered)
                                 : plan_gather(a, sm_count(), res);
    if (!p.valid) return cudaErrorInvalidValue;  // the caller splits the batch
    if (p.kernel == Kernel::kTma) return launch_kv_pipe_gather(a, stream);
    GatherParts parts;
    std::memcpy(parts.base, a.part_base, size_t(a.nparts) * sizeof(uint64_t));
    const GroupRelease rel{a.group_flags, a.group_counters, a.group_seq, a.group_parts};
    const auto go = [&](auto* kernel) {
        kernel<<<p.ctas, T, 0, stream>>>(a.descs, parts, a.n, a.nparts, a.part_bytes, a.first_part,
                                         p.chunk, p.cpb, a.write, publish_of(a, a.write),
                                         layer_of(a), rel);
        return cudaGetLastError();
    };
    switch (p.kernel) {
        case Kernel::kLdSt1:
            return layered ? go(kv_gather_ldst_kernel<1, true>) : go(kv_gather_ldst_kernel<1>);
        case Kernel::kLdSt32:
            return layered ? go(kv_gather_ldst_kernel<32, true>) : go(kv_gather_ldst_kernel<32>);
        default:
            return layered ? go(kv_gather_ldst_kernel<16, true>) : go(kv_gather_ldst_kernel<16>);
    }
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
