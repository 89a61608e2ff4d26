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
//                  fp8 pages end to end (launch_kv_gather_fp8, fp8_pages.cuh), in every part
//                  shape.  With row geometry (GatherLaunch::rows) a read dequantises rows (and
//                  slices) of each stored page, a write quantises a stored page whose rows are
//                  loaded from a strided local layout (e.g. a head-major page); with
//                  rows.pieces > 1 each block's rows are in runs at the offsets of its row of
//                  the piece table.  Reads walk their items in gather_items.cuh
//                  (scatter_items), writes in write_fp8 below.
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

#include "common.cuh"
#include "fp8_pages.cuh"
#include "fp8_row.cuh"
#include "gather_items.cuh"
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

// Where a lane's 16-byte bf16 load comes from: byte offset from the page's local address of
// elements 8 * hl .. 8 * hl + 7 of 128-element row `row` of the stored page.  A template
// policy rather than a runtime branch, so the existing kernels' loop is compiled as before.
//   DenseRows  the page is contiguous bf16 (kv_write_fp8 and whole gathered parts).
//   SlicedRows a row-sliced write (GatherLaunch::rows): PartRows::write_offset of the vector's
//              byte in the part's bf16 view; the geometry is in multiples of 16 bytes, so the 8
//              elements never straddle two slices.
//   PiecedRows a row-sliced write with pieces (rows.pieces > 1): the pieced write_offset, plus
//              the piece's offset from block b's row of the piece table (block(b)).
//              Pieces split at row boundaries, rows are multiples of 8 elements, so a vector
//              never straddles two pieces; a 128-element scale group may, and each of its
//              vectors is placed on its own.
// block(b) is the policy for the items of block b.
struct DenseRows {
    __device__ __forceinline__ size_t operator()(uint32_t row, uint32_t hl) const {
        return (size_t(row) * kRow + hl * 8) * 2;
    }
    __device__ __forceinline__ DenseRows block(uint32_t) const { return *this; }
};
struct SlicedRows {
    PartRows g;
    __device__ __forceinline__ size_t operator()(uint32_t row, uint32_t hl) const {
        return g.write_offset((row * kRow + hl * 8) * 2);
    }
    __device__ __forceinline__ SlicedRows block(uint32_t) const { return *this; }
};
struct PiecedRows {
    PartRows g;
    uint32_t piece_rows;  // g.rows / g.pieces
    const uint64_t* off;  // block b's row of the piece table once bound by block(b)
    __device__ __forceinline__ size_t operator()(uint32_t row, uint32_t hl) const {
        const PairOffsets p = g.write_offset((row * kRow + hl * 8) * 2, piece_rows);
        return off[p.piece] + p.dst;
    }
    __device__ __forceinline__ PiecedRows block(uint32_t b) const {
        PiecedRows r = *this;
        r.off += uint64_t(b) * g.pieces;
        return r;
    }
};

// Threads [0, 256) quantise + store; warp 8 is the control warp (in-band commit).  Work item
// k is chunk k % cpp of page k / cpp (`pages`, fp8_pages.cuh); n blocks of pages.nparts pages.
// `load_at` places each lane's bf16 load (DenseRows / SlicedRows above).
template <typename Pages, typename LoadAt = DenseRows>
__device__ __forceinline__ void write_fp8(const CopyDesc* __restrict__ descs, uint32_t n,
                                          uint32_t elems, uint32_t chunk, uint32_t cpp,
                                          const Publish& pub, const Pages& pages,
                                          const LoadAt& load_at = {}) {
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
        const LoadAt at = load_at.block(item / cpb);
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
                if (r < rows) v[u] = ld_u4(src + at(row0 + r, hl));
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

// Gathered writes (launch_kv_gather_fp8): n blocks of nparts parts, cpp items per part, the
// part bases in the kernel parameters; write_fp8's items and commit (BlockParts<true>), each
// lane's bf16 vector placed by `load_at`: DenseRows for whole parts, SlicedRows with
// GatherLaunch::rows, PiecedRows with rows.pieces > 1.
template <typename LoadAt>
__global__ void __launch_bounds__(kThreads + 32)
    kv_write_fp8_gather_kernel(const CopyDesc* __restrict__ descs,
                               const __grid_constant__ GatherParts parts, uint32_t n,
                               uint32_t nparts, uint32_t elems, uint32_t chunk, uint32_t cpp,
                               uint32_t first_part, uint64_t stride, LoadAt load_at, Publish pub,
                               LayerCommit lc) {
    write_fp8(descs, n, elems, chunk, cpp, pub,
              BlockParts<true>{&parts, nparts, first_part, stride, lc}, load_at);
}

// ---------------------------------------------------------------- gathered reads
// The units of the fp8 reads' row loops: a geometry's source side (row_bytes, src_pitch,
// src_col) in elements of the part's bf16 view, its destination side in bytes.  Built once per
// launch from its byte geometry (GatherLaunch::rows): derived inside the kernel, the halved
// values took registers that the parameter bank holds for free.
PartRows fp8_source_elems(const PartRows& g) {
    PartRows e = g;
    e.row_bytes = g.row_bytes / 2;
    e.src_pitch = g.src_pitch / 2;
    e.src_col = g.src_col / 2;
    return e;
}

constexpr int kRowVecs = 4;  // (row, vector) pairs in flight per thread: 4 x 16 B of bf16

// `nrows` rows of one stored fp8 part `q` (scales at q + elems) from element e0 on, dequantised
// to dst, in the units of fp8_source_elems: row r of the run takes e.row_bytes / 8 8-element
// vectors from element e0 + r * e.src_pitch and lands at r * e.dst_pitch bytes from dst.  The
// 256 threads walk the (row, vector) pairs flattened together, as copy_rows (copy_span.cuh)
// does, so one 128-element KV head (16 vectors) per row keeps every thread busy.  A vector is 8
// e4m3 bytes at q + e and the scale of its group at scales[e / 128]: the geometry keeps e a
// multiple of 8, so a vector never straddles two scale groups.
// SLICED (rows.slices > 1): dst is the part's destination and the nrows units are the (slice,
// row) pairs e0 .. e0 + nrows - 1 of the part, placed by e.pair: (slice, row, vector) triples
// flattened.
template <bool SLICED = false>
__device__ __forceinline__ void read_fp8_rows(uint8_t* dst, const uint8_t* q, const float* scales,
                                              uint32_t e0, uint32_t nrows, const PartRows& e) {
    const uint32_t vpr = e.row_bytes / 8;
    const uint32_t nvec = nrows * vpr;
    for (uint32_t i = threadIdx.x; i < nvec; i += kRowVecs * kThreads) {
        uint2 v[kRowVecs];
        float sc[kRowVecs];
        // a sliced destination lies within 32 bits (PartRows::ok), plain rows may not
        std::conditional_t<SLICED, uint32_t, size_t> out[kRowVecs];
#pragma unroll
        for (int u = 0; u < kRowVecs; ++u) {
            const uint32_t k = i + u * kThreads;
            if (k >= nvec) continue;
            const uint32_t p = k / vpr, c = k - p * vpr;
            uint32_t el;
            if constexpr (SLICED) {
                const PairOffsets o = e.pair(e0 + p);
                el = o.src + 8 * c;
                out[u] = o.dst + 16 * c;
            } else {
                el = e0 + p * e.src_pitch + 8 * c;
                out[u] = size_t(p) * e.dst_pitch + 16 * c;
            }
            v[u] = ld_u2(q + el);
            sc[u] = __uint_as_float(ld_u1(scales + el / kRow));
        }
#pragma unroll
        for (int u = 0; u < kRowVecs; ++u) {
            if (i + u * kThreads >= nvec) continue;
            *reinterpret_cast<uint4*>(dst + out[u]) = dequant8(v[u], sc[u]);
        }
    }
}

// Reads: gather_items.cuh's scatter_items walk, one body per part shape.  Item chunk c of part s
// of block b reads stored part first_part + s, at desc.src + (first_part + s) * stride, into
// local parts.base[s] + desc.dst:
//   kWhole   rows [c * chunk, +chunk) / 128 of the page, a half-warp per 128-element row as in
//            kv_read_fp8_kernel;
//   kRows    rows [c * chunk, +chunk) (GatherLaunch::rows: read_fp8_rows);
//   kSlices  (slice, row) pairs [c * chunk, +chunk), numbered slice-major (read_fp8_rows<true>);
//   kPieces  the same pairs (rows.pieces > 1, any slices), cut where q / piece_rows changes as
//            in kv_copy.cu's kv_scatter_ldst_kernel; each cut is read as plain rows to desc.dst +
//            piece_off[block * pieces + t] + the place PartRows::pair gives its first pair - one
//            piece-offset load per cut.
// `e` is the launch's row geometry in fp8_source_elems' units.
// (This kernel and kv_read_fp8_kernel share the row maths, not the loop: inlining one loop body
// into both changed how the compiler schedules kv_read_fp8_kernel.)
static_assert(kThreads == kLdStThreads, "scatter_items releases groups on kLdStThreads threads");
template <bool LAYERED, PartShape S>
__global__ void __launch_bounds__(kThreads)
    kv_read_fp8_scatter_kernel(const CopyDesc* __restrict__ descs,
                               const __grid_constant__ GatherParts parts, uint32_t n,
                               uint32_t nparts, uint32_t first_part, uint32_t chunk, uint32_t cpp,
                               uint64_t stride, uint32_t elems, PartRows e,
                               const uint64_t* piece_off, uint32_t* status, GroupRelease rel) {
    scatter_items<LAYERED>(descs, n, nparts, cpp, status, rel, [&](const CopyDesc& d,
                                                                  const LayeredItem& it) {
        const uint8_t* q =
            reinterpret_cast<const uint8_t*>(d.src + uint64_t(first_part + it.part) * stride);
        const float* scales = reinterpret_cast<const float*>(q + elems);
        uint8_t* dst = reinterpret_cast<uint8_t*>(parts.base[it.part] + d.dst);
        if constexpr (S == PartShape::kWhole) {
            const uint32_t warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
            const uint32_t half = lane >> 4, hl = lane & 15;
            constexpr uint32_t kStep = 2 * kRowPairs;
            const uint32_t e0 = it.chunk * chunk;
            const uint32_t rows = min(chunk, elems - e0) / kRow;
            const uint32_t row0 = e0 / kRow;
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
        } else if constexpr (S == PartShape::kRows) {
            const uint32_t r0 = it.chunk * chunk;
            read_fp8_rows(dst + uint64_t(r0) * e.dst_pitch, q, scales, r0 * e.src_pitch + e.src_col,
                          min(chunk, e.rows - r0), e);
        } else if constexpr (S == PartShape::kSlices) {
            const uint32_t q0 = it.chunk * chunk;
            read_fp8_rows<true>(dst, q, scales, q0, min(chunk, e.rows * e.slices - q0), e);
        } else {
            const uint32_t piece_rows = e.rows / e.pieces;
            const uint32_t q0 = it.chunk * chunk, q1 = min(q0 + chunk, e.rows * e.slices);
            const uint64_t* off = piece_off + uint64_t(it.block) * e.pieces;
            for (uint32_t p = q0; p < q1;) {
                const uint32_t end = min(q1, (p / piece_rows + 1) * piece_rows);
                const PairOffsets o = e.pair(p, piece_rows);
                read_fp8_rows(dst + off[o.piece] + o.dst, q, scales, o.src, end - p, e);
                p = end;
            }
        }
    });
}

// One gathered fp8 ld/st launch of shape S: its plan (whole pages may take the TMA pipeline of
// kv_fp8_pipe.cu), then the kernel.  The row plans' grid follows the launched kernel's residency.
template <bool WRITE, bool LAYERED, PartShape S>
cudaError_t launch_fp8_gather(const GatherLaunch& a, uint32_t elems, int variant,
                              const GatherParts& parts, cudaStream_t stream) {
    const uint64_t stride = fp8_gather_bytes(1, elems);
    const auto load_at = [&] {
        if constexpr (S == PartShape::kWhole)
            return DenseRows{};
        else if constexpr (S == PartShape::kRows)
            return SlicedRows{a.rows};
        else
            return PiecedRows{a.rows, a.rows.rows / a.rows.pieces, a.piece_off};
    }();
    using LoadAt = std::decay_t<decltype(load_at)>;
    LaunchPlan p;
    if constexpr (S == PartShape::kWhole) {
        p = plan_gather_fp8(a, elems, variant, sm_count());
    } else if constexpr (WRITE) {
        p = plan_gather_fp8_rows_write(
            a, elems, sm_count(),
            cached_resident<kv_write_fp8_gather_kernel<LoadAt>, kv_write_fp8_gather_kernel<LoadAt>,
                            kThreads + 32>());
    } else {
        p = plan_gather_fp8_rows(
            a, elems, sm_count(),
            cached_resident<kv_read_fp8_scatter_kernel<LAYERED, S>,
                            kv_read_fp8_scatter_kernel<LAYERED, S>, kThreads>());
    }
    if (!p.valid) return cudaErrorInvalidValue;  // the caller checks the geometry and splits
    if (p.kernel != Kernel::kLdStFp8) return launch_kv_fp8_pipe_gather(a, elems, stream);
    if constexpr (WRITE) {
        kv_write_fp8_gather_kernel<<<p.ctas, kThreads + 32, 0, stream>>>(
            a.descs, parts, a.n, a.nparts, elems, p.chunk, p.cpb, a.first_part, stride, load_at,
            publish_of(a, true), layer_of(a));
    } else {
        kv_read_fp8_scatter_kernel<LAYERED, S><<<p.ctas, kThreads, 0, stream>>>(
            a.descs, parts, a.n, a.nparts, a.first_part, p.chunk, p.cpb, stride, elems,
            fp8_source_elems(a.rows), a.piece_off, a.status, release_of(a));
    }
    return cudaGetLastError();
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
    if (a.part_scale) return launch_kv_gather_e4m3(a, elems, stream);
    if (a.records.latent) return launch_kv_gather_fp8_records(a, elems, stream);
    if (a.n == 0) return cudaSuccess;
    if (!a.part_base) return cudaErrorInvalidValue;
    const bool layered = a.group_flags != nullptr;
    if (layered && !a.group_counters) return cudaErrorInvalidValue;
    // pieces split rows, at the offsets of the piece table
    if (a.rows.pieces != 1 && (!a.rows.rows || !a.piece_off)) return cudaErrorInvalidValue;
    const GatherParts parts = parts_of(a);
    if (a.write)
        return with_shape<true>(a, [&](auto s) {
            return launch_fp8_gather<true, false, decltype(s)::value>(a, elems, variant, parts,
                                                                      stream);
        });
    return with_shape<false>(a, [&](auto s) {
        constexpr PartShape S = decltype(s)::value;
        return layered ? launch_fp8_gather<false, true, S>(a, elems, variant, parts, stream)
                       : launch_fp8_gather<false, false, S>(a, elems, variant, parts, stream);
    });
}

}  // namespace istore::kernels
