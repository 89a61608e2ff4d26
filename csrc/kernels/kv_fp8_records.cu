// fp8 token records (Fp8Records, kernels.h): the gathered fp8 movers of MLA latent pages.
//
//   kv_write_fp8_records : bf16 part [token][latent + rope] -> one record per token,
//                          [latent x e4m3][latent / 128 x fp32 scale][rope x bf16], written
//                          straight into the (peer) pool block, then the in-band commit
//                          (gather_items' control warp: one-shot or a layered writer's).
//   kv_read_fp8_records  : records -> bf16 part, plain or layered (scatter_items).
//   kv_{write,read}_fp8_records_pieces : the same with pieces (GatherLaunch::rows.pieces = k >
//                          1): each part's tokens are k runs of tokens / k tokens, run t of
//                          block b at its local offset + piece_off[b * k + t] - a chunk of k
//                          engine pages stored as the records of one page of k times the tokens.
//
// The latent is quantised in 128-element rows of the fp8 row contract (fp8_row.cuh): a
// half-warp owns one row per step as in kv_fp8.cu's write_fp8 (lane l: elements 8l..8l+7, one
// 16-byte load), reduces |x| max with shuffles inside the half and stores 8 e4m3 bytes per lane.
// The rope elements are copied in 16-byte vectors, NaN payloads included.  A read dequantises
// each 8-element e4m3 vector with its row's scale into one 16-byte store, and copies the rope
// back.  Reads and writes use ld/st only, for local and peer pools alike.
#include <cuda_bf16.h>

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

constexpr int kThreads = kLdStThreads;
constexpr int kWarps = kThreads / 32;
constexpr uint32_t kRow = 128;  // latent elements sharing a scale
constexpr int kRowPairs = 4;    // 8 rows = 2 KB of bf16 in flight per warp, as in write_fp8
constexpr int kVecs = 4;        // 16-byte vectors in flight per thread in the other loops

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

// The rope elements of nt tokens: 16-byte vectors from `src` (token pitch sp bytes) to `dst`
// (token pitch dp bytes), vpt vectors per token, kVecs in flight per thread.
__device__ __forceinline__ void copy_rope(uint8_t* dst, uint32_t dp, const uint8_t* src,
                                          uint32_t sp, uint32_t nt, uint32_t vpt) {
    const uint32_t nvec = nt * vpt;
    for (uint32_t i = threadIdx.x; i < nvec; i += kVecs * kThreads) {
        uint4 v[kVecs];
        uint32_t out[kVecs];
#pragma unroll
        for (int u = 0; u < kVecs; ++u) {
            const uint32_t k = i + u * kThreads;
            if (k >= nvec) continue;
            const uint32_t t = k / vpt, c = k - t * vpt;
            v[u] = ld_stream_v4(src + t * sp + 16 * c);
            out[u] = t * dp + 16 * c;
        }
#pragma unroll
        for (int u = 0; u < kVecs; ++u)
            if (i + u * kThreads < nvec) st_v4(dst + out[u], v[u]);
    }
}

// nt tokens from `src` (bf16, token pitch 2 * token_elems bytes) as records at `rec`.  Row k of
// the run is latent row g = k % G of token k / G (G = latent / 128 rows per token); the row
// loop is write_fp8's.  nt * token_elems stays below 2^31 (plan_gather_fp8_records' items).
__device__ __forceinline__ void write_records(uint8_t* rec, const uint8_t* src, uint32_t nt,
                                              const Fp8Records& r) {
    const uint32_t G = r.latent / kRow, tb = 2 * r.token_elems(), rb = r.record_bytes();
    const uint32_t rows = nt * G;
    const uint32_t warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const uint32_t half = lane >> 4, hl = lane & 15;
    constexpr uint32_t kStep = 2 * kRowPairs;
    for (uint32_t r0 = warp * kStep; r0 < rows; r0 += kWarps * kStep) {
        uint4 v[kRowPairs];
#pragma unroll
        for (int u = 0; u < kRowPairs; ++u) {
            const uint32_t k = r0 + 2 * u + half;
            const uint32_t t = k / G, g = k - t * G;
            if (k < rows) v[u] = ld_stream_v4(src + t * tb + g * (2 * kRow) + hl * 16);
        }
#pragma unroll
        for (int u = 0; u < kRowPairs; ++u) {
            const uint32_t k = r0 + 2 * u + half;
            const bool live = k < rows;
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
            const uint32_t t = k / G, g = k - t * G;
            uint8_t* q = rec + t * rb;
            *reinterpret_cast<uint2*>(q + g * kRow + hl * 8) = quant8(f, 1.f / scale);
            if (hl == 0) *reinterpret_cast<float*>(q + r.scale_offset() + 4 * g) = scale;
        }
    }
    copy_rope(rec + r.rope_offset(), rb, src + 2 * r.latent, tb, nt, r.rope / 8);
}

// nt records at `rec` dequantised to bf16 tokens at `dst` (token pitch 2 * token_elems bytes):
// the (token, 8-element vector) pairs of the latent flattened over the CTA, each vector an
// 8-byte e4m3 load inside one row and the scale of that row, then the rope.
__device__ __forceinline__ void read_records(uint8_t* dst, const uint8_t* rec, uint32_t nt,
                                             const Fp8Records& r) {
    const uint32_t vpt = r.latent / 8, tb = 2 * r.token_elems(), rb = r.record_bytes();
    const uint32_t nvec = nt * vpt;
    for (uint32_t i = threadIdx.x; i < nvec; i += kVecs * kThreads) {
        uint2 v[kVecs];
        float sc[kVecs];
        uint32_t out[kVecs];
#pragma unroll
        for (int u = 0; u < kVecs; ++u) {
            const uint32_t k = i + u * kThreads;
            if (k >= nvec) continue;
            const uint32_t t = k / vpt, c = k - t * vpt;
            const uint8_t* q = rec + t * rb;
            v[u] = ld_u2(q + 8 * c);
            sc[u] = __uint_as_float(ld_u1(q + r.scale_offset() + 4 * (c / (kRow / 8))));
            out[u] = t * tb + 16 * c;
        }
#pragma unroll
        for (int u = 0; u < kVecs; ++u)
            if (i + u * kThreads < nvec)
                *reinterpret_cast<uint4*>(dst + out[u]) = dequant8(v[u], sc[u]);
    }
    copy_rope(dst + 2 * r.latent, tb, rec + r.rope_offset(), rb, nt, r.rope / 8);
}

// Writes: gather_items' walk over (block, part, run of `chunk` tokens); part s of block b is
// loaded from parts.base[s] + desc.src and stored as part first_part + s of the pool block.
// Warp 8 is the control warp: the in-band commit, or a layered writer's LayerCommit.
__global__ void __launch_bounds__(kThreads + 32)
    kv_write_fp8_records_kernel(const CopyDesc* __restrict__ descs,
                                const __grid_constant__ GatherParts parts, uint32_t n,
                                uint32_t nparts, uint32_t tokens, uint32_t chunk, uint32_t cpp,
                                uint32_t first_part, Fp8Records r, Publish pub, LayerCommit lc) {
    gather_items(descs, n, nparts, tokens, chunk, cpp, pub, lc,
                 [&](const CopyDesc& d, uint32_t, uint32_t s, uint32_t t0, uint32_t nt) {
                     const uint8_t* src = reinterpret_cast<const uint8_t*>(parts.base[s] + d.src) +
                                          size_t(t0) * 2 * r.token_elems();
                     uint8_t* rec = reinterpret_cast<uint8_t*>(
                         d.dst + fp8_record_offset(r, tokens, first_part + s, t0));
                     write_records(rec, src, nt, r);
                 });
}

// Reads: scatter_items' walk (misses counted once per block, parts left untouched; LAYERED:
// group-major items and group releases).  Stored part first_part + s lands at parts.base[s] +
// desc.dst.
template <bool LAYERED>
__global__ void __launch_bounds__(kThreads)
    kv_read_fp8_records_kernel(const CopyDesc* __restrict__ descs,
                               const __grid_constant__ GatherParts parts, uint32_t n,
                               uint32_t nparts, uint32_t tokens, uint32_t chunk, uint32_t cpp,
                               uint32_t first_part, Fp8Records r, uint32_t* status,
                               GroupRelease rel) {
    scatter_items<LAYERED>(descs, n, nparts, cpp, status, rel, [&](const CopyDesc& d,
                                                                  const LayeredItem& it) {
        const uint32_t t0 = it.chunk * chunk;
        const uint8_t* rec = reinterpret_cast<const uint8_t*>(
            d.src + fp8_record_offset(r, tokens, first_part + it.part, t0));
        uint8_t* dst = reinterpret_cast<uint8_t*>(parts.base[it.part] + d.dst) +
                       size_t(t0) * 2 * r.token_elems();
        read_records(dst, rec, min(chunk, tokens - t0), r);
    });
}

// With pieces: the items of the whole-part kernels (runs of `chunk` tokens, which need not line
// up with the pieces: at 512 + 64 a run is 14 tokens) are cut where the piece t / pt changes
// (pt = tokens / pieces), and each cut runs the whole-part body from its piece's place in the
// caller's part: piece_off[block * pieces + t / pt] + (t % pt) tokens, one piece-offset load per
// cut.  A record, and so a scale row, never crosses a token, so a cut never splits one.  The
// reads' minimum of 3 CTAs per SM lets ptxas give them 80 registers; without it the layered
// read was held to 64 and spilled.
__global__ void __launch_bounds__(kThreads + 32)
    kv_write_fp8_records_pieces_kernel(const CopyDesc* __restrict__ descs,
                                       const __grid_constant__ GatherParts parts, uint32_t n,
                                       uint32_t nparts, uint32_t tokens, uint32_t chunk,
                                       uint32_t cpp, uint32_t first_part, Fp8Records r,
                                       const uint64_t* __restrict__ piece_off, uint32_t pieces,
                                       Publish pub, LayerCommit lc) {
    gather_items(descs, n, nparts, tokens, chunk, cpp, pub, lc,
                 [&](const CopyDesc& d, uint32_t block, uint32_t s, uint32_t t0, uint32_t nt) {
                     const uint32_t pt = tokens / pieces, tb = 2 * r.token_elems();
                     const uint64_t* off = piece_off + uint64_t(block) * pieces;
                     const uint64_t src = parts.base[s] + d.src;
                     uint8_t* rec = reinterpret_cast<uint8_t*>(
                         d.dst + fp8_record_offset(r, tokens, first_part + s, t0));
                     for (uint32_t t = t0; t < t0 + nt;) {
                         const uint32_t p = t / pt, e = min(t0 + nt, (p + 1) * pt);
                         write_records(rec + size_t(t - t0) * r.record_bytes(),
                                       reinterpret_cast<const uint8_t*>(src + off[p]) +
                                           size_t(t - p * pt) * tb,
                                       e - t, r);
                         t = e;
                     }
                 });
}

template <bool LAYERED>
__global__ void __launch_bounds__(kThreads, 3)
    kv_read_fp8_records_pieces_kernel(const CopyDesc* __restrict__ descs,
                                      const __grid_constant__ GatherParts parts, uint32_t n,
                                      uint32_t nparts, uint32_t tokens, uint32_t chunk,
                                      uint32_t cpp, uint32_t first_part, Fp8Records r,
                                      const uint64_t* __restrict__ piece_off, uint32_t pieces,
                                      uint32_t* status, GroupRelease rel) {
    scatter_items<LAYERED>(descs, n, nparts, cpp, status, rel, [&](const CopyDesc& d,
                                                                  const LayeredItem& it) {
        const uint32_t pt = tokens / pieces, tb = 2 * r.token_elems();
        const uint32_t t0 = it.chunk * chunk, t1 = min(t0 + chunk, tokens);
        const uint64_t* off = piece_off + uint64_t(it.block) * pieces;
        const uint64_t dst = parts.base[it.part] + d.dst;
        const uint8_t* rec = reinterpret_cast<const uint8_t*>(
            d.src + fp8_record_offset(r, tokens, first_part + it.part, t0));
        for (uint32_t t = t0; t < t1;) {
            const uint32_t p = t / pt, e = min(t1, (p + 1) * pt);
            read_records(reinterpret_cast<uint8_t*>(dst + off[p]) + size_t(t - p * pt) * tb,
                         rec + size_t(t - t0) * r.record_bytes(), e - t, r);
            t = e;
        }
    });
}

template <bool WRITE, bool LAYERED>
cudaError_t launch_records(const GatherLaunch& a, uint32_t elems, cudaStream_t stream) {
    const LaunchPlan p =
        WRITE ? plan_gather_fp8_records(
                    a, elems, sm_count(),
                    cached_resident<kv_write_fp8_records_kernel, kv_write_fp8_records_kernel,
                                    kThreads + 32>())
              : plan_gather_fp8_records(
                    a, elems, sm_count(),
                    cached_resident<kv_read_fp8_records_kernel<LAYERED>,
                                    kv_read_fp8_records_kernel<LAYERED>, kThreads>());
    if (!p.valid) return cudaErrorInvalidValue;
    const GatherParts parts = parts_of(a);
    const uint32_t tokens = elems / a.records.token_elems();
    if constexpr (WRITE)
        kv_write_fp8_records_kernel<<<p.ctas, kThreads + 32, 0, stream>>>(
            a.descs, parts, a.n, a.nparts, tokens, p.chunk, p.cpb, a.first_part, a.records,
            publish_of(a, true), layer_of(a));
    else
        kv_read_fp8_records_kernel<LAYERED><<<p.ctas, kThreads, 0, stream>>>(
            a.descs, parts, a.n, a.nparts, tokens, p.chunk, p.cpb, a.first_part, a.records,
            a.status, release_of(a));
    return cudaGetLastError();
}

// The same plan and grid for pieces, with the residency of the pieces kernels.
template <bool WRITE, bool LAYERED>
cudaError_t launch_records_pieces(const GatherLaunch& a, uint32_t elems, cudaStream_t stream) {
    const LaunchPlan p =
        WRITE ? plan_gather_fp8_records(
                    a, elems, sm_count(),
                    cached_resident<kv_write_fp8_records_pieces_kernel,
                                    kv_write_fp8_records_pieces_kernel, kThreads + 32>())
              : plan_gather_fp8_records(
                    a, elems, sm_count(),
                    cached_resident<kv_read_fp8_records_pieces_kernel<LAYERED>,
                                    kv_read_fp8_records_pieces_kernel<LAYERED>, kThreads>());
    if (!p.valid) return cudaErrorInvalidValue;
    const GatherParts parts = parts_of(a);
    const uint32_t tokens = elems / a.records.token_elems();
    if constexpr (WRITE)
        kv_write_fp8_records_pieces_kernel<<<p.ctas, kThreads + 32, 0, stream>>>(
            a.descs, parts, a.n, a.nparts, tokens, p.chunk, p.cpb, a.first_part, a.records,
            a.piece_off, a.rows.pieces, publish_of(a, true), layer_of(a));
    else
        kv_read_fp8_records_pieces_kernel<LAYERED><<<p.ctas, kThreads, 0, stream>>>(
            a.descs, parts, a.n, a.nparts, tokens, p.chunk, p.cpb, a.first_part, a.records,
            a.piece_off, a.rows.pieces, a.status, release_of(a));
    return cudaGetLastError();
}

}  // namespace

cudaError_t launch_kv_gather_fp8_records(const GatherLaunch& a, uint32_t elems,
                                         cudaStream_t stream) {
    if (a.n == 0) return cudaSuccess;
    if (!a.part_base) return cudaErrorInvalidValue;
    const bool layered = a.group_flags != nullptr;
    if (layered && !a.group_counters) return cudaErrorInvalidValue;
    if (a.rows.pieces > 1) {  // pieces of whole tokens, at the offsets of the piece table
        if (!a.piece_off) return cudaErrorInvalidValue;
        if (a.write) return launch_records_pieces<true, false>(a, elems, stream);
        return layered ? launch_records_pieces<false, true>(a, elems, stream)
                       : launch_records_pieces<false, false>(a, elems, stream);
    }
    if (a.write) return launch_records<true, false>(a, elems, stream);
    return layered ? launch_records<false, true>(a, elems, stream)
                   : launch_records<false, false>(a, elems, stream);
}

}  // namespace istore::kernels
