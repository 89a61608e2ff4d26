// fp8 KV path on the TMA pipeline: quantise / dequantise between two bulk-async copies.
//
//   write : bf16 page --cp.async.bulk--> SMEM tile (64 rows x 128)   [loader warp]
//           4 compute warps: per-row amax, e4m3 cast, scale           (shared -> shared)
//           SMEM payload + scales --cp.async.bulk--> pool block       [storer warp]
//           then the in-band commit                                   [control warp]
//   read  : payload + scales --cp.async.bulk--> SMEM, dequantise to bf16 in SMEM,
//           --cp.async.bulk--> destination page.
//   fused read : the (otherwise idle) third warp is the RESOLVER of resolve.cuh - it hashes the
//           keys, probes the HBM index and feeds {pool block, destination} to loader and storer
//           through the shared-memory queue, then re-checks the entries after the copy:
//           read_cache_fp8 through the device index is ONE launch instead of lookup +
//           read + validate.
// Compared with kv_fp8.cu (every thread loads 16 bytes, stores 8, one scalar store per row
// for the scale): the fabric sees whole 8 KB / 256 B bulk requests instead of 8-byte stores,
// the scales of a tile travel as one vector, and the global loads no longer sit in the
// dependency chain of the conversion.  Half the NVLink bytes of a bf16 write and no separate
// cast kernel - the reference moves opaque bytes only (infinistore/lib.py:377-379).
//
// Pool block layout (unchanged): [elems x e4m3][elems/128 x fp32 scale].
// Needs elems % 512 == 0 (scale vectors of a tile are 16-byte multiples); launch_kv_{write,
// read}_fp8 fall back to kv_fp8.cu otherwise.  Pages that are not 16-byte aligned are refused
// by plan_fp8 for both flavours.  The row maths are fp8_row.cuh's, shared with kv_fp8.cu.
#include <cuda_bf16.h>
#include <cuda_fp16.h>

#include <cstring>
#include <type_traits>

#include "common.cuh"
#include "fp8_pages.cuh"
#include "fp8_row.cuh"
#include "kernels.h"
#include "launch_plan.h"
#include "publish.cuh"
#include "resolve.cuh"

namespace istore::kernels {

namespace {

using namespace dev;
using namespace fp8row;

constexpr uint32_t kRow = 128;                  // elements sharing a scale
constexpr uint32_t kTileRows = 64;              // rows per tile
constexpr uint32_t kTileElems = kRow * kTileRows;
static_assert(kTileElems == kFp8Chunk, "plan_fp8 cuts pages into whole tiles");
constexpr uint32_t kTileBf16 = kTileElems * 2;  // 16 KB
constexpr uint32_t kTileQ = kTileElems;         // 8 KB
constexpr uint32_t kTileScale = kTileRows * 4;  // 256 B
constexpr int kInStages = 4, kOutStages = 3, kLag = 2;

struct Smem {
    // [kInStages][in tile] then [kOutStages][out tile]; sizes depend on the direction
    uint64_t full_in[kInStages], empty_in[kInStages], full_out[kOutStages], empty_out[kOutStages];
};

// Work schedule: item k of a CTA = chunk (item % cpb) of page (item / cpb); a chunk is a run
// of whole tiles (the last tile of a page may be short: rows % 4 == 0 is guaranteed).
struct Fp8Shape {
    uint32_t n, elems, chunk_elems, cpb;
};

// NCW compute warps (4 or 8) besides the loader, storer and control / resolver warps.
// FUSED (reads only): descriptors come from the resolver warp's queue instead of `descs`.
// `pages` (fp8_pages.cuh) maps page item / sh.cpb to its descriptor: sh.n pages, grouped into
// blocks of pages.nparts for the commit and the miss count.
template <bool WRITE, int NCW, bool FUSED, typename Pages>
__device__ __forceinline__ void fp8_pipe(const CopyDesc* __restrict__ descs, const Fp8Shape& sh,
                                         const Publish& pub, uint32_t* status,
                                         const ResolveArgs& ra, const Pages& pages) {
    static_assert(!(WRITE && FUSED), "only reads resolve keys");
    static_assert(!(FUSED && Pages::nparts != 1), "the resolver feeds whole pages");
    extern __shared__ __align__(128) uint8_t smem[];
    __shared__ Smem bars;
    __shared__ __align__(16) ResolveQueue rq;
    constexpr uint32_t kInTile = WRITE ? kTileBf16 : (kTileQ + kTileScale);
    constexpr uint32_t kOutTile = WRITE ? (kTileQ + kTileScale) : kTileBf16;
    uint8_t* in_ring = smem;
    uint8_t* out_ring = smem + kInStages * kInTile;
    const uint32_t total = sh.n * sh.cpb;
    const uint32_t grid = gridDim.x;
    const uint32_t nitems = blockIdx.x < total ? (total - blockIdx.x + grid - 1) / grid : 0;
    const uint32_t warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    if (threadIdx.x == 0) {
        for (int s = 0; s < kInStages; ++s) {
            mbar_init(&bars.full_in[s], 1);
            mbar_init(&bars.empty_in[s], NCW);
        }
        for (int t = 0; t < kOutStages; ++t) {
            mbar_init(&bars.full_out[t], NCW);
            mbar_init(&bars.empty_out[t], 1);
        }
        if (FUSED) resolve_queue_init(rq);
        mbar_fence_init();
    }
    __syncthreads();
    if (warp == 2) {  // control warp: in-band commit (writes) / resolver (fused reads)
        if (WRITE && pub.recs)
            pages.commit(pub, lane, blockIdx.x, nitems, grid, sh.cpb * pages.nparts, 64);
        if (FUSED)
            resolver_warp(ra, rq, sh.elems + sh.elems / kRow * 4, blockIdx.x, grid,
                          sh.cpb, nitems, lane);
        return;
    }
    // Every role walks the same sequence of tiles.  `role`: 0 loader, 1 storer (hands queue
    // halves back to the resolver), 2 compute (never looks at a descriptor when FUSED: a
    // missing block's tile is converted from whatever the slot holds and not stored).
    auto for_each_tile = [&](auto role, auto&& fn) {
        [[maybe_unused]] constexpr int kRole = decltype(role)::value;
        uint32_t q = 0;  // running tile number of this CTA
        for (uint32_t k = 0; k < nitems; ++k) {
            const uint32_t item = blockIdx.x + k * grid;
            CopyDesc d;
            bool head = true;  // a block's first page: its first tile counts a miss
            if constexpr (!FUSED) {
                d = pages.at(descs, item / sh.cpb);
                head = pages.head(item / sh.cpb);
            }
            else if constexpr (kRole == 2)
                d = CopyDesc{1, 0};
            else  // one lane per role makes this call: not warp wide
                d = resolved_desc<kRole == 1, false>(rq, k, 0);
            const uint32_t e0 = (item % sh.cpb) * sh.chunk_elems;
            const uint32_t e1 = min(sh.elems, e0 + sh.chunk_elems);
            for (uint32_t e = e0; e < e1; e += kTileElems, ++q)
                fn(q, d, e, min(kTileElems, e1 - e) / kRow, head && e == 0);
        }
    };
    if (warp == 0) {  // ---- loader
        if (lane != 0) return;
        for_each_tile(std::integral_constant<int, 0>{},
                      [&](uint32_t q, const CopyDesc& d, uint32_t e, uint32_t rows, bool) {
            const uint32_t s = q % kInStages, use = q / kInStages;
            if (use) mbar_wait(&bars.empty_in[s], (use - 1) & 1);
            uint8_t* tile = in_ring + s * kInTile;
            if (!d.src) {
                mbar_arrive(&bars.full_in[s]);
                return;
            }
            const uint8_t* src = reinterpret_cast<const uint8_t*>(d.src);
            if constexpr (WRITE) {
                mbar_expect_tx(&bars.full_in[s], rows * kRow * 2);
                bulk_g2s(tile, src + size_t(e) * 2, rows * kRow * 2, &bars.full_in[s]);
            } else {
                mbar_expect_tx(&bars.full_in[s], rows * kRow + rows * 4);
                bulk_g2s(tile, src + e, rows * kRow, &bars.full_in[s]);
                bulk_g2s(tile + kTileQ, src + sh.elems + size_t(e / kRow) * 4, rows * 4,
                         &bars.full_in[s]);
            }
        });
        return;
    }
    if (warp == 1) {  // ---- storer
        if (lane == 0) {
            uint32_t released = 0;
            for_each_tile(std::integral_constant<int, 1>{},
                          [&](uint32_t q, const CopyDesc& d, uint32_t e, uint32_t rows, bool first) {
                const uint32_t t = q % kOutStages;
                if (!d.src && first && status) atomicAdd(status + kStatMiss, 1u);
                mbar_wait(&bars.full_out[t], (q / kOutStages) & 1);
                const uint8_t* tile = out_ring + t * kOutTile;
                if (d.src) {
                    uint8_t* dst = reinterpret_cast<uint8_t*>(d.dst);
                    if constexpr (WRITE) {
                        bulk_s2g(dst + e, tile, rows * kRow);
                        bulk_s2g(dst + sh.elems + size_t(e / kRow) * 4, tile + kTileQ, rows * 4);
                    } else {
                        bulk_s2g(dst + size_t(e) * 2, tile, rows * kRow * 2);
                    }
                }
                bulk_commit();
                bulk_wait_read<kLag>();
                if (q >= uint32_t(kLag)) {
                    mbar_arrive(&bars.empty_out[released % kOutStages]);
                    ++released;
                }
            });
            bulk_wait<0>();
            fence_proxy_async();
            if (FUSED) resolved_done(rq, nitems, 0);
        }
        __syncwarp();
        if (WRITE && pub.recs) ctrl_barrier_arrive(64);
        return;
    }
    // ---- compute warps: half-warp per row, two rows per step
    const uint32_t cw = warp - 3;
    const uint32_t half = lane >> 4, hl = lane & 15;
    for_each_tile(std::integral_constant<int, 2>{},
                  [&](uint32_t q, const CopyDesc& d, uint32_t, uint32_t rows, bool) {
        const uint32_t s = q % kInStages, t = q % kOutStages;
        mbar_wait(&bars.full_in[s], (q / kInStages) & 1);
        if (q >= uint32_t(kOutStages)) mbar_wait(&bars.empty_out[t], (q / kOutStages - 1) & 1);
        const uint8_t* in = in_ring + s * kInTile;
        uint8_t* out = out_ring + t * kOutTile;
        if (d.src) {
            for (uint32_t r = cw * 2 + half; r < rows; r += NCW * 2) {
                if constexpr (WRITE) {
                    const uint4 v = *reinterpret_cast<const uint4*>(in + (size_t(r) * kRow + hl * 8) * 2);
                    float2 f[4];
                    float amax = load8(v, f);
                    // the 16 lanes of this half own the row; rows r and r^1 of the two halves
                    // are both live or the loop bound differs only in the last step
                    const uint32_t mask = half ? 0xffff0000u : 0x0000ffffu;
#pragma unroll
                    for (int o = 8; o > 0; o >>= 1) amax = fmaxf(amax, __shfl_xor_sync(mask, amax, o));
                    if (has_inf(amax)) {  // rare: the row holds +-inf (uniform in the half)
                        amax = drop_inf8(f);
#pragma unroll
                        for (int o = 8; o > 0; o >>= 1)
                            amax = fmaxf(amax, __shfl_xor_sync(mask, amax, o));
                    }
                    const float scale = row_scale(amax);
                    *reinterpret_cast<uint2*>(out + size_t(r) * kRow + hl * 8) =
                        quant8(f, 1.f / scale);
                    if (hl == 0) *reinterpret_cast<float*>(out + kTileQ + r * 4) = scale;
                } else {
                    const uint2 v = *reinterpret_cast<const uint2*>(in + size_t(r) * kRow + hl * 8);
                    const float sc = *reinterpret_cast<const float*>(in + kTileQ + r * 4);
                    *reinterpret_cast<uint4*>(out + (size_t(r) * kRow + hl * 8) * 2) =
                        dequant8(v, sc);
                }
            }
        }
        // this warp's reads of the input tile and writes of the output tile are done: make the
        // generic-proxy writes visible to the bulk store, then signal both rings
        fence_proxy_async();
        __syncwarp();
        if (lane == 0) {
            mbar_arrive(&bars.empty_in[s]);
            mbar_arrive(&bars.full_out[t]);
        }
    });
}

template <bool WRITE, int NCW, bool FUSED>
__global__ void __launch_bounds__((3 + NCW) * 32)
    kv_fp8_pipe_kernel(const CopyDesc* __restrict__ descs, const Fp8Shape sh, Publish pub,
                       uint32_t* status, const __grid_constant__ ResolveArgs ra) {
    fp8_pipe<WRITE, NCW, FUSED>(descs, sh, pub, status, ra, OnePage{});
}

// Gathered blocks (launch_kv_fp8_pipe_gather): part s of block b is page b * nparts + s, the
// way kv_pipe_gather treats it as a virtual block; sh.n = blocks * nparts, sh.cpb = items per
// part.  The part bases travel in the kernel parameters.
template <bool WRITE>
__global__ void __launch_bounds__((3 + 8) * 32)
    kv_fp8_pipe_gather_kernel(const CopyDesc* __restrict__ descs, const Fp8Shape sh, Publish pub,
                              uint32_t* status, const __grid_constant__ GatherParts parts,
                              uint32_t nparts, uint32_t first_part, uint64_t stride,
                              LayerCommit lc) {
    fp8_pipe<WRITE, 8, false>(descs, sh, pub, status, ResolveArgs{},
                              BlockParts<WRITE>{&parts, nparts, first_part, stride, lc});
}

constexpr size_t kSmemWrite = kInStages * kTileBf16 + kOutStages * (kTileQ + kTileScale);
constexpr size_t kSmemRead = kInStages * (kTileQ + kTileScale) + kOutStages * kTileBf16;

cudaError_t ensure_attrs() {
    static bool done[64] = {false};
    return set_smem_limits_once(
        done,
        {{reinterpret_cast<const void*>(kv_fp8_pipe_kernel<true, 4, false>), int(kSmemWrite)},
         {reinterpret_cast<const void*>(kv_fp8_pipe_kernel<true, 8, false>), int(kSmemWrite)},
         {reinterpret_cast<const void*>(kv_fp8_pipe_kernel<false, 4, false>), int(kSmemRead)},
         {reinterpret_cast<const void*>(kv_fp8_pipe_kernel<false, 8, false>), int(kSmemRead)},
         {reinterpret_cast<const void*>(kv_fp8_pipe_kernel<false, 8, true>), int(kSmemRead)},
         {reinterpret_cast<const void*>(kv_fp8_pipe_gather_kernel<true>), int(kSmemWrite)},
         {reinterpret_cast<const void*>(kv_fp8_pipe_gather_kernel<false>), int(kSmemRead)}});
}

}  // namespace

cudaError_t launch_kv_fp8_pipe(const Fp8Launch& a, bool write, cudaStream_t stream) {
    if (a.n == 0) return cudaSuccess;
    if (!fp8_pipe_supported(a)) return cudaErrorInvalidValue;
    cudaError_t e = ensure_attrs();
    if (e != cudaSuccess) return e;
    const Publish pub = publish_of(a, write);
    const LaunchPlan p = plan_fp8_pipe(a, sm_count());
    const Fp8Shape sh{a.n, a.elems, p.chunk, p.cpb};
    const ResolveArgs none{};
    const auto go = [&](auto* kernel, int warps, size_t smem) {
        kernel<<<p.ctas, warps * 32, smem, stream>>>(a.descs, sh, pub, a.status, none);
        return cudaGetLastError();
    };
    if (write)
        return p.kernel == Kernel::kTma4 ? go(kv_fp8_pipe_kernel<true, 4, false>, 3 + 4, kSmemWrite)
                                         : go(kv_fp8_pipe_kernel<true, 8, false>, 3 + 8, kSmemWrite);
    return p.kernel == Kernel::kTma4 ? go(kv_fp8_pipe_kernel<false, 4, false>, 3 + 4, kSmemRead)
                                     : go(kv_fp8_pipe_kernel<false, 8, false>, 3 + 8, kSmemRead);
}

cudaError_t launch_kv_fp8_pipe_gather(const GatherLaunch& a, uint32_t elems, cudaStream_t stream) {
    if (a.n == 0) return cudaSuccess;
    if (!a.part_base) return cudaErrorInvalidValue;
    const LaunchPlan p = plan_gather_fp8(a, elems, kFp8Auto, sm_count());
    if (!p.valid) return cudaErrorInvalidValue;  // the caller splits the batch
    cudaError_t e = ensure_attrs();
    if (e != cudaSuccess) return e;
    GatherParts parts;
    std::memcpy(parts.base, a.part_base, size_t(a.nparts) * sizeof(uint64_t));
    const Fp8Shape sh{a.n * a.nparts, elems, p.chunk, p.cpb};
    const uint64_t stride = fp8_gather_bytes(1, elems);
    if (a.write)
        kv_fp8_pipe_gather_kernel<true><<<p.ctas, (3 + 8) * 32, kSmemWrite, stream>>>(
            a.descs, sh, publish_of(a, true), a.status, parts, a.nparts, a.first_part, stride,
            layer_of(a));
    else
        kv_fp8_pipe_gather_kernel<false><<<p.ctas, (3 + 8) * 32, kSmemRead, stream>>>(
            a.descs, sh, Publish{}, a.status, parts, a.nparts, a.first_part, stride,
            LayerCommit{});
    return cudaGetLastError();
}

// read_cache_fp8 through the device index in one launch: keys -> (resolver warp) -> pool
// blocks -> dequantised pages.  Same contract as launch_kv_read_fused (misses and entries that
// changed under the copy are counted in status[kStatMiss] / [kStatStale]).
bool fp8_read_fused_supported(const ReadFusedLaunch& a, uint32_t elems) {
    return elems > 0 && elems % 512 == 0 && (a.align_or & 15) == 0;
}

cudaError_t launch_kv_fp8_read_fused(const ReadFusedLaunch& a, uint32_t elems, cudaStream_t stream) {
    if (a.n == 0) return cudaSuccess;
    if (!fp8_read_fused_supported(a, elems)) return cudaErrorInvalidValue;
    cudaError_t e = ensure_attrs();
    if (e != cudaSuccess) return e;
    Fp8Launch f;  // the shape of an fp8 pipeline read of these pages
    f.n = a.n;
    f.elems = elems;
    f.max_ctas = a.max_ctas;
    const LaunchPlan p = plan_fp8_pipe(f, sm_count());
    kv_fp8_pipe_kernel<false, 8, true><<<p.ctas, (3 + 8) * 32, kSmemRead, stream>>>(
        nullptr, Fp8Shape{f.n, f.elems, p.chunk, p.cpb}, Publish{}, a.status, resolve_args(a));
    return cudaGetLastError();
}

}  // namespace istore::kernels
