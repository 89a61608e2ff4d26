// Position-free KV segments (GatherLaunch::rope): the gathered bf16 ld/st movers with a RoPE
// shift applied to the keys inside the copy, so an all-layer page is stored at position 0 and
// read back at any position.
//
//   kv_write_rope_gather        : caller's parts -> pool block, rotated by the call's table
//                                 (the engine passes the shift -p0), then the in-band commit
//                                 (gather_items' control warp: one-shot or a layered writer's
//                                 LayerCommit).
//   kv_read_rope_scatter<LAYERED>: pool block -> caller's parts, rotated by the call's table
//                                 (+p1); plain or layered (scatter_items: misses counted once,
//                                 parts of a miss untouched, group releases).
//
// Contract (docs/kernels.md, "RoPE shift contract").  A part is a run of heads of head_elems
// bf16 elements.  The rotary pairs lie in elements [rot_offset, rot_offset + rot_dim) of every
// head: pair i is (i, i + rot_dim / 2) (neox) or (2i, 2i + 1) (interleaved) of that range.
// For K/V caches a head is a KV head and rot_offset = 0; for an MLA latent part a head is a
// token and rot_offset = latent_dim.  The table holds, for a shift of d positions,
// c_i = f32(cos(f64(d) * inv_freq_i)) and s_i = f32(sin(f64(d) * inv_freq_i)), built on the host
// (no trig runs here).  With a, b the pair's bf16 values widened to f32, and no FMA contraction:
//   a' = bf16_rne(rn32(rn32(a * c_i) - rn32(b * s_i)))
//   b' = bf16_rne(rn32(rn32(a * s_i) + rn32(b * c_i)))
// (a NaN in gives a NaN out).  Every other byte moves verbatim: the non-rotary elements, and
// every part that does not rotate (RopeShift::even_parts: the V parts, counted from the stored
// part index first_part + s).  launch_kv_gather never calls these for a table whose every pair
// is (1, 0): that call is copied verbatim by the plain movers.
//
// A thread owns whole pairs: a neox pair spans two 16-byte vectors of one head (element i
// and i + rot_dim / 2), so one work unit is that pair of vectors, or one non-rotary vector, or
// (interleaved) one vector of four pairs.  Items are runs of whole heads (plan_gather_rope), and
// the (c, s) table is staged in shared memory once per CTA.
#include <cuda_bf16.h>

#include "common.cuh"
#include "copy_span.cuh"
#include "gather_items.cuh"
#include "kernels.h"
#include "launch_plan.h"
#include "publish.cuh"

namespace istore::kernels {

namespace {

constexpr int kThreads = kLdStThreads;
constexpr int kUnits = 4;  // work units in flight per thread

// The head geometry of a launch in 16-byte vectors.
struct RopeGeom {
    uint32_t vph;   // vectors per head
    uint32_t r0;    // first rotary vector of a head
    uint32_t rv;    // rotary vectors of a head
    uint32_t ru;    // rotary units of a head: rv / 2 (neox pairs of vectors) or rv
    uint32_t uph;   // units per head: ru + the non-rotary vectors
    bool neox;
};

__device__ __forceinline__ RopeGeom geom_of(const RopeShift& r) {
    RopeGeom g;
    g.vph = r.head_elems / 8;
    g.r0 = r.rot_offset / 8;
    g.rv = r.rot_dim / 8;
    g.neox = r.interleaved == 0;
    g.ru = g.neox ? g.rv / 2 : g.rv;
    g.uph = g.vph - g.rv + g.ru;
    return g;
}

// Every thread of the CTA (the write's control warp included) stages the table; call before
// the item walk.
__device__ __forceinline__ void stage_table(const RopeShift& r, float2* tab) {
    for (uint32_t i = threadIdx.x; i < r.rot_dim / 2; i += blockDim.x)
        tab[i] = make_float2(r.c[i], r.s[i]);
    __syncthreads();
}

// Pair (a, b) turned by (c, s), as the contract writes it: no FMA contraction.
__device__ __forceinline__ void turn(float& a, float& b, float2 cs) {
    const float x = __fsub_rn(__fmul_rn(a, cs.x), __fmul_rn(b, cs.y));
    const float y = __fadd_rn(__fmul_rn(a, cs.y), __fmul_rn(b, cs.x));
    a = x;
    b = y;
}

__device__ __forceinline__ float lo_of(uint32_t w) { return __uint_as_float(w << 16); }
__device__ __forceinline__ float hi_of(uint32_t w) { return __uint_as_float(w & 0xffff0000u); }
__device__ __forceinline__ uint32_t pack_rne(float lo, float hi) {
    const __nv_bfloat162 v = __floats2bfloat162_rn(lo, hi);  // .x = lo, .y = hi, RNE
    return *reinterpret_cast<const uint32_t*>(&v);
}

// Neox: word k of vectors a and b holds pairs 2k and 2k + 1 of the 8 the two vectors carry,
// pair index i0 + 2k (low halves) and i0 + 2k + 1 (high halves).
__device__ __forceinline__ void turn_word_pair(uint32_t& wa, uint32_t& wb, const float2* tab,
                                               uint32_t i) {
    float al = lo_of(wa), bl = lo_of(wb), ah = hi_of(wa), bh = hi_of(wb);
    turn(al, bl, tab[i]);
    turn(ah, bh, tab[i + 1]);
    wa = pack_rne(al, ah);
    wb = pack_rne(bl, bh);
}

// Interleaved: word k of a vector is pair i0 + k, (low, high).
__device__ __forceinline__ uint32_t turn_word(uint32_t w, float2 cs) {
    float a = lo_of(w), b = hi_of(w);
    turn(a, b, cs);
    return pack_rne(a, b);
}

// Moves `len` bytes (whole heads) from src to dst, turning the rotary pairs of every head.
__device__ __forceinline__ void rope_span(uint8_t* dst, const uint8_t* src, uint32_t len,
                                          const RopeGeom& g, const float2* tab) {
    const uint32_t units = len / (16 * g.vph) * g.uph;
    for (uint32_t u0 = threadIdx.x; u0 < units; u0 += kUnits * kThreads) {
        uint4 va[kUnits], vb[kUnits];
        uint32_t at[kUnits], w[kUnits];
#pragma unroll
        for (int k = 0; k < kUnits; ++k) {
            const uint32_t u = u0 + k * kThreads;
            if (u >= units) continue;
            const uint32_t h = u / g.uph;
            w[k] = u - h * g.uph;
            const uint32_t x = w[k] - g.ru;  // the non-rotary vector's rank when w >= ru
            at[k] = h * g.vph + (w[k] < g.ru ? g.r0 + w[k] : x < g.r0 ? x : x + g.rv);
            va[k] = ld_stream_v4(src + size_t(at[k]) * 16);
            if (g.neox && w[k] < g.ru) vb[k] = ld_stream_v4(src + size_t(at[k] + g.ru) * 16);
        }
#pragma unroll
        for (int k = 0; k < kUnits; ++k) {
            const uint32_t u = u0 + k * kThreads;
            if (u >= units) continue;
            if (w[k] < g.ru) {
                if (g.neox) {
                    const uint32_t i = w[k] * 8;
                    turn_word_pair(va[k].x, vb[k].x, tab, i);
                    turn_word_pair(va[k].y, vb[k].y, tab, i + 2);
                    turn_word_pair(va[k].z, vb[k].z, tab, i + 4);
                    turn_word_pair(va[k].w, vb[k].w, tab, i + 6);
                    st_v4(dst + size_t(at[k] + g.ru) * 16, vb[k]);
                } else {
                    const uint32_t i = w[k] * 4;
                    va[k].x = turn_word(va[k].x, tab[i]);
                    va[k].y = turn_word(va[k].y, tab[i + 1]);
                    va[k].z = turn_word(va[k].z, tab[i + 2]);
                    va[k].w = turn_word(va[k].w, tab[i + 3]);
                }
            }
            st_v4(dst + size_t(at[k]) * 16, va[k]);
        }
    }
}

__device__ __forceinline__ bool rotates(const RopeShift& r, uint32_t stored_part) {
    return !r.even_parts || (stored_part & 1u) == 0;
}

// Writes: gather_items' walk over (block, part, run of whole heads); run [off, off + len) of
// part s is loaded from parts.base[s] + desc.src + off and stored into stored part
// first_part + s, turned when that part rotates.
__global__ void __launch_bounds__(kThreads + 32)
    kv_write_rope_gather_kernel(const CopyDesc* __restrict__ descs,
                                const __grid_constant__ GatherParts parts,
                                const __grid_constant__ RopeShift rope, uint32_t n,
                                uint32_t nparts, uint32_t part_bytes, uint32_t chunk, uint32_t cpp,
                                uint32_t first_part, Publish pub, LayerCommit lc) {
    __shared__ float2 tab[kRopeMaxPairs];
    stage_table(rope, tab);
    const RopeGeom g = geom_of(rope);
    gather_items(descs, n, nparts, part_bytes, chunk, cpp, pub, lc,
                 [&](const CopyDesc& d, uint32_t, uint32_t s, uint32_t off, uint32_t len) {
                     uint8_t* dst = reinterpret_cast<uint8_t*>(
                                        d.dst + uint64_t(first_part + s) * part_bytes) + off;
                     const uint8_t* src =
                         reinterpret_cast<const uint8_t*>(parts.base[s] + d.src) + off;
                     if (rotates(rope, first_part + s))
                         rope_span(dst, src, len, g, tab);
                     else
                         copy_span<16>(dst, src, len);
                 });
}

// Reads: scatter_items' walk (LAYERED: group-major items and group releases); item chunk c of
// part s moves bytes [c * chunk, +chunk) of stored part first_part + s to parts.base[s] +
// desc.dst, turned when that stored part rotates.
template <bool LAYERED>
__global__ void __launch_bounds__(kThreads)
    kv_read_rope_scatter_kernel(const CopyDesc* __restrict__ descs,
                                const __grid_constant__ GatherParts parts,
                                const __grid_constant__ RopeShift rope, uint32_t n,
                                uint32_t nparts, uint32_t part_bytes, uint32_t chunk, uint32_t cpp,
                                uint32_t first_part, uint32_t* status, GroupRelease rel) {
    __shared__ float2 tab[kRopeMaxPairs];
    stage_table(rope, tab);
    const RopeGeom g = geom_of(rope);
    scatter_items<LAYERED>(descs, n, nparts, cpp, status, rel, [&](const CopyDesc& d,
                                                                  const LayeredItem& it) {
        const uint32_t off = it.chunk * chunk;
        const uint32_t len = min(chunk, part_bytes - off);
        const uint8_t* src =
            reinterpret_cast<const uint8_t*>(d.src + uint64_t(first_part + it.part) * part_bytes) +
            off;
        uint8_t* dst = reinterpret_cast<uint8_t*>(parts.base[it.part] + d.dst) + off;
        if (rotates(rope, first_part + it.part))
            rope_span(dst, src, len, g, tab);
        else
            copy_span<16>(dst, src, len);
    });
}

template <bool WRITE, bool LAYERED>
cudaError_t launch_rope(const GatherLaunch& a, cudaStream_t stream) {
    const LaunchPlan p =
        WRITE ? plan_gather_rope(a, sm_count(),
                                 cached_resident<kv_write_rope_gather_kernel,
                                                 kv_write_rope_gather_kernel, kThreads + 32>())
              : plan_gather_rope(a, sm_count(),
                                 cached_resident<kv_read_rope_scatter_kernel<LAYERED>,
                                                 kv_read_rope_scatter_kernel<LAYERED>, kThreads>());
    if (!p.valid) return cudaErrorInvalidValue;
    const GatherParts parts = parts_of(a);
    if constexpr (WRITE)
        kv_write_rope_gather_kernel<<<p.ctas, kThreads + 32, 0, stream>>>(
            a.descs, parts, *a.rope, a.n, a.nparts, a.part_bytes, p.chunk, p.cpb, a.first_part,
            publish_of(a, true), layer_of(a));
    else
        kv_read_rope_scatter_kernel<LAYERED><<<p.ctas, kThreads, 0, stream>>>(
            a.descs, parts, *a.rope, a.n, a.nparts, a.part_bytes, p.chunk, p.cpb, a.first_part,
            a.status, release_of(a));
    return cudaGetLastError();
}

}  // namespace

cudaError_t launch_kv_gather_rope(const GatherLaunch& a, cudaStream_t stream) {
    if (a.n == 0) return cudaSuccess;
    if (!a.part_base || !a.rope) return cudaErrorInvalidValue;
    if (uint64_t(a.first_part + a.nparts) * a.part_bytes > 0xffffffffull)
        return cudaErrorInvalidValue;
    const bool layered = a.group_flags != nullptr;
    if (layered && !a.group_counters) return cudaErrorInvalidValue;
    if (a.write) return launch_rope<true, false>(a, stream);
    return layered ? launch_rope<false, true>(a, stream) : launch_rope<false, false>(a, stream);
}

}  // namespace istore::kernels
