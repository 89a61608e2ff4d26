// Which kernel a page-mover launcher runs, how it cuts the batch into work items and on how
// many CTAs.  No CUDA in here: the launchers (kv_copy.cu, kv_read_fused.cu, kv_pipe.cu,
// kv_fp8.cu, kv_fp8_pipe.cu) pass in the SM count and the CTAs per SM the ld/st kernels keep
// resident (occupancy API), so the choice is unit-tested on the CPU
// (_infinistore.testing.plan_copy / plan_gather / plan_read_fused / plan_fp8 /
// plan_gather_fp8 / plan_gather_layered / plan_gather_rows).
#pragma once

#include <algorithm>
#include <cstddef>
#include <cstdint>

#include "balance.h"
#include "kernels.h"

namespace istore::kernels {

enum class Kernel : int {
    kLdSt1,     // ld/st kernel, byte loop: unaligned blocks
    kLdSt16,    // ld/st kernel, 16-byte vectors, four in flight per thread
    kLdSt32,    // ld/st kernel for 32-byte aligned blocks: eight 16-byte vectors in flight
    kLdSt16Mc,  // kv_copy_ldst storing its 16-byte vectors with multimem.st (NVLS multicast)
    kTma,       // the TMA pipeline (kv_pipe.cu; fp8: kv_fp8_pipe.cu with 8 compute warps)
    kTma4,      // the fp8 TMA pipeline with 4 compute warps
    kLdStFp8,   // the fp8 ld/st kernels (kv_fp8.cu)
};

struct PipeGeometry {
    uint32_t stage_bytes = 0;
    uint32_t stages = 0;
    size_t smem = 0;
};

struct LaunchPlan {
    Kernel kernel = Kernel::kLdSt16;
    bool valid = true;   // false: the launcher returns cudaErrorInvalidValue
    bool param = false;  // the block descriptors travel in the kernel parameters
    uint32_t chunk = 0;  // bytes (fp8: elements) per work item; a block's last may be shorter
    uint32_t cpb = 0;    // items per block (gathers: per part)
    int ctas = 0;
    PipeGeometry geo;    // ring of kv_pipe.cu's kernels (kTma outside the fp8 family)
};

// CTAs per SM the 16- and 32-byte flavours of an ld/st kernel keep resident (occupancy API).
struct LdStResident {
    int r16 = 1, r32 = 1;
};

constexpr uint32_t kLdStChunk = 32u << 10;  // work item of the ld/st kernels
constexpr uint32_t kFp8Chunk = 8192;        // elements: work item of the fp8 ld/st kernels, and
                                            // the tile of the fp8 pipeline (64 rows of 128)
// Descriptors of small batches travel in the kernel parameters (constant bank): reading them
// from the pinned host ring costs a PCIe round trip at the start of every launch.
constexpr int kParamDescs = 256;
constexpr int kPipeMaxStages = 32;
constexpr int kStoreLag = 2;  // bulk-store groups that may still be reading a ring slot

// Ring geometry: slots of up to `stage` bytes (16-byte multiple), as many as fit `ring` bytes.
// 16 KB slots, 4 of them (64 KB per CTA), ONE CTA per SM per launch: a single launch then may
// run below the best single-kernel geometry (larger slots per CTA), but three such kernels fit
// an SM side by side, and that is what the API needs - the calls of a phase go round-robin over
// the connection's streams, and the next kernel must be able to start (descriptor fetch, index
// claims) while the previous one drains (store acknowledgements, system fence, commit).
inline PipeGeometry pipe_geometry(uint32_t bytes, uint32_t stage_pref, uint32_t ring_pref) {
    PipeGeometry g;
    const uint32_t stage_cap = stage_pref ? stage_pref : (16u << 10);
    const uint32_t ring = ring_pref ? ring_pref : (64u << 10);
    g.stage_bytes = std::min(stage_cap, (bytes + 15u) & ~15u);
    g.stages = std::max<uint32_t>(kStoreLag + 1,
                                  std::min<uint32_t>(kPipeMaxStages, ring / g.stage_bytes));
    g.smem = size_t(g.stages) * g.stage_bytes;
    return g;
}

// ---------------------------------------------------------------- rules shared by the plans
// No more CTAs than work items.
inline int clamp_grid(int ctas, uint64_t items) {
    return int(std::min<uint64_t>(uint64_t(ctas), items));
}

// The caller's cap (max_ctas > 0) bounded by `limit`, else `limit`: the TMA kernels.
inline int capped_grid(int max_ctas, int limit) {
    return max_ctas > 0 ? std::min(max_ctas, limit) : limit;
}

// ld/st work item: `piece` units, or a whole block once there are at least as many blocks as
// SMs and a block is at most `whole_max` units.  A block is then moved by a single CTA: its
// commit needs no cross-CTA counter (claim, one fence, one store) and a reader resolves every
// key exactly once.
inline void ldst_items(LaunchPlan& p, uint64_t blocks, uint32_t units, uint32_t piece,
                       uint32_t whole_max, int sms) {
    p.chunk = blocks >= uint64_t(sms) && units <= whole_max ? units : std::min(units, piece);
    p.cpb = (units + p.chunk - 1) / p.chunk;
}

// Pipelined work item: whole `unit`s (ring slots, fp8 tiles), min_units to max_units of them,
// balanced over `ctas` (balance.h): a whole block when that keeps the grid evenly busy.
inline void unit_items(LaunchPlan& p, uint32_t blocks, uint32_t size, uint32_t unit,
                       uint32_t min_units, uint32_t max_units, int ctas) {
    const ChunkPlan c = plan_chunks(blocks, (size + unit - 1) / unit, min_units, max_units,
                                    uint32_t(ctas));
    p.chunk = std::min(size, c.chunk * unit);
    p.cpb = (size + p.chunk - 1) / p.chunk;
}

// The TMA pipeline of kv_pipe.cu: ONE CTA per SM (the rest of the SM's shared memory is for
// the kernels of the connection's other streams, see pipe_geometry), a caller's cap is bounded
// by it; items of at least four ring slots and at most 1 MB.
inline LaunchPlan pipe_plan(uint32_t blocks, uint32_t bytes, uint32_t stage_pref,
                            uint32_t ring_pref, int max_ctas, int sms) {
    LaunchPlan p;
    p.kernel = Kernel::kTma;
    p.geo = pipe_geometry(bytes, stage_pref, ring_pref);
    const int ctas = capped_grid(max_ctas, sms);
    unit_items(p, blocks, bytes, p.geo.stage_bytes, 4, std::max(4u, (1u << 20) / p.geo.stage_bytes),
               ctas);
    p.ctas = clamp_grid(ctas, uint64_t(blocks) * p.cpb);
    return p;
}

// An ld/st kernel fills every SM with the CTAs it keeps resident (one wave: every CTA loops
// over its items, so the commit epilogue runs once per CTA).  A caller's cap is NOT bounded by
// that grid.
inline int ldst_grid(const LaunchPlan& p, int max_ctas, LdStResident res, int sms,
                     uint64_t items) {
    const int per_sm = p.kernel == Kernel::kLdSt32 ? res.r32 : res.r16;
    return clamp_grid(max_ctas > 0 ? max_ctas : per_sm * sms, items);
}

inline bool aligned_to(uint32_t bytes, uint64_t align_or, uint32_t a) {
    return bytes % a == 0 && (align_or & (a - 1)) == 0;
}

inline LaunchPlan invalid_plan() {
    LaunchPlan p;
    p.valid = false;
    return p;
}

// ---------------------------------------------------------------- launch_kv_copy
// launch_kv_pipe_copy: the caller has checked alignment and multicast.  Descriptors go in the
// parameters whenever the host sees them: unlike the ld/st path, with no alignment condition.
inline LaunchPlan plan_pipe_copy(const CopyLaunch& a, int sms) {
    LaunchPlan p = pipe_plan(a.n, a.bytes, a.stage_bytes, a.ring_bytes, a.max_ctas, sms);
    p.param = a.descs_host != nullptr && a.n <= uint32_t(kParamDescs);
    return p;
}

inline LaunchPlan plan_copy(const CopyLaunch& a, int sms, LdStResident res) {
    // bulk copies need 16-byte aligned addresses and sizes (the caller ORs every local address
    // into align_or; pool blocks are granule aligned)
    const bool aligned16 = aligned_to(a.bytes, a.align_or, 16);
    const bool aligned32 = aligned_to(a.bytes, a.align_or, 32);
    int variant = a.variant;
    if (a.multicast) {
        if (!aligned16) return invalid_plan();  // multimem.st moves 16-byte vectors
        variant = kCopyLdSt;
    }
    // auto: the TMA pipeline from kPipeMinBytes up (3 warps per CTA); small blocks are bound by
    // per-block issue cost, where 256 threads win
    if (variant == kCopyAuto)
        variant = aligned16 && a.bytes >= kPipeMinBytes ? kCopyTma
                  : aligned32                           ? kCopyLdSt256
                                                        : kCopyLdSt;
    // an unaligned tma / ldst256 request, and ldst256 without 32-byte alignment, fall to ldst,
    // which runs the byte kernel on an unaligned batch
    if (!aligned16 && (variant == kCopyTma || variant == kCopyLdSt256)) variant = kCopyLdSt;
    if (variant == kCopyLdSt256 && !aligned32) variant = kCopyLdSt;
    if (variant == kCopyTma) return plan_pipe_copy(a, sms);
    LaunchPlan p;
    p.kernel = a.multicast                ? Kernel::kLdSt16Mc
               : !aligned16               ? Kernel::kLdSt1
               : variant == kCopyLdSt256  ? Kernel::kLdSt32
                                          : Kernel::kLdSt16;
    p.param = a.descs_host != nullptr && a.n <= uint32_t(kParamDescs) && aligned16;
    ldst_items(p, a.n, a.bytes, kLdStChunk, 1u << 20, sms);
    p.ctas = ldst_grid(p, a.max_ctas, res, sms, uint64_t(a.n) * p.cpb);
    return p;
}

// ---------------------------------------------------------------- launch_kv_gather
// More than 2^31 - 1 work items are refused: the caller splits the batch.
constexpr uint64_t kMaxItems = 0x7fffffffull;

inline LaunchPlan plan_pipe_gather(const GatherLaunch& a, int sms) {
    // chunks of one part, balanced over the grid as for whole blocks
    const uint64_t parts = uint64_t(a.n) * a.nparts;
    if (parts > kMaxItems) return invalid_plan();
    LaunchPlan p = pipe_plan(uint32_t(parts), a.part_bytes, a.stage_bytes, a.ring_bytes,
                             a.max_ctas, sms);
    if (parts * p.cpb > kMaxItems) return invalid_plan();
    return p;
}

// Gathers take no variant: 16-byte aligned parts of at least kPipeMinBytes go to the TMA
// pipeline (the per-part form of launch_kv_copy's auto rule), even on a local pool or an ldst
// connection.
inline LaunchPlan plan_gather(const GatherLaunch& a, int sms, LdStResident res) {
    const bool aligned16 = aligned_to(a.part_bytes, a.align_or, 16);
    const bool aligned32 = aligned_to(a.part_bytes, a.align_or, 32);
    if (aligned16 && a.part_bytes >= kPipeMinBytes) return plan_pipe_gather(a, sms);
    LaunchPlan p;
    p.kernel = !aligned16 ? Kernel::kLdSt1 : aligned32 ? Kernel::kLdSt32 : Kernel::kLdSt16;
    const uint64_t parts = uint64_t(a.n) * a.nparts;
    ldst_items(p, parts, a.part_bytes, kLdStChunk, 1u << 20, sms);  // whole parts as items
    if (parts * p.cpb > kMaxItems) return invalid_plan();
    p.ctas = ldst_grid(p, a.max_ctas, res, sms, parts * p.cpb);
    return p;
}

// ---------------------------------------------------------------- layered reads
// A layered read (GatherLaunch::group_flags) numbers its work items group-major, so that the
// persistent grid's stride walks the groups roughly in order:
//   item = ((g * n + block) * gp + p) * cpp + chunk,   part = g * gp + p,
// with gp parts per group and G = nparts / gp groups.  Group g's items are the contiguous
// range [g * n * gp * cpp, (g + 1) * n * gp * cpp).  The kernels (kv_copy.cu, kv_fp8.cu) and
// the CPU tests (_infinistore.testing.layered_item) share these two functions.
struct LayeredItem {
    uint32_t group, block, part, chunk;
};
ISTORE_KHD inline LayeredItem layered_item(uint32_t item, uint32_t n, uint32_t gp, uint32_t cpp) {
    const uint32_t chunk = item % cpp;
    const uint32_t q = item / cpp;
    const uint32_t r = q / gp;
    const uint32_t g = r / n;
    return LayeredItem{g, r % n, g * gp + q % gp, chunk};
}

// How many of the items first, first + stride, ... (a CTA's stream) lie in [lo, hi).
ISTORE_KHD inline uint32_t cta_items_below(uint32_t end, uint32_t first, uint32_t stride) {
    return end > first ? (end - first + stride - 1) / stride : 0u;
}
ISTORE_KHD inline uint32_t cta_items(uint32_t lo, uint32_t hi, uint32_t first, uint32_t stride) {
    return cta_items_below(hi, first, stride) - cta_items_below(lo, first, stride);
}

// The layered read runs the ld/st kernels whatever the part size (the TMA pipelines have no
// layered flavour): 16- or 32-byte vectors, the byte kernel on an unaligned batch.  Whole
// parts as items as in plan_gather; group_parts must divide nparts.
inline LaunchPlan plan_gather_layered(const GatherLaunch& a, int sms, LdStResident res) {
    if (a.nparts == 0 || a.nparts > kGatherMaxParts || a.group_parts == 0 ||
        a.nparts % a.group_parts != 0 || a.write)
        return invalid_plan();
    const bool aligned16 = aligned_to(a.part_bytes, a.align_or, 16);
    const bool aligned32 = aligned_to(a.part_bytes, a.align_or, 32);
    LaunchPlan p;
    p.kernel = !aligned16 ? Kernel::kLdSt1 : aligned32 ? Kernel::kLdSt32 : Kernel::kLdSt16;
    const uint64_t parts = uint64_t(a.n) * a.nparts;
    ldst_items(p, parts, a.part_bytes, kLdStChunk, 1u << 20, sms);
    if (parts * p.cpb > kMaxItems) return invalid_plan();
    p.ctas = ldst_grid(p, a.max_ctas, res, sms, parts * p.cpb);
    return p;
}

// ---------------------------------------------------------------- row-sliced reads
// kv_scatter_rows (GatherLaunch::rows != 0), plain or layered: always the ld/st kernels (the
// TMA pipelines have no row form).  The vector width is the one the OR of row_bytes, both
// pitches, src_col, the part bases and the local offsets allows (pool blocks are granule
// aligned and part_bytes is a multiple of src_pitch).  A work item is a run of `chunk` rows of
// one part, about kLdStChunk of payload, or all of a part's rows under ldst_items' rule; cpb
// is runs per part, and a layered read numbers items with layered_item as whole parts do.
inline LaunchPlan plan_gather_rows(const GatherLaunch& a, int sms, LdStResident res) {
    if (a.write || a.rows == 0 || a.row_bytes == 0 || a.nparts == 0 ||
        a.nparts > kGatherMaxParts || uint64_t(a.src_col) + a.row_bytes > a.src_pitch ||
        uint64_t(a.rows) * a.src_pitch != a.part_bytes ||
        (a.group_flags && (a.group_parts == 0 || a.nparts % a.group_parts != 0)))
        return invalid_plan();
    const uint64_t geo_or = a.align_or | a.src_pitch | a.src_col | a.dst_pitch;
    const bool aligned16 = aligned_to(a.row_bytes, geo_or, 16);
    const bool aligned32 = aligned_to(a.row_bytes, geo_or, 32);
    LaunchPlan p;
    p.kernel = !aligned16 ? Kernel::kLdSt1 : aligned32 ? Kernel::kLdSt32 : Kernel::kLdSt16;
    const uint64_t parts = uint64_t(a.n) * a.nparts;
    ldst_items(p, parts, a.rows, std::max(1u, kLdStChunk / a.row_bytes),
               std::max(1u, (1u << 20) / a.row_bytes), sms);
    if (parts * p.cpb > kMaxItems) return invalid_plan();
    p.ctas = ldst_grid(p, a.max_ctas, res, sms, parts * p.cpb);
    return p;
}

// ---------------------------------------------------------------- launch_kv_read_fused
inline bool pipe_read_supported(const ReadFusedLaunch& a) {
    return aligned_to(a.bytes, a.align_or, 16);
}

// A block that is split over several CTAs is resolved by each of them.
inline LaunchPlan plan_pipe_read(const ReadFusedLaunch& a, int sms) {
    return pipe_plan(a.n, a.bytes, a.stage_bytes, a.ring_bytes, a.max_ctas, sms);
}

// Resolver warp + TMA pipeline for kCopyTma, and for kCopyAuto from kPipeMinBytes up, when the
// batch is 16-byte aligned; the ld/st kernel otherwise.  kCopyLdSt is the 16-byte ld/st kernel,
// as in launch_kv_copy; anything else takes 32-byte vectors when the batch allows them.
inline LaunchPlan plan_read_fused(const ReadFusedLaunch& a, int sms, LdStResident res) {
    const bool aligned16 = aligned_to(a.bytes, a.align_or, 16);
    const bool aligned32 = aligned_to(a.bytes, a.align_or, 32);
    if ((a.variant == kCopyTma || (a.variant == kCopyAuto && a.bytes >= kPipeMinBytes)) &&
        aligned16)
        return plan_pipe_read(a, sms);
    LaunchPlan p;
    p.kernel = !aligned16                             ? Kernel::kLdSt1
               : aligned32 && a.variant != kCopyLdSt  ? Kernel::kLdSt32
                                                      : Kernel::kLdSt16;
    ldst_items(p, a.n, a.bytes, kLdStChunk, 1u << 20, sms);
    p.ctas = ldst_grid(p, a.max_ctas, res, sms, uint64_t(a.n) * p.cpb);
    return p;
}

// launch_kv_pipe_scatter_read: a CTA per block, the TMA grid with no item clamp (the launch
// needs at least as many blocks as CTAs, scatter_read_fused_supported).
inline int scatter_read_ctas(const ReadFusedLaunch& r, int sms) {
    return capped_grid(r.max_ctas, sms);
}

// ---------------------------------------------------------------- launch_kv_{write,read}_fp8
inline bool fp8_pipe_supported(const Fp8Launch& a) {
    return a.group == 128 && a.elems % 512 == 0 && a.elems > 0 && a.aligned16;
}

// The fp8 pipeline (~90 KB of shared memory): two CTAs per SM, a caller's cap bounded by
// that.  Whole pages per CTA when that keeps the grid evenly busy (single-CTA commit), else
// chunks of at least two tiles; never more than 64 tiles (512 K elements) per item.
inline LaunchPlan plan_fp8_pipe(const Fp8Launch& a, int sms) {
    LaunchPlan p;
    p.kernel = a.variant == kFp8Tma4 ? Kernel::kTma4 : Kernel::kTma;
    const int ctas = capped_grid(a.max_ctas, 2 * sms);
    unit_items(p, a.n, a.elems, kFp8Chunk, 2, 64, ctas);
    p.ctas = clamp_grid(ctas, uint64_t(a.n) * p.cpb);
    return p;
}

// The pipeline unless the ld/st kernels are asked for or the pages do not suit it.  The ld/st
// kernels: whole pages per CTA when there are enough of them, six CTAs per SM, a caller's cap
// not bounded.  Pages that are not 16-byte aligned are refused: every fp8 kernel moves bf16
// in 16-byte vectors (the ld/st kernels' loads and stores, the pipeline's bulk copies).
inline LaunchPlan plan_fp8(const Fp8Launch& a, int sms) {
    if (!a.aligned16) return invalid_plan();
    if (a.variant != kFp8LdSt && fp8_pipe_supported(a)) return plan_fp8_pipe(a, sms);
    LaunchPlan p;
    p.kernel = Kernel::kLdStFp8;
    ldst_items(p, a.n, a.elems, kFp8Chunk, 1u << 19, sms);
    p.ctas = clamp_grid(a.max_ctas > 0 ? a.max_ctas : 6 * sms, uint64_t(a.n) * p.cpb);
    return p;
}

// ---------------------------------------------------------------- launch_kv_gather_fp8
// Every part of every block is one fp8 page, so the rules of plan_fp8 apply with n * nparts
// pages: cpb is the items per part.  kFp8LdSt picks the ld/st kernels, anything else the
// pipeline with 8 compute warps.  Parts of a multiple of 512 elements and 16-byte aligned part
// bases and offsets only (the pipeline's precondition, and every part starts 16-byte aligned);
// more than kMaxItems work items are refused (the caller splits the batch).
inline LaunchPlan plan_gather_fp8(const GatherLaunch& a, uint32_t elems, int variant, int sms) {
    const uint64_t parts = uint64_t(a.n) * a.nparts;
    if (a.nparts == 0 || a.nparts > kGatherMaxParts || elems == 0 || elems % 512 != 0 ||
        (a.align_or & 15) != 0 || parts > kMaxItems)
        return invalid_plan();
    Fp8Launch f;
    f.n = uint32_t(parts);
    f.elems = elems;
    f.max_ctas = a.max_ctas;
    f.variant = variant == kFp8LdSt ? kFp8LdSt : kFp8Auto;
    LaunchPlan p = plan_fp8(f, sms);
    if (parts * p.cpb > kMaxItems) return invalid_plan();
    return p;
}

}  // namespace istore::kernels
