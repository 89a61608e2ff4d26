// Which kernels a read through the device index runs (Connection::read_via_device_index).  No
// CUDA in here: the two support checks that need the kernels' launch structs are evaluated by
// the caller, so the choice is unit-tested on the CPU (_infinistore.testing.plan_device_read).
#pragma once

#include <algorithm>
#include <cstddef>
#include <cstdint>

#include "../kernels/kernels.h"

namespace istore {

struct DeviceReadIn {
    size_t n = 0;              // blocks in the batch
    uint32_t block_bytes = 0;  // all parts of a gathered block
    uint32_t fp8_elems = 0;    // bf16 elements per page of an fp8 read, 0 otherwise
    bool gather = false;
    bool fp8_fused_ok = false, scatter_fused_ok = false;  // kernels::*_read_fused_supported
    int copy_variant = kernels::kCopyAuto;
    // over every known segment (up to kMaxSegs), not only the batch's: intentional
    bool all_local = false, all_remote = false;
    int max_ctas = 0, sm_count = 0;  // max_ctas: the connection's grid cap, 0 = none
    bool layered = false;  // a layered read of gathered blocks (GatherLaunch::group_flags)
    bool rows = false;     // a row-sliced read of gathered blocks (GatherLaunch::rows)
};

enum class ReadPath {
    kFusedCopy,     // kv_read_fused: hash + probe + copy + re-check in one launch
    kFusedFp8,      // kv_fp8_read_fused: the same, dequantising
    kFusedScatter,  // kv_pipe_scatter_read: the same into the parts of gathered blocks
    kLookupCopy,    // index_lookup, kv_copy, index_validate
    kLookupFp8,     // index_lookup, kv_read_fp8, index_validate
    kLookupGather,  // index_lookup, kv_gather, index_validate
    kLookupGatherFp8,  // index_lookup, kv_gather_fp8, index_validate
};

struct DeviceReadPlan {
    ReadPath path = ReadPath::kLookupCopy;
    int variant = kernels::kCopyAuto;  // of the launch that moves the pages (unused by bf16 gathers)
    int grid_cap = 0;                  // max_ctas of every launch
    bool fused() const { return path <= ReadPath::kFusedScatter; }
};

// fp8 pages over NVLink: reads one CTA per SM, writes two per SM.  A grid choice not
// re-measured on H100: bench/configs.py fp8 --max-ctas N compares grid caps.
inline int device_read_grid_cap(int max_ctas, bool all_remote, bool fp8, int sm_count) {
    return max_ctas ? max_ctas : all_remote ? (fp8 ? 1 : 2) * sm_count : 0;
}

// `auto` for pages in this GPU's own HBM: the ld/st kernels (256 copy threads per CTA, every
// SM filled, 128 bytes in flight per thread) against the TMA pipeline's one issuing thread per
// role.  On H100 they move the flagship's 128 KB pages HBM to HBM faster, most of it in the
// read phase (docs/kernels.md); pools behind NVLink keep the TMA pipeline.
inline int local_auto_variant(int variant, bool local) {
    return variant == kernels::kCopyAuto && local ? int(kernels::kCopyLdSt256) : variant;
}

// What a row-sliced read of one stored fp8 part counts in bytes_read: the pool bytes it reads,
// which are the e4m3 bytes of its rows plus 4 bytes for every 128-element scale group they
// touch, each group counted once however many rows share it.  The geometry is in bytes of the
// part's bf16 view (GatherLaunch::rows); rows never overlap and come in increasing order.
// Full-width rows touch every group once: fp8_block_bytes(elems, 128), what a read of the
// whole part counts.
inline uint64_t fp8_rows_read_bytes(uint32_t rows, uint32_t row_bytes, uint32_t src_pitch,
                                    uint32_t src_col) {
    const uint64_t width = row_bytes / 2, pitch = src_pitch / 2, col = src_col / 2;
    if (rows == 0 || width == 0) return 0;
    uint64_t groups = 0, next = 0;  // next: the first group not counted yet
    for (uint64_t r = 0; r < rows; ++r) {
        const uint64_t lo = std::max((r * pitch + col) / 128, next);
        const uint64_t hi = (r * pitch + col + width - 1) / 128;
        if (hi >= lo) groups += hi - lo + 1;
        next = std::max(next, hi + 1);
    }
    return uint64_t(rows) * width + 4 * groups;
}

inline DeviceReadPlan plan_device_read(const DeviceReadIn& in) {
    DeviceReadPlan p;
    p.grid_cap = device_read_grid_cap(in.max_ctas, in.all_remote, in.fp8_elems != 0, in.sm_count);
    // The fused kernels resolve a key in every CTA that moves a piece of its block, reading
    // the key bytes from the pinned ring each time: right for a batch of blocks (items are
    // whole blocks, or chunks when that balances the grid better - kernels/balance.h),
    // wasteful when a few LARGE blocks are split over many CTAs - then resolve each key
    // once with the lookup kernel and feed the descriptors to kv_copy.
    // A handful of blocks (<= 4 MB in all): latency matters, not bandwidth.  One launch of
    // the ld/st flavour, which splits a block into 32 KB chunks over CTAs (each resolves its
    // block's key itself - a few redundant probes) and re-checks the entries in the same
    // kernel: lookup + copy + validate would be three launches.
    const bool small_batch = in.n * size_t(in.block_bytes) <= (4u << 20);
    const bool whole_blocks = !small_batch && in.block_bytes <= (1u << 20) && in.n >= 32;
    // gathered blocks: one launch (resolver warp + gather pipeline, a CTA per block) once
    // every CTA has a block of its own; fewer blocks: lookup + gather + validate.
    // fp8 pages: the resolver rides in the dequantising TMA pipeline (one launch instead of
    // lookup + read + validate: 32 calls of 512 pages were launch-bound).
    // gathered fp8 blocks: each key is probed once by the lookup kernel and re-checked after the
    // dequantising scatter; never the bf16 scatter pipeline.
    // layered reads: lookup, the layered ld/st scatter (the only kernels that release groups),
    // validate - each key probed once, by the lookup kernel.  Row-sliced reads the same way:
    // only the ld/st scatter has a row form.
    if (in.gather && (in.layered || in.rows)) {
        p.path = in.fp8_elems ? ReadPath::kLookupGatherFp8 : ReadPath::kLookupGather;
        p.variant = in.fp8_elems ? int(kernels::kFp8LdSt) : int(kernels::kCopyLdSt);
        return p;
    }
    if (in.gather && in.fp8_elems)
        p.path = ReadPath::kLookupGatherFp8;
    else if (in.gather)
        p.path = in.scatter_fused_ok ? ReadPath::kFusedScatter : ReadPath::kLookupGather;
    else if (in.fp8_elems)
        p.path = in.fp8_fused_ok ? ReadPath::kFusedFp8 : ReadPath::kLookupFp8;
    else
        p.path = whole_blocks || small_batch ? ReadPath::kFusedCopy : ReadPath::kLookupCopy;
    // lookup then fp8 (per-page or gathered): the TMA pipeline when every segment is remote,
    // the ld/st kernels otherwise.  Intentional: move_blocks' rule is all_local ? ld/st : TMA,
    // and the two differ for a pool that mixes local and remote segments.
    if (p.path == ReadPath::kLookupFp8 || p.path == ReadPath::kLookupGatherFp8)
        p.variant = in.all_remote ? kernels::kFp8Auto : kernels::kFp8LdSt;
    else if (p.path == ReadPath::kFusedCopy && in.copy_variant == kernels::kCopyLdSt)
        p.variant = kernels::kCopyLdSt;  // the 16-byte ld/st read kernel (launch_plan.h)
    else
        p.variant = p.fused() && small_batch ? int(kernels::kCopyLdSt256)
                                             : local_auto_variant(in.copy_variant, in.all_local);
    return p;
}

}  // namespace istore
