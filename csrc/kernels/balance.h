// How to cut a batch of equal-sized blocks into work items for a persistent grid.
//
// A CTA takes items first, first + grid, first + 2 * grid, ...  With whole blocks as items the
// batch finishes when the CTAs with ceil(n / grid) blocks finish: 512 blocks on 264 CTAs keep
// 248 CTAs busy for two blocks and 16 for one - 97 % of the grid's throughput, and the ring
// benchmarks issue exactly such batches (one layer's pages per call).  Splitting a block into
// `cpb` chunks makes the items finer; a chunk costs a descriptor (fused reads: a probe of the
// index) and, on writes, one more arrival at the block's commit counter, so the coarsest
// split within a few percent of the best makespan is taken.
#pragma once

#include <algorithm>
#include <cstdint>

namespace istore::kernels {

struct ChunkPlan {
    uint32_t chunk;  // units per item (the last item of a block may be shorter)
    uint32_t cpb;    // items per block
};

// `units` per block (ring slots, fp8 tiles), chunks are whole units and at least `min_units`
// (unless the block is shorter), at most `max_units`; `ctas` CTAs share n * cpb items.
inline ChunkPlan plan_chunks(uint32_t n, uint32_t units, uint32_t min_units, uint32_t max_units,
                             uint32_t ctas) {
    units = std::max(units, 1u);
    ctas = std::max(ctas, 1u);
    min_units = std::min(std::max(min_units, 1u), units);
    max_units = std::max(max_units, min_units);
    auto makespan = [&](uint32_t chunk) {  // units the busiest CTA moves
        const uint64_t cpb = (units + chunk - 1) / chunk;
        const uint64_t rounds = (uint64_t(n) * cpb + ctas - 1) / ctas;
        return rounds * chunk;
    };
    uint64_t best = ~0ull;
    for (uint32_t chunk = min_units; chunk <= std::min(units, max_units); ++chunk)
        best = std::min(best, makespan(chunk));
    uint32_t pick = min_units;
    for (uint32_t chunk = std::min(units, max_units); chunk >= min_units; --chunk) {
        if (makespan(chunk) * 100 <= best * 104) {  // coarsest within 4 % of the best
            pick = chunk;
            break;
        }
    }
    return ChunkPlan{pick, (units + pick - 1) / pick};
}

}  // namespace istore::kernels
