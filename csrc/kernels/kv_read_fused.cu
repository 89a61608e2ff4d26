// kv_read_fused: read_cache in ONE kernel — hash the keys, probe the HBM-resident index
// over NVLink, and move the pages, with no server round trip and no separate lookup launch.
//
// This is the "read fused with the lookup/gather" end of the north star: the reference
// answers a read by a CPU hash-map probe per key on the server followed by RDMA_WRITE work
// requests pushed towards the client (src/infinistore.cpp:424-533).  Here every CTA has a
// RESOLVER warp that runs ahead of the copy warps: lane l hashes the key of the CTA's l-th
// work item (core/hash.h), probes the index (ld.acquire.sys on peer memory) and hands the
// pool address to the 256 copy threads through shared memory, double-buffered in rounds of
// 32 items with named barriers.  The lookup latency (2 NVLink round trips) is paid once
// per CTA, overlapped with the copies of other CTAs and of kernels in other streams.
// With a store that evicts (a.validate) the resolver re-checks every entry after its copy:
// an optimistic read that reports a block evicted underneath it as a miss.
#include "../core/hash.h"
#include "copy_span.cuh"
#include "index.cuh"
#include "kernels.h"

namespace istore::kernels {

namespace {

constexpr int kRound = 32;
// named barriers: full[p] (resolver -> copy warps), empty[p] (copy warps -> resolver)
constexpr int kBarFull0 = 2, kBarEmpty0 = 4;
constexpr int kThreads = kLdStThreads + 32;

__device__ __forceinline__ void bar_sync(int id) {
    asm volatile("bar.sync %0, %1;" ::"r"(id), "n"(kThreads) : "memory");
}
__device__ __forceinline__ void bar_arrive(int id) {
    asm volatile("bar.arrive %0, %1;" ::"r"(id), "n"(kThreads) : "memory");
}

struct Resolved {
    uint64_t src;  // mapped pool address, 0 = miss
    uint32_t slot_plus1;
    uint32_t tag;
};

__device__ Resolved resolve(const ReadFusedLaunch& a, uint32_t block) {
    const KeyHash kh = hash_key(a.key_bytes + a.key_off[block], a.key_len[block]);
    const idx::TableRef t = idx::select_shard(a.table, a.table_mask, a.shards, kh.h2);
    idx::Found f = idx::find<false>(t.table, t.mask, kh);
    f.slot_plus1 = idx::pack_slot(t.shard, f.slot_plus1);
    if (!f.slot_plus1) return Resolved{0, 0, 0};
    const uint32_t seg = uint32_t(f.addr >> 44) - 1;
    if (f.size < a.bytes || seg >= a.nsegs || !a.seg_base[seg]) return Resolved{0, 0, 0};
    return Resolved{a.seg_base[seg] + (f.addr & ((1ull << 44) - 1)), f.slot_plus1, f.tag};
}

template <int VEC>
__global__ void __launch_bounds__(kThreads)
    kv_read_fused_kernel(const __grid_constant__ ReadFusedLaunch a, uint32_t chunk, uint32_t cpb) {
    __shared__ uint64_t src_of[2][kRound];
    const uint32_t total = a.n * cpb;
    const uint32_t count = blockIdx.x < total ? (total - blockIdx.x + gridDim.x - 1) / gridDim.x : 0;
    const uint32_t rounds = (count + kRound - 1) / kRound;

    if (threadIdx.x >= kLdStThreads) {  // ---- resolver warp
        const uint32_t lane = threadIdx.x - kLdStThreads;
        // what this lane resolved in the two rounds in flight, re-checked once the copy warps
        // are done with the round (a.validate: the server may evict a block under a reader)
        uint32_t slot0 = 0, tag0 = 0, slot1 = 0, tag1 = 0;  // scalars: no local memory
        auto recheck = [&](uint32_t p) {
            const uint32_t slot = p ? slot1 : slot0, tag = p ? tag1 : tag0;
            if (slot && !idx::still_valid(idx::table_of_slot(a.table, a.shards, slot),
                                          idx::slot_local(slot), tag)) {
                atomicAdd(a.status + kStatMiss, 1u);
                atomicAdd(a.status + kStatStale, 1u);
            }
            if (p)
                slot1 = 0;
            else
                slot0 = 0;
        };
        for (uint32_t r = 0; r < rounds; ++r) {
            const uint32_t p = r & 1;
            if (r >= 2) {
                bar_sync(kBarEmpty0 + p);  // copy warps are done with this buffer
                if (a.validate) recheck(p);
            }
            const uint32_t k = r * kRound + lane;
            if (k < count) {
                const uint32_t item = blockIdx.x + k * gridDim.x;
                const Resolved res = resolve(a, item / cpb);
                src_of[p][lane] = res.src;
                if (res.src == 0 && item % cpb == 0 && a.status) atomicAdd(a.status + kStatMiss, 1u);
                // every chunk of a block is copied at a different time: each item re-checks
                // the entry after its own copy
                if (p) {
                    slot1 = res.slot_plus1;
                    tag1 = res.tag;
                } else {
                    slot0 = res.slot_plus1;
                    tag0 = res.tag;
                }
            }
            bar_arrive(kBarFull0 + p);
        }
        if (a.validate) {  // the last (up to) two rounds
            for (uint32_t r = rounds >= 2 ? rounds - 2 : 0; r < rounds; ++r) {
                bar_sync(kBarEmpty0 + (r & 1));
                recheck(r & 1);
            }
        }
        return;
    }
    // ---- copy warps
    for (uint32_t r = 0; r < rounds; ++r) {
        const uint32_t p = r & 1;
        bar_sync(kBarFull0 + p);
        const uint32_t kend = min(count, (r + 1) * kRound);
        for (uint32_t k = r * kRound; k < kend; ++k) {
            const uint64_t base = src_of[p][k - r * kRound];
            if (base == 0) continue;  // key not found: counted by the resolver
            const uint32_t item = blockIdx.x + k * gridDim.x;
            const uint32_t off = (item % cpb) * chunk;
            const uint32_t len = min(chunk, a.bytes - off);
            uint8_t* dst = reinterpret_cast<uint8_t*>(a.dst_base + a.dst_off[item / cpb]) + off;
            const uint8_t* src = reinterpret_cast<const uint8_t*>(base) + off;
            if constexpr (VEC == 1) {
                for (uint32_t b = threadIdx.x; b < len; b += kLdStThreads) dst[b] = src[b];
            } else {
                copy_span<VEC>(dst, src, len);
            }
        }
        if (r + 2 < rounds || a.validate) bar_arrive(kBarEmpty0 + p);
    }
}

}  // namespace

cudaError_t launch_kv_read_fused(const ReadFusedLaunch& a, cudaStream_t stream) {
    if (a.n == 0 || a.bytes == 0) return cudaSuccess;
    static const LdStResident res =
        ldst_resident(kv_read_fused_kernel<16>, kv_read_fused_kernel<32>, kThreads);
    const LaunchPlan p = plan_read_fused(a, sm_count(), res);
    // default: resolver warp + TMA pipeline (kv_pipe.cu); this file's ld/st kernel serves
    // small or unaligned pages.  Both re-check every entry after its copy.
    if (p.kernel == Kernel::kTma) return launch_kv_pipe_read(a, stream);
    const auto go = [&](auto* kernel) {
        kernel<<<p.ctas, kThreads, 0, stream>>>(a, p.chunk, p.cpb);
        return cudaGetLastError();
    };
    switch (p.kernel) {
        case Kernel::kLdSt1:
            return go(kv_read_fused_kernel<1>);
        case Kernel::kLdSt32:
            return go(kv_read_fused_kernel<32>);
        default:
            return go(kv_read_fused_kernel<16>);
    }
}

}  // namespace istore::kernels
