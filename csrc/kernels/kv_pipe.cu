// kv_pipe: the Hopper-native page movers — warp-specialised TMA pipelines.
//
// This is the default data path of write_cache / read_cache: every byte moves
//     global (local HBM or a peer GPU over NVLink 4) --cp.async.bulk--> SMEM ring
//     SMEM ring --cp.async.bulk--> global (peer pool or local KV cache)
// with no register staging and two or three warps per CTA, so a transfer that overlaps
// prefill leaves the SM's issue slots and register file to the model's kernels.  It
// replaces, per batch, the reference's N cudaMemcpyAsync calls (src/infinistore.cpp:623-624,
// 747-748), its RDMA_WRITE work-request chains (src/libinfinistore.cpp:905-970,
// src/infinistore.cpp:456-530) and the COMMIT / lookup messages around them.
//
// Roles (one warp each, lane 0 issues, all lanes prefetch descriptors):
//   loader   : waits for a free ring slot (empty[s]), arms full[s] with the byte count
//              (mbarrier expect_tx) and issues the global->shared bulk copy   UBLKCP.S.G
//   storer   : waits for full[s] (SYNCS...TRYWAIT), issues the shared->global bulk copy
//              (UBLKCP.G.S) as its own bulk group, and releases slots whose stores have
//              finished READING shared memory (wait_group.read) kStoreLag groups behind, so
//              neither thread ever waits for the copy it has just issued
//   control  : (writes) the in-band commit of publish.cuh: claim early, one system fence once
//              the storer reports every bulk store complete, tag stores
//   resolver : (fused reads) hashes the keys of the CTA's items, probes the HBM index over
//              NVLink and feeds {pool address, destination} to loader and storer through a
//              double-buffered SMEM queue guarded by mbarriers - read_cache in ONE launch
//              with no server round trip, now on the bulk-async path as well.
//
// kv_pipe_mcast: thread-block CLUSTER variant (2 or 4 CTAs).  One pool block is fetched over
// NVLink ONCE by the cluster's leader with cp.async.bulk ... .multicast::cluster, which lands
// the tile in the shared memory of every CTA of the cluster; each CTA then stores it to its
// own destination (the same KV page wanted by several TP ranks / beams).  Slots are handed
// back to the leader with remote mbarrier arrivals (DSMEM), the cluster barrier closes the
// kernel.  NVLink bytes: 1x instead of Kx.
#include <cuda.h>  // CUtensorMap + enums only: the encoder is fetched through cudart at run time

#include <algorithm>
#include <cstring>

#include "../core/hash.h"
#include "common.cuh"
#include "index.cuh"
#include "kernels.h"
#include "launch_plan.h"
#include "publish.cuh"
#include "resolve.cuh"

namespace istore::kernels {

namespace {

using namespace dev;

constexpr int kPipeThreads = 96;

template <int N>
struct PipeDescParam {
    CopyDesc d[N];
};

// Static schedule shared by every role of a CTA: item k of this CTA is global item
// first + k * stride = chunk (item % cpb) of block (item / cpb); a chunk is moved in pieces
// of at most stage_bytes through consecutive ring slots.
struct Shape {
    uint32_t n, bytes, chunk, cpb, stage_bytes, stages;
};

// 64 descriptors in registers per warp (two coalesced fetches of 32), handed out by shuffle:
// descriptors may live in pinned host memory, one PCIe read per 32 items instead of one each.
template <bool PARAM>
struct DescWindow {
    const CopyDesc* descs;
    const PipeDescParam<PARAM ? kParamDescs : 1>* pd;
    uint32_t first, stride, cpb, nitems, lane;
    CopyDesc cur, nxt;
    uint32_t window = 0;
    __device__ __forceinline__ CopyDesc fetch(uint32_t k0) const {
        const uint32_t k = k0 + lane;
        if (k >= nitems) return CopyDesc{0, 0};
        const uint32_t block = (first + k * stride) / cpb;
        if constexpr (PARAM)
            return pd->d[block];
        else
            return descs[block];
    }
    __device__ __forceinline__ void init() {
        cur = fetch(0);
        nxt = fetch(32);
    }
    __device__ __forceinline__ CopyDesc at(uint32_t k) {  // k non-decreasing, warp-uniform
        if (k >= window + 32) {
            window += 32;
            cur = nxt;
            nxt = fetch(window + 32);
        }
        const uint32_t l = (k - window) & 31;
        CopyDesc r;
        r.src = __shfl_sync(0xffffffffu, cur.src, l);
        r.dst = __shfl_sync(0xffffffffu, cur.dst, l);
        return r;
    }
};

// ---------------------------------------------------------------- loader / storer bodies
// `desc_at(k)` returns the descriptor of the CTA's k-th item (warp-collective call).
template <typename DescAt>
__device__ __forceinline__ void loader_body(const Shape& sh, uint32_t first, uint32_t stride,
                                            uint32_t nitems, uint32_t lane, uint8_t* ring,
                                            uint64_t* full, uint64_t* empty, DescAt&& desc_at) {
    uint32_t s = 0, use = 0;  // ring slot and how many times it has been used
    for (uint32_t k = 0; k < nitems; ++k) {
        const CopyDesc d = desc_at(k);
        const uint32_t item = first + k * stride;
        const uint32_t off0 = (item % sh.cpb) * sh.chunk;
        const uint32_t len = min(sh.chunk, sh.bytes - off0);
        for (uint32_t o = 0; o < len; o += sh.stage_bytes) {
            if (lane == 0) {
                if (use) mbar_wait(&empty[s], (use - 1) & 1);
                const uint32_t plen = min(sh.stage_bytes, len - o);
                if (d.src) {
                    mbar_expect_tx(&full[s], plen);
                    bulk_g2s(ring + size_t(s) * sh.stage_bytes,
                             reinterpret_cast<const uint8_t*>(d.src) + off0 + o, plen, &full[s]);
                } else {
                    mbar_arrive(&full[s]);  // a miss: nothing to move, keep the ring in step
                }
            }
            if (++s == sh.stages) {
                s = 0;
                ++use;
            }
        }
    }
}

// Fan-out: every piece is stored to `n` destinations, dst + delta[r] (one load, n stores from
// the same ring slot - the multi-destination read when the source sits behind NVLink).
struct FanOut {
    uint32_t n = 1;
    int64_t delta[4] = {0, 0, 0, 0};
};

template <typename DescAt>
__device__ __forceinline__ void storer_body(const Shape& sh, uint32_t first, uint32_t stride,
                                            uint32_t nitems, uint32_t lane, uint8_t* ring,
                                            uint64_t* full, uint64_t* empty, uint32_t* status,
                                            DescAt&& desc_at, const FanOut fan = FanOut{}) {
    uint32_t s = 0, ph = 0;  // slot being stored and its full-phase parity
    uint32_t sf = 0;         // slot to release next
    uint32_t q = 0;          // pieces issued
    for (uint32_t k = 0; k < nitems; ++k) {
        const CopyDesc d = desc_at(k);
        const uint32_t item = first + k * stride;
        const uint32_t off0 = (item % sh.cpb) * sh.chunk;
        const uint32_t len = min(sh.chunk, sh.bytes - off0);
        if (lane == 0 && d.src == 0 && off0 == 0 && status) atomicAdd(status + kStatMiss, 1u);
        for (uint32_t o = 0; o < len; o += sh.stage_bytes, ++q) {
            if (lane == 0) {
                mbar_wait(&full[s], ph);
                if (d.src) {
                    const uint32_t plen = min(sh.stage_bytes, len - o);
                    for (uint32_t r = 0; r < fan.n; ++r)  // delta[0] == 0 without fan-out
                        bulk_s2g(reinterpret_cast<uint8_t*>(int64_t(d.dst) + fan.delta[r]) + off0 + o,
                                 ring + size_t(s) * sh.stage_bytes, plen);
                }
                bulk_commit();  // one group per piece (an empty one for a miss)
                bulk_wait_read<kStoreLag>();  // pieces <= q - kStoreLag have left the ring
                if (q >= uint32_t(kStoreLag)) {
                    mbar_arrive(&empty[sf]);
                    if (++sf == sh.stages) sf = 0;
                }
            }
            if (++s == sh.stages) {
                s = 0;
                ph ^= 1;
            }
        }
    }
    if (lane == 0) {
        bulk_wait<0>();       // every bulk store of this CTA has completed its writes
        fence_proxy_async();  // async-proxy writes before the generic-proxy commit / exit
    }
    __syncwarp();
}

// ---------------------------------------------------------------- kv_pipe_copy
template <bool PARAM>
__global__ void __launch_bounds__(kPipeThreads)
    kv_pipe_copy_kernel(const CopyDesc* __restrict__ descs,
                        const __grid_constant__ PipeDescParam<PARAM ? kParamDescs : 1> pd,
                        const Shape sh, Publish pub, const FanOut fan) {
    extern __shared__ __align__(128) uint8_t ring[];
    __shared__ __align__(8) uint64_t full[kPipeMaxStages];
    __shared__ __align__(8) uint64_t empty[kPipeMaxStages];
    const uint32_t total = sh.n * sh.cpb;
    const uint32_t grid = gridDim.x;
    const uint32_t nitems = blockIdx.x < total ? (total - blockIdx.x + grid - 1) / grid : 0;
    const uint32_t warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    if (threadIdx.x == 0) {
        for (uint32_t s = 0; s < sh.stages; ++s) {
            mbar_init(&full[s], 1);
            mbar_init(&empty[s], 1);
        }
        mbar_fence_init();
    }
    __syncthreads();
    if (warp == 2) {  // control warp: in-band commit
        if (pub.recs) control_warp(pub, lane, blockIdx.x, nitems, grid, sh.cpb, 64);
        return;
    }
    DescWindow<PARAM> win{descs, &pd, blockIdx.x, grid, sh.cpb, nitems, lane};
    win.init();
    auto desc_at = [&](uint32_t k) { return win.at(k); };
    if (warp == 0) {
        loader_body(sh, blockIdx.x, grid, nitems, lane, ring, full, empty, desc_at);
    } else {
        storer_body(sh, blockIdx.x, grid, nitems, lane, ring, full, empty, pub.status, desc_at, fan);
        if (pub.recs) ctrl_barrier_arrive(64);
    }
}

// ---------------------------------------------------------------- kv_pipe_gather
// Gathered blocks (GatherLaunch) through the same loader / storer bodies: part s of block b is
// the virtual block b * nparts + s of part_bytes (sh.n virtual blocks, sh.cpb chunks each), so
// global item numbers are those of GatherLaunch and the control warp counts nparts * sh.cpb
// arrivals per real block.  The descriptor window walks the real blocks' descriptors.
// LAYERED: a layered write's launch (publish.cuh: control_warp_layered).  It is a separate
// instantiation because with both control-warp bodies in one kernel ptxas spilled registers.
template <bool LAYERED>
__global__ void __launch_bounds__(kPipeThreads)
    kv_pipe_gather_kernel(const CopyDesc* __restrict__ descs,
                          const __grid_constant__ GatherParts parts, const Shape sh,
                          uint32_t nparts, uint32_t first_part, bool write, Publish pub,
                          LayerCommit lc) {
    extern __shared__ __align__(128) uint8_t ring[];
    __shared__ __align__(8) uint64_t full[kPipeMaxStages];
    __shared__ __align__(8) uint64_t empty[kPipeMaxStages];
    const uint32_t cpb = nparts * sh.cpb;  // items per real block
    const uint32_t total = sh.n * sh.cpb;
    const uint32_t grid = gridDim.x;
    const uint32_t nitems = blockIdx.x < total ? (total - blockIdx.x + grid - 1) / grid : 0;
    const uint32_t warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    if (threadIdx.x == 0) {
        for (uint32_t s = 0; s < sh.stages; ++s) {
            mbar_init(&full[s], 1);
            mbar_init(&empty[s], 1);
        }
        mbar_fence_init();
    }
    __syncthreads();
    if (warp == 2) {  // control warp: in-band commit
        if (!pub.recs) return;
        if constexpr (LAYERED)
            control_warp_layered(pub, lc, lane, blockIdx.x, nitems, grid, cpb, nparts, 64);
        else
            control_warp(pub, lane, blockIdx.x, nitems, grid, cpb, 64);
        return;
    }
    DescWindow<false> win{descs, nullptr, blockIdx.x, grid, cpb, nitems, lane};
    win.init();
    auto desc_at = [&](uint32_t k) {
        const CopyDesc b = win.at(k);
        const uint32_t item = blockIdx.x + k * grid;
        const uint32_t s = (item % cpb) / sh.cpb;
        CopyDesc d;
        if (write) {
            d.src = parts.base[s] + b.src;
            d.dst = b.dst + uint64_t(first_part + s) * sh.bytes;
        } else {
            d.src = b.src ? b.src + uint64_t(first_part + s) * sh.bytes : 0;
            d.dst = parts.base[s] + b.dst;
        }
        return d;
    };
    if (warp == 0) {
        loader_body(sh, blockIdx.x, grid, nitems, lane, ring, full, empty, desc_at);
    } else {
        // misses are counted here, once per block, not by storer_body once per part
        storer_body(sh, blockIdx.x, grid, nitems, lane, ring, full, empty, nullptr,
                    [&](uint32_t k) {
                        const CopyDesc d = desc_at(k);
                        if (lane == 0 && d.src == 0 && (blockIdx.x + k * grid) % cpb == 0 &&
                            pub.status)
                            atomicAdd(pub.status + kStatMiss, 1u);
                        return d;
                    });
        if (pub.recs) ctrl_barrier_arrive(64);
    }
}

// ---------------------------------------------------------------- kv_pipe_read (fused)
// resolver warp + queue: resolve.cuh
__global__ void __launch_bounds__(kPipeThreads)
    kv_pipe_read_kernel(const __grid_constant__ ResolveArgs a, const Shape sh) {
    extern __shared__ __align__(128) uint8_t ring[];
    __shared__ __align__(8) uint64_t full[kPipeMaxStages];
    __shared__ __align__(8) uint64_t empty[kPipeMaxStages];
    __shared__ __align__(16) ResolveQueue rq;
    const uint32_t total = sh.n * sh.cpb;
    const uint32_t grid = gridDim.x;
    const uint32_t nitems = blockIdx.x < total ? (total - blockIdx.x + grid - 1) / grid : 0;
    const uint32_t warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    if (threadIdx.x == 0) {
        for (uint32_t s = 0; s < sh.stages; ++s) {
            mbar_init(&full[s], 1);
            mbar_init(&empty[s], 1);
        }
        resolve_queue_init(rq);
        mbar_fence_init();
    }
    __syncthreads();
    if (warp == 2) {  // ---- resolver: runs ahead of the copy by up to two batches
        resolver_warp(a, rq, sh.bytes, blockIdx.x, grid, sh.cpb, nitems, lane);
        return;
    }
    // Loader and storer read their descriptors from the queue.  The storer hands a half back
    // when it moves on to the next batch (or finishes): every load of the half's blocks has
    // completed by then, which is what the resolver's re-check relies on.
    if (warp == 0) {
        loader_body(sh, blockIdx.x, grid, nitems, lane, ring, full, empty,
                    [&](uint32_t k) { return resolved_desc<false, true>(rq, k, lane); });
    } else {
        storer_body(sh, blockIdx.x, grid, nitems, lane, ring, full, empty, a.status,
                    [&](uint32_t k) { return resolved_desc<true, true>(rq, k, lane); });
        resolved_done(rq, nitems, lane);
    }
}

// ---------------------------------------------------------------- kv_pipe_scatter_read (fused)
// CTA c owns blocks c, c + grid, ...; the resolver warp resolves them in that order, one probe
// per key.  Loader and storer walk the CTA's local items k = 0, 1, ...: part (k / cpb) % nparts
// (sh.cpb chunks per part) of the CTA's block k / (nparts * sh.cpb), so every part of a block
// is moved by the CTA that resolved it.  The resolver re-checks each entry once the storer has
// handed its queue half back (every load of those blocks has completed by then).
__global__ void __launch_bounds__(kPipeThreads)
    kv_pipe_scatter_read_kernel(const __grid_constant__ ResolveArgs a,
                                const __grid_constant__ GatherParts parts, const Shape sh,
                                uint32_t nparts, uint32_t first_part) {
    extern __shared__ __align__(128) uint8_t ring[];
    __shared__ __align__(8) uint64_t full[kPipeMaxStages];
    __shared__ __align__(8) uint64_t empty[kPipeMaxStages];
    __shared__ __align__(16) ResolveQueue rq;
    const uint32_t grid = gridDim.x;
    const uint32_t nblocks = blockIdx.x < sh.n ? (sh.n - blockIdx.x + grid - 1) / grid : 0;
    const uint32_t per_block = nparts * sh.cpb;
    const uint32_t warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    if (threadIdx.x == 0) {
        for (uint32_t s = 0; s < sh.stages; ++s) {
            mbar_init(&full[s], 1);
            mbar_init(&empty[s], 1);
        }
        resolve_queue_init(rq);
        mbar_fence_init();
    }
    __syncthreads();
    if (warp == 2) {  // ---- resolver: a hit must hold every part asked for
        resolver_warp(a, rq, (first_part + nparts) * sh.bytes, blockIdx.x, grid, 1, nblocks, lane);
        return;
    }
    const bool storer = warp == 1;
    uint32_t cur_j = ~0u;  // the CTA's block whose descriptor `cur` holds
    CopyDesc cur{0, 0};
    auto desc_at = [&](uint32_t k) {  // warp-wide; k non-decreasing, so j advances one by one
        const uint32_t j = k / per_block;
        if (j != cur_j) {
            cur = storer ? resolved_desc<true, true>(rq, j, lane) : resolved_desc<false, true>(rq, j, lane);
            cur_j = j;
            // a missing key is one miss, whatever the number of parts
            if (storer && lane == 0 && cur.src == 0 && a.status) atomicAdd(a.status + kStatMiss, 1u);
        }
        const uint32_t s = (k / sh.cpb) % nparts;
        return CopyDesc{cur.src ? cur.src + uint64_t(first_part + s) * sh.bytes : 0,
                        parts.base[s] + cur.dst};
    };
    if (warp == 0) {
        loader_body(sh, 0, 1, nblocks * per_block, lane, ring, full, empty, desc_at);
    } else {
        storer_body(sh, 0, 1, nblocks * per_block, lane, ring, full, empty, nullptr, desc_at);
        resolved_done(rq, nblocks, lane);
    }
}

// ---------------------------------------------------------------- kv_pipe_mcast (clusters)
__device__ __forceinline__ uint32_t cluster_ctarank() {
    uint32_t r;
    asm volatile("mov.u32 %0, %%cluster_ctarank;" : "=r"(r));
    return r;
}
__device__ __forceinline__ void cluster_sync_all() {  // UCGABAR_ARV / UCGABAR_WAIT
    asm volatile("barrier.cluster.arrive.release.aligned;" ::: "memory");
    asm volatile("barrier.cluster.wait.acquire.aligned;" ::: "memory");
}
// arrive on the barrier at the same shared-memory offset in CTA `rank` of the cluster
__device__ __forceinline__ void mbar_arrive_remote(uint64_t* bar, uint32_t rank) {
    uint32_t remote;
    asm volatile("mapa.shared::cluster.u32 %0, %1, %2;" : "=r"(remote) : "r"(smem_u32(bar)), "r"(rank));
    asm volatile("mbarrier.arrive.release.cluster.shared::cluster.b64 _, [%0];" ::"r"(remote)
                 : "memory");
}
__device__ __forceinline__ void mbar_wait_cluster(uint64_t* bar, uint32_t parity) {
    const uint32_t addr = smem_u32(bar);
    uint32_t done = 0;
    long long start = 0;
    for (uint32_t spins = 0;; ++spins) {
        asm volatile(
            "{\n\t"
            ".reg .pred p;\n\t"
            "mbarrier.try_wait.parity.acquire.cluster.shared::cta.b64 p, [%1], %2;\n\t"
            "selp.u32 %0, 1, 0, p;\n\t"
            "}"
            : "=r"(done)
            : "r"(addr), "r"(parity)
            : "memory");
        if (done) return;
        if (spins == 64) start = clock64();
        if (spins > 64 && (spins & 1023) == 0 && clock64() - start > 8000000000ll) __trap();
    }
}
// global -> the shared memory of every CTA in `mask`, completing on the barrier at the same
// offset in each of them                                        UBLKCP.S.G ... MULTICAST
__device__ __forceinline__ void bulk_g2s_multicast(void* smem_dst, const void* gsrc,
                                                   uint32_t bytes, uint64_t* bar, uint16_t mask) {
    asm volatile(
        "cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes.multicast::cluster "
        "[%0], [%1], %2, [%3], %4;" ::"r"(smem_u32(smem_dst)),
        "l"(gsrc), "r"(bytes), "r"(smem_u32(bar)), "h"(mask)
        : "memory");
}

struct McastArgs {
    const CopyDesc* descs;  // src = pool block, dst = its place in destination 0
    uint32_t n, bytes, stage_bytes, stages;
    int64_t delta[4];  // destination r = dst + delta[r]   (delta[0] = 0)
    uint32_t* status;
};

template <int K>
__global__ void __launch_bounds__(64)
    kv_pipe_mcast_kernel(const __grid_constant__ McastArgs a) {
    extern __shared__ __align__(128) uint8_t ring[];
    __shared__ __align__(8) uint64_t full[kPipeMaxStages];   // per CTA: the tile has landed here
    __shared__ __align__(8) uint64_t empty[kPipeMaxStages];  // leader only: K CTAs released it
    const uint32_t rank = cluster_ctarank();
    const uint32_t cluster = blockIdx.x / K, nclusters = gridDim.x / K;
    const uint32_t nitems = cluster < a.n ? (a.n - cluster + nclusters - 1) / nclusters : 0;
    const uint32_t warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    if (threadIdx.x == 0) {
        for (uint32_t s = 0; s < a.stages; ++s) {
            mbar_init(&full[s], 1);
            mbar_init(&empty[s], K);
        }
        mbar_fence_init();
    }
    cluster_sync_all();  // every CTA's barriers exist before the leader multicasts into them
    DescWindow<false> win{a.descs, nullptr, cluster, nclusters, 1, nitems, lane};
    win.init();
    if (warp == 0) {
        if (rank == 0) {  // ---- leader's loader: one fetch over NVLink feeds K CTAs
            uint32_t s = 0, use = 0;
            for (uint32_t k = 0; k < nitems; ++k) {
                const CopyDesc d = win.at(k);
                for (uint32_t o = 0; o < a.bytes; o += a.stage_bytes) {
                    if (lane == 0) {
                        if (use) mbar_wait_cluster(&empty[s], (use - 1) & 1);
                        if (d.src)
                            bulk_g2s_multicast(ring + size_t(s) * a.stage_bytes,
                                               reinterpret_cast<const uint8_t*>(d.src) + o,
                                               min(a.stage_bytes, a.bytes - o), &full[s],
                                               uint16_t((1u << K) - 1));
                    }
                    if (++s == a.stages) {
                        s = 0;
                        ++use;
                    }
                }
            }
        }
    } else {  // ---- every CTA: store the tile to its own destination
        uint32_t s = 0, ph = 0, sf = 0, q = 0;
        for (uint32_t k = 0; k < nitems; ++k) {
            const CopyDesc d = win.at(k);
            if (lane == 0 && rank == 0 && d.src == 0 && a.status) atomicAdd(a.status + kStatMiss, 1u);
            for (uint32_t o = 0; o < a.bytes; o += a.stage_bytes, ++q) {
                if (lane == 0) {
                    const uint32_t plen = min(a.stage_bytes, a.bytes - o);
                    if (d.src) {
                        // arm this CTA's barrier for the bytes the leader multicasts (they may
                        // already have landed: the phase completes once both have happened)
                        mbar_expect_tx(&full[s], plen);
                        mbar_wait(&full[s], ph);
                        bulk_s2g(reinterpret_cast<uint8_t*>(int64_t(d.dst) + a.delta[rank]) + o,
                                 ring + size_t(s) * a.stage_bytes, plen);
                    } else {
                        // a miss: complete the phase to keep the parities in step - and wait for
                        // it like for any other (returns at once; synccheck insists that a
                        // completed phase has been waited for before the barrier is used again)
                        mbar_arrive(&full[s]);
                        mbar_wait(&full[s], ph);
                    }
                    bulk_commit();
                    bulk_wait_read<kStoreLag>();
                    if (q >= uint32_t(kStoreLag)) {
                        mbar_arrive_remote(&empty[sf], 0);  // DSMEM: hand the slot back to the leader
                        if (++sf == a.stages) sf = 0;
                    }
                }
                if (++s == a.stages) {
                    s = 0;
                    ph ^= 1;
                }
            }
        }
        if (lane == 0) {
            bulk_wait<0>();
            fence_proxy_async();
        }
    }
    __syncwarp();
    cluster_sync_all();  // nobody leaves while a sibling may still arrive on its barriers
}

// ---------------------------------------------------------------- kv_pipe_hnd (layout swizzle)
// read_cache fused with the layout change the attention consumer wants: pool pages are
// token-major, [tok][head][dim]; the destination KV cache is head-major, [page][head][tok][dim]
// (contiguous per head: what a paged-attention kernel streams).  The tile is loaded with one
// 1-D bulk copy (the pool page is contiguous) and STORED with a 4-D tensor-map TMA whose
// dimensions are declared in the order (dim, head, tok, page): the box (D, H, Tt, 1) then
// enumerates shared memory as [tok][head][dim] - exactly the source order - while the tensor
// map's strides scatter every (tok, head) row to its head-major place.  The transposition is
// done by the TMA unit: no thread touches the data, no separate pack/unpack kernel.
//   SASS: UBLKCP.S.G (load) + UTMASTG.4D (store).
__device__ __forceinline__ void tma_store_4d(const CUtensorMap* map, const void* smem_src,
                                             int32_t c0, int32_t c1, int32_t c2, int32_t c3) {
    asm volatile(
        "cp.async.bulk.tensor.4d.global.shared::cta.bulk_group [%0, {%1, %2, %3, %4}], [%5];" ::
            "l"(reinterpret_cast<uint64_t>(map)),
        "r"(c0), "r"(c1), "r"(c2), "r"(c3), "r"(smem_u32(smem_src))
        : "memory");
}

struct HndArgs {
    const CopyDesc* descs;  // src = pool page (mapped), dst = destination page index
    uint32_t n;
    uint32_t page_bytes;   // T * H * D * elem_size
    uint32_t tile_bytes;   // Tt * H * D * elem_size (one ring slot)
    uint32_t tile_tokens;  // Tt
    uint32_t stages;
    uint32_t* status;
};

__global__ void __launch_bounds__(64)
    kv_pipe_hnd_kernel(const __grid_constant__ CUtensorMap tmap, const HndArgs a) {
    extern __shared__ __align__(128) uint8_t ring[];
    __shared__ __align__(8) uint64_t full[kPipeMaxStages];
    __shared__ __align__(8) uint64_t empty[kPipeMaxStages];
    const uint32_t grid = gridDim.x;
    const uint32_t nitems = blockIdx.x < a.n ? (a.n - blockIdx.x + grid - 1) / grid : 0;
    const uint32_t warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    if (threadIdx.x == 0) {
        for (uint32_t s = 0; s < a.stages; ++s) {
            mbar_init(&full[s], 1);
            mbar_init(&empty[s], 1);
        }
        mbar_fence_init();
        asm volatile("prefetch.tensormap [%0];" ::"l"(reinterpret_cast<uint64_t>(&tmap)) : "memory");
    }
    __syncthreads();
    const Shape sh{a.n, a.page_bytes, a.page_bytes, 1, a.tile_bytes, a.stages};
    DescWindow<false> win{a.descs, nullptr, blockIdx.x, grid, 1, nitems, lane};
    win.init();
    if (warp == 0) {
        loader_body(sh, blockIdx.x, grid, nitems, lane, ring, full, empty,
                    [&](uint32_t k) { return win.at(k); });
        return;
    }
    uint32_t s = 0, ph = 0, sf = 0, q = 0;
    for (uint32_t k = 0; k < nitems; ++k) {
        const CopyDesc d = win.at(k);
        if (lane == 0 && d.src == 0 && a.status) atomicAdd(a.status + kStatMiss, 1u);
        uint32_t t0 = 0;
        for (uint32_t o = 0; o < a.page_bytes; o += a.tile_bytes, t0 += a.tile_tokens, ++q) {
            if (lane == 0) {
                mbar_wait(&full[s], ph);
                if (d.src)  // box (D, H, Tt, 1) at (0, 0, t0, page): tokens beyond T are clipped
                    tma_store_4d(&tmap, ring + size_t(s) * a.tile_bytes, 0, 0, int32_t(t0),
                                 int32_t(d.dst));
                bulk_commit();
                bulk_wait_read<kStoreLag>();
                if (q >= uint32_t(kStoreLag)) {
                    mbar_arrive(&empty[sf]);
                    if (++sf == a.stages) sf = 0;
                }
            }
            if (++s == a.stages) {
                s = 0;
                ph ^= 1;
            }
        }
    }
    if (lane == 0) {
        bulk_wait<0>();
        fence_proxy_async();
    }
}

cudaError_t ensure_pipe_attrs() {
    static bool done[64] = {false};
    const int kMax = 200 << 10;
    return set_smem_limits_once(
        done, {{reinterpret_cast<const void*>(kv_pipe_copy_kernel<false>), kMax},
               {reinterpret_cast<const void*>(kv_pipe_copy_kernel<true>), kMax},
               {reinterpret_cast<const void*>(kv_pipe_read_kernel), kMax},
               {reinterpret_cast<const void*>(kv_pipe_gather_kernel<false>), kMax},
               {reinterpret_cast<const void*>(kv_pipe_gather_kernel<true>), kMax},
               {reinterpret_cast<const void*>(kv_pipe_scatter_read_kernel), kMax},
               {reinterpret_cast<const void*>(kv_pipe_mcast_kernel<2>), kMax},
               {reinterpret_cast<const void*>(kv_pipe_mcast_kernel<4>), kMax},
               {reinterpret_cast<const void*>(kv_pipe_hnd_kernel), kMax}});
}

// cuTensorMapEncodeTiled through the runtime's driver-entry-point lookup: the module links
// cudart statically and must import on hosts without libcuda (CPU-only CI).
using EncodeTiledFn = CUresult (*)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*,
                                   const cuuint64_t*, const cuuint64_t*, const cuuint32_t*,
                                   const cuuint32_t*, CUtensorMapInterleave, CUtensorMapSwizzle,
                                   CUtensorMapL2promotion, CUtensorMapFloatOOBfill);
EncodeTiledFn encode_tiled_fn() {
    static EncodeTiledFn fn = [] {
        void* p = nullptr;
        cudaDriverEntryPointQueryResult q{};
        if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &p, cudaEnableDefault, &q) !=
                cudaSuccess ||
            q != cudaDriverEntryPointSuccess)
            p = nullptr;
        (void)cudaGetLastError();
        return reinterpret_cast<EncodeTiledFn>(p);
    }();
    return fn;
}

}  // namespace

cudaError_t launch_kv_pipe_copy(const CopyLaunch& a, cudaStream_t stream) {
    if (a.n == 0 || a.bytes == 0) return cudaSuccess;
    if ((a.bytes % 16) != 0 || (a.align_or & 15) != 0 || a.multicast) return cudaErrorInvalidValue;
    cudaError_t e = ensure_pipe_attrs();
    if (e != cudaSuccess) return e;
    const Publish pub = publish_of(a, true, a.trace, a.debug);
    FanOut fan;
    if (a.fan_n > 1) {
        if (a.fan_n > 4 || pub.recs) return cudaErrorInvalidValue;  // reads only
        fan.n = uint32_t(a.fan_n);
        for (int r = 0; r < a.fan_n; ++r) fan.delta[r] = a.fan_delta[r];
    }
    const LaunchPlan p = plan_pipe_copy(a, sm_count());
    const Shape sh{a.n, a.bytes, p.chunk, p.cpb, p.geo.stage_bytes, p.geo.stages};
    if (p.param) {
        PipeDescParam<kParamDescs> pd;
        std::memcpy(pd.d, a.descs_host, size_t(a.n) * sizeof(CopyDesc));
        kv_pipe_copy_kernel<true><<<p.ctas, kPipeThreads, p.geo.smem, stream>>>(a.descs, pd, sh, pub, fan);
    } else {
        const PipeDescParam<1> none{};
        kv_pipe_copy_kernel<false><<<p.ctas, kPipeThreads, p.geo.smem, stream>>>(a.descs, none, sh, pub, fan);
    }
    return cudaGetLastError();
}

cudaError_t launch_kv_pipe_gather(const GatherLaunch& a, cudaStream_t stream) {
    if (a.n == 0 || a.part_bytes == 0) return cudaSuccess;
    if (a.nparts == 0 || a.nparts > kGatherMaxParts || !a.part_base || (a.part_bytes % 16) != 0 ||
        (a.align_or & 15) != 0)
        return cudaErrorInvalidValue;
    cudaError_t e = ensure_pipe_attrs();
    if (e != cudaSuccess) return e;
    const LaunchPlan p = plan_pipe_gather(a, sm_count());
    if (!p.valid) return cudaErrorInvalidValue;  // the caller splits the batch
    const Shape sh{a.n * a.nparts, a.part_bytes, p.chunk, p.cpb, p.geo.stage_bytes, p.geo.stages};
    GatherParts parts;
    std::memcpy(parts.base, a.part_base, size_t(a.nparts) * sizeof(uint64_t));
    const LayerCommit lc = layer_of(a);
    auto* kernel = lc.state ? kv_pipe_gather_kernel<true> : kv_pipe_gather_kernel<false>;
    kernel<<<p.ctas, kPipeThreads, p.geo.smem, stream>>>(a.descs, parts, sh, a.nparts, a.first_part,
                                                         a.write, publish_of(a, a.write), lc);
    return cudaGetLastError();
}

bool scatter_read_fused_supported(const ReadFusedLaunch& r, const GatherLaunch& g) {
    return g.rows == 0 && g.nparts >= 1 && g.nparts <= kGatherMaxParts && g.part_base && g.part_bytes &&
           (g.part_bytes % 16) == 0 && (g.align_or & 15) == 0 &&
           r.n >= uint32_t(scatter_read_ctas(r, sm_count()));
}

cudaError_t launch_kv_pipe_scatter_read(const ReadFusedLaunch& r, const GatherLaunch& g,
                                        cudaStream_t stream) {
    if (r.n == 0) return cudaSuccess;
    if (!scatter_read_fused_supported(r, g) ||
        uint64_t(g.first_part + g.nparts) * g.part_bytes > 0xffffffffull ||
        uint64_t(r.n) * g.nparts > 0x7fffffffull)
        return cudaErrorInvalidValue;
    cudaError_t e = ensure_pipe_attrs();
    if (e != cudaSuccess) return e;
    const PipeGeometry geo = pipe_geometry(g.part_bytes, r.stage_bytes, r.ring_bytes);
    GatherParts parts;
    std::memcpy(parts.base, g.part_base, size_t(g.nparts) * sizeof(uint64_t));
    // whole parts as items: a CTA moves whole blocks, the ring cuts them into pieces
    const Shape sh{r.n, g.part_bytes, g.part_bytes, 1, geo.stage_bytes, geo.stages};
    kv_pipe_scatter_read_kernel<<<scatter_read_ctas(r, sm_count()), kPipeThreads, geo.smem, stream>>>(
        resolve_args(r), parts, sh, g.nparts, g.first_part);
    return cudaGetLastError();
}

cudaError_t launch_kv_pipe_read(const ReadFusedLaunch& a, cudaStream_t stream) {
    if (a.n == 0 || a.bytes == 0) return cudaSuccess;
    if (!pipe_read_supported(a)) return cudaErrorInvalidValue;
    cudaError_t e = ensure_pipe_attrs();
    if (e != cudaSuccess) return e;
    const LaunchPlan p = plan_pipe_read(a, sm_count());
    const Shape sh{a.n, a.bytes, p.chunk, p.cpb, p.geo.stage_bytes, p.geo.stages};
    kv_pipe_read_kernel<<<p.ctas, kPipeThreads, p.geo.smem, stream>>>(resolve_args(a), sh);
    return cudaGetLastError();
}

cudaError_t launch_kv_pipe_hnd(const HndLaunch& a, cudaStream_t stream) {
    if (a.n == 0) return cudaSuccess;
    const uint64_t row = uint64_t(a.dim) * a.elem_size;          // one (tok, head) row
    const uint64_t tok_bytes = row * a.heads;                      // one token of a pool page
    const uint64_t page_bytes = tok_bytes * a.tokens;
    if (!a.tokens || !a.heads || !a.dim || a.dim > 256 || a.heads > 256 || row % 16 ||
        (a.elem_size != 1 && a.elem_size != 2 && a.elem_size != 4) || page_bytes > (1ull << 30) ||
        (a.dst_base & 15) || !a.num_pages)
        return cudaErrorInvalidValue;
    EncodeTiledFn encode = encode_tiled_fn();
    if (!encode) return cudaErrorNotSupported;
    cudaError_t e = ensure_pipe_attrs();
    if (e != cudaSuccess) return e;
    // ring slot = as many whole tokens as fit 16 KB (at least one), box dims are <= 256
    const uint32_t stage_cap = a.stage_bytes ? a.stage_bytes : (16u << 10);
    uint32_t tt = uint32_t(std::max<uint64_t>(1, stage_cap / tok_bytes));
    tt = std::min<uint32_t>({tt, a.tokens, 256u});
    const uint32_t tile_bytes = uint32_t(tt * tok_bytes);
    if (tile_bytes > (96u << 10)) return cudaErrorInvalidValue;  // one token must fit a slot
    const uint32_t ring = a.ring_bytes ? a.ring_bytes : (64u << 10);
    const uint32_t stages = std::max<uint32_t>(kStoreLag + 1,
                                               std::min<uint32_t>(kPipeMaxStages, ring / tile_bytes));
    CUtensorMap tmap;
    const CUtensorMapDataType dt = a.elem_size == 2 ? CU_TENSOR_MAP_DATA_TYPE_UINT16
                                   : a.elem_size == 4 ? CU_TENSOR_MAP_DATA_TYPE_UINT32
                                                      : CU_TENSOR_MAP_DATA_TYPE_UINT8;
    // destination [page][head][tok][dim], declared as (dim, head, tok, page)
    const cuuint64_t gdim[4] = {a.dim, a.heads, a.tokens, a.num_pages};
    const cuuint64_t gstr[3] = {uint64_t(a.tokens) * row, row, page_bytes};
    const cuuint32_t box[4] = {a.dim, a.heads, tt, 1};
    const cuuint32_t estr[4] = {1, 1, 1, 1};
    if (encode(&tmap, dt, 4, reinterpret_cast<void*>(a.dst_base), gdim, gstr, box, estr,
               CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_NONE,
               CU_TENSOR_MAP_L2_PROMOTION_L2_256B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE) != CUDA_SUCCESS)
        return cudaErrorInvalidValue;
    HndArgs h{};
    h.descs = a.descs;
    h.n = a.n;
    h.page_bytes = uint32_t(page_bytes);
    h.tile_bytes = tile_bytes;
    h.tile_tokens = tt;
    h.stages = stages;
    h.status = a.status;
    const size_t smem = size_t(stages) * tile_bytes;
    const int ctas = clamp_grid(capped_grid(a.max_ctas, sm_count()), a.n);
    kv_pipe_hnd_kernel<<<ctas, 64, smem, stream>>>(tmap, h);
    return cudaGetLastError();
}

cudaError_t launch_kv_pipe_mcast(const McastLaunch& a, cudaStream_t stream) {
    if (a.n == 0 || a.bytes == 0) return cudaSuccess;
    if ((a.ndst != 2 && a.ndst != 4) || (a.bytes % 16) != 0 || (a.align_or & 15) != 0)
        return cudaErrorInvalidValue;
    // The multicast bulk load is used on LOCAL sources only: with a peer-mapped source
    // (NVLink aperture) the launch once wedged a GPU - the fabric path
    // of multicast TMA reads is not something this store relies on.  Peer sources take the
    // fan-out flavour of kv_pipe_copy instead (one load, K stores per CTA).
    if (!a.src_local) return cudaErrorNotSupported;
    cudaError_t e = ensure_pipe_attrs();
    if (e != cudaSuccess) return e;
    // two CTAs of a cluster may share an SM: keep the ring at half the usual size
    const PipeGeometry g = pipe_geometry(a.bytes, a.stage_bytes, a.ring_bytes ? a.ring_bytes : (64u << 10));
    McastArgs m{};
    m.descs = a.descs;
    m.n = a.n;
    m.bytes = a.bytes;
    m.stage_bytes = g.stage_bytes;
    m.stages = g.stages;
    for (int r = 0; r < 4; ++r) m.delta[r] = r < a.ndst ? a.delta[r] : 0;
    m.status = a.status;
    // a caller's cluster count is not bounded by the SM count
    const int clusters = clamp_grid(a.max_clusters > 0 ? a.max_clusters : sm_count() / a.ndst, a.n);
    cudaLaunchConfig_t cfg{};
    cfg.gridDim = dim3(unsigned(clusters * a.ndst));
    cfg.blockDim = dim3(64);
    cfg.dynamicSmemBytes = g.smem;
    cfg.stream = stream;
    cudaLaunchAttribute attr[1];
    attr[0].id = cudaLaunchAttributeClusterDimension;
    attr[0].val.clusterDim.x = unsigned(a.ndst);
    attr[0].val.clusterDim.y = 1;
    attr[0].val.clusterDim.z = 1;
    cfg.attrs = attr;
    cfg.numAttrs = 1;
    if (a.ndst == 2) return cudaLaunchKernelEx(&cfg, kv_pipe_mcast_kernel<2>, m);
    return cudaLaunchKernelEx(&cfg, kv_pipe_mcast_kernel<4>, m);
}

}  // namespace istore::kernels
