// kv_doorbell: a persistent worker CTA for single-block operations (the latency path).
//
// A write or read of ONE block through the ordinary path costs a kernel launch, an event
// record + wait when it runs on an internal stream, and a completion that the host detects by
// polling the stream; for a 4 KB block the data movement is the smallest part.  With
// ClientConfig(doorbell=True) the client keeps ONE CTA resident that polls a request ring in
// pinned host memory:
//
//   host   : fills a 64-byte request line {seq|op, local address, pool address, key
//            fingerprint, block address / generation / size, checksum} - seq last - and
//            later spins on `done_seq` in the same pinned page
//   worker : lanes 0..7 of the control warp read the line with one coalesced request over
//            PCIe; a line whose sequence number or checksum does not match is "nothing yet".
//            WRITE: control lane claims the key's way in the HBM index (CAS over NVLink)
//                   while the copy warps move the block with 128-bit L2-only loads; then
//                   st.release.sys of the tag (MEMBAR.SYS + store: the in-band commit)
//            READ : control lane probes the index, copy warps pull the block, the tag is
//                   re-checked after the copy (purge / eviction safe, as on every device path)
//            both : status word, then st.release.sys of done_seq into host memory
//
// The worker leaves when no request arrived for `idle_ns` (so a device-wide synchronise
// never waits longer than that) and says so in `state`; the host relaunches it with the next
// request.  One block per request, at most kDoorbellMaxBytes; anything else takes the
// ordinary path.  Replaces, for this case, the reference's per-request stream + event +
// cudaMemcpyAsync + cudaEventSynchronize (src/infinistore.cpp:570-804) and its COMMIT message.
#include <algorithm>

#include "../core/hash.h"
#include "common.cuh"
#include "index.cuh"
#include "kernels.h"
#include "publish.cuh"

namespace istore::kernels {

namespace {

using namespace dev;

constexpr int kThreads = 1024;      // warp 0: control, warps 1..31: copy (62 KB in flight per round)
constexpr int kCopyThreads = kThreads - 32;
constexpr int kBarAll = 2;          // named barrier: control + copy warps

__device__ __forceinline__ void bar_all() {
    asm volatile("bar.sync %0, %1;" ::"n"(kBarAll), "n"(kThreads) : "memory");
}
__device__ __forceinline__ void st_release_sys_u64(uint64_t* p, uint64_t v) {
    asm volatile("st.release.sys.global.u64 [%0], %1;" ::"l"(p), "l"(v) : "memory");
}
__device__ __forceinline__ void st_relaxed_sys_u32(uint32_t* p, uint32_t v) {
    asm volatile("st.relaxed.sys.global.u32 [%0], %1;" ::"l"(p), "r"(v) : "memory");
}

// L2-only load: the worker outlives the caller's rewrites of a buffer (and the pool's reuse of
// a block), so nothing it copies may come out of this SM's L1            LDG.E.128.STRONG.GPU
__device__ __forceinline__ uint4 ld_cg_v4(const void* p) {
    uint4 r;
    asm volatile("ld.global.cg.v4.u32 {%0,%1,%2,%3}, [%4];"
                 : "=r"(r.x), "=r"(r.y), "=r"(r.z), "=r"(r.w)
                 : "l"(p)
                 : "memory");
    return r;
}
__device__ __forceinline__ uint8_t ld_cg_u8(const void* p) {
    uint32_t r;
    asm volatile("ld.global.cg.u8 %0, [%1];" : "=r"(r) : "l"(p) : "memory");
    return uint8_t(r);
}

// `len` bytes, src -> dst, by the copy warps (tid = 0 .. kCopyThreads-1)
__device__ __forceinline__ void copy_block(uint8_t* dst, const uint8_t* src, uint32_t len,
                                           uint32_t tid) {
    const uint64_t a = reinterpret_cast<uint64_t>(dst) | reinterpret_cast<uint64_t>(src) | len;
    if ((a & 15) == 0) {
        constexpr int U = 4;
        const uint32_t nvec = len / 16;
        uint32_t i = tid;
        for (; i + (U - 1) * kCopyThreads < nvec; i += U * kCopyThreads) {
            uint4 v[U];
#pragma unroll
            for (int u = 0; u < U; ++u) v[u] = ld_cg_v4(src + size_t(i + u * kCopyThreads) * 16);
#pragma unroll
            for (int u = 0; u < U; ++u) st_v4(dst + size_t(i + u * kCopyThreads) * 16, v[u]);
        }
        for (; i < nvec; i += kCopyThreads) st_v4(dst + size_t(i) * 16, ld_cg_v4(src + size_t(i) * 16));
    } else {
        for (uint32_t i = tid; i < len; i += kCopyThreads) dst[i] = ld_cg_u8(src + i);
    }
}

struct Shared {
    uint64_t q[8];       // the request line
    uint32_t have;       // 1: q holds request `next`; 2: leave
    uint64_t pool_addr;  // READ: resolved source (0 = miss)
    uint32_t slot, tag;  // READ: what the probe resolved (for the re-check)
};

__global__ void __launch_bounds__(kThreads)
    kv_doorbell_kernel(const __grid_constant__ DoorbellLaunch a) {
    __shared__ Shared sh;
    const uint32_t warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    uint64_t next = a.first_seq;
    unsigned long long idle_since = globaltimer_ns();
    if (threadIdx.x == 0)
        st_release_sys_u64(&a.ctl->state, doorbell_state(a.epoch, next, kDoorbellRunning));
    Publish pub{};
    pub.table = a.table;
    pub.mask = a.table_mask;
    pub.status = nullptr;
    pub.sys = a.sys;
    pub.shards = a.shards;
    for (;;) {
        // ---- poll: one coalesced 64-byte read of the request line over PCIe
        if (warp == 0) {
            const uint64_t* line = a.ring[next % a.slots].q;
            uint64_t v = lane < 8 ? ld_relaxed_sys_u64(line + lane) : 0;
            uint64_t x = lane < 7 ? v : 0;  // checksum over q0..q6
#pragma unroll
            for (int o = 4; o > 0; o >>= 1) x ^= __shfl_xor_sync(0xffffffffu, x, o);
            x = __shfl_sync(0xffffffffu, x, 0);
            const uint64_t q0 = __shfl_sync(0xffffffffu, v, 0);
            const uint64_t q7 = __shfl_sync(0xffffffffu, v, 7);
            const bool ok = (q0 >> 2) == next && q7 == (x ^ kDoorbellMagic);
            if (lane < 8) sh.q[lane] = v;
            uint32_t have = ok ? 1u : 0u;
            if (!ok && lane == 0 && globaltimer_ns() - idle_since > a.idle_ns) have = 2;
            have = __shfl_sync(0xffffffffu, have, 0);
            if (lane == 0) sh.have = have;
        }
        bar_all();
        const uint32_t have = sh.have;
        if (have == 2 || (have == 1 && (sh.q[0] & 3) == kDoorbellStop)) {
            if (threadIdx.x == 0) {
                const uint64_t at = have == 1 ? next + 1 : next;  // a STOP request is consumed
                if (have == 1) {
                    st_relaxed_sys_u32(&a.ctl->status[next % a.slots], kDoorbellOk);
                    st_release_sys_u64(&a.ctl->done_seq, next);
                }
                st_release_sys_u64(&a.ctl->state, doorbell_state(a.epoch, at, kDoorbellExited));
            }
            return;
        }
        if (have == 0) {
            bar_all();  // sh is rewritten by the next poll
            continue;
        }
        // ---- a request
        const uint32_t op = uint32_t(sh.q[0] & 3);
        const uint64_t local = sh.q[1];
        const uint32_t bytes = uint32_t(sh.q[6] >> 32);
        uint32_t status = kDoorbellOk;
        if (op == kDoorbellWrite) {
            uint32_t slot = 0;
            const IndexEntry rec{sh.q[3], sh.q[4], sh.q[5], uint32_t(sh.q[6]), bytes};
            if (warp == 0) {
                // claim (one CAS round trip) while the copy warps move the block
                if (lane == 0 && a.table && rec.h1) {
                    bool full = false;
                    const idx::TableRef t = idx::select_shard(pub.table, pub.mask, pub.shards, rec.h2);
                    slot = idx::pack_slot(t.shard, idx::claim(t.table, t.mask, rec, pub.sys, &full));
                    if (full) status = kDoorbellIndexFull;
                }
            } else {
                copy_block(reinterpret_cast<uint8_t*>(sh.q[2]), reinterpret_cast<const uint8_t*>(local),
                           bytes, threadIdx.x - 32);
            }
            bar_all();  // the copy warps' stores are ordered before the release below (CTA scope)
            if (threadIdx.x == 0) {
                // In-band commit.  st.release.sys = MEMBAR.SYS + store: cumulative over the
                // stores of the whole CTA (they happen-before through the barrier), so a reader
                // on any GPU that observes the tag observes the block.
                if (slot) {
                    IndexBucket* tb = idx::table_of_slot(pub.table, pub.shards, slot);
                    st_release_sys(&idx::way_of(tb, idx::slot_local(slot) - 1)->tag, rec.tag);
                } else {
                    fence_sys();  // no index entry (server-only visibility): the data all the same
                }
            }
        } else {  // kDoorbellRead
            if (threadIdx.x == 0) {
                const KeyHash kh{sh.q[3], sh.q[4]};
                const idx::TableRef t = idx::select_shard(a.table, a.table_mask, a.shards, kh.h2);
                idx::Found f = idx::find<false>(t.table, t.mask, kh);
                f.slot_plus1 = idx::pack_slot(t.shard, f.slot_plus1);
                uint64_t src = 0;
                if (f.slot_plus1) {
                    const uint32_t seg = uint32_t(f.addr >> 44) - 1;
                    if (f.size >= bytes && seg < a.nsegs && a.seg_base[seg])
                        src = a.seg_base[seg] + (f.addr & ((1ull << 44) - 1));
                }
                sh.pool_addr = src;
                sh.slot = src ? f.slot_plus1 : 0;
                sh.tag = f.tag;
            }
            bar_all();
            const uint64_t src = sh.pool_addr;
            if (warp != 0 && src)
                copy_block(reinterpret_cast<uint8_t*>(local), reinterpret_cast<const uint8_t*>(src),
                           bytes, threadIdx.x - 32);
            bar_all();
            if (threadIdx.x == 0) {
                if (!src)
                    status = kDoorbellMiss;
                else if (!idx::still_valid(idx::table_of_slot(a.table, a.shards, sh.slot),
                                           idx::slot_local(sh.slot), sh.tag))
                    status = kDoorbellStale;
            }
        }
        if (threadIdx.x == 0) {
            st_relaxed_sys_u32(&a.ctl->status[next % a.slots], status);
            // release: the tag store (writes) / the local data stores (reads) are performed
            // before the host can see the request as done
            st_release_sys_u64(&a.ctl->done_seq, next);
            idle_since = globaltimer_ns();
        }
        ++next;
        bar_all();  // sh is rewritten by the next poll
    }
}

}  // namespace

cudaError_t launch_kv_doorbell(const DoorbellLaunch& a, cudaStream_t stream) {
    if (!a.ring || !a.ctl || a.slots == 0 || a.slots > uint32_t(kDoorbellMaxSlots))
        return cudaErrorInvalidValue;
    kv_doorbell_kernel<<<1, kThreads, 0, stream>>>(a);
    return cudaGetLastError();
}

}  // namespace istore::kernels
