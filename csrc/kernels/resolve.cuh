// The resolver warp of the fused reads (kv_pipe_read, kv_fp8_pipe<read, fused>).
//
// One warp of the CTA turns keys into {pool address, destination}: lane l hashes the key of
// the CTA's l-th item of the current batch of 32, probes the (sharded) HBM index - over
// NVLink when the pool is remote - and writes the descriptor into one half of a
// double-buffered shared-memory queue.  mbarriers hand the halves to the consumers (loader and
// storer) and back, so resolution runs up to two batches ahead of the copy and the copy
// never waits for a probe except at the very start.  This is what makes read_cache ONE launch
// with no server round trip; the reference resolves keys in the server's map and answers with
// a message (src/infinistore.cpp:424-533).
//
// Optimistic read: no lease is taken.  With ReadFusedLaunch::validate (and a status array),
// once the storer has handed a half back - every byte of its items has been read from the pool
// by then - the resolver re-loads the tags it resolved.  An item whose block was purged or
// evicted meanwhile (its space may already belong to another key) shows a changed tag and is
// reported as a miss (kStatMiss + kStatStale), once per item: a block split into several
// chunks counts once for each chunk that saw the change.
#pragma once

#include "../core/hash.h"
#include "common.cuh"
#include "index.cuh"
#include "kernels.h"

namespace istore::kernels {

struct ResolveArgs {
    const uint8_t* key_bytes;  // packed keys (pinned ring), 8-byte aligned and zero padded
    const uint32_t* key_off;
    const uint32_t* key_len;
    const uint64_t* dst_off;
    uint64_t dst_base;
    const IndexBucket* table;
    uint64_t table_mask;
    IndexShards shards;
    uint64_t seg_base[ReadFusedLaunch::kMaxSegs];
    uint32_t nsegs;
    uint32_t* status;
    bool validate;  // re-check every resolved entry after its copy
};

inline ResolveArgs resolve_args(const ReadFusedLaunch& a) {
    ResolveArgs r{};
    r.key_bytes = a.key_bytes;
    r.key_off = a.key_off;
    r.key_len = a.key_len;
    r.dst_off = a.dst_off;
    r.dst_base = a.dst_base;
    r.table = a.table;
    r.table_mask = a.table_mask;
    r.shards = a.shards;
    r.nsegs = a.nsegs;
    for (uint32_t s = 0; s < a.nsegs && s < uint32_t(ReadFusedLaunch::kMaxSegs); ++s)
        r.seg_base[s] = a.seg_base[s];
    r.status = a.status;
    r.validate = a.validate;
    return r;
}

constexpr int kResolveBatch = 32;  // descriptors per queue half: one per resolver lane

struct ResolveQueue {
    uint64_t qfull[2];
    uint64_t qempty[2];
    CopyDesc queue[2][kResolveBatch];
};

namespace dev {

__device__ __forceinline__ void resolve_queue_init(ResolveQueue& q) {  // one thread, before the CTA barrier
    mbar_init(&q.qfull[0], 1);
    mbar_init(&q.qfull[1], 1);
    mbar_init(&q.qempty[0], 1);
    mbar_init(&q.qempty[1], 1);
}

// Item k of the CTA is global item first + k * stride = chunk (item % cpb) of block
// (item / cpb).  A block that is split over several CTAs is resolved (and re-checked) by each
// of them: a few redundant probes instead of a second launch.
__device__ __forceinline__ void resolver_warp(const ResolveArgs& a, ResolveQueue& q,
                                              uint32_t need_bytes, uint32_t first, uint32_t stride,
                                              uint32_t cpb, uint32_t nitems, uint32_t lane) {
    const uint32_t nbatches = (nitems + kResolveBatch - 1) / kResolveBatch;
    uint32_t vslot0 = 0, vtag0 = 0, vslot1 = 0, vtag1 = 0;  // scalars: no local memory
    auto recheck = [&](uint32_t p) {
        const uint32_t slot = p ? vslot1 : vslot0, tag = p ? vtag1 : vtag0;
        if (slot && a.validate && a.status &&
            !idx::still_valid(idx::table_of_slot(a.table, a.shards, slot), idx::slot_local(slot), tag)) {
            atomicAdd(a.status + kStatMiss, 1u);
            atomicAdd(a.status + kStatStale, 1u);
        }
        if (p)
            vslot1 = 0;
        else
            vslot0 = 0;
    };
    for (uint32_t b = 0; b < nbatches; ++b) {
        const uint32_t p = b & 1;
        if (b >= 2) {
            mbar_wait(&q.qempty[p], ((b >> 1) - 1) & 1);
            recheck(p);
        }
        const uint32_t k = b * kResolveBatch + lane;
        if (k < nitems) {
            const uint32_t block = (first + k * stride) / cpb;
            const KeyHash kh = hash_key(a.key_bytes + a.key_off[block], a.key_len[block]);
            const idx::TableRef t = idx::select_shard(a.table, a.table_mask, a.shards, kh.h2);
            idx::Found f = idx::find<false>(t.table, t.mask, kh);
            f.slot_plus1 = idx::pack_slot(t.shard, f.slot_plus1);
            uint64_t src = 0;
            if (f.slot_plus1) {
                const uint32_t seg = uint32_t(f.addr >> 44) - 1;
                if (f.size >= need_bytes && seg < a.nsegs && a.seg_base[seg])
                    src = a.seg_base[seg] + (f.addr & ((1ull << 44) - 1));
            }
            q.queue[p][lane] = CopyDesc{src, a.dst_base + a.dst_off[block]};
            if (p) {
                vslot1 = src ? f.slot_plus1 : 0;
                vtag1 = f.tag;
            } else {
                vslot0 = src ? f.slot_plus1 : 0;
                vtag0 = f.tag;
            }
        }
        __syncwarp();
        if (lane == 0) mbar_arrive(&q.qfull[p]);  // release: the queue half is visible
    }
    for (uint32_t b = nbatches >= 2 ? nbatches - 2 : 0; b < nbatches; ++b) {  // the tail
        mbar_wait(&q.qempty[b & 1], (b >> 1) & 1);
        recheck(b & 1);
    }
}

// Consumer side.  Loader and storer walk k = 0, 1, 2, ... in order.  The RELEASING consumer
// (the storer: the last one to need a descriptor, and the one that knows when the loads of a
// block have completed) hands the previous half back when it enters a new one and calls
// resolved_done() after its last item.  kWarpWide: all 32 lanes of the consumer warp make the
// call (and read the queue), so they are joined before a half is released.
template <bool kReleases, bool kWarpWide>
__device__ __forceinline__ CopyDesc resolved_desc(ResolveQueue& q, uint32_t k, uint32_t lane) {
    const uint32_t b = k / kResolveBatch, p = b & 1;
    if (k % kResolveBatch == 0) {
        if (kReleases && k) {
            if (kWarpWide) __syncwarp();
            if (lane == 0) mbar_arrive(&q.qempty[p ^ 1]);
        }
        mbar_wait(&q.qfull[p], (b >> 1) & 1);
    }
    return q.queue[p][k % kResolveBatch];
}
__device__ __forceinline__ void resolved_done(ResolveQueue& q, uint32_t nitems, uint32_t lane) {
    if (lane == 0 && nitems) mbar_arrive(&q.qempty[((nitems - 1) / kResolveBatch) & 1]);
}

}  // namespace dev
}  // namespace istore::kernels
