// In-band commit: how a writer kernel makes a block visible in the HBM-resident index.
//
// Replaces the reference's COMMIT control message (client SEND after the RDMA writes,
// src/libinfinistore.cpp:362-395; server flips `committed`, src/infinistore.cpp:255-271)
// with a release-ordered publication from the kernel that moved the data: a reader on any
// GPU that observes the entry's tag (ld.acquire.sys) is guaranteed to observe the block.
//
// Two phases, run by a dedicated CONTROL WARP of every CTA so that the copy warps never
// wait on a fabric round trip (doing the whole insertion after the data would add the
// claim's NVLink round trips to every launch's tail):
//   claim  (kernel start, overlaps the copy): CAS a way's h1 from 0 (one NVLink round
//          trip), fill h2/addr/size with posted stores; tag stays 0 = invisible.
//   commit (after the block's last chunk has landed): one posted st.release.sys of the tag.
// Chunks of one block may be moved by several CTAs: completion is counted with
// client-local atomics; slot and tag travel through client-local scratch.
#pragma once

#include "common.cuh"
#include "index.cuh"
#include "kernels.h"

namespace istore::kernels {

using namespace dev;

struct Publish {
    const IndexEntry* recs;  // one record per block (device-addressable, may be host memory)
    IndexBucket* table;
    uint64_t mask;  // bucket mask
    uint32_t* scratch;  // 3*n zeroed u32 in client-local device memory: done | slot+1 | tag
    uint32_t* status;
    uint32_t n;
    unsigned long long* trace = nullptr;  // optional: 8 %globaltimer stamps per CTA (bench only)
    // true: some destination (pool block or index table) is NOT in this GPU's own HBM, so
    // "performed" must mean acknowledged across NVLink: fence.acq_rel.sys (MEMBAR.SYS +
    // ERRBAR).  false: everything is local; the local L2 is the point of coherence
    // for local memory, also for peers reading it over NVLink, so gpu scope suffices.
    bool sys = true;
    uint32_t debug = 0;  // bench only: 1 = skip claim, 2 = skip fence, 4 = skip commit store
    IndexShards shards;  // further index shards (shard 0 = table / mask)
};

__device__ inline unsigned long long globaltimer_ns() {
    unsigned long long t;
    asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t));
    return t;
}

// Reserve a way for `rec` (index.cuh).  Returns slot + 1, or 0 when nothing is to be
// committed (the key is already published - first writer wins - or its buckets are full).
__device__ inline uint32_t claim_entry(const Publish& pub, const IndexEntry& rec) {
    bool full = false;
    const idx::TableRef t = idx::select_shard(pub.table, pub.mask, pub.shards, rec.h2);
    const uint32_t s = idx::claim(t.table, t.mask, rec, pub.sys, &full);
    if (full && pub.status) atomicAdd(pub.status + kStatPublishFail, 1u);
    return idx::pack_slot(t.shard, s);
}

// The caller has just executed fence.acq_rel.sys; fence + relaxed store is a release
// pattern, so the tag needs no second MEMBAR.SYS/ERRBAR (the most expensive instruction of
// the epilogue).
__device__ inline void commit_entry(const Publish& pub, uint32_t slot_plus1, uint32_t tag) {
    if (!slot_plus1 || (pub.debug & 4)) return;
    idx::commit(idx::table_of_slot(pub.table, pub.shards, slot_plus1), idx::slot_local(slot_plus1),
                tag, pub.sys);
}

constexpr int kCtrlBarrier = 1;  // named barrier shared by the copy warps and the control warp

__device__ inline void ctrl_barrier_arrive(uint32_t threads) {
    asm volatile("bar.arrive %0, %1;" ::"n"(kCtrlBarrier), "r"(threads) : "memory");
}
__device__ inline void ctrl_barrier_sync(uint32_t threads) {
    asm volatile("bar.sync %0, %1;" ::"n"(kCtrlBarrier), "r"(threads) : "memory");
}

// Body of the control warp.  The CTA moves items first, first+stride, ... (count of them);
// item i is chunk i % cpb of block i / cpb.  `cta_threads` = copy threads + 32.
// Ordering: the copy threads' bar.arrive orders their data stores before the control warp's
// bar.sync at CTA scope; each lane then issues ONE cumulative fence.acq_rel.sys before its
// counter increments, so the whole CTA's stores are performed system-wide first (one fence
// per lane of one warp, not one per copy thread: MEMBAR.SYS is the expensive part).
__device__ inline void control_warp(const Publish& pub, uint32_t lane, uint32_t first,
                                    uint32_t count, uint32_t stride, uint32_t cpb,
                                    uint32_t cta_threads) {
    unsigned long long* tr = pub.trace && lane == 0 ? pub.trace + size_t(blockIdx.x) * 8 : nullptr;
    if (tr) tr[0] = globaltimer_ns();
    uint32_t* done = pub.scratch;
    uint32_t* slot_of = pub.scratch + pub.n;
    uint32_t* tag_of = pub.scratch + 2 * size_t(pub.n);
    // ---- claim (overlaps the copy)
    uint32_t my_slot = 0, my_tag = 0;  // valid for this lane's first claimed item (cpb == 1 path)
    for (uint32_t k = lane; k < count; k += 32) {
        const uint32_t item = first + k * stride;
        if (item % cpb) continue;
        const uint32_t block = item / cpb;
        const IndexEntry rec = pub.recs[block];
        const uint32_t s = (pub.debug & 1) ? uint32_t(rec.h1 & pub.mask) + 1 : claim_entry(pub, rec);
        if (cpb == 1 && count <= 32) {
            my_slot = s;
            my_tag = rec.tag;
        } else {
            slot_of[block] = s;
            tag_of[block] = rec.tag;
        }
    }
    if (tr) tr[1] = globaltimer_ns();  // claims done
    // ---- wait until every copy thread of this CTA has issued its last store
    ctrl_barrier_sync(cta_threads);
    if (tr) tr[2] = globaltimer_ns();  // copy warps done issuing
    // The ONE expensive fence of the epilogue: when it completes, every data store of this
    // CTA (and the claim's field stores) has been performed where its readers will look.
    if (pub.debug & 2) {
    } else if (pub.sys)
        fence_sys();
    else
        fence_gpu();
    if (tr) tr[3] = globaltimer_ns();  // stores performed
    // ---- commit
    if (cpb == 1 && count <= 32) {
        if (lane < count) commit_entry(pub, my_slot, my_tag);
        if (tr) tr[4] = globaltimer_ns();
        return;
    }
    for (uint32_t k = lane; k < count; k += 32) {
        const uint32_t block = (first + k * stride) / cpb;
        // acq_rel counter in local memory: every arriver fenced its stores BEFORE its
        // increment, so when the last arriver observes the full count all chunks of the block
        // are already performed; its tag store is issued after that in program order
        // (no second MEMBAR.SYS).
        const uint32_t arrived = cpb == 1 ? 1 : atom_add_acq_rel_gpu(done + block, 1u) + 1;
        if (arrived != cpb) continue;
        const uint32_t s = __ldcg(slot_of + block);
        const uint32_t t = __ldcg(tag_of + block);
        done[block] = 0;  // leave the scratch zeroed for the next launch
        slot_of[block] = 0;
        tag_of[block] = 0;
        commit_entry(pub, s, t);
    }
    if (tr) tr[4] = globaltimer_ns();
}

}  // namespace istore::kernels
