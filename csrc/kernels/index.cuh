// The key index algorithm: claim / find / erase / validate on the bucketed table
// (kernels.h: IndexBucket).  Written once for both sides: the sm_90a kernels run it with
// system-scope PTX memory operations on (usually peer-mapped) HBM, the native unit tests
// run the same code on the CPU with __atomic builtins, threads standing in for GPUs.
//
// Replaces the reference's std::unordered_map<string> probes on the server CPU
// (src/infinistore.cpp:63-65, 1077-1108) for every client that reads through the device
// path; the server's host map stays the authority for allocation and first-writer-wins.
//
// Concurrency contract
//   writer : claim (CAS h1 0 -> fingerprint) ... data stores ... fence ... tag := gen
//   reader : find  (fingerprints, tag with acquire, then the fields) ... copy ...
//            validate (tag unchanged)   [validate only when the server evicts]
//   evictor: tag := 0, fence, h1 := 0   (server, before the block's space is reused)
// A reader that loses a race against evictor + new writer of the same way reads fields or
// bytes of another block; the changed tag exposes it and the read is reported as a miss.
#pragma once

#include <cstdint>

#include "../core/hash.h"
#include "kernels.h"

#if defined(__CUDACC__)
#include "common.cuh"
#endif

namespace istore::kernels::idx {

// ---------------------------------------------------------------- memory primitives
IS_HD uint64_t ld_u64(const uint64_t* p) {
#if defined(__CUDA_ARCH__)
    return dev::ld_relaxed_sys_u64(p);
#else
    return __atomic_load_n(p, __ATOMIC_RELAXED);
#endif
}
IS_HD uint32_t ld_u32(const uint32_t* p) {
#if defined(__CUDA_ARCH__)
    uint32_t v;
    asm volatile("ld.relaxed.sys.global.u32 %0, [%1];" : "=r"(v) : "l"(p) : "memory");
    return v;
#else
    return __atomic_load_n(p, __ATOMIC_RELAXED);
#endif
}
IS_HD uint32_t ld_acquire_u32(const uint32_t* p) {
#if defined(__CUDA_ARCH__)
    return dev::ld_acquire_sys(p);
#else
    return __atomic_load_n(p, __ATOMIC_ACQUIRE);
#endif
}
// the eight fingerprints of a bucket: four 16-byte loads, one 64-byte line
IS_HD void ld_fingerprints(const IndexBucket* b, uint64_t (&h)[kIndexWays]) {
#if defined(__CUDA_ARCH__)
#pragma unroll
    for (int i = 0; i < int(kIndexWays); i += 2)
        asm volatile("ld.relaxed.sys.global.v2.u64 {%0,%1}, [%2];"
                     : "=l"(h[i]), "=l"(h[i + 1])
                     : "l"(&b->h1[i])
                     : "memory");
#else
    for (uint32_t i = 0; i < kIndexWays; ++i) h[i] = __atomic_load_n(&b->h1[i], __ATOMIC_RELAXED);
#endif
}
IS_HD uint64_t cas_u64(uint64_t* p, uint64_t cmp, uint64_t val, bool sys) {
#if defined(__CUDA_ARCH__)
    // Atomics on one address are serialised at the L2 that owns it whatever the scope
    // qualifier, so a table in this GPU's own HBM may be claimed at gpu scope.
    return sys ? dev::cas_relaxed_sys_u64(p, cmp, val) : dev::cas_relaxed_gpu_u64(p, cmp, val);
#else
    (void)sys;
    __atomic_compare_exchange_n(p, &cmp, val, false, __ATOMIC_RELAXED, __ATOMIC_RELAXED);
    return cmp;
#endif
}
IS_HD void st_u64(uint64_t* p, uint64_t v) {
#if defined(__CUDA_ARCH__)
    dev::st_relaxed_sys_u64(p, v);
#else
    __atomic_store_n(p, v, __ATOMIC_RELAXED);
#endif
}
IS_HD void st_u32(uint32_t* p, uint32_t v, bool sys) {
#if defined(__CUDA_ARCH__)
    if (sys)
        asm volatile("st.relaxed.sys.global.u32 [%0], %1;" ::"l"(p), "r"(v) : "memory");
    else
        asm volatile("st.relaxed.gpu.global.u32 [%0], %1;" ::"l"(p), "r"(v) : "memory");
#else
    (void)sys;
    __atomic_store_n(p, v, __ATOMIC_RELAXED);
#endif
}
IS_HD void fence(bool sys) {
#if defined(__CUDA_ARCH__)
    if (sys)
        dev::fence_sys();
    else
        dev::fence_gpu();
#else
    (void)sys;
    __atomic_thread_fence(__ATOMIC_SEQ_CST);
#endif
}

// ---------------------------------------------------------------- shards
struct TableRef {
    IndexBucket* table;
    uint64_t mask;
    uint32_t shard;
};
// The table a key lives in (kernels.h: IndexShards).
IS_HD TableRef select_shard(const IndexBucket* t0, uint64_t m0, const IndexShards& sh, uint64_t h2) {
    const uint32_t s = index_shard_of(h2, sh.n);
    if (s == 0) return TableRef{const_cast<IndexBucket*>(t0), m0, 0};
    return TableRef{sh.table[s - 1], sh.mask[s - 1], s};
}
// slot ids that leave a kernel (or a kernel phase) carry their shard in the top 3 bits
IS_HD uint32_t pack_slot(uint32_t shard, uint32_t slot_plus1) {
    return slot_plus1 ? (shard << kSlotShardShift) | slot_plus1 : 0u;
}
IS_HD uint32_t slot_local(uint32_t packed) { return packed & ((1u << kSlotShardShift) - 1); }
IS_HD IndexBucket* table_of_slot(const IndexBucket* t0, const IndexShards& sh, uint32_t packed) {
    const uint32_t s = packed >> kSlotShardShift;
    return s == 0 ? const_cast<IndexBucket*>(t0) : sh.table[s - 1];
}

// ---------------------------------------------------------------- placement
IS_HD uint64_t bucket_a(uint64_t h1, uint64_t mask) { return h1 & mask; }
IS_HD uint64_t bucket_b(uint64_t h1, uint64_t h2, uint64_t mask) {
    uint64_t b = ((h1 >> 32) ^ h2) & mask;
    if (b == (h1 & mask)) b = (b + 1) & mask;  // equal only for a one-bucket table
    return b;
}
IS_HD uint32_t first_way(uint64_t h2) { return uint32_t(h2 >> 61); }
IS_HD uint32_t slot_id(uint64_t bucket, uint32_t way) { return uint32_t(bucket * kIndexWays + way); }
IS_HD IndexWay* way_of(IndexBucket* table, uint32_t slot) {
    return &table[slot / kIndexWays].way[slot % kIndexWays];
}
IS_HD const IndexWay* way_of(const IndexBucket* table, uint32_t slot) {
    return &table[slot / kIndexWays].way[slot % kIndexWays];
}

// ---------------------------------------------------------------- writer
// Reserve a way for `rec`.  Returns slot + 1, or 0 when nothing is to be committed: the key
// is already published (first writer wins) or both buckets are full (*full set).
// Fast path: one CAS on the key's preferred way of bucket A - ONE fabric round trip for an
// insertion into a lightly loaded table; the fields follow as posted stores, tag stays 0.
// Slow path (that way is taken): read the fingerprints of A, then of B, and take a free way
// of the emptier bucket.  Two-choice placement keeps "both buckets full" out of reach at the
// load the server sizes the table for (<= 0.5): none in 4e4 simulated insertions at load
// 0.5, 3e-4 at 0.75.  The buckets are scanned one after the other (16 live registers, not
// 32): this code is inlined into the copy kernels and must not cost them occupancy.
IS_HD uint32_t take_way(IndexBucket* bk, uint64_t bi, uint32_t w, const IndexEntry& rec,
                        bool sys) {
    // posted stores, published by the writer's fence + tag store; the tag stays 0
#if defined(__CUDA_ARCH__)
    (void)sys;
    bk->way[w].h2 = rec.h2;
    bk->way[w].addr = rec.addr;
    bk->way[w].size = rec.size;
#else
    st_u64(&bk->way[w].h2, rec.h2);
    st_u64(&bk->way[w].addr, rec.addr);
    st_u32(&bk->way[w].size, rec.size, sys);
#endif
    return slot_id(bi, w) + 1;
}
IS_HD bool published_as(const IndexBucket* bk, uint32_t w, const IndexEntry& rec) {
    // same fingerprint: the same key (already published: first writer wins) or a 64-bit
    // collision with another key; the authoritative copy is the server's map either way
    return ld_acquire_u32(&bk->way[w].tag) != 0 && ld_u64(&bk->way[w].h2) == rec.h2;
}
// bit w set: way w of `bk` is free; bit 8 + w set: way w carries `h1` already.  Pure ALU on
// one 64-byte read; kept small on purpose - this is inlined into the copy kernels, whose
// control warp pays for every extra instruction-cache line on its critical path.
IS_HD uint32_t scan_ways(const IndexBucket* bk, uint64_t h1) {
    uint64_t h[kIndexWays];
    ld_fingerprints(bk, h);
    uint32_t m = 0;
#if defined(__CUDA_ARCH__)
#pragma unroll
#endif
    for (uint32_t w = 0; w < kIndexWays; ++w) {
        m |= (h[w] == 0 ? 1u : 0u) << w;
        m |= (h[w] == h1 ? 0x100u : 0u) << w;
    }
    return m;
}
// does one of the ways flagged in `same` (bits 0..7) hold `rec`'s key, committed?
IS_HD bool any_published(const IndexBucket* bk, uint32_t same, const IndexEntry& rec) {
#if defined(__CUDA_ARCH__)
#pragma unroll 1
#endif
    for (uint32_t w = 0; same; ++w, same >>= 1)
        if ((same & 1u) && published_as(bk, w, rec)) return true;
    return false;
}
IS_HD uint32_t popcount8(uint32_t m) {
    m = (m & 0x55u) + ((m >> 1) & 0x55u);
    m = (m & 0x33u) + ((m >> 2) & 0x33u);
    return (m & 0x0fu) + (m >> 4);
}
// The slow path of claim() below: both buckets are read, the emptier one is used.
#define IDX_SLOW_PATH IS_HD
IDX_SLOW_PATH uint32_t claim_slow(IndexBucket* table, uint64_t mask, const IndexEntry& rec,
                                  bool sys, bool* full) {
    const uint64_t a = bucket_a(rec.h1, mask), b = bucket_b(rec.h1, rec.h2, mask);
    IndexBucket* ba = table + a;
    IndexBucket* bb = table + b;
#if defined(__CUDA_ARCH__)
#pragma unroll 1
#endif
    for (int attempt = 0; attempt < 4; ++attempt) {  // retried only when a CAS loses a race
        const uint32_t ma = scan_ways(ba, rec.h1);
        const uint32_t mb = b != a ? scan_ways(bb, rec.h1) : 0u;
        if (((ma | mb) >> 8) &&
            (any_published(ba, ma >> 8, rec) || any_published(bb, mb >> 8, rec)))
            return 0;
        const uint32_t free_a = ma & 0xffu, free_b = mb & 0xffu;
        if ((free_a | free_b) == 0) break;
        const bool use_b = popcount8(free_b) > popcount8(free_a);
        IndexBucket* bk = use_b ? bb : ba;
        uint32_t m = use_b ? free_b : free_a;
#if defined(__CUDA_ARCH__)
#pragma unroll 1
#endif
        for (uint32_t w = 0; w < kIndexWays; ++w, m >>= 1) {
            if (!(m & 1u)) continue;
            if (cas_u64(&bk->h1[w], 0, rec.h1, sys) == 0)
                return take_way(bk, use_b ? b : a, w, rec, sys);
        }
    }
    *full = true;
    return 0;
}

IS_HD uint32_t claim(IndexBucket* table, uint64_t mask, const IndexEntry& rec, bool sys,
                     bool* full) {
    const uint64_t a = bucket_a(rec.h1, mask);
    const uint32_t w0 = first_way(rec.h2);
    IndexBucket* ba = table + a;
    const uint64_t cur = cas_u64(&ba->h1[w0], 0, rec.h1, sys);
    if (cur == 0) return take_way(ba, a, w0, rec, sys);
    if (cur == rec.h1 && published_as(ba, w0, rec)) return 0;
    return claim_slow(table, mask, rec, sys, full);
}

// The caller has fenced the block's data stores (and the claim's field stores): fence +
// relaxed store is a release pattern, the tag needs no second MEMBAR.
IS_HD void commit(IndexBucket* table, uint32_t slot_plus1, uint32_t tag, bool sys) {
    if (slot_plus1) st_u32(&way_of(table, slot_plus1 - 1)->tag, tag, sys);
}

// ---------------------------------------------------------------- reader
struct Found {
    uint32_t slot_plus1;  // 0 = not found (absent, or reserved by a writer still copying)
    uint32_t tag;
    uint64_t addr;
    uint32_t size;
};

// bit w set: way w carries the fingerprint h1
IS_HD uint32_t match_mask(const uint64_t (&h)[kIndexWays], uint64_t h1) {
    uint32_t m = 0;
#if defined(__CUDA_ARCH__)
#pragma unroll
#endif
    for (uint32_t w = 0; w < kIndexWays; ++w) m |= (h[w] == h1 ? 1u : 0u) << w;
    return m;
}
IS_HD uint32_t lowest_bit(uint32_t m) {
#if defined(__CUDA_ARCH__)
    return uint32_t(__ffs(int(m))) - 1u;
#else
    return uint32_t(__builtin_ctz(m));
#endif
}

// Check the ways of one bucket whose fingerprint matched (`m`).  `tag0`: the already loaded
// tag of way `w0` (pass w0 >= kIndexWays when none was loaded).  A rolled loop on purpose:
// almost always one iteration, and the unrolled form cost every reader kilobytes of
// instruction fetch on a cold kernel.
// kAcceptClaimed: a way that a writer has claimed but not yet committed (tag == 0) counts
// as a hit (returned with tag 0).  That is the reference's rule for get_match_last_index -
// a key is "present" from the moment it is reserved, committed or not
// (src/infinistore.cpp:1097) - and ONLY for it: reads and check_exist need the commit.
template <bool kAcceptClaimed = false>
IS_HD Found match_bucket(const IndexBucket* bk, uint64_t bi, uint32_t m, const KeyHash& kh,
                         uint32_t w0, uint32_t tag0) {
#if defined(__CUDA_ARCH__)
#pragma unroll 1
#endif
    for (; m; m &= m - 1) {
        const uint32_t w = lowest_bit(m);
        const IndexWay* wy = &bk->way[w];
        const uint32_t tag = w == w0 ? tag0 : ld_acquire_u32(&wy->tag);
        if (!kAcceptClaimed && tag == 0) continue;  // claimed, not committed
        // all three fields in flight together: ONE round trip after the tag, not two
        const uint64_t h2 = ld_u64(&wy->h2);
        const uint64_t addr = ld_u64(&wy->addr);
        const uint32_t size = ld_u32(&wy->size);
        if (h2 != kh.h2) continue;
        return Found{slot_id(bi, w) + 1, tag, addr, size};
    }
    return Found{0, 0, 0, 0};
}

// Round trip 1: the fingerprints of bucket A and, speculatively, the tag of the key's
// preferred way (where it sits unless that way was taken when it was written).  Round trip 2:
// the fields.  kBothAtOnce also fetches bucket B in round trip 1: a miss then costs one
// round trip instead of two - right for get_match_last_index, which probes mostly absent
// keys; the read path, whose keys are almost always in bucket A, skips those four loads.
template <bool kBothAtOnce, bool kAcceptClaimed = false>
IS_HD Found find(const IndexBucket* table, uint64_t mask, const KeyHash& kh) {
    const uint64_t a = bucket_a(kh.h1, mask), b = bucket_b(kh.h1, kh.h2, mask);
    const uint32_t w0 = first_way(kh.h2);
    uint32_t ma, mb = 0;
    uint32_t tag0;
    {
        uint64_t ha[kIndexWays];
        ld_fingerprints(table + a, ha);
        if constexpr (kBothAtOnce) {
            uint64_t hb[kIndexWays];
            ld_fingerprints(table + b, hb);
            tag0 = ld_acquire_u32(&table[a].way[w0].tag);
            mb = match_mask(hb, kh.h1);
        } else {
            tag0 = ld_acquire_u32(&table[a].way[w0].tag);
        }
        ma = match_mask(ha, kh.h1);
    }
    const Found f = match_bucket<kAcceptClaimed>(table + a, a, ma, kh, w0, tag0);
    if (f.slot_plus1 || b == a) return f;
    if constexpr (!kBothAtOnce) {
        uint64_t hb[kIndexWays];
        ld_fingerprints(table + b, hb);
        mb = match_mask(hb, kh.h1);
    }
    return match_bucket<kAcceptClaimed>(table + b, b, mb, kh, kIndexWays, 0);
}

// After the copy: is the entry the reader resolved still the one in the table?
IS_HD bool still_valid(const IndexBucket* table, uint32_t slot_plus1, uint32_t tag) {
    return ld_acquire_u32(&way_of(table, slot_plus1 - 1)->tag) == tag;
}

// ---------------------------------------------------------------- evictor
// Empty the way that holds (h1, h2, addr).  tag := 0 first, so a reader sees "not
// committed" before the way can be claimed by another key.  false: no such entry.
IS_HD bool erase(IndexBucket* table, uint64_t mask, uint64_t h1, uint64_t h2, uint64_t addr) {
    const uint64_t a = bucket_a(h1, mask), b = bucket_b(h1, h2, mask);
    for (int which = 0; which < 2; ++which) {
        if (which && b == a) break;
        IndexBucket* bk = table + (which ? b : a);
        for (uint32_t w = 0; w < kIndexWays; ++w) {
            if (ld_u64(&bk->h1[w]) != h1) continue;
            if (ld_u64(&bk->way[w].h2) != h2 || ld_u64(&bk->way[w].addr) != addr) continue;
            st_u32(&bk->way[w].tag, 0u, true);
            fence(true);
            st_u64(&bk->h1[w], 0);
            return true;
        }
    }
    return false;
}

}  // namespace istore::kernels::idx
