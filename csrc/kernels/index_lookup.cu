// kv_index_lookup: hash + probe + compare of the HBM-resident key index on the GPU.
//
// Serves three API calls that the reference answers on the server CPU with
// std::unordered_map<string> probes (src/infinistore.cpp:1077-1108, 436-446):
//   * read_cache        : resolve every key of the batch to a pool address and emit the
//                         copy descriptors consumed by kv_copy in the same stream;
//   * get_match_last_index : presence bitmap over the key list, then the last CTA replays
//                         the reference's binary search over that bitmap, bit-exact on any
//                         (also non-monotone) input (SURVEY §2.5-C7);
//   * check_exist       : the same with one key.
// One thread per key, keys staged per warp through shared memory: the key bytes are hashed
// twice (core/hash.h, identical on host and device) and the key's two buckets of the table -
// which lives in the pool GPU's HBM and is usually a PEER mapping read over NVLink - are
// searched (index.cuh).  For reads and check_exist an entry counts only once its tag has been
// published with release semantics by the writer's kernel; get_match_last_index also counts
// ways that a writer has claimed but not committed yet (reference visibility rule C3).
// Also here: the eviction kernels (erase on the server side, post-copy validation on the
// reader side).
#include "../core/hash.h"
#include "common.cuh"
#include "index.cuh"
#include "kernels.h"

namespace istore::kernels {

namespace {

using namespace dev;

// One warp per CTA: a batch of lookups spreads over many SMs instead of queueing hundreds of
// fabric loads behind one SM's load unit.
//
// Key bytes usually sit in the client's pinned ring (PCIe): a thread that walked its own key
// with serial 8-byte loads paid one PCIe round trip per 8 bytes.  The warp's 32 keys are packed back to back, so the warp first stages their whole
// byte range into shared memory with coalesced 8-byte loads - a handful of PCIe reads in
// flight at once - and every thread then hashes its key from shared memory.
constexpr int kLookupThreads = 32;
constexpr uint32_t kStageBytes = 8192;  // shared staging per warp; longer ranges hash from global

template <bool kAcceptClaimed>
__device__ __forceinline__ idx::Found probe(const LookupLaunch& a, const KeyHash& kh) {
    const idx::TableRef t = idx::select_shard(a.table, a.table_mask, a.shards, kh.h2);
    // reads resolve present keys (bucket A first), match / exist probes mostly absent ones
    idx::Found f = a.present ? idx::find<true, kAcceptClaimed>(t.table, t.mask, kh)
                             : idx::find<false, kAcceptClaimed>(t.table, t.mask, kh);
    f.slot_plus1 = idx::pack_slot(t.shard, f.slot_plus1);
    return f;
}

__global__ void __launch_bounds__(kLookupThreads)
    kv_index_lookup_kernel(const __grid_constant__ LookupLaunch a) {
    __shared__ __align__(8) uint8_t stage[kStageBytes];
    const uint32_t first = blockIdx.x * kLookupThreads;
    const uint32_t i = first + threadIdx.x;
    const uint32_t last = min(first + kLookupThreads, a.n) - 1;
    // byte range of this warp's keys (each key starts 8-byte aligned, zero padded)
    const uint32_t lo = a.key_off[first];
    const uint32_t hi = a.key_off[last] + ((max(a.key_len[last], 1u) + 7u) & ~7u);
    const bool staged = hi > lo && hi - lo <= kStageBytes;
    if (staged) {
        const uint64_t* g = reinterpret_cast<const uint64_t*>(a.key_bytes + lo);
        uint64_t* sm = reinterpret_cast<uint64_t*>(stage);
        for (uint32_t w = threadIdx.x; w < (hi - lo) / 8; w += kLookupThreads) sm[w] = g[w];
        __syncwarp();
    }
    bool found = false;
    if (i < a.n) {
        const uint32_t off = a.key_off[i];
        const uint8_t* kp = staged ? stage + (off - lo) : a.key_bytes + off;
        const KeyHash kh = hash_key(kp, a.key_len[i]);
        const idx::Found h = a.accept_claimed ? probe<true>(a, kh) : probe<false>(a, kh);
        found = h.slot_plus1 != 0;
        if (a.out_descs) {
            uint64_t src = 0;
            if (found && h.tag != 0 && h.size >= a.need_bytes) {
                const uint32_t seg = uint32_t(h.addr >> 44) - 1;
                if (seg < a.nsegs && a.seg_base[seg])
                    src = a.seg_base[seg] + (h.addr & ((1ull << 44) - 1));
            }
            a.out_descs[i] = CopyDesc{src, a.dst_base + a.dst_off[i]};
            if (a.found_at)
                a.found_at[i] = LookupLaunch::FoundAt{src ? h.slot_plus1 : 0u, h.tag};
        }
    }
    if (!a.present) return;
    // 32 consecutive keys per warp -> one bitmap word, no atomics
    const uint32_t word = __ballot_sync(0xffffffffu, found);
    if ((threadIdx.x & 31) == 0 && i < a.n) a.present[i >> 5] = word;
    if (!a.want_match) return;

    // elect the last CTA; it sees every CTA's bitmap words
    __shared__ bool is_last;
    __threadfence();
    __syncthreads();
    if (threadIdx.x == 0) {
        const uint32_t t = atomicAdd(a.ticket, 1u);
        is_last = t == gridDim.x - 1;
        if (is_last) *a.ticket = 0;  // self-cleaning for the next launch
    }
    __syncthreads();
    if (!is_last || threadIdx.x != 0) return;
    __threadfence();
    const volatile uint32_t* present = a.present;
    // Exact replay of the reference's search (src/infinistore.cpp:1093-1104).
    int left = 0, right = int(a.n);
    while (left < right) {
        const int mid = left + (right - left) / 2;
        if ((present[mid >> 5] >> (mid & 31)) & 1u)
            left = mid + 1;
        else
            right = mid;
    }
    a.status[kStatMatch] = uint32_t(left - 1);
    __threadfence_system();
}

// One thread per block that was read: the tag must be unchanged (see ValidateLaunch).
__global__ void __launch_bounds__(kLookupThreads)
    kv_index_validate_kernel(const __grid_constant__ ValidateLaunch a) {
    const uint32_t i = blockIdx.x * kLookupThreads + threadIdx.x;
    if (i >= a.n) return;
    const LookupLaunch::FoundAt f = a.found_at[i];
    if (!f.slot_plus1) return;  // a miss was counted by the lookup
    if (!idx::still_valid(idx::table_of_slot(a.table, a.shards, f.slot_plus1),
                          idx::slot_local(f.slot_plus1), f.tag)) {
        atomicAdd(a.status + kStatMiss, 1u);
        atomicAdd(a.status + kStatStale, 1u);
    }
}

// One thread per evicted block (index.cuh: tag := 0, fence, h1 := 0).
__global__ void __launch_bounds__(kLookupThreads)
    kv_index_erase_kernel(const __grid_constant__ EraseLaunch a) {
    const uint32_t i = blockIdx.x * kLookupThreads + threadIdx.x;
    if (i >= a.n) return;
    const EraseRec r = a.recs[i];
    idx::erase(a.table, a.table_mask, r.h1, r.h2, r.addr);
}

}  // namespace

cudaError_t launch_index_validate(const ValidateLaunch& a, cudaStream_t stream) {
    if (a.n == 0) return cudaSuccess;
    const unsigned grid = (a.n + kLookupThreads - 1) / kLookupThreads;
    kv_index_validate_kernel<<<grid, kLookupThreads, 0, stream>>>(a);
    return cudaGetLastError();
}

cudaError_t launch_index_erase(const EraseLaunch& a, cudaStream_t stream) {
    if (a.n == 0) return cudaSuccess;
    const unsigned grid = (a.n + kLookupThreads - 1) / kLookupThreads;
    kv_index_erase_kernel<<<grid, kLookupThreads, 0, stream>>>(a);
    return cudaGetLastError();
}

cudaError_t launch_index_lookup(const LookupLaunch& a, cudaStream_t stream) {
    if (a.n == 0) return cudaSuccess;
    const unsigned grid = (a.n + kLookupThreads - 1) / kLookupThreads;
    kv_index_lookup_kernel<<<grid, kLookupThreads, 0, stream>>>(a);
    return cudaGetLastError();
}

}  // namespace istore::kernels
