// Host-callable launchers of the sm_90a data-plane kernels.
//
// These kernels replace every byte-moving / lookup call site of the reference, which has
// no device code at all (SURVEY §2.2): per-block cudaMemcpyAsync (src/infinistore.cpp:
// 623-624,747-748), ibv_post_send RDMA_WRITE chains (src/libinfinistore.cpp:916-981,
// src/infinistore.cpp:471-501), the COMMIT message (src/libinfinistore.cpp:362-395) and
// the get_match_last_index / check_key CPU probes (src/infinistore.cpp:1077-1108).
#pragma once

#include <cuda_runtime_api.h>

#include <cstdint>
#include <initializer_list>

namespace istore::kernels {

// One block to move: absolute, device-addressable source and destination.  For a write
// `dst` is a peer-mapped pool address, for a read `src` is.  src == 0 marks a block the
// device lookup did not find: it is skipped and counted in status[kStatMiss].
struct CopyDesc {
    uint64_t src;
    uint64_t dst;
};

// Record a writer publishes for one block once its data is visible system-wide.
struct IndexEntry {
    uint64_t h1;    // 128-bit key fingerprint (core/hash.h)
    uint64_t h2;
    uint64_t addr;  // global block address: (segment+1) << 44 | offset
    uint32_t tag;   // allocation generation (never 0)
    uint32_t size;
};
static_assert(sizeof(IndexEntry) == 32, "index records are 32 bytes");

// The HBM-resident key index: an array of 256-byte, 8-way buckets.  A key lives in one of
// two buckets chosen by its fingerprint (index.cuh), in any way.  There are no probe chains,
// so an evicted block's way simply becomes empty again - no tombstones, no degradation
// under the steady churn of a full cache.
//   h1[w] : claimed with a 64-bit CAS from 0 (empty).  All eight fingerprints of a bucket
//           are one 64-byte read.
//   tag   : written last with release semantics; 0 = claimed but not yet committed.
//           Generations are unique per allocation, so "the tag I resolved is still there"
//           proves that the block was not evicted (and the way reused) during a read.
constexpr uint32_t kIndexWays = 8;
struct IndexWay {
    uint64_t h2;
    uint64_t addr;
    uint32_t tag;
    uint32_t size;
};
struct alignas(64) IndexBucket {
    uint64_t h1[kIndexWays];
    IndexWay way[kIndexWays];
};
static_assert(sizeof(IndexWay) == 24 && sizeof(IndexBucket) == 256, "index bucket layout");
// An index of `slots` entries (a power of two, >= 8) has slots / 8 buckets; kernels take
// the bucket mask.
inline uint64_t index_bucket_mask(uint64_t slots) { return slots / kIndexWays - 1; }

// Sharded index.  A server with several pool GPUs (--pool-devices 0,1,...) keeps one table
// per initial HBM segment; a key lives in the table its fingerprint selects - independent of
// where its block lives - so probes and claims spread over the pool GPUs instead of all
// landing on segment 0's.  Launch structs carry shard 0 as `table` / `table_mask` and the
// others here (n <= 1: unsharded).  Slot ids handed around by the kernels carry the shard in
// their top 3 bits.
constexpr uint32_t kMaxIndexShards = 8;
constexpr uint32_t kSlotShardShift = 29;
struct IndexShards {
    uint32_t n = 0;  // total number of shards including shard 0
    IndexBucket* table[kMaxIndexShards - 1] = {nullptr, nullptr, nullptr, nullptr, nullptr, nullptr, nullptr};
    uint64_t mask[kMaxIndexShards - 1] = {0, 0, 0, 0, 0, 0, 0};
};
#if defined(__CUDACC__)
__host__ __device__
#endif
inline uint32_t index_shard_of(uint64_t h2, uint32_t nshards) {
    // bits 20..52 of the verifier half: not used by the way preference (top 3 bits) and only
    // mixed into the bucket choice
    return nshards <= 1 ? 0u : uint32_t((h2 >> 20) % nshards);
}

enum Status : int {
    kStatMiss = 0,         // blocks skipped by a read because the key was not in the index
    kStatPublishFail = 1,  // index insertions that found the table full
    kStatMatch = 2,        // result of the last match_last_index launch (int32)
    kStatStale = 3,        // blocks whose index entry changed while they were read (evicted)
    kStatWords = 8,
};

enum CopyVariant : int {
    kCopyAuto = 0,
    kCopyLdSt = 1,  // 128-bit ld/st, all threads: LDG.128 / STG.128 on (peer) global memory
    kCopyTma = 2,   // warp-specialised TMA pipeline (kv_pipe.cu): UBLKCP.S.G / UBLKCP.G.S + mbarriers
    kCopyLdSt256 = 3,  // 32-byte aligned ld/st: 128-bit vectors, eight in flight per thread
};

struct CopyLaunch {
    const CopyDesc* descs = nullptr;  // device-addressable (device memory or mapped pinned host)
    const CopyDesc* descs_host = nullptr;  // same array as seen by the CPU, if it is host memory:
                                           // small batches are then passed as kernel parameters
    uint32_t n = 0;                   // blocks
    uint32_t bytes = 0;               // bytes per block
    uint64_t align_or = 0;            // OR of every local address (pool blocks are granule aligned)
    // optional in-band commit (writes): publish recs[i] once block i has landed
    const IndexEntry* recs = nullptr;
    IndexBucket* table = nullptr;
    uint64_t table_mask = 0;  // bucket mask
    uint32_t* done = nullptr;         // 3*n zeroed u32 of client-local device scratch
    uint32_t* status = nullptr;       // kStatWords u32, device-addressable
    int variant = kCopyAuto;
    int max_ctas = 0;                 // 0 = pick from the problem size
    unsigned long long* trace = nullptr;  // optional per-CTA %globaltimer stamps (bench only)
    bool all_local = false;  // every destination and the index table are in this GPU's own HBM
    IndexShards shards;      // further index shards (shard 0 = table / table_mask)
    uint32_t debug = 0;      // bench only, see publish.cuh
    bool multicast = false;  // every dst is an NVLS multicast address: store with multimem.st
    // TMA pipeline geometry (0 = default: 16 KB slots, 128 KB ring per CTA)
    uint32_t stage_bytes = 0;
    uint32_t ring_bytes = 0;
    // TMA pipeline only, reads only: store every block to fan_n destinations,
    // desc.dst + fan_delta[r] (one load over the fabric, fan_n local stores)
    int fan_n = 1;
    int64_t fan_delta[4] = {0, 0, 0, 0};
};
// Picks the data path (CopyVariant) and launches it.  kCopyAuto: the TMA pipeline for every
// 16-byte aligned transfer of blocks >= kPipeMinBytes, ld/st below that (one issuing thread
// per CTA cannot keep up with the per-block work of small blocks; bench/sweep_copy.py
// compares the variants per block size).
cudaError_t launch_kv_copy(const CopyLaunch& a, cudaStream_t stream);
constexpr uint32_t kPipeMinBytes = 64u << 10;
// The TMA pipeline itself (kv_pipe.cu); needs 16-byte aligned addresses and sizes.
cudaError_t launch_kv_pipe_copy(const CopyLaunch& a, cudaStream_t stream);

// Gathered blocks: pool block i is the concatenation of `nparts` parts of part_bytes each,
// part s taken from (write) or scattered to (read) part_base[s] + the block's local offset -
// one page of every layer of a paged KV cache under one key, with no pack/unpack kernel.
// first_part shifts which stored parts a launch covers, on both sides.
// Work item = (block, part, chunk), numbered block * nparts * cpp + part * cpp + chunk, so a
// chunk never crosses a part and the in-band commit (publish.cuh) counts nparts * cpp
// arrivals per block.  The part bases travel in the kernel parameters.
constexpr uint32_t kGatherMaxParts = 256;
struct GatherLaunch {
    // per block, device-addressable: write {local byte offset, pool address},
    // read {pool address or 0 = miss, local byte offset}
    const CopyDesc* descs = nullptr;
    uint32_t n = 0;
    bool write = false;
    const uint64_t* part_base = nullptr;  // host array of nparts absolute addresses
    uint32_t nparts = 0;
    uint32_t part_bytes = 0;
    // reads: pool part first_part + s lands in part s; writes: part s is stored as pool part
    // first_part + s (a layered write, below, stores a block's parts over several launches)
    uint32_t first_part = 0;
    uint64_t align_or = 0;    // OR of every part base and local offset
    // optional in-band commit (writes), as in CopyLaunch; recs[i].size covers all parts
    const IndexEntry* recs = nullptr;
    IndexBucket* table = nullptr;
    uint64_t table_mask = 0;
    uint32_t* done = nullptr;  // 3*n zeroed u32 of client-local device scratch
    uint32_t* status = nullptr;  // reads: a missing block counts once in kStatMiss
    int max_ctas = 0;
    bool all_local = false;
    IndexShards shards;
    uint32_t stage_bytes = 0;  // TMA pipeline geometry, 0 = default
    uint32_t ring_bytes = 0;
    // Layered write (with recs): this launch stores nparts of the layer_parts parts of each
    // block, and the block is published by whichever launch lands its last part
    // (publish.cuh: control_warp_layered).  layer_state: 3 u32 per block, kept by the writer
    // across its launches and zeroed before its first: slot + 1 | tag | parts landed.
    // layer_claim: this launch claims the blocks' index ways (the writer's first call).
    uint32_t* layer_state = nullptr;
    uint32_t layer_parts = 0;
    bool layer_claim = false;
    // Layered read (reads only, ld/st kernels only): the launch walks the parts in groups of
    // group_parts (2 = one layer's K and V), numbered group-major (launch_plan.h:
    // layered_item), and releases group g by storing group_seq to group_flags[g] once every
    // block's parts of g have landed (publish.cuh: leave_group).  A missing block's items count
    // as landed.  group_counters: nparts / group_parts zeroed u32, left zeroed.
    uint32_t* group_flags = nullptr;
    uint32_t* group_counters = nullptr;
    uint32_t group_seq = 0;
    uint32_t group_parts = 0;
    // Row-sliced read (reads only, ld/st kernels only; rows == 0: whole contiguous parts): the
    // reader's share of stored part s is `rows` rows of row_bytes at a pitch of src_pitch,
    // src_col bytes into each row (part_bytes == rows * src_pitch), and row r lands at
    // part_base[s] + desc.dst + r * dst_pitch - e.g. a decode rank's KV heads of a page that
    // a prefill rank at another tensor-parallel degree wrote.  Works with group_flags.
    uint32_t rows = 0;
    uint32_t row_bytes = 0;
    uint32_t src_pitch = 0;
    uint32_t src_col = 0;
    uint32_t dst_pitch = 0;
};
// The TMA pipeline for 16-byte aligned parts of at least kPipeMinBytes, the ld/st kernel
// (kv_copy.cu) otherwise: the same rule launch_kv_copy applies to whole blocks.  A row-sliced
// read runs kv_scatter_rows (kv_copy.cu).
cudaError_t launch_kv_gather(const GatherLaunch& a, cudaStream_t stream);
cudaError_t launch_kv_pipe_gather(const GatherLaunch& a, cudaStream_t stream);
struct GatherParts {
    uint64_t base[kGatherMaxParts];
};
struct ReadFusedLaunch;
// A scattered read through the device index in ONE launch (kv_pipe.cu): the resolver warp of
// kv_pipe_read feeding the gather pipeline.  CTA c owns blocks c, c + grid, ...: each key is
// probed once, by the CTA that moves all of its parts, and re-checked after the copy.  `r`
// carries keys, dst_off (local byte offsets; dst_base 0), index, segments, status, grid cap
// and ring geometry; `g` the parts (descs, recs and write are ignored).  Needs 16-byte aligned
// parts and at least as many blocks as CTAs (fewer: lookup + launch_kv_gather + validate).
bool scatter_read_fused_supported(const ReadFusedLaunch& r, const GatherLaunch& g);
cudaError_t launch_kv_pipe_scatter_read(const ReadFusedLaunch& r, const GatherLaunch& g,
                                        cudaStream_t stream);
// fp8 (e4m3) fused variants: the write converts bf16 pages to e4m3 with one fp32 scale
// per `group` elements (the head_dim row) and stores payload + scales into the pool block;
// the read dequantises back to bf16 while scattering into the paged KV cache.
struct Fp8Launch {
    const CopyDesc* descs = nullptr;
    uint32_t n = 0;
    uint32_t elems = 0;   // bf16 elements per page
    uint32_t group = 128; // elements sharing one scale
    const IndexEntry* recs = nullptr;
    IndexBucket* table = nullptr;
    uint64_t table_mask = 0;  // bucket mask
    uint32_t* done = nullptr;
    uint32_t* status = nullptr;
    int max_ctas = 0;
    bool all_local = false;
    IndexShards shards;     // further index shards (shard 0 = table / table_mask)
    bool aligned16 = true;  // every page address is 16-byte aligned (bulk copies need it)
    int variant = 0;        // Fp8Variant
};
enum Fp8Variant : int {
    kFp8Auto = 0,  // the TMA pipeline with 8 compute warps, ld/st kernels where it does not fit
    kFp8LdSt = 1,  // the ld/st kernels
    kFp8Tma4 = 2,  // the TMA pipeline with 4 compute warps (A/B)
};
// The TMA-pipelined flavour (kv_fp8_pipe.cu): needs elems % 512 == 0 and aligned pages.
cudaError_t launch_kv_fp8_pipe(const Fp8Launch& a, bool write, cudaStream_t stream);
// bytes a quantised page occupies in the pool: elems (e4m3) + 4 * elems/group (scales)
inline uint32_t fp8_block_bytes(uint32_t elems, uint32_t group) {
    return elems + 4u * (elems / group);
}
// Gathered fp8 blocks: nparts quantised pages end to end, part s at byte
// fp8_gather_bytes(s, elems) of the block; fp8_gather_bytes(nparts, elems) is the block's size
// (Llama-3-8B, 16-token pages: 64 parts of 16384 elements = 1,081,344 bytes).  elems % 512 == 0
// keeps every part 16-byte aligned inside a granule-aligned block.
inline uint64_t fp8_gather_bytes(uint32_t nparts, uint32_t elems) {
    return uint64_t(nparts) * fp8_block_bytes(elems, 128);
}
cudaError_t launch_kv_write_fp8(const Fp8Launch& a, cudaStream_t stream);
cudaError_t launch_kv_read_fp8(const Fp8Launch& a, cudaStream_t stream);
// The gathered form of the two above: each part of a GatherLaunch is a bf16 page of `elems`
// elements (a multiple of 512; part_bytes is not read) at part_base[s] + the block's local
// offset, and each is quantised into / dequantised from its own fp8 page of the pool block.
// Every part of a block is byte-identical to the block launch_kv_write_fp8 stores for that
// page.  variant kFp8LdSt: the ld/st kernels (kv_fp8.cu), anything else: the TMA pipeline with
// 8 compute warps (kv_fp8_pipe.cu).  Part bases and local offsets must be 16-byte aligned.
cudaError_t launch_kv_gather_fp8(const GatherLaunch& a, uint32_t elems, int variant,
                                 cudaStream_t stream);
cudaError_t launch_kv_fp8_pipe_gather(const GatherLaunch& a, uint32_t elems, cudaStream_t stream);

// Device-side key lookup: hash the packed key bytes, probe the index, and either build
// copy descriptors for a following kv_copy (read path) or produce a presence bitmap and
// replay the reference's binary search (get_match_last_index / check_exist).
struct LookupLaunch {
    const uint8_t* key_bytes = nullptr;  // every key starts 8-byte aligned, zero padded
    const uint32_t* key_off = nullptr;   // n byte offsets into key_bytes
    const uint32_t* key_len = nullptr;   // n lengths
    uint32_t n = 0;
    const IndexBucket* table = nullptr;
    uint64_t table_mask = 0;  // bucket mask
    IndexShards shards;       // further index shards
    // segment id -> mapped base pointer on the launching device
    static constexpr int kMaxSegs = 16;
    uint64_t seg_base[kMaxSegs] = {0};
    uint32_t nsegs = 0;
    // read path: out_descs[i] = {pool pointer or 0, dst_base + dst_off[i]}
    CopyDesc* out_descs = nullptr;
    const uint64_t* dst_off = nullptr;
    uint64_t dst_base = 0;
    uint32_t need_bytes = 0;             // a hit must hold at least this many bytes
    // match path: presence bitmap (n bits, device memory) + replayed binary search
    uint32_t* present = nullptr;         // ceil(n/32) words, zeroed by the kernel's caller
    uint32_t* status = nullptr;          // status[kStatMatch] receives the int32 result
    uint32_t* ticket = nullptr;          // zeroed u32 used to elect the last CTA
    bool want_match = false;
    // get_match_last_index: a way claimed by a writer that has not committed yet counts as
    // present (the reference counts reserved keys, src/infinistore.cpp:1097); never set for
    // reads or check_exist
    bool accept_claimed = false;
    // optional: where every hit was found, for launch_index_validate after the copy
    struct FoundAt {
        uint32_t slot_plus1;  // 0 = miss
        uint32_t tag;
    };
    FoundAt* found_at = nullptr;
};
cudaError_t launch_index_lookup(const LookupLaunch& a, cudaStream_t stream);

// Optimistic-read validation (stores with eviction): after the copy, every entry must still
// carry the tag the lookup saw; otherwise the block was evicted meanwhile and the bytes
// just read may be another key's - counted in status[kStatMiss] and status[kStatStale].
struct ValidateLaunch {
    const LookupLaunch::FoundAt* found_at = nullptr;
    uint32_t n = 0;
    const IndexBucket* table = nullptr;
    IndexShards shards;  // further index shards (found_at slots carry the shard)
    uint32_t* status = nullptr;
};
cudaError_t launch_index_validate(const ValidateLaunch& a, cudaStream_t stream);

// Eviction: empty the ways of evicted blocks.  Runs on the pool GPU, from the server,
// before the blocks' space is handed out again.
struct EraseRec {
    uint64_t h1;
    uint64_t h2;
    uint64_t addr;
};
struct EraseLaunch {
    const EraseRec* recs = nullptr;  // device-addressable
    uint32_t n = 0;
    IndexBucket* table = nullptr;
    uint64_t table_mask = 0;  // bucket mask
};
cudaError_t launch_index_erase(const EraseLaunch& a, cudaStream_t stream);

// read_cache in one kernel: resolve the keys in the HBM index and move the pages.
struct ReadFusedLaunch {
    const uint8_t* key_bytes = nullptr;  // packed as for LookupLaunch
    const uint32_t* key_off = nullptr;
    const uint32_t* key_len = nullptr;
    const uint64_t* dst_off = nullptr;   // byte offset of every page from dst_base
    uint64_t dst_base = 0;
    uint32_t n = 0;
    uint32_t bytes = 0;                  // bytes per page; an index hit must hold at least this
    uint64_t align_or = 0;               // OR of every destination address
    const IndexBucket* table = nullptr;
    uint64_t table_mask = 0;  // bucket mask
    IndexShards shards;       // further index shards
    static constexpr int kMaxSegs = 16;
    uint64_t seg_base[kMaxSegs] = {0};
    uint32_t nsegs = 0;
    uint32_t* status = nullptr;          // status[kStatMiss] counts keys that were not found
    int max_ctas = 0;
    bool validate = false;               // re-check every entry's tag after its copy (eviction)
    int variant = kCopyAuto;             // kCopyTma: resolver warp feeding the TMA pipeline
    uint32_t stage_bytes = 0;            // TMA pipeline geometry, 0 = default
    uint32_t ring_bytes = 0;
};
// kCopyAuto / kCopyTma run the TMA pipeline (kv_pipe.cu) when the transfer is 16-byte
// aligned and the blocks are >= kPipeMinBytes; the ld/st kernel otherwise.  Both re-check
// every entry after its copy.
cudaError_t launch_kv_read_fused(const ReadFusedLaunch& a, cudaStream_t stream);
cudaError_t launch_kv_pipe_read(const ReadFusedLaunch& a, cudaStream_t stream);
// The same for fp8 pages ([elems x e4m3][elems/128 x fp32 scale] in the pool, bf16 at the
// destination): resolver + dequantising TMA pipeline in one launch (kv_fp8_pipe.cu).
// `bytes` / `variant` / ring geometry of the launch are ignored.
bool fp8_read_fused_supported(const ReadFusedLaunch& a, uint32_t elems);
cudaError_t launch_kv_fp8_read_fused(const ReadFusedLaunch& a, uint32_t elems, cudaStream_t stream);

// One pool block -> 2 or 4 destinations with a thread-block cluster: the leader CTA fetches
// the tile once (cp.async.bulk ... .multicast::cluster lands it in every CTA's shared
// memory), each CTA stores it to its own destination.  Destination r of block i is
// descs[i].dst + delta[r] (the same page offset in every destination tensor).
struct McastLaunch {
    const CopyDesc* descs = nullptr;  // device memory (e.g. written by launch_index_lookup)
    uint32_t n = 0;
    uint32_t bytes = 0;
    uint64_t align_or = 0;  // OR of every destination base and offset
    int ndst = 2;           // 2 or 4 = cluster size
    int64_t delta[4] = {0, 0, 0, 0};
    bool src_local = false;  // every source is in the launching GPU's own HBM (required)
    uint32_t* status = nullptr;
    int max_clusters = 0;
    uint32_t stage_bytes = 0;
    uint32_t ring_bytes = 0;
};
cudaError_t launch_kv_pipe_mcast(const McastLaunch& a, cudaStream_t stream);

// read fused with the layout swizzle for the attention consumer: pool pages are token-major
// [tok][head][dim]; the destination is a head-major paged KV cache [page][head][tok][dim].
// The tile is loaded with a 1-D bulk copy and stored with a 4-D tensor-map TMA
// (cp.async.bulk.tensor, SASS UTMASTG) that performs the transposition in hardware.
struct HndLaunch {
    const CopyDesc* descs = nullptr;  // src = mapped pool page (0 = miss), dst = page INDEX
    uint32_t n = 0;
    uint32_t tokens = 0, heads = 0, dim = 0, elem_size = 2;
    uint64_t dst_base = 0;   // [num_pages][heads][tokens][dim]
    uint32_t num_pages = 0;
    uint32_t* status = nullptr;
    int max_ctas = 0;
    uint32_t stage_bytes = 0, ring_bytes = 0;
};
cudaError_t launch_kv_pipe_hnd(const HndLaunch& a, cudaStream_t stream);

// One writer -> all readers replication through an NVLS multicast mapping (multimem.st).
struct BcastLaunch {
    const CopyDesc* descs = nullptr;  // dst = address inside the multicast mapping
    uint32_t n = 0;
    uint32_t bytes = 0;
    int max_ctas = 0;
    // optional in-band readiness: u32 per block INSIDE the multicast mapping; the writer adds
    // 1 per finished chunk to every replica's copy (multimem.red.release.sys)
    uint32_t* flags_mc = nullptr;
};
cudaError_t launch_kv_bcast_nvls(const BcastLaunch& a, cudaStream_t stream);
// chunks the broadcast kernel splits a block of `bytes` into = what a block's flag reaches
uint32_t bcast_chunks_per_block(uint32_t bytes);

// Reader of an NVLS broadcast: waits for each block's flag in the LOCAL replica
// (ld.acquire.sys, no host sync) and then copies the block out of the local replica.
struct ReadyLaunch {
    const CopyDesc* descs = nullptr;      // src = local replica address, dst = destination
    uint32_t n = 0;
    uint32_t bytes = 0;
    const uint32_t* flags_local = nullptr;  // this GPU's replica of the flag array
    uint32_t ready_value = 0;               // flag value that means "block complete"
    uint32_t* status = nullptr;             // kStatMiss counts blocks that never became ready
    int max_ctas = 0;
};
cudaError_t launch_kv_read_when_ready(const ReadyLaunch& a, cudaStream_t stream);

// ---------------------------------------------------------------- doorbell worker (kv_doorbell.cu)
// One persistent CTA that serves single-block writes / reads posted into a ring in pinned
// host memory: no launch, no event, no stream poll on the caller's path.
#if defined(__CUDACC__)
#define ISTORE_KHD __host__ __device__
#else
#define ISTORE_KHD
#endif
constexpr int kDoorbellMaxSlots = 64;
constexpr uint32_t kDoorbellMaxBytes = 256u << 10;  // larger blocks want more than one CTA
constexpr uint64_t kDoorbellMagic = 0x646f6f7262656c6cull;
enum : uint32_t { kDoorbellWrite = 1, kDoorbellRead = 2, kDoorbellStop = 3 };
enum : uint32_t { kDoorbellOk = 0, kDoorbellMiss = 1, kDoorbellStale = 2, kDoorbellIndexFull = 3 };
enum : uint32_t { kDoorbellRunning = 1, kDoorbellExited = 2 };
// q0 = seq << 2 | op                 q1 = local address (write: source, read: destination)
// q2 = mapped pool address (write)   q3, q4 = key fingerprint (write: h1 = 0 -> not indexed)
// q5 = global block address (write)  q6 = generation | bytes << 32
// q7 = q0 ^ ... ^ q6 ^ kDoorbellMagic: a line the host is still writing never matches
struct alignas(64) DoorbellReq {
    uint64_t q[8];
};
struct DoorbellCtl {
    alignas(64) uint64_t done_seq;  // worker -> host: every request <= done_seq has completed
    alignas(64) uint64_t state;     // worker -> host: doorbell_state(epoch, next request, code)
    alignas(64) uint32_t status[kDoorbellMaxSlots];  // per ring slot, valid once done
};
ISTORE_KHD inline uint64_t doorbell_state(uint32_t epoch, uint64_t next, uint32_t code) {
    return (uint64_t(epoch & 0xfffffu) << 44) | ((next & ((1ull << 42) - 1)) << 2) | code;
}
struct DoorbellLaunch {
    const DoorbellReq* ring = nullptr;  // device address of the pinned ring
    DoorbellCtl* ctl = nullptr;         // device address of the pinned control block
    uint32_t slots = 0;
    uint32_t epoch = 0;      // launch number (the host tells launches apart in `state`)
    uint64_t first_seq = 1;  // first request this launch serves
    uint64_t idle_ns = 200000;
    IndexBucket* table = nullptr;  // shard 0 of the device index (nullptr: nothing is indexed)
    uint64_t table_mask = 0;
    IndexShards shards;
    static constexpr int kMaxSegs = 16;
    uint64_t seg_base[kMaxSegs] = {0};
    uint32_t nsegs = 0;
    bool sys = true;
};
cudaError_t launch_kv_doorbell(const DoorbellLaunch& a, cudaStream_t stream);

// Number of SMs of the current device (cached per device).
int sm_count();
// Later work on `stream` waits, on the GPU, until *addr >= value (cuStreamWaitValue32, GEQ):
// how a consumer waits for a layered read's group flags without a host round trip.
// cudaErrorNotSupported when the driver does not offer the entry point.
cudaError_t stream_wait_geq(const uint32_t* addr, uint32_t value, cudaStream_t stream);
// Raises the dynamic shared-memory limit of each kernel to its `bytes`, once per device:
// `done` holds the caller's flag of every device.
struct SmemLimit {
    const void* kernel;
    int bytes;
};
cudaError_t set_smem_limits_once(bool (&done)[64], std::initializer_list<SmemLimit> limits);

}  // namespace istore::kernels
