// Client connection: blocking control-plane socket + client-driven data plane.
//
// Capability parity with the reference's `Connection` (src/libinfinistore.h:34-122):
// init_connection, the fabric set-up that replaces setup_rdma, register_mr,
// allocate[_async], w_rdma[_async], r_rdma[_async], rw_local, sync_local, sync_rdma,
// check_exist, get_match_last_index.
//
// The data plane is redesigned for an NVSwitch box: instead of posting RDMA work requests
// to a NIC (reference: src/libinfinistore.cpp:860-1099) the client maps the server's HBM
// pool segments into its own address space and launches sm_90a kernels on ITS GPU that
// move a whole batch of pages with peer loads/stores over NVLink and publish the commit
// in-band (kernels/kv_copy.cu).  The server CPU only allocates and indexes.
#pragma once

#include <atomic>
#include <condition_variable>
#include <deque>
#include <functional>
#include <map>
#include <memory>
#include <mutex>
#include <string>
#include <string_view>
#include <thread>
#include <unordered_map>
#include <vector>

#include "../core/config.h"
#include "../core/hash.h"
#include "../fabric/segment.h"
#include "../wire/protocol.h"

namespace istore {

namespace kernels {
struct CopyDesc;
struct IndexShards;
struct LookupLaunch;
struct GatherLaunch;
}
using kernels_CopyDesc = kernels::CopyDesc;
using kernels_IndexShards = kernels::IndexShards;
struct KeyBatch;

// Non-owning: the key bytes must stay valid for the duration of the call.
struct KeyOffset {
    std::string_view key;
    uint64_t offset;  // bytes from the tensor base
};

// The keys of a batch in the layout the lookup kernels read: every key on an 8-byte boundary,
// zero padded to a multiple of 8 (an empty key occupies 8 zero bytes), offsets and lengths as
// u32 arrays.  A caller that already holds its keys like this (the Python binding's arena)
// passes the view along with the KeyOffset list and saves the client a second pass over them.
struct PackedKeys {
    const uint8_t* bytes = nullptr;
    size_t nbytes = 0;
    const uint32_t* off = nullptr;
    const uint32_t* len = nullptr;
    size_t n = 0;
};

// addr -> key fingerprint of blocks that were allocated but not written yet.
// Blocks are almost always written in the order they were allocated, so the entries sit in a
// FIFO and `take` pops the head (a few ns per block on the write hot path); anything out of
// order falls back to an open-addressing map with backward-shift deletion.
class PendingHashes {
   public:
    void put(uint64_t addr, const KeyHash& h) { fifo_.push_back(Entry{addr, h}); }
    bool take(uint64_t addr, KeyHash* out);  // find + erase
    size_t size() const { return (fifo_.size() - head_) + count_; }

   private:
    struct Entry {
        uint64_t addr = 0;  // 0 = empty (block addresses are never 0)
        KeyHash h{};
    };
    void spill();  // move the FIFO into the map
    void map_put(uint64_t addr, const KeyHash& h);
    bool map_take(uint64_t addr, KeyHash* out);
    void grow();
    static size_t mix(uint64_t a) { return size_t((a * 0x9e3779b97f4a7c15ull) >> 20); }
    std::vector<Entry> fifo_;
    size_t head_ = 0;
    std::vector<Entry> slots_;
    size_t count_ = 0;
};

struct ClientStats {
    uint64_t kernel_launches = 0;   // data-plane kernels launched by this connection
    uint64_t bytes_written = 0;
    uint64_t bytes_read = 0;
    uint64_t ctrl_requests = 0;
    uint64_t host_copies = 0;       // blocks moved with memcpy (CPU tensors / host pool)
    // host-side time of the data-plane calls, nanoseconds (tracing aid, see docs/design.md)
    uint64_t ns_build = 0;    // descriptor / record / key packing loops
    uint64_t ns_streams = 0;  // stream selection + cross-stream event dependencies
    uint64_t ns_launch = 0;   // cudaLaunchKernel and friends
    uint64_t calls = 0;
    uint64_t doorbell_ops = 0;      // single-block operations served by the persistent worker
    uint64_t doorbell_launches = 0;  // (re)launches of the worker
    // staging allocations (descriptors, records, keys, counters) that had to block the host
    // until an earlier launch of this connection completed before reusing its bytes
    uint64_t drains = 0;
};

class Connection {
   public:
    Connection();
    ~Connection();
    Connection(const Connection&) = delete;
    Connection& operator=(const Connection&) = delete;

    // --- connection management
    int init_connection(const ClientConfig& cfg);  // TCP connect + 'E' exchange
    int setup_rdma(const ClientConfig& cfg);       // fetch the pool map (fabric set-up)
    void close();
    bool connected() const { return fd_ >= 0; }
    bool server_has_hbm() const { return server_hbm_; }
    bool server_evicts() const { return server_evicts_; }
    bool index_incomplete() const { return index_incomplete_.load(); }

    // --- metadata
    int check_exist(const std::string& key);  // 0 = exists & committed, 1 = not, <0 error
    int get_match_last_index(const std::vector<std::string_view>& keys);  // index, -1 none, <-1 error
    // Recency hint for a store that evicts: the blocks of `keys` were just used (e.g. read
    // through the device index, which the server does not see).  Returns the number of
    // blocks refreshed, < 0 on error.
    int touch(const std::vector<std::string_view>& keys);
    int sync_local();  // remaining server-side tasks (always 0 here) or <0
    int sync_rdma();   // drain kernels + async ops, commit, control-plane barrier

    // --- data plane.  `device` is the CUDA ordinal owning base_ptr, -1 for host memory;
    //     `stream` is a cudaStream_t to order after (0 = the connection's own stream).
    int register_mr(uint64_t ptr, size_t size, int device);
    // Forget a registered region; host memory is unpinned once no kernel can still read it.
    // Must be called before registered HOST memory is freed: a stale pin would keep mapping
    // the old physical pages at that virtual address.
    int unregister_mr(uint64_t ptr);
    // hint: pool device to prefer, kReplicaDevice (-2) for the NVLS-replicated region,
    // kHintDefault for the connection's configured pool_hint
    static constexpr int kHintDefault = -1000;
    int allocate(const std::vector<std::string_view>& keys, int block_size,
                 std::vector<RemoteBlock>& out, int hint = kHintDefault);
    // offsets[i] * scale = byte offset of block i (scale lets callers pass element offsets)
    // What one data-plane call did: the stream (and device) its kernels were launched on,
    // and - for writes, when `commits` is set - the addresses of exactly the blocks it wrote
    // (otherwise they join the connection-wide list that the next sync() commits).
    struct MoveResult {
        std::vector<uint64_t>* commits = nullptr;
        void* stream = nullptr;  // cudaStream_t
        int device = -1;
        bool launched = false;
    };
    int w_rdma(const uint64_t* offsets, size_t noffsets, uint64_t scale, int block_size,
               const RemoteBlock* blocks, size_t nblocks, uint64_t base_ptr, int device,
               uint64_t stream, MoveResult* res = nullptr);
    int r_rdma(const std::vector<KeyOffset>& blocks, int block_size, uint64_t base_ptr, int device,
               uint64_t stream, MoveResult* res = nullptr, const PackedKeys* packed = nullptr);
    int rw_local(char op, const std::vector<KeyOffset>& blocks, int block_size, uint64_t base_ptr,
                 int device, uint64_t stream);
    // read the same pages into several destination tensors of one device: each pool block
    // crosses the fabric once and is fanned out by a thread-block cluster (TMA multicast)
    int r_rdma_multi(const std::vector<KeyOffset>& blocks, int block_size,
                     const std::vector<uint64_t>& bases, int device, uint64_t stream);
    // read fused with the attention consumer's layout: token-major pool pages
    // ([tokens][heads][dim]) land head-major in base_ptr = [num_pages][heads][tokens][dim];
    // blocks[i].offset is the destination page index (TMA tensor-map store)
    int r_rdma_hnd(const std::vector<KeyOffset>& blocks, int tokens, int heads, int dim,
                   int elem_size, uint64_t base_ptr, uint64_t num_pages, int device,
                   uint64_t stream);
    // fp8 KV path: pages are bf16 in the caller's tensor (`elems` elements each) and
    // e4m3 + per-128 fp32 scales in the pool (kernels::fp8_block_bytes(elems) bytes, which is
    // the size to allocate).  The cast is fused into the page mover.
    int w_rdma_fp8(const uint64_t* offsets, size_t noffsets, uint64_t scale, int elems,
                   const RemoteBlock* blocks, size_t nblocks, uint64_t base_ptr, int device,
                   uint64_t stream);
    int r_rdma_fp8(const std::vector<KeyOffset>& blocks, int elems, uint64_t base_ptr, int device,
                   uint64_t stream);
    // A layered read's groups (r_rdma_scatter with GatherSpec::reader).  wait_layered(r, g,
    // stream) makes later work on `stream` wait on the GPU until group g has landed
    // (cuStreamWaitValue32), with no host synchronisation.
    struct ScatterReader {
        uint32_t groups = 0;
        uint32_t group_parts = 0;
        int device = -1;
        uint64_t seq = 0;                 // 0: nothing was launched (no blocks); waits are no-ops
        const uint32_t* flags = nullptr;  // device: one word per group, in the reader's slot
        bool failed = false;              // refused or failed: every wait is refused
        uint64_t session = 0;             // the connection session whose device flags it uses
    };
    // Gathered blocks (kernels::GatherLaunch): a block is `nparts` parts, part s at
    // part_base[s] + the block's local byte offset (one page of every layer under one key).
    struct GatherSpec {
        const uint64_t* part_base = nullptr;  // absolute addresses, all on `device` (or host)
        uint32_t nparts = 0;
        uint32_t part_bytes = 0;  // bytes of a raw part (not read when fp8_elems > 0)
        // > 0: every part is a bf16 page of fp8_elems elements (a multiple of 512) in the
        // caller's CUDA tensors and an fp8 page in the pool; part bases and offsets 16-byte
        // aligned
        uint32_t fp8_elems = 0;
        uint32_t first_part = 0;  // stored part first_part + s is part s (one-shot writes: 0)
        // reads: a layered read, whose parts are released to `reader`'s waits in groups of
        // group_parts (which must divide nparts)
        ScatterReader* reader = nullptr;
        uint32_t group_parts = 0;
        // reads: row-sliced parts (kernels::GatherLaunch::rows, bytes); rows == 0: whole parts
        uint32_t rows = 0, row_bytes = 0, src_pitch = 0, src_col = 0, dst_pitch = 0;
        // pool bytes of a part: part_bytes, or kernels::fp8_gather_bytes(1, fp8_elems)
        uint64_t pool_part_bytes() const;
        // bytes a stored block must hold to serve a read: parts 0 .. first_part + nparts - 1
        uint64_t need_bytes() const { return (uint64_t(first_part) + nparts) * pool_part_bytes(); }
    };
    // Layered gathered write: a fixed set of allocated gathered blocks whose parts are stored
    // over several calls (write_layered), each a contiguous range of parts of every block -
    // typically one layer's K and V as prefill produces them.  A block is published (device
    // index) by the launch that lands its last part, and its server commit is staged by the
    // call that completes the writer.  Not thread-safe: one caller at a time.
    struct GatherWriter {
        std::vector<RemoteBlock> blocks;  // blocks to write (the "already exists" ones dropped)
        std::vector<uint64_t> offsets;    // their local offsets (elements until the first call)
        std::vector<KeyHash> hashes;      // their key fingerprints from allocate
        bool indexed = true;              // every block has a fingerprint: it can be published
        uint32_t nparts = 0;              // S: parts of a block
        std::vector<uint8_t> written;     // per part: stored by an earlier call
        uint32_t parts_written = 0;
        uint32_t calls = 0;               // calls that launched (the first one claims)
        int device = -2;                  // fixed by the first call (-1: host tensors)
        uint64_t scale = 0;               // bytes per offset unit, fixed by the first call
        uint32_t fp8_elems = 0;           // fp8 elements per part (0: raw bytes), first call
        uint32_t part_bytes = 0;          // pool bytes of a part, first call
        bool failed = false;
        void* event = nullptr;            // cudaEvent_t recorded after the last launch
        uint32_t* state = nullptr;        // device: 3 u32 per block (kernels::GatherLaunch)
        uint64_t session = 0;             // the connection session that allocated the blocks
        bool complete() const { return parts_written == nparts; }
        ~GatherWriter();
    };
    // Takes the blocks' fingerprints out of the allocation record, once.
    std::shared_ptr<GatherWriter> gather_writer(const RemoteBlock* blocks, const uint64_t* offsets,
                                                size_t n, uint32_t nparts);
    // Stores parts g.first_part .. g.first_part + g.nparts - 1 of every block of `w`; offsets
    // are scaled by `scale`.  Refuses part ranges written before, a device, scale, fp8_elems
    // or part size other than the first call's, a complete or failed writer, and a writer made
    // before the connection was last closed (its blocks and index ways were released).  A
    // refused call leaves the writer as it was.
    int write_layered(GatherWriter& w, const GatherSpec& g, uint64_t scale, int device,
                      uint64_t stream);
    // offsets in bytes; blocks allocated with nparts * g.pool_part_bytes() bytes (trusted)
    int w_rdma_gather(const GatherSpec& g, const uint64_t* offsets, size_t noffsets,
                      const RemoteBlock* blocks, size_t nblocks, int device, uint64_t stream);
    // A stored block must hold g.need_bytes() bytes, else it is a miss.  Row-sliced (g.rows):
    // bf16 only, rows >= 1, src_col + row_bytes <= src_pitch and part_bytes == rows *
    // src_pitch.  With g.reader, a layered read: one call whose last page-mover launch
    // releases the parts group by group, each by storing `seq` to its flag word, and each key
    // is resolved once; CUDA tensors of an HBM pool only, not on a doorbell connection, and on
    // failure the reader is failed.  Every refusal comes before anything is enqueued.
    int r_rdma_scatter(const GatherSpec& g, const std::vector<KeyOffset>& blocks, int device,
                       uint64_t stream);
    // Later work on `stream` waits on the GPU until group `group` of `r` has landed.  0; -1
    // (and *err) when refused: a failed reader, a group outside the read, or a reader made
    // before the connection was last closed (its flags were freed with the device context);
    // -2 (and *err) when the driver refuses the wait.  Nothing is enqueued unless 0.
    int wait_layered(const ScatterReader& r, uint32_t group, uint64_t stream, std::string* err);

    // --- async flavours: the callback runs on the connection's completion thread
    int allocate_async(const std::vector<std::string>& keys, int block_size,
                       std::function<void(std::vector<RemoteBlock>)> cb);
    int w_rdma_async(const std::vector<uint64_t>& offsets, int block_size,
                     const RemoteBlock* blocks, size_t nblocks, uint64_t base_ptr, int device,
                     uint64_t stream, std::function<void(int)> cb);
    int r_rdma_async(const std::vector<KeyOffset>& blocks, int block_size, uint64_t base_ptr,
                     int device, uint64_t stream, std::function<void(int)> cb);

    // --- tuning / introspection
    void set_copy_variant(int v) { copy_variant_ = v; }
    void set_max_ctas(int n) { max_ctas_ = n; }
    // TMA pipeline ring geometry: slot bytes and ring bytes per CTA (0 = kernel default)
    void set_pipe_geometry(uint32_t stage_bytes, uint32_t ring_bytes) {
        pipe_stage_ = stage_bytes;
        pipe_ring_ = ring_bytes;
    }
    void set_device_lookup(bool on) { device_lookup_ = on; }
    // 0: launch in the caller's stream; n >= 1: round-robin over n internal streams that
    // wait for the caller's stream (kernels of successive calls overlap)
    void set_streams(int n) { streams_ = n < 0 ? 0 : (n > 8 ? 8 : n); }
    bool device_lookup() const { return device_lookup_; }
    ClientStats stats() const;
    std::vector<SegmentInfo> segments() const { return segs_; }
    const std::string& last_error() const { return last_error_; }

   private:
    struct DevCtx;
    struct Task;
    struct LaunchScope;

    // control plane
    int transact(char op, const void* body, size_t len, int32_t* code,
                 std::vector<uint8_t>* payload, size_t fixed_payload,
                 const std::vector<uint8_t>* prefix = nullptr);
    int send_raw(const void* framed, size_t len);  // already framed, reply-less message(s)
    int send_only(char op, const void* body, size_t len);
    int refresh_pool_map();
    int lookup_blocks(char op, const std::vector<KeyOffset>& blocks, int block_size,
                      std::vector<RemoteBlock>& out);
    int flush_commits();
    uint32_t take_publish_failures();
    void refresh_index_state();
    // doorbell worker (latency mode); all under mu_
    bool doorbell_ready(DevCtx* ctx, uint64_t user_stream, size_t bytes);
    int doorbell_post(DevCtx* ctx, uint32_t op, const uint64_t (&q)[6]);
    int doorbell_start(DevCtx* ctx);
    int doorbell_wait(DevCtx* ctx);
    int doorbell_quiesce(DevCtx* ctx);
    void doorbell_collect(DevCtx* ctx);
    void doorbell_stop(DevCtx* ctx);
    int send_commit(const uint64_t* addrs, size_t count);

    // data plane
    DevCtx* dev_ctx(int device);
    std::shared_ptr<fabric::Mapping> mapping(uint32_t seg, int device);
    int move_blocks(bool write, const uint64_t* local_off, uint64_t scale,
                    const RemoteBlock* blocks, size_t n, int block_size, uint64_t base_ptr,
                    int device, uint64_t stream, int fp8_elems = 0, MoveResult* res = nullptr,
                    const GatherSpec* gather = nullptr, GatherWriter* layered = nullptr);
    // tell the server that the blocks at `addrs` were not (completely) written: it releases
    // them, device-index entries included
    int discard_blocks(const uint64_t* addrs, size_t count);
    uint8_t* seg_dev_ptr(DevCtx* ctx, uint32_t seg);
    kernels_IndexShards index_shards(DevCtx* ctx, bool* all_local);
    kernels::GatherLaunch gather_launch(const GatherSpec& g, uint32_t n, uint64_t align_or,
                                        uint32_t* status, int max_ctas);
    // why a gathered call is refused (nullptr: it is not); `w`: a layered writer's call
    const char* gather_refusal(const GatherSpec& g, const uint64_t* offs, size_t n, int device,
                               bool write, const GatherWriter* w = nullptr) const;
    // a layered read's last launch: takes the reader's slot (0 on failure, else its seq)
    uint64_t arm_reader(DevCtx* ctx, const ScatterReader& r, kernels::GatherLaunch& G);
    int reader_launched(DevCtx* ctx, ScatterReader& r, uint64_t seq, void* stream);
    struct ReaderHold;
    template <typename Launch>
    bool set_index(DevCtx* ctx, Launch& L, bool segs = true);
    const kernels_CopyDesc* resolve_descs(DevCtx* ctx, const std::vector<KeyOffset>& blocks,
                                          size_t base, const KeyBatch& b, const PackedKeys* packed,
                                          uint32_t need_bytes, uint64_t dst_base,
                                          const std::vector<RemoteBlock>* rb, void* stream,
                                          kernels::LookupLaunch* checked = nullptr);
    template <typename Launch>
    int read_resolved(const std::vector<KeyOffset>& blocks, int block_size, int device,
                      uint64_t stream, uint64_t dst_base, const char* what, Launch&& launch);
    int read_blocks(char op, const std::vector<KeyOffset>& blocks, int block_size,
                    uint64_t base_ptr, int device, uint64_t stream, int fp8_elems = 0,
                    MoveResult* res = nullptr, const PackedKeys* packed = nullptr,
                    const GatherSpec* gather = nullptr);
    int read_via_device_index(const std::vector<KeyOffset>& blocks, int block_size,
                              uint64_t base_ptr, int device, uint64_t stream, int fp8_elems = 0,
                              MoveResult* res = nullptr, const PackedKeys* packed = nullptr,
                              const GatherSpec* gather = nullptr);
    int match_via_device_index(const std::vector<std::string_view>& keys, bool exist_only);
    int ensure_host_registered(uint64_t ptr, size_t bytes, int device, bool temporary);
    void release_temporary_host_regs();
    int drain_devices(bool* device_error = nullptr);
    bool device_index_usable();
    void fail(const std::string& msg);

    // completion thread
    void worker();
    void post(Task&& t);

    ClientConfig cfg_;
    int fd_ = -1;
    std::mutex sock_mu_;  // one request/response transaction at a time
    std::mutex sync_mu_;  // one sync() at a time (staged commit + SYNC form a pair)
    bool server_cuda_ = false;
    bool server_hbm_ = false;
    uint8_t server_uuid_[16] = {0};
    std::vector<SegmentInfo> segs_;

    std::mutex mu_;  // guards the data-plane state below
    std::map<int, std::unique_ptr<DevCtx>> devs_;
    std::vector<std::shared_ptr<fabric::Mapping>> host_maps_;  // CPU view of host segments
    PendingHashes pending_hash_;  // allocated addr -> key fingerprint
    std::vector<uint64_t> pending_commit_;
    bool ctrl_dirty_ = false;  // the server holds state (leases) that the next SYNC releases
    struct HostReg {
        size_t bytes;
        bool registered;
        bool temporary;  // pinned implicitly for one transfer: released at the next sync()
    };
    std::map<uint64_t, HostReg> host_regs_;  // register_mr'ed host ranges by base pointer
    std::map<uint64_t, size_t> mrs_;         // registered regions by base pointer (C10)
    int copy_variant_ = 0;
    int max_ctas_ = 0;
    uint32_t pipe_stage_ = 0, pipe_ring_ = 0;
    bool device_lookup_ = false;
    bool server_evicts_ = false;
    // set when any writer failed to publish a block in the HBM index (learnt from own kernels,
    // the server's exchange flags or a SYNC reply): reads then resolve through the server
    std::atomic<bool> index_incomplete_{false};
    uint32_t publish_failures_ = 0;  // own failures not yet reported to the server
    int streams_ = 4;
    int default_device_ = -1;
    uint64_t session_ = 0;  // under mu_: close() ends a session (GatherWriter::session)
    ClientStats stats_;
    std::string last_error_;

    std::thread worker_;
    std::mutex q_mu_;
    std::condition_variable q_cv_, idle_cv_;
    std::deque<Task> queue_;
    size_t inflight_async_ = 0;
    bool stop_ = false;
};

}  // namespace istore
