// Control-plane server: an epoll reactor on its own thread that owns the allocator, the
// key index and the pool segments.
//
// Role parity with the reference's libuv front-end + server bootstrap
// (src/infinistore.cpp:1113-1298): accept, 2-state header/body stream parser tolerant of
// arbitrary TCP segmentation, per-op dispatch, replies of `int code + payload`.  It is
// NOT a libuv port: libuv headers do not exist on the target image, and this design
// moves all data movement to client-side kernels, so the server never touches CUDA on a
// request path (no per-request stream/event/IPC-open as in the reference's local path).
//
// Hardening relative to the reference (SURVEY §2.5 D7, D11, D12): body_size is capped, an
// unknown op is answered with 400 and the connection is closed instead of spinning,
// every flatbuffer is verified, the exchange body must be exactly 30 bytes, the listen
// address is honoured, and uncommitted reservations of a dead client are released.
#pragma once

#include <atomic>
#include <cstdint>
#include <map>
#include <memory>
#include <mutex>
#include <string>
#include <thread>
#include <utility>
#include <vector>

#include "../core/config.h"
#include "../core/kv_store.h"
#include "../core/mempool.h"
#include "../fabric/segment.h"

namespace istore {

namespace kernels {
struct IndexBucket;
struct IndexShards;
}  // namespace kernels

// Service-time histogram of one opcode: bucket b counts requests that took < 2^b microseconds
// (bucket 0: < 1 us ... bucket 23: everything longer than ~4 s).
struct OpTiming {
    static constexpr int kBuckets = 24;
    uint64_t count = 0;
    uint64_t sum_us = 0;
    uint64_t max_us = 0;
    uint64_t bucket[kBuckets] = {0};
    void add(uint64_t us) {
        ++count;
        sum_us += us;
        if (us > max_us) max_us = us;
        int b = 0;
        while (b < kBuckets - 1 && (uint64_t(1) << b) <= us) ++b;
        ++bucket[b];
    }
    // upper bound (us) of the bucket that holds quantile q in (0, 1]
    uint64_t quantile_us(double q) const {
        if (!count) return 0;
        const uint64_t want = uint64_t(q * double(count) + 0.999999);
        uint64_t seen = 0;
        for (int b = 0; b < kBuckets; ++b) {
            seen += bucket[b];
            if (seen >= want) return b == kBuckets - 1 ? max_us : (uint64_t(1) << b);
        }
        return max_us;
    }
};

struct ServerStats {
    uint64_t connections = 0;       // currently open
    uint64_t accepted = 0;          // total accepted
    uint64_t requests = 0;
    uint64_t bad_requests = 0;
    uint64_t keys = 0;
    uint64_t inflight = 0;
    uint64_t pool_bytes = 0;
    uint64_t used_bytes = 0;
    uint64_t segments = 0;
    uint64_t evicted = 0;           // blocks evicted since start
    uint64_t lookup_hits = 0;       // keys resolved by server-mediated reads
    uint64_t lookup_misses = 0;     // server-mediated read requests answered 404
    uint64_t dedup_skips = 0;       // allocate requests for keys that already existed
    uint64_t index_overflows = 0;   // blocks writers could not insert into the HBM index
    uint64_t ops[128] = {0};        // per opcode
    OpTiming timing[128];           // per opcode service time (reactor thread, decode -> reply queued)
};

class Server {
   public:
    explicit Server(const ServerConfig& cfg);
    ~Server();

    // Creates the pool, binds and starts the reactor thread.  0 on success.
    int start(std::string* err);
    void stop();
    bool running() const { return running_.load(); }
    int port() const { return port_; }

    size_t kvmap_len();
    size_t purge();
    ServerStats stats();
    std::vector<SegmentInfo> segments();
    // Shard 0 of the device index: its address on the pool GPU and its slots ({0, 0} when the
    // pool keeps no device index).  Lets tests of an in-process server inspect the index.
    std::pair<uint64_t, uint64_t> index_table();

    // Checkpoint / resume (the reference has none: a restart loses everything, SURVEY §5.4).
    // dump: every committed block (key, size, bytes) to one file.  load: re-reserve, copy the
    // bytes into the pool and commit; keys that already exist are skipped (first writer wins).
    // For an HBM pool the bytes go through the kv_copy kernel, which also publishes the
    // device index.  Both return the number of blocks, or -1 with `err` set.
    long dump(const std::string& path, std::string* err);
    long load(const std::string& path, std::string* err);

    // Fault injection for tests: close a connection instead of answering the n-th request
    // from now (0 = off).
    void inject_drop_after(uint64_t n) { drop_after_.store(n); }
    // Fault injection for tests: stall the reactor for `ms` before serving each of the next
    // `count` requests (a slow / overloaded server).
    void inject_delay(uint32_t ms, uint64_t count) {
        delay_ms_.store(ms);
        delay_count_.store(count);
    }

   private:
    struct Conn;
    void loop();
    void on_accept();
    void on_readable(Conn* c);
    void on_writable(Conn* c);
    void close_conn(Conn* c);
    bool dispatch(Conn* c);  // false => close the connection
    void reply(Conn* c, int32_t code, const void* payload = nullptr, size_t len = 0);
    void reply_blob(Conn* c, int32_t code, const void* blob, size_t len);
    bool add_segment(std::string* err);
    bool maybe_extend();
    // Evict least-recently-used committed blocks covering `want` bytes: out of the map, out
    // of the device index (erase kernel, synchronised), then back to the pool.
    bool evict_some(size_t want, bool replica);
    bool erase_from_device_index(const std::vector<KVStore::Victim>& victims);
    // Uncommitted blocks taken out of the map: erase their device-index ways, then free them
    // (or quarantine them when the erase cannot be confirmed).
    void release_dropped(std::vector<KVStore::Victim>& victims);
    void note_publish_failures(uint32_t n);
    void fill_index_view(kernels::IndexBucket** table, uint64_t* mask,
                         kernels::IndexShards* shards) const;

    int handle_exchange(Conn* c);
    int handle_pool_map(Conn* c);
    int handle_allocate(Conn* c, bool local);
    int handle_lookup(Conn* c, bool local);
    int handle_commit(Conn* c);
    int handle_stage_commit(Conn* c);
    int handle_check_exist(Conn* c);
    int handle_match(Conn* c);
    int handle_touch(Conn* c);

    ServerConfig cfg_;
    int port_ = 0;
    int listen_fd_ = -1;
    int epoll_fd_ = -1;
    int wake_fd_ = -1;
    std::thread thread_;
    std::atomic<bool> running_{false};
    std::atomic<bool> stop_{false};
    std::atomic<uint64_t> drop_after_{0};
    std::atomic<uint32_t> delay_ms_{0};
    std::atomic<uint64_t> delay_count_{0};

    std::mutex mu_;  // guards everything below (reactor thread vs. manage-plane callers)
    MM mm_;
    std::unique_ptr<KVStore> store_;
    std::vector<std::unique_ptr<fabric::SegmentOwner>> segs_;
    std::map<int, std::unique_ptr<Conn>> conns_;
    uint64_t next_conn_id_ = 1;
    size_t next_pool_dev_ = 0;
    bool use_hbm_ = false;
    bool index_incomplete_ = false;  // some block is in the host map but not in the HBM index
    ServerStats stats_;
    std::vector<uint8_t> scratch_;  // reply serialisation buffer
    // segment ids that carry an index shard, in shard order (shard k = index_shards_[k])
    std::vector<uint32_t> index_shards_;
    struct EraseCtx {  // per shard: device staging + stream of the erase kernel
        int device = -1;
        void* buf = nullptr;
        size_t cap = 0;        // records
        void* stream = nullptr;  // cudaStream_t
    };
    std::vector<EraseCtx> erase_;
    // evicted blocks whose index entries could not be erased: their space stays reserved
    std::vector<KVStore::Victim> quarantine_;
};

}  // namespace istore
