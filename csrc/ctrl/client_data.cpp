// Data plane of the client: pool mappings, page-mover launches, device-index reads.
#include "client.h"

#include <cuda_runtime_api.h>

#include <algorithm>
#include <atomic>
#include <cerrno>
#include <cfloat>
#include <chrono>
#include <cstring>
#include <mutex>

#include "../core/log.h"
#include "../core/trace.h"
#include "../kernels/kernels.h"
#include "../kernels/launch_plan.h"
#include "../wire/messages.h"
#include "client_dev.h"
#include "read_plan.h"

namespace istore {

Connection::DevCtx* Connection::dev_ctx(int device) {
    auto it = devs_.find(device);
    if (it != devs_.end()) return it->second.get();
    if (device < 0 || device >= fabric::cuda_device_count()) {
        fail("no such CUDA device: " + std::to_string(device));
        return nullptr;
    }
    DeviceGuard g(device);
    auto ctx = std::make_unique<DevCtx>();
    ctx->device = device;
    ctx->drains = &stats_.drains;
    void* dp = nullptr;
    if (cudaStreamCreateWithFlags(&ctx->stream, cudaStreamNonBlocking) != cudaSuccess ||
        cudaHostAlloc(reinterpret_cast<void**>(&ctx->ring_h), kRingBytes,
                      cudaHostAllocMapped | cudaHostAllocPortable) != cudaSuccess ||
        cudaHostGetDevicePointer(&dp, ctx->ring_h, 0) != cudaSuccess) {
        fail(std::string("device context: ") + cudaGetErrorString(cudaGetLastError()));
        return nullptr;
    }
    ctx->ring_d = static_cast<uint8_t*>(dp);
    if (cudaHostAlloc(reinterpret_cast<void**>(&ctx->status_h), 256,
                      cudaHostAllocMapped | cudaHostAllocPortable) != cudaSuccess ||
        cudaHostGetDevicePointer(&dp, ctx->status_h, 0) != cudaSuccess ||
        cudaMalloc(reinterpret_cast<void**>(&ctx->scratch), kScratchBytes) != cudaSuccess ||
        cudaMalloc(reinterpret_cast<void**>(&ctx->zeros), kZeroBytes) != cudaSuccess ||
        cudaMemset(ctx->zeros, 0, kZeroBytes) != cudaSuccess) {
        fail(std::string("device context: ") + cudaGetErrorString(cudaGetLastError()));
        return nullptr;
    }
    ctx->status_d = static_cast<uint32_t*>(dp);
    std::memset(ctx->status_h, 0, 256);
    if (default_device_ < 0) default_device_ = device;
    DevCtx* raw = ctx.get();
    devs_[device] = std::move(ctx);
    return raw;
}

std::shared_ptr<fabric::Mapping> Connection::mapping(uint32_t seg, int device) {
    if (seg >= segs_.size() && refresh_pool_map() != 0) return nullptr;
    if (seg >= segs_.size()) {
        fail("server referenced unknown pool segment " + std::to_string(seg));
        return nullptr;
    }
    if (device >= 0) {
        DevCtx* ctx = dev_ctx(device);
        if (!ctx) return nullptr;
        if (ctx->maps.size() <= seg) ctx->maps.resize(seg + 1);
        if (!ctx->maps[seg]) {
            std::string err;
            ctx->maps[seg] = fabric::map_segment(segs_[seg], device, &err);
            if (!ctx->maps[seg]) fail("cannot map pool segment: " + err);
        }
        return ctx->maps[seg];
    }
    // host-only mapping (CPU tensors against a host pool)
    if (host_maps_.size() <= seg) host_maps_.resize(seg + 1);
    if (!host_maps_[seg]) {
        std::string err;
        host_maps_[seg] = fabric::map_segment(segs_[seg], -1, &err);
        if (!host_maps_[seg]) fail("cannot map pool segment: " + err);
    }
    return host_maps_[seg];
}

int Connection::ensure_host_registered(uint64_t ptr, size_t bytes, int device, bool temporary) {
    auto it = host_regs_.upper_bound(ptr);
    if (it != host_regs_.begin()) {
        --it;
        if (ptr >= it->first && ptr + bytes <= it->first + it->second.bytes &&
            it->second.registered)
            return 0;
    }
    DeviceGuard g(device);
    const cudaError_t e = cudaHostRegister(reinterpret_cast<void*>(ptr), bytes,
                                           cudaHostRegisterMapped | cudaHostRegisterPortable);
    if (e != cudaSuccess && e != cudaErrorHostMemoryAlreadyRegistered) {
        (void)cudaGetLastError();
        return -1;
    }
    (void)cudaGetLastError();
    host_regs_[ptr] = HostReg{bytes, e == cudaSuccess, temporary};
    return 0;
}

// Implicit pins (a CPU tensor that was never register_mr'ed) live for one transfer only: the
// caller may free the tensor after sync(), and a pin that outlives its memory would map stale
// physical pages if the address is reused.
void Connection::release_temporary_host_regs() {
    for (auto it = host_regs_.begin(); it != host_regs_.end();) {
        if (it->second.temporary) {
            if (it->second.registered) cudaHostUnregister(reinterpret_cast<void*>(it->first));
            (void)cudaGetLastError();
            it = host_regs_.erase(it);
        } else {
            ++it;
        }
    }
}

int Connection::unregister_mr(uint64_t ptr) {
    if (drain_devices() != 0) { /* report via the next sync; still unpin below */ }
    std::lock_guard<std::mutex> lk(mu_);
    mrs_.erase(ptr);
    auto it = host_regs_.find(ptr);
    if (it != host_regs_.end()) {
        if (it->second.registered) cudaHostUnregister(reinterpret_cast<void*>(ptr));
        (void)cudaGetLastError();
        host_regs_.erase(it);
    }
    return 0;
}

int Connection::register_mr(uint64_t ptr, size_t size, int device) {
    std::lock_guard<std::mutex> lk(mu_);
    mrs_[ptr] = size;  // re-registering the same base replaces the old entry
    if (device < 0 && fabric::cuda_available() && server_hbm_) {
        // Pin + map host memory so that kernels can stream it over PCIe (the role
        // ibv_reg_mr plays for CPU tensors in the reference).
        const int kd = cfg_.device >= 0 ? cfg_.device : std::max(default_device_, 0);
        if (ensure_host_registered(ptr, size, kd, false) != 0)
            LOG_WARN("register_mr: could not pin host memory, falling back to staged copies");
    }
    if (device >= 0 && !dev_ctx(device)) return -1;
    return 1;
}

// Resolve the device pointer of a pool segment for `ctx` (slow path: map it first).
uint8_t* Connection::seg_dev_ptr(DevCtx* ctx, uint32_t seg) {
    if (seg < ctx->seg_ptr.size() && ctx->seg_ptr[seg]) return ctx->seg_ptr[seg];
    auto mp = mapping(seg, ctx->device);
    if (!mp || (!mp->dev_ptr && !mp->mc_ptr)) {
        fail("pool segment " + std::to_string(seg) + " is not addressable from device " +
             std::to_string(ctx->device));
        return nullptr;
    }
    if (ctx->seg_ptr.size() <= seg) {
        ctx->seg_ptr.resize(seg + 1, nullptr);
        ctx->seg_remote.resize(seg + 1, 1);
        ctx->seg_mc.resize(seg + 1, nullptr);
    }
    ctx->seg_ptr[seg] = mp->dev_ptr;
    ctx->seg_mc[seg] = mp->mc_ptr;
    // NVLink (or PCIe) on the path?  Such transfers are link-bound: a small grid saturates
    // them and leaves the SMs to whatever else runs on this GPU.
    cudaPointerAttributes attr{};
    bool local = false;
    if (cudaPointerGetAttributes(&attr, mp->dev_ptr) == cudaSuccess)
        local = attr.type == cudaMemoryTypeDevice && attr.device == ctx->device;
    (void)cudaGetLastError();
    ctx->seg_remote[seg] = local ? 0 : 1;
    return mp->dev_ptr;
}

// The index shards beyond shard 0 as seen from `ctx`'s device: the k-th HBM segment (in id
// order) that carries a table is shard k.  *all_local is cleared when a shard's table lives
// on another GPU.
kernels::IndexShards Connection::index_shards(DevCtx* ctx, bool* all_local) {
    kernels::IndexShards sh;
    uint32_t n = 0;
    for (uint32_t id = 0; id < segs_.size() && n < kernels::kMaxIndexShards; ++id) {
        if (segs_[id].kind != kSegDeviceIpc || !segs_[id].index_slots) continue;
        if (n > 0) {
            uint8_t* base = seg_dev_ptr(ctx, id);
            if (!base) break;  // cannot map it: stay with the shards found so far
            sh.table[n - 1] = reinterpret_cast<kernels::IndexBucket*>(base + segs_[id].index_off);
            sh.mask[n - 1] = kernels::index_bucket_mask(segs_[id].index_slots);
            if (all_local && ctx->seg_remote[id]) *all_local = false;
        }
        ++n;
    }
    sh.n = n;
    return sh;
}

// Shard 0 of the device index (segment 0's table) and the further shards as seen from ctx's
// device, and with `segs` the segment bases the lookup kernels turn hits into addresses with.
// false when segment 0 carries no index this device can reach.
template <typename Launch>
bool Connection::set_index(DevCtx* ctx, Launch& L, bool segs) {
    auto m0 = mapping(0, ctx->device);
    if (!m0 || !m0->dev_ptr || !segs_[0].index_slots) return false;
    if (segs) {
        L.nsegs = uint32_t(std::min<size_t>(segs_.size(), Launch::kMaxSegs));
        for (uint32_t s = 0; s < L.nsegs; ++s)
            L.seg_base[s] = reinterpret_cast<uint64_t>(seg_dev_ptr(ctx, s));
    }
    L.table = reinterpret_cast<kernels::IndexBucket*>(m0->dev_ptr + segs_[0].index_off);
    L.table_mask = kernels::index_bucket_mask(segs_[0].index_slots);
    L.shards = index_shards(ctx, nullptr);
    return true;
}

// The steps around the launches of one data-plane call.  The constructor makes the device
// context current for the scope; the doorbell fast paths go between it and begin(), which
// quiesces the doorbell worker and picks the launch stream.  launched() follows each batch.
struct Connection::LaunchScope {
    Connection& c;
    DevCtx* ctx;
    DeviceGuard guard;
    MoveResult* res;
    cudaStream_t stream = nullptr;

    LaunchScope(Connection& conn, int device, MoveResult* r)
        : c(conn), ctx(conn.dev_ctx(device)), guard(ctx ? device : -1), res(r) {}
    int begin(uint64_t stream_in, bool write) {
        if (c.doorbell_quiesce(ctx) != 0) return -1;
        const uint64_t t_pick0 = now_ns();
        stream = ctx->pick(reinterpret_cast<cudaStream_t>(stream_in), write, c.streams_);
        c.stats_.ns_streams += now_ns() - t_pick0;
        c.stats_.calls++;
        if (res) {
            res->stream = stream;
            res->device = ctx->device;
        }
        return 0;
    }
    // -1 when the batch's launches failed (reported as `what` and the CUDA error); otherwise
    // sync() waits for them, and they are counted.
    int launched(cudaError_t e, const char* what, uint32_t launches, bool write, uint64_t bytes) {
        if (e != cudaSuccess) {
            c.fail(std::string(what) + cudaGetErrorString(e));
            return -1;
        }
        ctx->mark(stream);
        if (res) res->launched = true;
        c.stats_.kernel_launches += launches;
        (write ? c.stats_.bytes_written : c.stats_.bytes_read) += bytes;
        return 0;
    }
};

// A layered read's slot from arm_reader on (seq != 0).  Whichever way the call ends, the slot
// is marked live with an event recorded behind everything the call enqueued, so that the next
// reader of the slot waits for the flagged launch whenever it was enqueued: a later failure
// (the validate launch, a failed batch) must not hand the slot on while that launch may still
// store its smaller seq over the next reader's flags.  done() ends a call that succeeded.
struct Connection::ReaderHold {
    Connection& c;
    DevCtx* ctx;
    ScatterReader* r;
    cudaStream_t stream;
    uint64_t seq = 0;
    int done() {
        const uint64_t s = seq;
        seq = 0;
        return c.reader_launched(ctx, *r, s, stream);
    }
    ~ReaderHold() {
        if (seq) c.reader_launched(ctx, *r, seq, stream);  // the call failed: r is failed too
    }
};

// The parts of a gathered launch of n blocks whose local offsets OR to `align_or` (the part
// bases' alignment counts with theirs); descriptors and commit fields are the caller's.
kernels::GatherLaunch Connection::gather_launch(const GatherSpec& g, uint32_t n, uint64_t align_or,
                                                uint32_t* status, int max_ctas) {
    kernels::GatherLaunch G;
    G.n = n;
    G.part_base = g.part_base;
    G.nparts = g.nparts;
    // a row-sliced read's geometry counts bytes of the caller's view of a part (bf16 for fp8)
    G.part_bytes = uint32_t(g.rows.rows ? g.view_part_bytes() : g.pool_part_bytes());
    G.first_part = g.first_part;
    G.align_or = align_or;
    for (uint32_t s = 0; s < g.nparts; ++s) G.align_or |= g.part_base[s];
    G.status = status;
    G.max_ctas = max_ctas;
    G.stage_bytes = pipe_stage_;
    G.ring_bytes = pipe_ring_;
    G.rows = g.rows;  // the caller stages the piece table beside the descriptors
    G.records = g.records;
    G.part_scale = g.part_scale;
    G.rope = g.rope;
    return G;
}

// Bytes one block of a gathered call moves: its parts, or their rows when a read is row-sliced
// (of fp8 parts: the pool bytes of those rows, read_plan.h: fp8_rows_read_bytes; a row's slices
// are adjacent in the stored row, so they count as one run of slices * row_bytes).  A
// row-sliced write fills whole stored parts, so it counts them as the write without rows does.
static uint64_t gather_moved_bytes(const Connection::GatherSpec& g, bool write) {
    const kernels::PartRows& r = g.rows;
    const uint64_t width = uint64_t(r.slices) * r.row_bytes;
    const uint64_t part = !r.rows || write ? g.pool_part_bytes()
                          : g.fp8_elems
                              ? fp8_rows_read_bytes(r.rows, uint32_t(width), r.src_pitch, r.src_col)
                              : uint64_t(r.rows) * width;
    return uint64_t(g.nparts) * part;
}

// Layered writers' state (GatherWriter::state), allocated stream-ordered from a memory pool of
// the process that keeps up to 64 MB (about 5.6 M blocks' state) once freed.  The device's
// default pool hands freed memory back to the driver at every synchronise, and mapping it
// again on a writer's first call stalled that call by up to a few hundred milliseconds
// (bench/layerwise_gather.py).  The pool lives as long as the process, so a writer that
// outlives its connection still frees into it.
static cudaError_t writer_state_alloc(void** p, size_t bytes, int device, cudaStream_t s) {
    static std::mutex mu;
    static cudaMemPool_t pools[64] = {};
    if (device < 0 || device >= 64) return cudaErrorInvalidDevice;
    cudaMemPool_t pool;
    {
        std::lock_guard<std::mutex> lk(mu);
        if (!pools[device]) {
            cudaMemPoolProps props{};
            props.allocType = cudaMemAllocationTypePinned;
            props.location.type = cudaMemLocationTypeDevice;
            props.location.id = device;
            const cudaError_t e = cudaMemPoolCreate(&pools[device], &props);
            if (e != cudaSuccess) {
                pools[device] = nullptr;
                return e;
            }
            uint64_t keep = 64ull << 20;
            cudaMemPoolSetAttribute(pools[device], cudaMemPoolAttrReleaseThreshold, &keep);
        }
        pool = pools[device];
    }
    return cudaMallocFromPoolAsync(p, bytes, pool, s);
}

// Blocks per launch of a gathered call (staging.h: gather_max_blocks).  fp8 parts are counted
// in bf16 bytes: the fp8 kernels cut a part into chunks of at least kFp8Chunk elements (16 KB
// of bf16), or take it whole.
// A piece table (GatherSpec::rows.pieces) bounds it to the blocks whose tables fit
// kPieceRingBytes.
static size_t gather_batch_cap(const Connection::GatherSpec& g) {
    const size_t cap =
        gather_max_blocks(kMaxBatch, g.nparts, g.fp8_elems ? 2 * g.fp8_elems : g.part_bytes);
    const uint32_t k = g.rows.pieces;
    return k > 1 ? std::min(cap, kPieceRingBytes / (sizeof(uint64_t) * k)) : cap;
}

// The blocks of blocks[base, ...) that the next launch stages (staging.h: key_batch) within
// half the ring, so that a launch's placements never come round to each other.  *packed is
// kept only when it covers the call and the call fits in one launch.  n == 0: one key is
// longer than the ring.
static KeyBatch next_key_batch(const std::vector<KeyOffset>& blocks, size_t base,
                               size_t max_blocks, const PackedKeys** packed = nullptr) {
    const size_t left = blocks.size() - base;
    const PackedKeys* p = packed ? *packed : nullptr;
    if (p && base == 0 && p->n == left && left <= max_blocks &&
        p->nbytes + 16 * left <= kRingBytes / 2)
        return KeyBatch{left, p->nbytes};
    if (packed) *packed = nullptr;
    const KeyBatch b = key_batch(left, max_blocks, kRingBytes / 2,
                                 [&](size_t i) { return blocks[base + i].key.size(); });
    // a lone key must not reach its own offsets after a wrap: ring_alloc rounds each of the
    // four placements up to 64 bytes: at most 56 + 60 + 60 + 56 < 256 bytes beyond key_bytes + 16n
    return b.key_bytes + 16 * b.n + 256 > kRingBytes ? KeyBatch{} : b;
}

// Move n blocks between the caller's tensor and the pool.  local_off[i] * scale is the
// byte offset of block i from base_ptr.  With `gather` (base_ptr 0), block i is
// gather->nparts parts, part s at gather->part_base[s] + local_off[i] * scale, and
// block_size = nparts * part_bytes.
// `layered` (with `gather`): a call of a layered writer, whose blocks are exactly `blocks`.
int Connection::move_blocks(bool write, const uint64_t* local_off, uint64_t scale,
                            const RemoteBlock* blocks, size_t n, int block_size,
                            uint64_t base_ptr, int device, uint64_t stream_in, int fp8_elems,
                            MoveResult* res, const GatherSpec* gather, GatherWriter* layered) {
    NvtxRange nvtx(write ? "istore.write_blocks" : "istore.read_blocks");
    std::lock_guard<std::mutex> lk(mu_);
    if (n == 0) return 0;
    // Where the addresses to COMMIT go: the connection-wide list shipped by the next sync(),
    // or the caller's own list (async writes commit exactly their own blocks when THEIR
    // kernels have finished, reference: src/libinfinistore.cpp:362-395).  An address is
    // appended only after the launch that writes the block has succeeded; every error return
    // below leaves the sink exactly as the last successful launch left it.
    std::vector<uint64_t>& sink = (res && res->commits) ? *res->commits : pending_commit_;
    std::vector<uint64_t> batch_commits;
    // a layered writer's blocks are committed by the call that writes their last parts
    const bool commit_now = !layered || layered->parts_written + gather->nparts == layered->nparts;
    // bytes moved per block: a gathered call moves its parts, which are the whole block
    // unless the call is layered
    const uint64_t moved =
        gather ? gather_moved_bytes(*gather, write) : uint64_t(uint32_t(block_size));
    int kd = device;
    if (device < 0 && fp8_elems) {
        fail("the fp8 KV path needs a CUDA tensor");
        return -1;
    }
    if (device < 0) {
        // host tensor: memcpy when every target segment is host memory, else a kernel on
        // the connection's default device reads / writes the (pinned) host tensor
        bool all_host_segs = true;
        size_t live = 0;
        uint64_t max_off = 0;
        for (size_t i = 0; i < n; ++i) {
            if (write && is_fake_block(blocks[i])) continue;  // dedup: first writer wins
            const uint32_t seg = addr_seg(blocks[i].remote_addr);
            if (seg >= segs_.size() && refresh_pool_map() != 0) return -1;
            if (seg >= segs_.size()) {
                fail("block refers to unknown segment");
                return -1;
            }
            if (segs_[seg].kind != kSegHostShm) all_host_segs = false;
            max_off = std::max(max_off, local_off[i] * scale);
            ++live;
        }
        if (live == 0) return 0;
        if (all_host_segs) {
            for (size_t i = 0; i < n; ++i) {
                if (write && is_fake_block(blocks[i])) continue;
                auto m = mapping(addr_seg(blocks[i].remote_addr), -1);
                if (!m || !m->host_ptr) return -1;
                uint8_t* pool = m->host_ptr + addr_off(blocks[i].remote_addr);
                if (gather) {  // one memcpy per part, or per (row, slice) of a row-sliced call
                    const size_t pb = gather->pool_part_bytes();
                    const kernels::PartRows& R = gather->rows;
                    for (uint32_t s = 0; s < gather->nparts; ++s) {
                        uint8_t* local =
                            reinterpret_cast<uint8_t*>(gather->part_base[s] + local_off[i] * scale);
                        if (R.rows) {  // as the kernels do: runs of rows of one slice and piece
                            uint8_t* stored = pool + (gather->first_part + s) * pb;
                            const uint32_t pr = R.rows / R.pieces;
                            for (uint32_t q = 0; q < R.rows * R.slices; q += pr) {
                                const kernels::PairOffsets o = R.pair(q, pr);
                                uint8_t* l = local + o.dst;
                                if (R.pieces > 1)
                                    l += gather->piece_off[i * R.pieces + o.piece] * scale;
                                for (uint32_t r = 0; r < pr; ++r) {
                                    uint8_t* lr = l + size_t(r) * R.dst_pitch;
                                    uint8_t* p = stored + o.src + size_t(r) * R.src_pitch;
                                    if (write)
                                        std::memcpy(p, lr, R.row_bytes);
                                    else
                                        std::memcpy(lr, p, R.row_bytes);
                                }
                            }
                        } else if (write)
                            std::memcpy(pool + (gather->first_part + s) * pb, local, pb);
                        else
                            std::memcpy(local, pool + (gather->first_part + s) * pb, pb);
                    }
                } else {
                    uint8_t* local = reinterpret_cast<uint8_t*>(base_ptr + local_off[i] * scale);
                    if (write)
                        std::memcpy(pool, local, size_t(block_size));
                    else
                        std::memcpy(local, pool, size_t(block_size));
                }
                if (write && commit_now) sink.push_back(blocks[i].remote_addr);
                stats_.host_copies++;
            }
            (write ? stats_.bytes_written : stats_.bytes_read) += live * moved;
            return 0;
        }
        if (gather) {
            fail("gathered blocks of CPU tensors need a host-memory pool (--pool-backend host)");
            return -1;
        }
        if (!fabric::cuda_available()) {
            fail("a CUDA device is required to reach an HBM pool");
            return -1;
        }
        kd = cfg_.device >= 0 ? cfg_.device : std::max(default_device_, 0);
        auto mr = mrs_.find(base_ptr);
        const size_t span = mr != mrs_.end() ? mr->second : size_t(max_off) + size_t(block_size);
        if (ensure_host_registered(base_ptr, span, kd, mr == mrs_.end()) != 0) {
            fail("cannot pin the host tensor for the GPU data path");
            return -1;
        }
    }

    // --- kernel path on `kd`
    LaunchScope scope(*this, kd, res);
    DevCtx* ctx = scope.ctx;
    if (!ctx) return -1;
    if (cfg_.doorbell && write && n == 1 && device >= 0 && !fp8_elems && !res && !gather &&
        !is_fake_block(blocks[0])) {
        // latency mode: one block, handed to the persistent worker (no launch, no event)
        const RemoteBlock& rb = blocks[0];
        const uint32_t seg = addr_seg(rb.remote_addr);
        uint8_t* segbase =
            (seg < segs_.size() || refresh_pool_map() == 0) ? seg_dev_ptr(ctx, seg) : nullptr;
        const bool replicated = seg < ctx->seg_mc.size() && ctx->seg_mc[seg];
        if (segbase && !replicated && doorbell_ready(ctx, stream_in, size_t(block_size))) {
            KeyHash kh{0, 0};  // h1 == 0: not allocated through this connection, not indexed
            if (!segs_[0].index_slots || !pending_hash_.take(rb.remote_addr, &kh)) kh = KeyHash{0, 0};
            const uint64_t q[6] = {base_ptr + local_off[0] * scale,
                                   reinterpret_cast<uint64_t>(segbase) + addr_off(rb.remote_addr),
                                   kh.h1, kh.h2, rb.remote_addr,
                                   uint64_t(rb.gen) | (uint64_t(uint32_t(block_size)) << 32)};
            if (doorbell_post(ctx, kernels::kDoorbellWrite, q) != 0) return -1;
            sink.push_back(rb.remote_addr);
            stats_.calls++;
            stats_.bytes_written += uint64_t(block_size);
            return 0;
        }
    }
    if (scope.begin(stream_in, write) != 0) return -1;
    ReaderHold hold{*this, ctx, gather ? gather->reader : nullptr, scope.stream};
    if (layered && layered->event &&
        cudaStreamWaitEvent(scope.stream, static_cast<cudaEvent_t>(layered->event), 0) !=
            cudaSuccess) {
        fail(std::string("layered write: ") + cudaGetErrorString(cudaGetLastError()));
        return -1;
    }

    // the device index lives in segment 0
    kernels::IndexBucket* table = nullptr;
    uint64_t table_mask = 0;
    if (write && !segs_.empty() && segs_[0].index_slots) {
        if (uint8_t* p0 = seg_dev_ptr(ctx, 0)) {
            table = reinterpret_cast<kernels::IndexBucket*>(p0 + segs_[0].index_off);
            table_mask = kernels::index_bucket_mask(segs_[0].index_slots);
        }
    }

    const size_t max_batch = gather ? gather_batch_cap(*gather) : kMaxBatch;
    size_t i = 0;
    while (i < n) {
        const uint64_t t_build0 = now_ns();
        const size_t batch_cap = std::min(max_batch, n - i);
        const size_t at_desc = ctx->ring_alloc(batch_cap * sizeof(kernels::CopyDesc));
        auto* descs = reinterpret_cast<kernels::CopyDesc*>(ctx->ring_h + at_desc);
        size_t at_rec = 0;
        kernels::IndexEntry* recs = nullptr;
        if (table) {
            at_rec = ctx->ring_alloc(batch_cap * sizeof(kernels::IndexEntry));
            recs = reinterpret_cast<kernels::IndexEntry*>(ctx->ring_h + at_rec);
        }
        const uint32_t k = gather ? gather->rows.pieces : 1;  // piece table: one row per descriptor
        size_t at_piece = 0;
        uint64_t* pieces = nullptr;
        if (k > 1) {
            at_piece = ctx->ring_alloc(batch_cap * k * sizeof(uint64_t));
            pieces = reinterpret_cast<uint64_t*>(ctx->ring_h + at_piece);
        }
        uint32_t m = 0;
        const size_t batch0 = i;  // a layered writer's blocks: its state index of descs[0]
        batch_commits.clear();
        uint32_t n_mc = 0;  // blocks of this batch that live in the NVLS-replicated region
        bool can_publish = table != nullptr && (!layered || layered->indexed);
        bool all_remote = true;
        bool all_local = !ctx->seg_remote.empty() && !ctx->seg_remote[0];  // index table (segment 0)
        uint64_t align_or = 0;
        const size_t nseg = ctx->seg_ptr.size();
        uint8_t* const* seg_ptr = ctx->seg_ptr.data();
        for (; i < n && m < batch_cap; ++i) {
            const RemoteBlock& rb = blocks[i];
            if (write && is_fake_block(rb)) continue;
            const uint32_t seg = addr_seg(rb.remote_addr);
            uint8_t* segbase = seg < nseg ? seg_ptr[seg] : nullptr;
            if (!segbase) {
                segbase = seg_dev_ptr(ctx, seg);
                if (!segbase && !(seg < ctx->seg_mc.size() && ctx->seg_mc[seg])) return -1;
                seg_ptr = ctx->seg_ptr.data();
            }
            if (gather && seg < ctx->seg_mc.size() && ctx->seg_mc[seg]) {
                fail("gathered blocks cannot live in the replicated (NVLS) region");
                return -1;
            }
            if (write && seg < ctx->seg_mc.size() && ctx->seg_mc[seg]) {
                segbase = ctx->seg_mc[seg];  // replicated block: write through the multicast VA
                ++n_mc;
            } else if (!segbase) {
                fail("no local replica of the NVLS region on device " + std::to_string(kd));
                return -1;
            }
            const uint64_t pool = reinterpret_cast<uint64_t>(segbase) + addr_off(rb.remote_addr);
            const uint64_t local = base_ptr + local_off[i] * scale;
            all_remote = all_remote && ctx->seg_remote[seg];
            all_local = all_local && !ctx->seg_remote[seg];
            align_or |= local;
            descs[m].src = write ? local : pool;
            descs[m].dst = write ? pool : local;
            for (uint32_t t = 0; t < k && pieces; ++t) {
                pieces[size_t(m) * k + t] = gather->piece_off[i * k + t] * scale;
                align_or |= pieces[size_t(m) * k + t];
            }
            if (write) {
                if (recs) {
                    KeyHash kh;
                    if (layered) kh = layered->hashes[i];
                    if (layered || pending_hash_.take(rb.remote_addr, &kh))
                        recs[m] = kernels::IndexEntry{kh.h1, kh.h2, rb.remote_addr, rb.gen,
                                                      uint32_t(block_size)};
                    else
                        can_publish = false;  // not allocated through this connection
                }
                batch_commits.push_back(rb.remote_addr);
            }
            ++m;
        }
        if (m == 0) break;
        if (n_mc && n_mc != m) {
            fail("a write batch must not mix replicated and ordinary blocks");
            return -1;
        }
        kernels::CopyLaunch L;
        L.multicast = n_mc != 0;
        L.descs = reinterpret_cast<const kernels::CopyDesc*>(ctx->ring_d + at_desc);
        L.descs_host = descs;
        L.n = m;
        L.bytes = uint32_t(block_size);
        L.align_or = align_or;
        L.status = ctx->status_d;
        L.variant = local_auto_variant(copy_variant_, all_local && !L.multicast);
        L.stage_bytes = pipe_stage_;
        L.ring_bytes = pipe_ring_;
        L.max_ctas = max_ctas_ ? max_ctas_ : (all_remote ? 2 * kernels::sm_count() : 0);
        L.all_local = all_local && !L.multicast;
        if (L.multicast && fp8_elems) {
            fail("the fp8 path does not write to the replicated region");
            return -1;
        }
        if (can_publish) {
            L.recs = reinterpret_cast<const kernels::IndexEntry*>(ctx->ring_d + at_rec);
            L.table = table;
            L.table_mask = table_mask;
            bool shards_local = true;
            L.shards = index_shards(ctx, &shards_local);
            L.all_local = L.all_local && shards_local;
            all_local = all_local && shards_local;
            L.done = reinterpret_cast<uint32_t*>(ctx->zeros + ctx->zeros_alloc(size_t(m) * 12));
        }
        const uint64_t t_launch0 = now_ns();
        stats_.ns_build += t_launch0 - t_build0;
        cudaError_t e;
        if (gather) {
            kernels::GatherLaunch G = gather_launch(*gather, m, align_or, L.status, L.max_ctas);
            G.descs = L.descs;
            if (pieces) G.piece_off = reinterpret_cast<const uint64_t*>(ctx->ring_d + at_piece);
            G.write = write;
            G.recs = L.recs;
            G.table = L.table;
            G.table_mask = L.table_mask;
            G.done = L.done;
            G.all_local = L.all_local;
            G.shards = L.shards;
            if (layered && L.recs) {
                if (!layered->state) {  // zeroed behind the caller's pages, before any launch
                    const size_t bytes = layered->blocks.size() * 3 * sizeof(uint32_t);
                    void* p = nullptr;
                    cudaError_t ea = writer_state_alloc(&p, bytes, ctx->device, scope.stream);
                    if (ea == cudaSuccess) ea = cudaMemsetAsync(p, 0, bytes, scope.stream);
                    if (ea != cudaSuccess) {
                        if (p) cudaFreeAsync(p, scope.stream);
                        fail(std::string("layered write state: ") + cudaGetErrorString(ea));
                        return -1;
                    }
                    layered->state = static_cast<uint32_t*>(p);
                }
                G.layer_state = layered->state + 3 * batch0;
                G.layer_parts = layered->nparts;
                G.layer_claim = layered->calls == 0;
            }
            if (gather->reader && i >= n) {  // a layered read's flags ride on its last launch
                hold.seq = arm_reader(ctx, *gather->reader, G);
                if (!hold.seq) return -1;
            }
            // fp8 parts: the variant rule of the per-page fp8 path below
            e = fp8_elems ? kernels::launch_kv_gather_fp8(G, uint32_t(fp8_elems),
                                                          all_local ? kernels::kFp8LdSt
                                                                    : kernels::kFp8Auto,
                                                          scope.stream)
                          : kernels::launch_kv_gather(G, scope.stream);
        } else if (fp8_elems) {
            kernels::Fp8Launch F;
            F.descs = L.descs;
            F.n = m;
            F.elems = uint32_t(fp8_elems);
            F.recs = L.recs;
            F.table = L.table;
            F.table_mask = L.table_mask;
            F.shards = L.shards;
            F.done = L.done;
            F.status = L.status;
            F.max_ctas = L.max_ctas;
            F.all_local = all_local;
            F.aligned16 = (align_or & 15) == 0;
            // TMA-pipelined flavour over NVLink, per-thread flavour on local HBM.  Intentional:
            // the lookup-then-fp8 read (read_plan.h) uses all_remote ? 0 : 1 instead, and the
            // two differ for a pool that mixes local and remote segments.
            F.variant = all_local ? 1 : 0;
            e = write ? kernels::launch_kv_write_fp8(F, scope.stream)
                      : kernels::launch_kv_read_fp8(F, scope.stream);
        } else {
            e = kernels::launch_kv_copy(L, scope.stream);
        }
        stats_.ns_launch += now_ns() - t_launch0;
        if (scope.launched(e, "page mover launch failed: ", 1, write, uint64_t(m) * moved) != 0)
            return -1;
        if (commit_now) sink.insert(sink.end(), batch_commits.begin(), batch_commits.end());
    }
    if (layered) {  // the writer's next call runs after these launches
        cudaEvent_t ev = static_cast<cudaEvent_t>(layered->event);
        cudaError_t e = ev ? cudaSuccess : cudaEventCreateWithFlags(&ev, cudaEventDisableTiming);
        if (e == cudaSuccess) {
            layered->event = ev;
            e = cudaEventRecord(ev, scope.stream);
        }
        if (e == cudaSuccess && commit_now && layered->state) {
            e = cudaFreeAsync(layered->state, scope.stream);
            layered->state = nullptr;
        }
        if (e != cudaSuccess) {
            fail(std::string("layered write: ") + cudaGetErrorString(e));
            return -1;
        }
    }
    if (hold.seq) return hold.done();
    return 0;
}

// The slot flags are zeroed, and the zeroing has completed, before any reader is handed a
// slot: a consumer's wait runs on its own stream and must never see uninitialised words.
uint64_t Connection::arm_reader(DevCtx* ctx, const ScatterReader& r, kernels::GatherLaunch& G) {
    if (!ctx->group_flags) {
        const size_t bytes = size_t(kReaderSlots) * kernels::kGatherMaxParts * sizeof(uint32_t);
        void* p = nullptr;
        cudaError_t e = cudaMalloc(&p, bytes);
        if (e == cudaSuccess) e = cudaMemsetAsync(p, 0, bytes, ctx->stream);
        if (e == cudaSuccess) e = cudaStreamSynchronize(ctx->stream);
        if (e != cudaSuccess) {
            if (p) cudaFree(p);
            fail(std::string("layered read flags: ") + cudaGetErrorString(e));
            return 0;
        }
        ctx->group_flags = static_cast<uint32_t*>(p);
    }
    // cuStreamWaitValue32's GEQ compares cyclically, (int32_t)(*addr - seq) >= 0: a word
    // that lags seq by 2^31 or more would satisfy the wait at once, so seq stays below 2^31
    if (ctx->readers.last() >= uint64_t(INT32_MAX)) {
        fail("layered read: a connection serves 2^31 - 1 layered reads per device");
        return 0;
    }
    const uint64_t seq = ctx->readers.take([ctx](cudaEvent_t ev) {
        if (cudaEventQuery(ev) != cudaErrorNotReady) return;  // done, or failed: sync() reports it
        cudaEventSynchronize(ev);
        if (ctx->drains) ++*ctx->drains;
    });
    G.group_flags = ctx->group_flags + size_t(ctx->readers.slot_of(seq)) * kernels::kGatherMaxParts;
    G.group_counters =
        reinterpret_cast<uint32_t*>(ctx->zeros + ctx->zeros_alloc(size_t(r.groups) * 4));
    G.group_seq = uint32_t(seq);
    G.group_parts = r.group_parts;
    return seq;
}

// After the call's last launch: the slot is held until the reader's launches complete.
int Connection::reader_launched(DevCtx* ctx, ScatterReader& r, uint64_t seq, void* stream) {
    const uint32_t slot = ctx->readers.slot_of(seq);
    cudaEvent_t& ev = ctx->reader_ev[slot];
    cudaError_t e = ev ? cudaSuccess : cudaEventCreateWithFlags(&ev, cudaEventDisableTiming);
    if (e == cudaSuccess) e = cudaEventRecord(ev, static_cast<cudaStream_t>(stream));
    if (e != cudaSuccess) {
        fail(std::string("layered read: ") + cudaGetErrorString(e));
        return -1;
    }
    ctx->readers.launched(seq, ev);
    r.seq = seq;
    r.flags = ctx->group_flags + size_t(slot) * kernels::kGatherMaxParts;
    return 0;
}

int Connection::wait_layered(const ScatterReader& r, uint32_t group, uint64_t stream,
                             std::string* err) {
    std::lock_guard<std::mutex> lk(mu_);  // close() cannot free the flags under the wait
    const char* bad = r.failed               ? "the read failed, so its groups are never released"
                      : group >= r.groups    ? "the group is outside the read"
                      : r.session != session_ ? "the connection was closed after the read"
                                             : nullptr;
    if (bad) {
        if (err) *err = bad;
        return -1;
    }
    if (r.seq == 0) return 0;  // nothing was read
    DeviceGuard g(r.device);
    const cudaError_t e = kernels::stream_wait_geq(r.flags + group, uint32_t(r.seq),
                                                   reinterpret_cast<cudaStream_t>(stream));
    if (e != cudaSuccess) {
        (void)cudaGetLastError();
        if (err) *err = std::string("stream wait: ") + cudaGetErrorString(e);
        return -2;
    }
    return 0;
}

int Connection::w_rdma(const uint64_t* offsets, size_t noffsets, uint64_t scale, int block_size,
                       const RemoteBlock* blocks, size_t nblocks, uint64_t base_ptr, int device,
                       uint64_t stream, MoveResult* res) {
    if (noffsets != nblocks) {
        fail("w_rdma: offsets and remote blocks differ in length");
        return -1;
    }
    return move_blocks(true, offsets, scale, blocks, nblocks, block_size, base_ptr, device,
                       stream, 0, res);
}

// Every fp8 kernel moves bf16 in 16-byte vectors: pages that are not 16-byte aligned are
// refused before anything is enqueued.
static bool fp8_pages_aligned(uint64_t base_ptr, const uint64_t* offs, size_t n, uint64_t scale) {
    uint64_t align_or = base_ptr;
    for (size_t i = 0; i < n; ++i) align_or |= offs[i] * scale;
    return (align_or & 15) == 0;
}

int Connection::w_rdma_fp8(const uint64_t* offsets, size_t noffsets, uint64_t scale, int elems,
                           const RemoteBlock* blocks, size_t nblocks, uint64_t base_ptr,
                           int device, uint64_t stream) {
    if (noffsets != nblocks || elems <= 0 || elems % 128) {
        fail("w_rdma_fp8: page size must be a positive multiple of 128 elements");
        return -1;
    }
    if (!fp8_pages_aligned(base_ptr, offsets, noffsets, scale)) {
        fail("w_rdma_fp8: pages must start 16-byte aligned");
        return -1;
    }
    return move_blocks(true, offsets, scale, blocks, nblocks,
                       int(kernels::fp8_block_bytes(uint32_t(elems), 128)), base_ptr, device,
                       stream, elems);
}

int Connection::r_rdma_fp8(const std::vector<KeyOffset>& blocks, int elems, uint64_t base_ptr,
                           int device, uint64_t stream) {
    if (blocks.empty()) return 0;
    if (elems <= 0 || elems % 128 || device < 0) {
        fail("r_rdma_fp8: needs a CUDA tensor and pages of a multiple of 128 elements");
        return -1;
    }
    std::vector<uint64_t> offs(blocks.size());
    for (size_t i = 0; i < blocks.size(); ++i) offs[i] = blocks[i].offset;
    if (!fp8_pages_aligned(base_ptr, offs.data(), offs.size(), 1)) {
        fail("r_rdma_fp8: pages must start 16-byte aligned");
        return -1;
    }
    return read_blocks(kOpReadLookup, blocks, int(kernels::fp8_block_bytes(uint32_t(elems), 128)),
                       base_ptr, device, stream, elems);
}

int Connection::r_rdma(const std::vector<KeyOffset>& blocks, int block_size, uint64_t base_ptr,
                       int device, uint64_t stream, MoveResult* res, const PackedKeys* packed) {
    if (blocks.empty()) return 0;
    return read_blocks(kOpReadLookup, blocks, block_size, base_ptr, device, stream, 0, res, packed);
}

uint64_t Connection::GatherSpec::pool_part_bytes() const {
    if (!fp8_elems) return part_bytes;
    return records.latent ? kernels::fp8_records_bytes(1, fp8_elems, records)
                          : kernels::fp8_gather_bytes(1, fp8_elems);
}

// Bytes a stored block must hold to serve the read: every part asked for.
static uint32_t need_bytes_of(int block_size, const Connection::GatherSpec* g) {
    return g ? uint32_t(g->need_bytes()) : uint32_t(block_size);
}

// A read through the device index when this connection can use it from `device`; otherwise
// the server resolves the keys (`op`) and move_blocks copies.
int Connection::read_blocks(char op, const std::vector<KeyOffset>& blocks, int block_size,
                            uint64_t base_ptr, int device, uint64_t stream, int fp8_elems,
                            MoveResult* res, const PackedKeys* packed, const GatherSpec* gather) {
    if (device_lookup_ && server_hbm_ && device >= 0 && device_index_usable())
        return read_via_device_index(blocks, block_size, base_ptr, device, stream, fp8_elems, res,
                                     packed, gather);
    std::vector<RemoteBlock> rb;
    const int r = lookup_blocks(op, blocks, int(need_bytes_of(block_size, gather)), rb);
    if (r != 0) return r;
    std::vector<uint64_t> offs(blocks.size());
    for (size_t i = 0; i < blocks.size(); ++i) offs[i] = blocks[i].offset;
    return move_blocks(false, offs.data(), 1, rb.data(), rb.size(), block_size, base_ptr, device,
                       stream, fp8_elems, res, gather);
}

// Every check that a launch would fail, or that would let it run past a block, made before
// anything is enqueued.  The parts a block holds: a one-shot write's nparts, a layered
// writer's w->nparts, or for a read, the first_part + nparts that a stored block must hold.
const char* Connection::gather_refusal(const GatherSpec& g, const uint64_t* offs, size_t n,
                                       int device, bool write, const GatherWriter* w) const {
    if (!g.part_base || g.nparts < 1 || g.nparts > kernels::kGatherMaxParts)
        return "bad parts list: 1 to GATHER_MAX_PARTS parts";
    if (g.part_scale) {  // e4m3 caches: whole fp8 pages of e4m3 parts at one scale each
        if (!g.fp8_elems) return "e4m3 parts (scales) need fp8 parts";
        if (g.records.latent || g.rows.rows || g.rows.pieces != 1 || g.piece_off)
            return "e4m3 parts (scales) take whole parts: no records, row geometry or pieces";
        for (uint32_t s = 0; s < g.nparts; ++s)
            if (!(g.part_scale[s] >= FLT_MIN && g.part_scale[s] <= FLT_MAX))
                return "bad scale for e4m3 parts: every scale must be finite, positive and normal";
        if (w && w->device != -2 && !w->e4m3)
            return "e4m3 parts (scales) differ from the writer's first call";
    } else if (w && w->device != -2 && w->e4m3) {
        return "parts without scales differ from the writer's first call, whose parts were e4m3";
    }
    if (g.rope) {  // RoPE-shifted segments: bf16 whole parts of whole heads on the GPU
        if (g.fp8_elems || g.records.latent || g.part_scale)
            return "a RoPE shift takes bf16 parts: no fp8, records or scales";
        if (g.rows.rows || g.rows.pieces != 1 || g.piece_off)
            return "a RoPE shift takes whole parts: no row geometry or pieces";
        if (!g.rope->ok())
            return "bad RoPE geometry: head_elems, rot_offset and rot_dim multiples of 8 (neox: "
                   "rot_dim of 16), 1 to 128 pairs, rot_offset + rot_dim <= head_elems";
        if (!g.part_bytes || g.part_bytes % (2ull * g.rope->head_elems))
            return "bad part size for a RoPE shift: a whole number of bf16 heads";
        if (!g.rope->finite()) return "bad RoPE table: every cos and sin must be finite";
        if (device < 0) return "a RoPE shift needs CUDA tensors";
        uint64_t align_or = 0;
        for (uint32_t s = 0; s < g.nparts; ++s) align_or |= g.part_base[s];
        for (size_t i = 0; i < n; ++i) align_or |= offs[i];
        if (align_or & 15) return "a RoPE shift needs 16-byte aligned part bases and offsets";
        if (w && w->device != -2 && !w->rope)
            return "a RoPE shift differs from the writer's first call, which had none";
    } else if (w && w->device != -2 && w->rope) {
        return "parts without a RoPE shift differ from the writer's first call, which had one";
    }
    if (g.records.latent) {  // token records: whole parts of whole tokens, bf16 in the tensors
        if (!g.fp8_elems) return "fp8 records need fp8 parts (bf16 elements in the tensors)";
        if (!g.records.ok())
            return "bad fp8 records: latent a positive multiple of 128, rope a multiple of 8, and "
                   "a record (latent + 4 * latent / 128 + 2 * rope bytes) a multiple of 16 bytes";
        if (g.fp8_elems % g.records.token_elems() || g.fp8_elems > uint32_t(INT32_MAX))
            return "bad part size for fp8 records: a whole number of tokens of latent + rope "
                   "elements";
        if (g.rows.rows || (g.rows.pieces == 1 && g.piece_off))
            return "fp8 records take whole parts: no row geometry or pieces";
        // pieces of whole tokens (kv_fp8_records.cu), at the offsets of the piece table
        if (g.rows.pieces > 1 && !g.piece_off) return "bad pieces: fp8 records need a piece table";
        if (g.rows.pieces > 1 && (g.fp8_elems / g.records.token_elems()) % g.rows.pieces)
            return "bad pieces: the piece count must divide a part's tokens";
    } else if (g.fp8_elems ? g.fp8_elems % 512 || g.fp8_elems > uint32_t(INT32_MAX)
                           : !g.part_bytes) {
        return "bad part size: raw parts of 1 byte or more, fp8 parts of a multiple of 512 "
               "elements";
    }
    const uint64_t end = uint64_t(g.first_part) + g.nparts;
    const uint64_t block_parts = w ? w->nparts : write ? g.nparts : end;
    if (end > block_parts) return "the part range runs past the block";
    if (block_parts > uint64_t(INT32_MAX) / g.pool_part_bytes())
        return "bad parts list: a block holds at most 2^31 - 1 bytes";
    const kernels::PartRows& r = g.rows;
    if (r.pieces == 0 || (r.pieces > 1 && ((!r.rows && !g.records.latent) || !g.piece_off)))
        return "bad pieces: pieces >= 1, and pieces > 1 need row geometry and a piece table";
    if (r.pieces > 1 && r.rows % r.pieces)
        return "bad pieces: the piece count must divide the rows";
    if (uint64_t(r.pieces) * sizeof(uint64_t) > kPieceRingBytes)
        return "bad pieces: one block's piece table does not fit the staging ring";
    if (r.rows && !r.ok(g.view_part_bytes()))
        return "bad row geometry (rows >= 1, slices >= 1, src_col + slices * row_bytes <= "
               "src_pitch, part_bytes == rows * src_pitch; with slices > 1, disjoint local "
               "slices within 2^32 bytes; with pieces, per piece)";
    // the in-band commit publishes whole blocks: a write fills every byte of a stored part
    if (r.rows && write && !r.covers())
        return "bad row geometry for a write: the rows must fill the stored part (src_col == 0, "
               "slices * row_bytes == src_pitch)";
    if (r.rows && g.fp8_elems && (r.align_or() & 15))
        return "bad row geometry for fp8 parts: row_bytes, src_pitch, src_col, dst_pitch and "
               "dst_slice_pitch must be multiples of 16 bytes (8 bf16 elements)";
    if (g.reader) {
        if (!g.group_parts || g.nparts % g.group_parts)
            return "a layered read needs group_parts that divides the part count";
        if (device < 0) return "a layered read needs CUDA tensors";
        if (!server_hbm_) return "a layered read needs a pool in GPU memory";
        if (cfg_.doorbell) return "a layered read is not available on a doorbell connection";
    }
    if (g.fp8_elems) {  // the fp8 kernels move bf16 in 16-byte vectors
        if (device < 0) return "fp8 parts need CUDA tensors";
        uint64_t align_or = 0;
        for (uint32_t s = 0; s < g.nparts; ++s) align_or |= g.part_base[s];
        for (size_t i = 0; i < n; ++i) align_or |= offs[i];
        if (r.pieces > 1)
            for (size_t i = 0; i < n * r.pieces; ++i) align_or |= g.piece_off[i];
        if (align_or & 15)
            return "fp8 parts need 16-byte aligned part bases, offsets and piece offsets";
    }
    return nullptr;
}

int Connection::w_rdma_gather(const GatherSpec& g, const uint64_t* offsets, size_t noffsets,
                              const RemoteBlock* blocks, size_t nblocks, int device,
                              uint64_t stream) {
    const char* bad = noffsets != nblocks ? "offsets and remote blocks differ in length"
                                          : gather_refusal(g, offsets, noffsets, device, true);
    if (bad) {
        fail(std::string("w_rdma_gather: ") + bad);
        return -1;
    }
    return move_blocks(true, offsets, 1, blocks, nblocks, int(g.nparts * g.pool_part_bytes()), 0,
                       device, stream, int(g.fp8_elems), nullptr, &g);
}

int Connection::r_rdma_scatter(const GatherSpec& g, const std::vector<KeyOffset>& blocks,
                               int device, uint64_t stream) {
    ScatterReader* r = g.reader;
    if (r) {
        *r = ScatterReader{};
        r->device = device;
        {
            std::lock_guard<std::mutex> lk(mu_);
            r->session = session_;
        }
        r->group_parts = g.group_parts;
        r->groups = g.group_parts && g.nparts % g.group_parts == 0 ? g.nparts / g.group_parts : 0;
    }
    std::vector<uint64_t> offs;  // only the fp8 and RoPE alignment checks read them
    if (g.fp8_elems || g.rope) {
        offs.resize(blocks.size());
        for (size_t i = 0; i < blocks.size(); ++i) offs[i] = blocks[i].offset;
    }
    const char* bad = gather_refusal(g, offs.data(), offs.size(), device, false);
    if (bad) fail(std::string("r_rdma_scatter: ") + bad);
    const int rc = bad              ? -1
                   : blocks.empty() ? 0
                                    : read_blocks(kOpReadLookup, blocks,
                                                  int(g.nparts * g.pool_part_bytes()), 0, device,
                                                  stream, int(g.fp8_elems), nullptr, nullptr, &g);
    if (rc != 0 && r) r->failed = true;
    return rc;
}

// Never waits for the device: an abandoned writer's state is freed on the per-thread stream
// behind the writer's last launch.  Destroying a recorded event is safe while work is queued.
Connection::GatherWriter::~GatherWriter() {
    if (!event && !state) return;
    DeviceGuard g(device);
    if (state) {
        if (event) cudaStreamWaitEvent(cudaStreamPerThread, static_cast<cudaEvent_t>(event), 0);
        cudaFreeAsync(state, cudaStreamPerThread);
    }
    if (event) cudaEventDestroy(static_cast<cudaEvent_t>(event));
    (void)cudaGetLastError();
}

std::shared_ptr<Connection::GatherWriter> Connection::gather_writer(const RemoteBlock* blocks,
                                                                    const uint64_t* offsets,
                                                                    size_t n, uint32_t nparts,
                                                                    const uint64_t* piece_off,
                                                                    uint32_t pieces) {
    auto w = std::make_shared<GatherWriter>();
    w->nparts = nparts;
    w->pieces = piece_off ? pieces : 1;
    w->written.assign(nparts, 0);
    std::lock_guard<std::mutex> lk(mu_);
    w->session = session_;
    for (size_t i = 0; i < n; ++i) {
        if (is_fake_block(blocks[i])) continue;  // dedup: first writer wins
        KeyHash kh{0, 0};
        if (!pending_hash_.take(blocks[i].remote_addr, &kh)) w->indexed = false;
        w->blocks.push_back(blocks[i]);
        w->offsets.push_back(offsets[i]);
        w->hashes.push_back(kh);
        if (w->pieces > 1)
            w->piece_off.insert(w->piece_off.end(), piece_off + i * pieces,
                                piece_off + (i + 1) * pieces);
    }
    return w;
}

int Connection::write_layered(GatherWriter& w, const GatherSpec& g, uint64_t scale, int device,
                              uint64_t stream) {
    const uint64_t end = uint64_t(g.first_part) + g.nparts;
    const bool first = w.device == -2;
    uint64_t session;
    {
        std::lock_guard<std::mutex> lk(mu_);
        session = session_;
    }
    const char* bad = nullptr;
    if (w.session != session)
        bad = "the connection was closed after the writer was made";
    else if (w.failed || w.complete())
        bad = "the writer is complete or has failed";
    else if (!first && (device != w.device || scale != w.scale || g.fp8_elems != w.fp8_elems ||
                        g.records.latent != w.records.latent || g.records.rope != w.records.rope ||
                        g.pool_part_bytes() != w.part_bytes))
        bad = "device, element size, records or part size differ from the writer's first call";
    // every check before the writer changes: the first call's offsets are still in elements
    std::vector<uint64_t> scaled, scaled_pieces;
    if (!bad && first) {
        scaled = w.offsets;
        for (uint64_t& o : scaled) o *= scale;
        scaled_pieces = w.piece_off;
        for (uint64_t& o : scaled_pieces) o *= scale;
    }
    const std::vector<uint64_t>& offs = first ? scaled : w.offsets;
    GatherSpec gp = g;  // the writer's piece table goes with every call
    if (!bad && (g.rows.pieces != 1 || g.piece_off))
        bad = "a layered writer takes its pieces when it is made";
    gp.rows.pieces = w.pieces;
    gp.piece_off = w.pieces > 1 ? (first ? scaled_pieces : w.piece_off).data() : nullptr;
    if (!bad) bad = gather_refusal(gp, offs.data(), offs.size(), device, true, &w);
    for (uint64_t s = g.first_part; !bad && s < end; ++s)
        if (w.written[s]) bad = "the part range overlaps parts written before";
    if (bad) {
        fail(std::string("write_layered: ") + bad);
        return -1;
    }
    if (first) {
        w.device = device;
        w.scale = scale;
        w.fp8_elems = g.fp8_elems;
        w.records = g.records;
        w.e4m3 = g.part_scale != nullptr;
        w.rope = g.rope != nullptr;
        w.part_bytes = uint32_t(g.pool_part_bytes());
        w.offsets.swap(scaled);
        w.piece_off.swap(scaled_pieces);
        if (w.pieces > 1) gp.piece_off = w.piece_off.data();
    }
    const int r = move_blocks(true, w.offsets.data(), 1, w.blocks.data(), w.blocks.size(),
                              int(w.nparts * w.part_bytes), 0, device, stream, int(g.fp8_elems),
                              nullptr, &gp, &w);
    if (r != 0) {
        w.failed = true;
        return r;
    }
    for (uint64_t s = g.first_part; s < end; ++s) w.written[s] = 1;
    w.parts_written += g.nparts;
    ++w.calls;
    return 0;
}

int Connection::rw_local(char op, const std::vector<KeyOffset>& blocks, int block_size,
                         uint64_t base_ptr, int device, uint64_t stream) {
    if (blocks.empty()) return 0;
    if (op != kOpLocalRead && op != kOpLocalWrite) return -1;
    if (op == kOpLocalRead) return read_blocks(op, blocks, block_size, base_ptr, device, stream);
    std::vector<RemoteBlock> rb;
    const int r = lookup_blocks(op, blocks, block_size, rb);
    if (r != 0) return r;
    if (server_hbm_) {
        std::lock_guard<std::mutex> lk(mu_);
        for (size_t i = 0; i < blocks.size(); ++i) {
            if (is_fake_block(rb[i])) continue;
            pending_hash_.put(rb[i].remote_addr,
                              hash_key(reinterpret_cast<const uint8_t*>(blocks[i].key.data()),
                                       blocks[i].key.size()));
        }
    }
    std::vector<uint64_t> offs(blocks.size());
    for (size_t i = 0; i < blocks.size(); ++i) offs[i] = blocks[i].offset;
    return move_blocks(true, offs.data(), 1, rb.data(), rb.size(), block_size, base_ptr, device,
                       stream);
}

int Connection::read_via_device_index(const std::vector<KeyOffset>& blocks, int block_size,
                                      uint64_t base_ptr, int device, uint64_t stream_in,
                                      int fp8_elems, MoveResult* res, const PackedKeys* packed,
                                      const GatherSpec* gather) {
    NvtxRange nvtx("istore.read_via_device_index");
    std::lock_guard<std::mutex> lk(mu_);
    LaunchScope scope(*this, device, res);
    DevCtx* ctx = scope.ctx;
    if (!ctx) return -1;
    auto m0 = mapping(0, device);
    if (!m0 || !m0->dev_ptr || !segs_[0].index_slots) {
        fail("the server exposes no device index");
        return -1;
    }
    if (cfg_.doorbell && blocks.size() == 1 && !fp8_elems && !res && !gather &&
        doorbell_ready(ctx, stream_in, size_t(block_size))) {
        // latency mode: the key is hashed here, the worker probes, copies and re-checks
        const KeyHash kh = hash_key(reinterpret_cast<const uint8_t*>(blocks[0].key.data()),
                                    blocks[0].key.size());
        const uint64_t q[6] = {base_ptr + blocks[0].offset, 0, kh.h1, kh.h2, 0,
                               uint64_t(uint32_t(block_size)) << 32};
        if (doorbell_post(ctx, kernels::kDoorbellRead, q) != 0) return -1;
        stats_.calls++;
        stats_.bytes_read += uint64_t(block_size);
        return 0;
    }
    if (scope.begin(stream_in, false) != 0) return -1;
    const size_t max_batch = gather ? gather_batch_cap(*gather) : kMaxBatch;
    const bool layered = gather && gather->reader;
    ReaderHold hold{*this, ctx, layered ? gather->reader : nullptr, scope.stream};
    KeyBatch b;
    for (size_t base = 0; base < blocks.size(); base += b.n) {
        const uint64_t t_build0 = now_ns();
        b = next_key_batch(blocks, base, max_batch, &packed);
        if (!b.n) {
            fail("read: a key does not fit the staging ring");
            return -1;
        }
        const size_t n = b.n;
        kernels::ReadFusedLaunch R;
        set_index(ctx, R);
        DeviceReadIn in{.n = n, .block_bytes = uint32_t(block_size),
                        .fp8_elems = uint32_t(fp8_elems), .gather = gather != nullptr,
                        .copy_variant = copy_variant_, .all_local = true, .all_remote = true,
                        .max_ctas = max_ctas_, .sm_count = kernels::sm_count(),
                        .layered = layered, .rows = gather && gather->rows.rows};
        // over every known segment, not only the ones this batch touches: intentional
        for (uint32_t s = 0; s < R.nsegs; ++s) {
            in.all_remote = in.all_remote && ctx->seg_remote[s];
            in.all_local = in.all_local && !ctx->seg_remote[s];
        }
        uint64_t align_or = base_ptr;
        for (size_t i = 0; i < n; ++i) align_or |= blocks[base + i].offset;
        const uint32_t k = gather ? gather->rows.pieces : 1;  // piece table, beside the keys
        const uint64_t* pieces_d = nullptr;
        if (k > 1) {
            const size_t at = ctx->ring_alloc(n * k * sizeof(uint64_t));
            auto* pieces = reinterpret_cast<uint64_t*>(ctx->ring_h + at);
            for (size_t t = 0; t < n * k; ++t) {
                pieces[t] = gather->piece_off[base * k + t];
                align_or |= pieces[t];
            }
            pieces_d = reinterpret_cast<const uint64_t*>(ctx->ring_d + at);
        }
        // the fused kernels' support checks see the batch as it would be launched
        R.n = uint32_t(n);
        R.align_or = align_or;
        R.max_ctas = device_read_grid_cap(max_ctas_, in.all_remote, fp8_elems != 0, in.sm_count);
        kernels::GatherLaunch G;
        if (gather) G = gather_launch(*gather, uint32_t(n), align_or, ctx->status_d, R.max_ctas);
        G.piece_off = pieces_d;
        in.fp8_fused_ok = fp8_elems && kernels::fp8_read_fused_supported(R, uint32_t(fp8_elems));
        in.scatter_fused_ok = gather && kernels::scatter_read_fused_supported(R, G);
        const DeviceReadPlan plan = plan_device_read(in);
        uint64_t t_launch0 = now_ns();
        cudaError_t e = cudaSuccess;
        if (plan.fused()) {
            // one kernel: hash + probe + move
            const StagedKeys keys = ctx->stage_keys(blocks, base, b, packed);
            R.key_bytes = keys.bytes;
            R.key_off = keys.off;
            R.key_len = keys.len;
            R.dst_off = keys.dst;
            R.dst_base = base_ptr;
            R.bytes = uint32_t(block_size);
            R.status = ctx->status_d;
            // always: a purge (or an eviction) may free a block while a device-path read is
            // copying it; the post-copy tag check turns that into a reported miss
            R.validate = true;
            R.variant = plan.variant;
            R.stage_bytes = pipe_stage_;
            R.ring_bytes = pipe_ring_;
            t_launch0 = now_ns();
            e = plan.path == ReadPath::kFusedScatter
                    ? kernels::launch_kv_pipe_scatter_read(R, G, scope.stream)
                : plan.path == ReadPath::kFusedFp8
                    ? kernels::launch_kv_fp8_read_fused(R, uint32_t(fp8_elems), scope.stream)
                    : kernels::launch_kv_read_fused(R, scope.stream);
        } else {
            // optimistic read: the entries are re-checked after the copy (purge / eviction)
            kernels::LookupLaunch Q;
            const kernels::CopyDesc* descs =
                resolve_descs(ctx, blocks, base, b, packed, need_bytes_of(block_size, gather),
                              base_ptr, nullptr, scope.stream, &Q);
            if (!descs) {
                fail("device-index read: cannot resolve the blocks");
                return -1;
            }
            if (layered && base + n == blocks.size()) {  // the flags ride on the last launch
                hold.seq = arm_reader(ctx, *gather->reader, G);
                if (!hold.seq) return -1;
            }
            if (plan.path == ReadPath::kLookupGather) {
                G.descs = descs;  // {pool address or 0, local byte offset} (dst_base 0)
                e = kernels::launch_kv_gather(G, scope.stream);
            } else if (plan.path == ReadPath::kLookupGatherFp8) {
                G.descs = descs;
                e = kernels::launch_kv_gather_fp8(G, uint32_t(fp8_elems), plan.variant,
                                                  scope.stream);
            } else if (plan.path == ReadPath::kLookupFp8) {
                kernels::Fp8Launch F;
                F.descs = descs;
                F.n = uint32_t(n);
                F.elems = uint32_t(fp8_elems);
                F.status = ctx->status_d;
                F.max_ctas = plan.grid_cap;
                F.aligned16 = (align_or & 15) == 0;
                F.variant = plan.variant;
                e = kernels::launch_kv_read_fp8(F, scope.stream);
            } else {
                kernels::CopyLaunch L;
                L.descs = descs;
                L.n = uint32_t(n);
                L.bytes = uint32_t(block_size);
                L.align_or = align_or;
                L.status = ctx->status_d;
                L.variant = plan.variant;
                L.stage_bytes = pipe_stage_;
                L.ring_bytes = pipe_ring_;
                L.max_ctas = plan.grid_cap;
                e = kernels::launch_kv_copy(L, scope.stream);
            }
            if (e == cudaSuccess) {
                // the server evicts: the entries must still be the ones the lookup resolved
                kernels::ValidateLaunch V;
                V.found_at = Q.found_at;
                V.n = uint32_t(n);
                V.table = Q.table;
                V.shards = Q.shards;
                V.status = ctx->status_d;
                e = kernels::launch_index_validate(V, scope.stream);
            }
        }
        stats_.ns_build += t_launch0 - t_build0;
        stats_.ns_launch += now_ns() - t_launch0;
        // lookup + copy + validate: resolve_descs counted the lookup
        const uint64_t moved = gather && gather->rows.rows ? gather_moved_bytes(*gather, false)
                                                           : uint64_t(block_size);
        if (scope.launched(e, "device-index read failed to launch: ", plan.fused() ? 1 : 2, false,
                           uint64_t(n) * moved) != 0)
            return -1;
    }
    if (hold.seq) return hold.done();
    return 0;
}

// Device-addressable copy descriptors {mapped pool address (0 = miss), dst_base + offset} for
// blocks[base, base + b.n): resolved on the GPU by the lookup kernel (rb == nullptr, the
// descriptors land in device scratch) or taken from a server lookup (rb, pinned ring).  With
// `checked`, the lookup also records where it found every hit (found_at), and *checked is
// left holding the launch, for a validate launch after the copy.
const kernels::CopyDesc* Connection::resolve_descs(DevCtx* ctx, const std::vector<KeyOffset>& blocks,
                                                   size_t base, const KeyBatch& b,
                                                   const PackedKeys* packed, uint32_t need_bytes,
                                                   uint64_t dst_base,
                                                   const std::vector<RemoteBlock>* rb,
                                                   void* stream, kernels::LookupLaunch* checked) {
    const size_t n = b.n;
    if (n == 0) return nullptr;
    if (rb) {
        const size_t at_desc = ctx->ring_alloc(n * sizeof(kernels::CopyDesc));
        auto* descs = reinterpret_cast<kernels::CopyDesc*>(ctx->ring_h + at_desc);
        for (size_t i = 0; i < n; ++i) {
            const RemoteBlock& rbi = (*rb)[base + i];
            uint8_t* segbase = seg_dev_ptr(ctx, addr_seg(rbi.remote_addr));
            if (!segbase) return nullptr;
            descs[i].src = reinterpret_cast<uint64_t>(segbase) + addr_off(rbi.remote_addr);
            descs[i].dst = dst_base + blocks[base + i].offset;
        }
        return reinterpret_cast<const kernels::CopyDesc*>(ctx->ring_d + at_desc);
    }
    kernels::LookupLaunch own;
    kernels::LookupLaunch& Q = checked ? *checked : own;
    if (!set_index(ctx, Q)) return nullptr;
    const StagedKeys keys = ctx->stage_keys(blocks, base, b, packed);
    Q.key_bytes = keys.bytes;
    Q.key_off = keys.off;
    Q.key_len = keys.len;
    Q.n = uint32_t(n);
    Q.out_descs = reinterpret_cast<kernels::CopyDesc*>(
        ctx->scratch + ctx->scratch_alloc(n * sizeof(kernels::CopyDesc)));
    Q.dst_off = keys.dst;
    Q.dst_base = dst_base;
    Q.need_bytes = need_bytes;
    Q.status = ctx->status_d;
    if (checked)
        Q.found_at = reinterpret_cast<kernels::LookupLaunch::FoundAt*>(
            ctx->scratch + ctx->scratch_alloc(n * sizeof(kernels::LookupLaunch::FoundAt)));
    if (kernels::launch_index_lookup(Q, static_cast<cudaStream_t>(stream)) != cudaSuccess)
        return nullptr;
    stats_.kernel_launches++;
    return Q.out_descs;
}

// The reads that resolve their blocks to descriptors first and launch their own kernels on
// them: launch(scope, descs, base, n) runs once per batch and returns 0 or -1.
template <typename Launch>
int Connection::read_resolved(const std::vector<KeyOffset>& blocks, int block_size, int device,
                              uint64_t stream_in, uint64_t dst_base, const char* what,
                              Launch&& launch) {
    const bool via_index = device_lookup_ && device_index_usable();
    std::vector<RemoteBlock> rb;
    if (!via_index) {
        const int r = lookup_blocks(kOpReadLookup, blocks, block_size, rb);
        if (r != 0) return r;
    }
    std::lock_guard<std::mutex> lk(mu_);
    LaunchScope scope(*this, device, nullptr);
    if (!scope.ctx || scope.begin(stream_in, false) != 0) return -1;
    KeyBatch b;
    for (size_t base = 0; base < blocks.size(); base += b.n) {
        b = next_key_batch(blocks, base, kMaxBatch);
        const kernels::CopyDesc* descs = resolve_descs(scope.ctx, blocks, base, b, nullptr,
                                                       uint32_t(block_size), dst_base,
                                                       via_index ? nullptr : &rb, scope.stream);
        if (!descs) {
            fail(std::string(what) + ": cannot resolve the blocks");
            return -1;
        }
        if (launch(scope, descs, base, b.n) != 0) return -1;
    }
    return 0;
}

// The same pages into several destination tensors (TP ranks / beams sharing a prefix): every
// pool block crosses NVLink once and is fanned out inside a thread-block cluster
// (kernels/kv_pipe.cu: cp.async.bulk ... .multicast::cluster).  bases[r] is the base pointer
// of destination r; every destination uses the same page offsets.
int Connection::r_rdma_multi(const std::vector<KeyOffset>& blocks, int block_size,
                             const std::vector<uint64_t>& bases, int device, uint64_t stream_in) {
    if (blocks.empty() || bases.empty()) return 0;
    if (device < 0 || !server_hbm_) {
        fail("read_cache_multi needs CUDA destinations and an HBM pool");
        return -1;
    }
    if (bases.size() == 1) return r_rdma(blocks, block_size, bases[0], device, stream_in);
    NvtxRange nvtx("istore.read_multi");
    uint64_t align_or = 0;
    for (uint64_t b : bases) align_or |= b;
    auto launch = [&](LaunchScope& scope, const kernels::CopyDesc* descs_d, size_t base,
                      size_t n) {
        for (size_t i = 0; i < n; ++i) align_or |= blocks[base + i].offset;
        // Local pool: thread-block clusters (multicast bulk load into 2 or 4 CTAs, one
        // destination each; an odd last destination shares a 2-cluster with its predecessor,
        // which is rewritten with the same bytes).  Pool behind NVLink: one load, K stores
        // per CTA (the fan-out flavour of the TMA pipeline) - the fabric still carries every
        // page once.
        bool src_local = true;
        for (size_t sgi = 0; sgi < scope.ctx->seg_remote.size(); ++sgi)
            if (scope.ctx->seg_ptr[sgi] && scope.ctx->seg_remote[sgi]) src_local = false;
        cudaError_t e = cudaSuccess;
        uint32_t launches = 0;
        size_t r = 0;
        while (e == cudaSuccess && r < bases.size()) {
            const size_t left = bases.size() - r;
            if (src_local) {
                kernels::McastLaunch M;
                M.descs = descs_d;
                M.n = uint32_t(n);
                M.bytes = uint32_t(block_size);
                M.align_or = align_or;
                M.src_local = true;
                M.status = r == 0 ? scope.ctx->status_d : nullptr;  // count a miss once
                const size_t first = left >= 2 ? r : r - 1;
                M.ndst = left >= 4 ? 4 : 2;
                for (int j = 0; j < M.ndst; ++j)
                    M.delta[j] = int64_t(bases[first + size_t(j)]) - int64_t(bases[0]);
                e = kernels::launch_kv_pipe_mcast(M, scope.stream);
                r = first + size_t(M.ndst);
            } else {
                kernels::CopyLaunch L;
                L.descs = descs_d;
                L.n = uint32_t(n);
                L.bytes = uint32_t(block_size);
                L.align_or = align_or;
                L.status = r == 0 ? scope.ctx->status_d : nullptr;
                L.variant = kernels::kCopyTma;
                L.max_ctas = max_ctas_;
                L.fan_n = int(std::min<size_t>(left, 4));
                for (int j = 0; j < L.fan_n; ++j)
                    L.fan_delta[j] = int64_t(bases[r + size_t(j)]) - int64_t(bases[0]);
                e = kernels::launch_kv_pipe_copy(L, scope.stream);
                r += size_t(L.fan_n);
            }
            ++launches;
        }
        return scope.launched(e, "multi-destination read failed to launch: ", launches, false,
                              uint64_t(n) * uint64_t(block_size) * bases.size());
    };
    return read_resolved(blocks, block_size, device, stream_in, bases[0],
                         "multi-destination read", launch);
}

// read_cache fused with the layout swizzle of the attention consumer: pages are stored
// token-major ([tok][head][dim], as the prefill wrote them) and land head-major in a paged KV
// cache [page][head][tok][dim]; blocks[i].offset is the destination PAGE INDEX.  The
// transposition is done by the TMA unit (4-D tensor-map store, kernels/kv_pipe.cu).
int Connection::r_rdma_hnd(const std::vector<KeyOffset>& blocks, int tokens, int heads, int dim,
                           int elem_size, uint64_t base_ptr, uint64_t num_pages, int device,
                           uint64_t stream_in) {
    if (blocks.empty()) return 0;
    if (device < 0 || !server_hbm_) {
        fail("read_cache_hnd needs a CUDA destination and an HBM pool");
        return -1;
    }
    const int block_size = tokens * heads * dim * elem_size;
    for (const KeyOffset& b : blocks)
        if (b.offset >= num_pages) {
            fail("read_cache_hnd: page index beyond the destination tensor");
            return -1;
        }
    NvtxRange nvtx("istore.read_hnd");
    // dst_base 0: the descriptor's dst field carries the page index
    return read_resolved(blocks, block_size, device, stream_in, 0, "read_cache_hnd",
                         [&](LaunchScope& scope, const kernels::CopyDesc* descs, size_t, size_t n) {
        kernels::HndLaunch H;
        H.descs = descs;
        H.n = uint32_t(n);
        H.tokens = uint32_t(tokens);
        H.heads = uint32_t(heads);
        H.dim = uint32_t(dim);
        H.elem_size = uint32_t(elem_size);
        H.dst_base = base_ptr;
        H.num_pages = uint32_t(num_pages);
        H.status = scope.ctx->status_d;
        H.max_ctas = max_ctas_;
        return scope.launched(kernels::launch_kv_pipe_hnd(H, scope.stream),
                              "layout-swizzling read failed to launch: ", 1, false,
                              uint64_t(n) * uint64_t(block_size));
    });
}

int Connection::match_via_device_index(const std::vector<std::string_view>& keys, bool exist_only) {
    std::lock_guard<std::mutex> lk(mu_);
    const int device = cfg_.device >= 0 ? cfg_.device : std::max(default_device_, 0);
    DevCtx* ctx = dev_ctx(device);
    if (!ctx) return -3;
    DeviceGuard g(device);
    kernels::LookupLaunch Q;
    if (!set_index(ctx, Q, false)) return -3;
    std::vector<KeyOffset> blocks(keys.size());
    for (size_t i = 0; i < keys.size(); ++i) blocks[i] = KeyOffset{keys[i], 0};
    const KeyBatch b = next_key_batch(blocks, 0, blocks.size());
    if (b.n < blocks.size()) return -3;  // more than one launch stages: use the control plane
    if (doorbell_quiesce(ctx) != 0) return -3;
    const StagedKeys staged = ctx->stage_keys(blocks, 0, b, nullptr);
    Q.key_bytes = staged.bytes;
    Q.key_off = staged.off;
    Q.key_len = staged.len;
    Q.n = uint32_t(b.n);
    const size_t words = (b.n + 31) / 32;
    Q.present = reinterpret_cast<uint32_t*>(ctx->scratch + ctx->scratch_alloc(words * 4));
    Q.ticket = reinterpret_cast<uint32_t*>(ctx->zeros + ctx->zeros_alloc(4));
    Q.status = ctx->status_d;
    Q.want_match = true;
    Q.accept_claimed = !exist_only;  // C3: reserved-but-uncommitted keys count for match only
    // The launch is ordered after this connection's writes on the same stream, so keys
    // written just before (even without sync) are visible, as in the reference.
    cudaStream_t stream = ctx->pick(nullptr, false, std::max(streams_, 1));
    const cudaError_t e = kernels::launch_index_lookup(Q, stream);
    if (e != cudaSuccess) {
        fail(std::string("match kernel failed to launch: ") + cudaGetErrorString(e));
        return -3;
    }
    stats_.kernel_launches++;
    // external streams may hold this connection's writes: wait for them too
    ctx->mark(stream);
    ctx->wait_all();
    return int32_t(ctx->status_h[kernels::kStatMatch]);
}

int Connection::drain_devices(bool* device_error) {
    std::lock_guard<std::mutex> lk(mu_);
    int rc = 0;
    if (device_error) *device_error = false;
    struct AtExit {
        Connection* c;
        ~AtExit() { c->release_temporary_host_regs(); }
    } at_exit{this};
    for (auto& kv : devs_) {
        DevCtx& ctx = *kv.second;
        if (!ctx.dirty) continue;
        if (ctx.db && ctx.db->posted > ctx.db->collected) {
            DeviceGuard g(ctx.device);
            if (doorbell_wait(&ctx) != 0) {
                rc = -1;
                if (device_error) *device_error = true;
            }
        }
        ctx.wait_all();
        if (ctx.db) {  // no kernel is adding to the status words now
            ctx.status_h[kernels::kStatMiss] += ctx.db->misses;
            ctx.status_h[kernels::kStatStale] += ctx.db->stale;
            ctx.status_h[kernels::kStatPublishFail] += ctx.db->publish_failures;
            ctx.db->misses = ctx.db->stale = ctx.db->publish_failures = 0;
        }
        const cudaError_t e = cudaGetLastError();
        if (e != cudaSuccess) {
            fail(std::string("device error during transfer: ") + cudaGetErrorString(e));
            rc = -1;
            if (device_error) *device_error = true;
        }
        if (ctx.status_h[kernels::kStatMiss]) {
            fail("read: " + std::to_string(ctx.status_h[kernels::kStatMiss]) +
                 " key(s) not found in the device index" +
                 (ctx.status_h[kernels::kStatStale]
                      ? " (" + std::to_string(ctx.status_h[kernels::kStatStale]) +
                            " evicted while being read)"
                      : std::string()));
            ctx.status_h[kernels::kStatMiss] = 0;
            ctx.status_h[kernels::kStatStale] = 0;
            rc = -kKeyNotFound;
        }
        if (ctx.status_h[kernels::kStatPublishFail]) {
            LOG_WARN("device index is full: %u block(s) are only reachable through the server; "
                     "reads fall back to server lookups",
                     ctx.status_h[kernels::kStatPublishFail]);
            publish_failures_ += ctx.status_h[kernels::kStatPublishFail];
            index_incomplete_.store(true, std::memory_order_relaxed);
            ctx.status_h[kernels::kStatPublishFail] = 0;
        }
    }
    return rc;
}

}  // namespace istore
