// Data plane of the client: pool mappings, page-mover launches, device-index reads.
#include "client.h"

#include <cuda_runtime_api.h>

#include <algorithm>
#include <atomic>
#include <cerrno>
#include <chrono>
#include <cstring>

#include "../core/log.h"
#include "../core/trace.h"
#include "../kernels/kernels.h"
#include "../wire/messages.h"
#include "client_dev.h"

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

// Move n blocks between the caller's tensor and the pool.  local_off[i] * scale is the
// byte offset of block i from base_ptr.
int Connection::move_blocks(bool write, const uint64_t* local_off, uint64_t scale,
                            const RemoteBlock* blocks, size_t n, int block_size,
                            uint64_t base_ptr, int device, uint64_t stream_in, int fp8_elems,
                            MoveResult* res) {
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
                uint8_t* local = reinterpret_cast<uint8_t*>(base_ptr + local_off[i] * scale);
                if (write)
                    std::memcpy(pool, local, size_t(block_size));
                else
                    std::memcpy(local, pool, size_t(block_size));
                if (write) sink.push_back(blocks[i].remote_addr);
                stats_.host_copies++;
            }
            (write ? stats_.bytes_written : stats_.bytes_read) += live * uint64_t(block_size);
            return 0;
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
    DevCtx* ctx = dev_ctx(kd);
    if (!ctx) return -1;
    DeviceGuard g(kd);
    if (cfg_.doorbell && write && n == 1 && device >= 0 && !fp8_elems && !res &&
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
    if (doorbell_quiesce(ctx) != 0) return -1;
    const uint64_t t_pick0 = now_ns();
    cudaStream_t stream = ctx->pick(reinterpret_cast<cudaStream_t>(stream_in), write, streams_);
    stats_.ns_streams += now_ns() - t_pick0;
    stats_.calls++;
    if (res) {
        res->stream = stream;
        res->device = kd;
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

    size_t i = 0;
    while (i < n) {
        const uint64_t t_build0 = now_ns();
        const size_t batch_cap = std::min(kMaxBatch, n - i);
        const size_t at_desc = ctx->ring_alloc(batch_cap * sizeof(kernels::CopyDesc));
        auto* descs = reinterpret_cast<kernels::CopyDesc*>(ctx->ring_h + at_desc);
        size_t at_rec = 0;
        kernels::IndexEntry* recs = nullptr;
        if (table) {
            at_rec = ctx->ring_alloc(batch_cap * sizeof(kernels::IndexEntry));
            recs = reinterpret_cast<kernels::IndexEntry*>(ctx->ring_h + at_rec);
        }
        uint32_t m = 0;
        batch_commits.clear();
        uint32_t n_mc = 0;  // blocks of this batch that live in the NVLS-replicated region
        bool can_publish = table != nullptr;
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
            if (write) {
                if (recs) {
                    KeyHash kh;
                    if (pending_hash_.take(rb.remote_addr, &kh))
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
        L.variant = copy_variant_;
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
        if (fp8_elems) {
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
            // TMA-pipelined flavour over NVLink, per-thread flavour on local HBM
            F.variant = all_local ? 1 : 0;
            e = write ? kernels::launch_kv_write_fp8(F, stream) : kernels::launch_kv_read_fp8(F, stream);
        } else {
            e = kernels::launch_kv_copy(L, stream);
        }
        stats_.ns_launch += now_ns() - t_launch0;
        if (e != cudaSuccess) {
            fail(std::string("page mover launch failed: ") + cudaGetErrorString(e));
            return -1;
        }
        ctx->mark(stream);
        if (res) res->launched = true;
        sink.insert(sink.end(), batch_commits.begin(), batch_commits.end());
        stats_.kernel_launches++;
        (write ? stats_.bytes_written : stats_.bytes_read) += uint64_t(m) * uint64_t(block_size);
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

int Connection::w_rdma_fp8(const uint64_t* offsets, size_t noffsets, uint64_t scale, int elems,
                           const RemoteBlock* blocks, size_t nblocks, uint64_t base_ptr,
                           int device, uint64_t stream) {
    if (noffsets != nblocks || elems <= 0 || elems % 128) {
        fail("w_rdma_fp8: page size must be a positive multiple of 128 elements");
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
    const int bytes = int(kernels::fp8_block_bytes(uint32_t(elems), 128));
    if (device_lookup_ && server_hbm_ && device_index_usable())
        return read_via_device_index(blocks, bytes, base_ptr, device, stream, elems);
    std::vector<RemoteBlock> rb;
    const int r = lookup_blocks(kOpReadLookup, blocks, bytes, rb);
    if (r != 0) return r;
    std::vector<uint64_t> offs(blocks.size());
    for (size_t i = 0; i < blocks.size(); ++i) offs[i] = blocks[i].offset;
    return move_blocks(false, offs.data(), 1, rb.data(), rb.size(), bytes, base_ptr, device,
                       stream, elems);
}

int Connection::r_rdma(const std::vector<KeyOffset>& blocks, int block_size, uint64_t base_ptr,
                       int device, uint64_t stream, MoveResult* res, const PackedKeys* packed) {
    if (blocks.empty()) return 0;
    if (device_lookup_ && server_hbm_ && device >= 0 && device_index_usable())
        return read_via_device_index(blocks, block_size, base_ptr, device, stream, 0, res, packed);
    std::vector<RemoteBlock> rb;
    const int r = lookup_blocks(kOpReadLookup, blocks, block_size, rb);
    if (r != 0) return r;
    std::vector<uint64_t> offs(blocks.size());
    for (size_t i = 0; i < blocks.size(); ++i) offs[i] = blocks[i].offset;
    return move_blocks(false, offs.data(), 1, rb.data(), rb.size(), block_size, base_ptr, device,
                       stream, 0, res);
}

int Connection::rw_local(char op, const std::vector<KeyOffset>& blocks, int block_size,
                         uint64_t base_ptr, int device, uint64_t stream) {
    if (blocks.empty()) return 0;
    if (op != kOpLocalRead && op != kOpLocalWrite) return -1;
    if (op == kOpLocalRead && device_lookup_ && server_hbm_ && device >= 0 && device_index_usable())
        return read_via_device_index(blocks, block_size, base_ptr, device, stream);
    std::vector<RemoteBlock> rb;
    const int r = lookup_blocks(op, blocks, block_size, rb);
    if (r != 0) return r;
    if (op == kOpLocalWrite && server_hbm_) {
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
    return move_blocks(op == kOpLocalWrite, offs.data(), 1, rb.data(), rb.size(), block_size,
                       base_ptr, device, stream);
}

// Pack keys into the pinned ring so that the lookup kernel can hash them: each key starts
// on an 8-byte boundary and is zero padded to a multiple of 8.
static size_t pack_keys(const std::string_view* keys, size_t n, uint8_t* bytes, uint32_t* off,
                        uint32_t* len) {
    size_t at = 0;
    for (size_t i = 0; i < n; ++i) {
        const std::string_view k = keys[i];
        off[i] = uint32_t(at);
        len[i] = uint32_t(k.size());
        const size_t padded = align_up(k.size() ? k.size() : 1, 8);
        std::memcpy(bytes + at, k.data(), k.size());
        std::memset(bytes + at + k.size(), 0, padded - k.size());
        at += padded;
    }
    return at;
}

int Connection::read_via_device_index(const std::vector<KeyOffset>& blocks, int block_size,
                                      uint64_t base_ptr, int device, uint64_t stream_in,
                                      int fp8_elems, MoveResult* res, const PackedKeys* packed) {
    NvtxRange nvtx("istore.read_via_device_index");
    std::lock_guard<std::mutex> lk(mu_);
    DevCtx* ctx = dev_ctx(device);
    if (!ctx) return -1;
    auto m0 = mapping(0, device);
    if (!m0 || !m0->dev_ptr || !segs_[0].index_slots) {
        fail("the server exposes no device index");
        return -1;
    }
    DeviceGuard g(device);
    if (cfg_.doorbell && blocks.size() == 1 && !fp8_elems && !res &&
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
    if (doorbell_quiesce(ctx) != 0) return -1;
    const uint64_t t_pick0 = now_ns();
    cudaStream_t stream = ctx->pick(reinterpret_cast<cudaStream_t>(stream_in), false, streams_);
    stats_.ns_streams += now_ns() - t_pick0;
    stats_.calls++;
    if (res) {
        res->stream = stream;
        res->device = device;
    }
    for (size_t base = 0; base < blocks.size(); base += kMaxBatch) {
        const uint64_t t_build0 = now_ns();
        const size_t n = std::min(kMaxBatch, blocks.size() - base);
        // keys into the pinned ring, in the layout the kernels hash them from; three memcpys
        // when the caller holds them like that already (one batch), a pass over the keys else
        const bool prepacked = packed && base == 0 && packed->n == blocks.size() && n == blocks.size();
        size_t key_bytes = 0;
        std::vector<std::string_view> kp;
        if (prepacked) {
            key_bytes = packed->nbytes;
        } else {
            kp.resize(n);
            for (size_t i = 0; i < n; ++i) {
                kp[i] = blocks[base + i].key;
                key_bytes += align_up(std::max<size_t>(kp[i].size(), 1), 8);
            }
        }
        const size_t at_bytes = ctx->ring_alloc(key_bytes);
        const size_t at_off = ctx->ring_alloc(n * 4);
        const size_t at_len = ctx->ring_alloc(n * 4);
        const size_t at_dst = ctx->ring_alloc(n * 8);
        if (prepacked) {
            std::memcpy(ctx->ring_h + at_bytes, packed->bytes, key_bytes);
            std::memcpy(ctx->ring_h + at_off, packed->off, n * 4);
            std::memcpy(ctx->ring_h + at_len, packed->len, n * 4);
        } else {
            pack_keys(kp.data(), n, ctx->ring_h + at_bytes,
                      reinterpret_cast<uint32_t*>(ctx->ring_h + at_off),
                      reinterpret_cast<uint32_t*>(ctx->ring_h + at_len));
        }
        auto* dst = reinterpret_cast<uint64_t*>(ctx->ring_h + at_dst);
        for (size_t i = 0; i < n; ++i) dst[i] = blocks[base + i].offset;

        const uint32_t nsegs =
            uint32_t(std::min<size_t>(segs_.size(), kernels::LookupLaunch::kMaxSegs));
        uint64_t seg_base[kernels::LookupLaunch::kMaxSegs] = {0};
        bool all_remote = true;
        for (uint32_t s = 0; s < nsegs; ++s) {
            seg_base[s] = reinterpret_cast<uint64_t>(seg_dev_ptr(ctx, s));
            all_remote = all_remote && ctx->seg_remote[s];
        }
        // fp8 pages over NVLink: reads one CTA per SM, writes two per SM.  A grid choice not
        // re-measured on H100: bench/configs.py fp8 --max-ctas N compares grid caps.
        const int grid_cap = max_ctas_ ? max_ctas_
                             : all_remote ? (fp8_elems ? 1 : 2) * kernels::sm_count()
                                          : 0;
        uint64_t align_or = base_ptr;
        for (size_t i = 0; i < n; ++i) align_or |= blocks[base + i].offset;
        const uint64_t t_launch0 = now_ns();
        stats_.ns_build += t_launch0 - t_build0;
        cudaError_t e;
        // The fused kernels resolve a key in every CTA that moves a piece of its block, reading
        // the key bytes from the pinned ring each time: right for a batch of blocks (items are
        // whole blocks, or chunks when that balances the grid better - kernels/balance.h),
        // wasteful when a few LARGE blocks are split over many CTAs - then resolve each key
        // once with the lookup kernel and feed the descriptors to kv_copy.
        // A handful of blocks (<= 4 MB in all): latency matters, not bandwidth.  One launch of
        // the ld/st flavour, which splits a block into 32 KB chunks over CTAs (each resolves its
        // block's key itself - a few redundant probes) and re-checks the entries in the same
        // kernel: lookup + copy + validate would be three launches.
        const bool small_batch = n * size_t(block_size) <= (4u << 20);
        const bool whole_blocks = !small_batch && uint32_t(block_size) <= (1u << 20) && n >= 32;
        kernels::ReadFusedLaunch R;
        R.align_or = align_or;
        const bool fp8_fused = fp8_elems && kernels::fp8_read_fused_supported(R, uint32_t(fp8_elems));
        if (fp8_fused || (!fp8_elems && (whole_blocks || small_batch))) {
            // one kernel: hash + probe + move
            R.key_bytes = ctx->ring_d + at_bytes;
            R.key_off = reinterpret_cast<const uint32_t*>(ctx->ring_d + at_off);
            R.key_len = reinterpret_cast<const uint32_t*>(ctx->ring_d + at_len);
            R.dst_off = reinterpret_cast<const uint64_t*>(ctx->ring_d + at_dst);
            R.dst_base = base_ptr;
            R.n = uint32_t(n);
            R.bytes = uint32_t(block_size);
            R.align_or = copy_variant_ == kernels::kCopyLdSt ? (align_or | 16) : align_or;
            R.table = reinterpret_cast<const kernels::IndexBucket*>(m0->dev_ptr + segs_[0].index_off);
            R.table_mask = kernels::index_bucket_mask(segs_[0].index_slots);
            R.shards = index_shards(ctx, nullptr);
            R.nsegs = nsegs;
            for (uint32_t s = 0; s < nsegs; ++s) R.seg_base[s] = seg_base[s];
            R.status = ctx->status_d;
            R.max_ctas = grid_cap;
            // always: a purge (or an eviction) may free a block while a device-path read is
            // copying it; the post-copy tag check turns that into a reported miss
            R.validate = true;
            R.variant = small_batch ? int(kernels::kCopyLdSt256) : copy_variant_;
            R.stage_bytes = pipe_stage_;
            R.ring_bytes = pipe_ring_;
            // fp8 pages: the resolver rides in the dequantising TMA pipeline (one launch
            // instead of lookup + read + validate: 32 calls of 512 pages were launch-bound)
            e = fp8_fused ? kernels::launch_kv_fp8_read_fused(R, uint32_t(fp8_elems), stream)
                          : kernels::launch_kv_read_fused(R, stream);
            stats_.kernel_launches += 1;
        } else {
            kernels::LookupLaunch Q;
            Q.key_bytes = ctx->ring_d + at_bytes;
            Q.key_off = reinterpret_cast<const uint32_t*>(ctx->ring_d + at_off);
            Q.key_len = reinterpret_cast<const uint32_t*>(ctx->ring_d + at_len);
            Q.n = uint32_t(n);
            Q.table = reinterpret_cast<const kernels::IndexBucket*>(m0->dev_ptr + segs_[0].index_off);
            Q.table_mask = kernels::index_bucket_mask(segs_[0].index_slots);
            Q.shards = index_shards(ctx, nullptr);
            Q.nsegs = nsegs;
            for (uint32_t s = 0; s < nsegs; ++s) Q.seg_base[s] = seg_base[s];
            auto* out = reinterpret_cast<kernels::CopyDesc*>(
                ctx->scratch + ctx->scratch_alloc(n * sizeof(kernels::CopyDesc)));
            Q.out_descs = out;
            Q.dst_off = reinterpret_cast<const uint64_t*>(ctx->ring_d + at_dst);
            Q.dst_base = base_ptr;
            Q.need_bytes = uint32_t(block_size);
            Q.status = ctx->status_d;
            // optimistic read: the entries are re-checked after the copy (purge / eviction)
            Q.found_at = reinterpret_cast<kernels::LookupLaunch::FoundAt*>(
                    ctx->scratch + ctx->scratch_alloc(n * sizeof(kernels::LookupLaunch::FoundAt)));
            e = kernels::launch_index_lookup(Q, stream);
            if (e == cudaSuccess && fp8_elems) {
                kernels::Fp8Launch F;
                F.descs = out;
                F.n = uint32_t(n);
                F.elems = uint32_t(fp8_elems);
                F.status = ctx->status_d;
                F.max_ctas = grid_cap;
                F.aligned16 = (align_or & 15) == 0;
                F.variant = all_remote ? 0 : 1;
                e = kernels::launch_kv_read_fp8(F, stream);
            } else if (e == cudaSuccess) {
                kernels::CopyLaunch L;
                L.descs = out;
                L.n = uint32_t(n);
                L.bytes = uint32_t(block_size);
                L.align_or = align_or;
                L.status = ctx->status_d;
                L.variant = copy_variant_;
                L.stage_bytes = pipe_stage_;
                L.ring_bytes = pipe_ring_;
                L.max_ctas = grid_cap;
                e = kernels::launch_kv_copy(L, stream);
            }
            stats_.kernel_launches += 2;
            if (e == cudaSuccess && Q.found_at) {
                // the server evicts: the entries must still be the ones the lookup resolved
                kernels::ValidateLaunch V;
                V.found_at = Q.found_at;
                V.n = uint32_t(n);
                V.table = Q.table;
                V.shards = Q.shards;
                V.status = ctx->status_d;
                e = kernels::launch_index_validate(V, stream);
                stats_.kernel_launches += 1;
            }
        }
        stats_.ns_launch += now_ns() - t_launch0;
        if (e != cudaSuccess) {
            fail(std::string("device-index read failed to launch: ") + cudaGetErrorString(e));
            return -1;
        }
        ctx->mark(stream);
        if (res) res->launched = true;
        stats_.bytes_read += uint64_t(n) * uint64_t(block_size);
    }
    return 0;
}

// Device-addressable copy descriptors {mapped pool address (0 = miss), dst_base + offset} for
// blocks[base, base + n): resolved on the GPU by the lookup kernel (rb == nullptr, the
// descriptors land in device scratch) or taken from a server lookup (rb, pinned ring).
const kernels::CopyDesc* Connection::resolve_descs(DevCtx* ctx, const std::vector<KeyOffset>& blocks,
                                                   size_t base, size_t n, int block_size,
                                                   uint64_t dst_base,
                                                   const std::vector<RemoteBlock>* rb,
                                                   void* stream_v) {
    cudaStream_t stream = static_cast<cudaStream_t>(stream_v);
    if (rb) {
        const size_t at_desc = ctx->ring_alloc(n * sizeof(kernels::CopyDesc));
        auto* descs = reinterpret_cast<kernels::CopyDesc*>(ctx->ring_h + at_desc);
        for (size_t i = 0; i < n; ++i) {
            const RemoteBlock& b = (*rb)[base + i];
            uint8_t* segbase = seg_dev_ptr(ctx, addr_seg(b.remote_addr));
            if (!segbase) return nullptr;
            descs[i].src = reinterpret_cast<uint64_t>(segbase) + addr_off(b.remote_addr);
            descs[i].dst = dst_base + blocks[base + i].offset;
        }
        return reinterpret_cast<const kernels::CopyDesc*>(ctx->ring_d + at_desc);
    }
    auto m0 = mapping(0, ctx->device);
    if (!m0 || !m0->dev_ptr) return nullptr;
    size_t key_bytes = 0;
    std::vector<std::string_view> kp(n);
    for (size_t i = 0; i < n; ++i) {
        kp[i] = blocks[base + i].key;
        key_bytes += align_up(std::max<size_t>(kp[i].size(), 1), 8);
    }
    const size_t at_bytes = ctx->ring_alloc(key_bytes);
    const size_t at_off = ctx->ring_alloc(n * 4);
    const size_t at_len = ctx->ring_alloc(n * 4);
    const size_t at_dst = ctx->ring_alloc(n * 8);
    pack_keys(kp.data(), n, ctx->ring_h + at_bytes, reinterpret_cast<uint32_t*>(ctx->ring_h + at_off),
              reinterpret_cast<uint32_t*>(ctx->ring_h + at_len));
    auto* dst = reinterpret_cast<uint64_t*>(ctx->ring_h + at_dst);
    for (size_t i = 0; i < n; ++i) dst[i] = blocks[base + i].offset;
    kernels::LookupLaunch Q;
    Q.key_bytes = ctx->ring_d + at_bytes;
    Q.key_off = reinterpret_cast<const uint32_t*>(ctx->ring_d + at_off);
    Q.key_len = reinterpret_cast<const uint32_t*>(ctx->ring_d + at_len);
    Q.n = uint32_t(n);
    Q.table = reinterpret_cast<const kernels::IndexBucket*>(m0->dev_ptr + segs_[0].index_off);
    Q.table_mask = kernels::index_bucket_mask(segs_[0].index_slots);
    Q.shards = index_shards(ctx, nullptr);
    Q.nsegs = uint32_t(std::min<size_t>(segs_.size(), kernels::LookupLaunch::kMaxSegs));
    for (uint32_t sgi = 0; sgi < Q.nsegs; ++sgi)
        Q.seg_base[sgi] = reinterpret_cast<uint64_t>(seg_dev_ptr(ctx, sgi));
    auto* out = reinterpret_cast<kernels::CopyDesc*>(
        ctx->scratch + ctx->scratch_alloc(n * sizeof(kernels::CopyDesc)));
    Q.out_descs = out;
    Q.dst_off = reinterpret_cast<const uint64_t*>(ctx->ring_d + at_dst);
    Q.dst_base = dst_base;
    Q.need_bytes = uint32_t(block_size);
    Q.status = ctx->status_d;
    if (kernels::launch_index_lookup(Q, stream) != cudaSuccess) return nullptr;
    stats_.kernel_launches++;
    return out;
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
    const bool via_index = device_lookup_ && device_index_usable();
    std::vector<RemoteBlock> rb;
    if (!via_index) {
        const int r = lookup_blocks(kOpReadLookup, blocks, block_size, rb);
        if (r != 0) return r;
    }
    NvtxRange nvtx("istore.read_multi");
    std::lock_guard<std::mutex> lk(mu_);
    DevCtx* ctx = dev_ctx(device);
    if (!ctx) return -1;
    DeviceGuard g(device);
    if (doorbell_quiesce(ctx) != 0) return -1;
    cudaStream_t stream = ctx->pick(reinterpret_cast<cudaStream_t>(stream_in), false, streams_);
    stats_.calls++;
    uint64_t align_or = 0;
    for (uint64_t b : bases) align_or |= b;
    for (size_t base = 0; base < blocks.size(); base += kMaxBatch) {
        const size_t n = std::min(kMaxBatch, blocks.size() - base);
        for (size_t i = 0; i < n; ++i) align_or |= blocks[base + i].offset;
        const kernels::CopyDesc* descs_d =
            resolve_descs(ctx, blocks, base, n, block_size, bases[0], via_index ? nullptr : &rb, stream);
        if (!descs_d) {
            fail("multi-destination read: cannot resolve the blocks");
            return -1;
        }
        // Local pool: thread-block clusters (multicast bulk load into 2 or 4 CTAs, one
        // destination each; an odd last destination shares a 2-cluster with its predecessor,
        // which is rewritten with the same bytes).  Pool behind NVLink: one load, K stores
        // per CTA (the fan-out flavour of the TMA pipeline) - the fabric still carries every
        // page once.
        bool src_local = true;
        for (size_t sgi = 0; sgi < ctx->seg_remote.size(); ++sgi)
            if (ctx->seg_ptr[sgi] && ctx->seg_remote[sgi]) src_local = false;
        cudaError_t e = cudaSuccess;
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
                M.status = r == 0 ? ctx->status_d : nullptr;  // count a miss once
                const size_t first = left >= 2 ? r : r - 1;
                M.ndst = left >= 4 ? 4 : 2;
                for (int j = 0; j < M.ndst; ++j)
                    M.delta[j] = int64_t(bases[first + size_t(j)]) - int64_t(bases[0]);
                e = kernels::launch_kv_pipe_mcast(M, stream);
                r = first + size_t(M.ndst);
            } else {
                kernels::CopyLaunch L;
                L.descs = descs_d;
                L.n = uint32_t(n);
                L.bytes = uint32_t(block_size);
                L.align_or = align_or;
                L.status = r == 0 ? ctx->status_d : nullptr;
                L.variant = kernels::kCopyTma;
                L.max_ctas = max_ctas_;
                L.fan_n = int(std::min<size_t>(left, 4));
                for (int j = 0; j < L.fan_n; ++j)
                    L.fan_delta[j] = int64_t(bases[r + size_t(j)]) - int64_t(bases[0]);
                e = kernels::launch_kv_pipe_copy(L, stream);
                r += size_t(L.fan_n);
            }
            stats_.kernel_launches++;
        }
        if (e != cudaSuccess) {
            fail(std::string("multi-destination read failed to launch: ") + cudaGetErrorString(e));
            return -1;
        }
        ctx->mark(stream);
        stats_.bytes_read += uint64_t(n) * uint64_t(block_size) * bases.size();
    }
    return 0;
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
    const bool via_index = device_lookup_ && device_index_usable();
    std::vector<RemoteBlock> rb;
    if (!via_index) {
        const int r = lookup_blocks(kOpReadLookup, blocks, block_size, rb);
        if (r != 0) return r;
    }
    NvtxRange nvtx("istore.read_hnd");
    std::lock_guard<std::mutex> lk(mu_);
    DevCtx* ctx = dev_ctx(device);
    if (!ctx) return -1;
    DeviceGuard g(device);
    if (doorbell_quiesce(ctx) != 0) return -1;
    cudaStream_t stream = ctx->pick(reinterpret_cast<cudaStream_t>(stream_in), false, streams_);
    stats_.calls++;
    for (size_t base = 0; base < blocks.size(); base += kMaxBatch) {
        const size_t n = std::min(kMaxBatch, blocks.size() - base);
        // dst_base 0: the descriptor's dst field carries the page index
        const kernels::CopyDesc* descs_d =
            resolve_descs(ctx, blocks, base, n, block_size, 0, via_index ? nullptr : &rb, stream);
        if (!descs_d) {
            fail("read_cache_hnd: cannot resolve the blocks");
            return -1;
        }
        kernels::HndLaunch H;
        H.descs = descs_d;
        H.n = uint32_t(n);
        H.tokens = uint32_t(tokens);
        H.heads = uint32_t(heads);
        H.dim = uint32_t(dim);
        H.elem_size = uint32_t(elem_size);
        H.dst_base = base_ptr;
        H.num_pages = uint32_t(num_pages);
        H.status = ctx->status_d;
        H.max_ctas = max_ctas_;
        const cudaError_t e = kernels::launch_kv_pipe_hnd(H, stream);
        if (e != cudaSuccess) {
            fail(std::string("layout-swizzling read failed to launch: ") + cudaGetErrorString(e));
            return -1;
        }
        stats_.kernel_launches++;
        ctx->mark(stream);
        stats_.bytes_read += uint64_t(n) * uint64_t(block_size);
    }
    return 0;
}

int Connection::match_via_device_index(const std::vector<std::string_view>& keys, bool exist_only) {
    std::lock_guard<std::mutex> lk(mu_);
    const int device = cfg_.device >= 0 ? cfg_.device : std::max(default_device_, 0);
    DevCtx* ctx = dev_ctx(device);
    if (!ctx) return -3;
    auto m0 = mapping(0, device);
    if (!m0 || !m0->dev_ptr || !segs_[0].index_slots) return -3;
    const size_t n = keys.size();
    size_t key_bytes = 0;
    std::vector<std::string_view> kp(n);
    for (size_t i = 0; i < n; ++i) {
        kp[i] = keys[i];
        key_bytes += align_up(std::max<size_t>(keys[i].size(), 1), 8);
    }
    if (key_bytes + n * 8 + 4096 > kRingBytes / 2) return -3;  // too large: use the control plane
    DeviceGuard g(device);
    if (doorbell_quiesce(ctx) != 0) return -3;
    const size_t at_bytes = ctx->ring_alloc(key_bytes);
    const size_t at_off = ctx->ring_alloc(n * 4);
    const size_t at_len = ctx->ring_alloc(n * 4);
    pack_keys(kp.data(), n, ctx->ring_h + at_bytes,
              reinterpret_cast<uint32_t*>(ctx->ring_h + at_off),
              reinterpret_cast<uint32_t*>(ctx->ring_h + at_len));
    kernels::LookupLaunch Q;
    Q.key_bytes = ctx->ring_d + at_bytes;
    Q.key_off = reinterpret_cast<const uint32_t*>(ctx->ring_d + at_off);
    Q.key_len = reinterpret_cast<const uint32_t*>(ctx->ring_d + at_len);
    Q.n = uint32_t(n);
    Q.table = reinterpret_cast<const kernels::IndexBucket*>(m0->dev_ptr + segs_[0].index_off);
    Q.table_mask = kernels::index_bucket_mask(segs_[0].index_slots);
    Q.shards = index_shards(ctx, nullptr);
    const size_t words = (n + 31) / 32;
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
