#include "server.h"

#include <arpa/inet.h>
#include <fcntl.h>
#include <netinet/in.h>
#include <netinet/tcp.h>
#include <sys/epoll.h>
#include <sys/eventfd.h>
#include <sys/socket.h>
#include <unistd.h>

#include <cerrno>
#include <chrono>
#include <cstring>

#include <cuda_runtime_api.h>

#include <cstdio>
#include <thread>

#include "../core/log.h"
#include "../kernels/kernels.h"
#include "../wire/messages.h"

namespace istore {

struct Server::Conn {
    int fd = -1;
    uint64_t id = 0;
    enum State { kHeader, kBody } state = kHeader;
    uint8_t hdr_buf[sizeof(Header)];
    size_t hdr_got = 0;
    Header hdr{};
    std::vector<uint8_t> body;
    size_t body_got = 0;
    std::vector<uint8_t> out;
    size_t out_off = 0;
    bool want_write = false;
    bool closing = false;  // flush pending output, then close
    ConnInfo peer{};
    std::vector<BlockPtr> leases;  // blocks pinned for this client's in-flight reads
    std::vector<uint64_t> staged;  // commit list received with 'U', applied at the next 'S'
    std::string addr;
};

namespace {
bool set_nonblock(int fd) {
    const int fl = fcntl(fd, F_GETFL, 0);
    return fl >= 0 && fcntl(fd, F_SETFL, fl | O_NONBLOCK) == 0;
}
struct DevGuard {
    int prev = -1;
    explicit DevGuard(int dev) {
        if (dev >= 0 && cudaGetDevice(&prev) == cudaSuccess && prev != dev) cudaSetDevice(dev);
    }
    ~DevGuard() {
        if (prev >= 0) cudaSetDevice(prev);
    }
};
size_t next_pow2(size_t v) {
    size_t p = 1;
    while (p < v) p <<= 1;
    return p;
}
}  // namespace

Server::Server(const ServerConfig& cfg) : cfg_(cfg) {
    store_ = std::make_unique<KVStore>(&mm_, cfg_.evict);
    scratch_.resize(64 << 10);
}

Server::~Server() { stop(); }

bool Server::add_segment(std::string* err) {
    const uint32_t id = uint32_t(segs_.size());
    const bool first_round = id < std::max<size_t>(1, cfg_.pool_devices.size());
    size_t bytes = cfg_.prealloc_bytes ? cfg_.prealloc_bytes
                                       : (first_round ? cfg_.prealloc_size : cfg_.extend_size) << 30;
    const uint32_t granule = uint32_t(cfg_.minimal_allocate_size) * 1024u;
    bytes = bytes / granule * granule;
    if (bytes == 0) {
        if (err) *err = "pool size is smaller than one allocation granule";
        return false;
    }
    std::unique_ptr<fabric::SegmentOwner> seg;
    int device = -1;
    if (use_hbm_) {
        device = cfg_.pool_devices.empty()
                     ? 0
                     : cfg_.pool_devices[next_pool_dev_++ % cfg_.pool_devices.size()];
        // 2 entries per block: at half load a key's two 8-way buckets are practically never
        // both full.  Every INITIAL segment (one per --pool-devices entry) carries a table:
        // the index is sharded by key fingerprint over them, so the probes and claims of all
        // clients spread over the pool GPUs instead of landing on segment 0's.  Together the
        // shards must also cover the blocks of segments added later by --auto-increase,
        // which carry no table (the shard count is fixed at start).
        const size_t growth = cfg_.auto_increase ? 8 : 1;
        size_t slots = cfg_.index_slots
                           ? next_pow2(cfg_.index_slots)
                           : next_pow2(std::max<size_t>(1024, 2 * growth * (bytes / granule)));
        if (!first_round || index_shards_.size() >= kernels::kMaxIndexShards) slots = 0;
        if (slots) index_shards_.push_back(id);
        seg = fabric::SegmentOwner::create_device(id, device, bytes, granule, slots, err);
    } else {
        seg = fabric::SegmentOwner::create_host(id, bytes, granule, port_, err);
    }
    if (!seg) return false;
    mm_.add_pool(bytes, granule, device);
    LOG_INFO("pool segment %u: %s, %.2f GiB, granule %u KiB, device %d", id,
             use_hbm_ ? "HBM" : "host shm", double(bytes) / double(1ull << 30), granule / 1024,
             device);
    segs_.push_back(std::move(seg));
    return true;
}

bool Server::maybe_extend() {
    if (!cfg_.auto_increase) return false;
    std::string err;
    // Done inline on the reactor thread: creating a segment is an allocation, not a
    // multi-second pin+register as in the reference, and it keeps the pool vector
    // single-threaded (the reference mutates it from a worker thread).
    if (!add_segment(&err)) {
        LOG_WARN("pool auto-increase failed: %s", err.c_str());
        return false;
    }
    LOG_INFO("pool extended to %zu segments", segs_.size());
    return true;
}

int Server::start(std::string* err) {
    if (running_.load()) return 0;
    port_ = cfg_.service_port;
    if (cfg_.pool_backend == "hbm")
        use_hbm_ = true;
    else if (cfg_.pool_backend == "host")
        use_hbm_ = false;
    else
        use_hbm_ = fabric::cuda_available();
    if (use_hbm_ && !fabric::cuda_available()) {
        if (err) *err = "pool backend 'hbm' requested but no CUDA device is usable";
        return -1;
    }

    listen_fd_ = socket(AF_INET, SOCK_STREAM | SOCK_CLOEXEC, 0);
    if (listen_fd_ < 0) {
        if (err) *err = std::string("socket: ") + std::strerror(errno);
        return -1;
    }
    int one = 1;
    setsockopt(listen_fd_, SOL_SOCKET, SO_REUSEADDR, &one, sizeof(one));
    sockaddr_in sa{};
    sa.sin_family = AF_INET;
    sa.sin_port = htons(uint16_t(cfg_.service_port));
    const std::string host = cfg_.host.empty() ? "0.0.0.0" : cfg_.host;
    if (inet_pton(AF_INET, host == "localhost" ? "127.0.0.1" : host.c_str(), &sa.sin_addr) != 1) {
        if (err) *err = "invalid listen address: " + host;
        close(listen_fd_);
        listen_fd_ = -1;
        return -1;
    }
    if (bind(listen_fd_, reinterpret_cast<sockaddr*>(&sa), sizeof(sa)) != 0 ||
        listen(listen_fd_, 128) != 0) {
        if (err)
            *err = "bind/listen on " + host + ":" + std::to_string(cfg_.service_port) + ": " +
                   std::strerror(errno);
        close(listen_fd_);
        listen_fd_ = -1;
        return -1;
    }
    if (cfg_.service_port == 0) {  // ephemeral port (tests)
        socklen_t sl = sizeof(sa);
        getsockname(listen_fd_, reinterpret_cast<sockaddr*>(&sa), &sl);
        port_ = ntohs(sa.sin_port);
    }
    set_nonblock(listen_fd_);

    {
        std::lock_guard<std::mutex> lk(mu_);
        const size_t initial = std::max<size_t>(1, use_hbm_ ? cfg_.pool_devices.size() : 1);
        for (size_t i = 0; i < initial; ++i) {
            if (!add_segment(err)) {
                close(listen_fd_);
                listen_fd_ = -1;
                segs_.clear();
                return -1;
            }
        }
    }

    if (use_hbm_ && cfg_.replica_bytes) {
        // NVLS-replicated region for one-writer / many-reader blocks (shared prompt prefixes)
        std::lock_guard<std::mutex> lk(mu_);
        std::vector<int> devs = cfg_.replica_devices;
        if (devs.empty())
            for (int d = 0; d < fabric::cuda_device_count(); ++d) devs.push_back(d);
        const uint32_t granule = uint32_t(cfg_.minimal_allocate_size) * 1024u;
        std::string rerr;
        auto seg = fabric::SegmentOwner::create_replica(uint32_t(segs_.size()), devs,
                                                        cfg_.replica_bytes, granule, port_, &rerr);
        if (seg) {
            mm_.add_pool(seg->info().bytes, granule, kReplicaDevice);
            LOG_INFO("NVLS replica segment %zu: %.2f GiB on %zu GPUs", segs_.size(),
                     double(seg->info().bytes) / double(1ull << 30), devs.size());
            segs_.push_back(std::move(seg));
        } else {
            LOG_WARN("no NVLS-replicated region: %s", rerr.c_str());
        }
    }

    epoll_fd_ = epoll_create1(EPOLL_CLOEXEC);
    wake_fd_ = eventfd(0, EFD_NONBLOCK | EFD_CLOEXEC);
    epoll_event ev{};
    ev.events = EPOLLIN;
    ev.data.fd = listen_fd_;
    epoll_ctl(epoll_fd_, EPOLL_CTL_ADD, listen_fd_, &ev);
    ev.data.fd = wake_fd_;
    epoll_ctl(epoll_fd_, EPOLL_CTL_ADD, wake_fd_, &ev);

    stop_.store(false);
    running_.store(true);
    thread_ = std::thread([this] { loop(); });
    LOG_INFO("control plane listening on %s:%d (%s pool)", host.c_str(), port_,
             use_hbm_ ? "HBM" : "host");
    return 0;
}

void Server::stop() {
    if (!running_.exchange(false)) return;
    stop_.store(true);
    uint64_t one = 1;
    (void)!write(wake_fd_, &one, sizeof(one));
    if (thread_.joinable()) thread_.join();
    std::lock_guard<std::mutex> lk(mu_);
    for (auto& kv : conns_) close(kv.second->fd);
    conns_.clear();
    if (listen_fd_ >= 0) close(listen_fd_);
    if (epoll_fd_ >= 0) close(epoll_fd_);
    if (wake_fd_ >= 0) close(wake_fd_);
    listen_fd_ = epoll_fd_ = wake_fd_ = -1;
    quarantine_.clear();
    store_->purge();
    for (EraseCtx& ec : erase_) {
        if (!ec.buf && !ec.stream) continue;
        DevGuard g(ec.device);
        if (ec.buf) cudaFree(ec.buf);
        if (ec.stream) cudaStreamDestroy(static_cast<cudaStream_t>(ec.stream));
    }
    erase_.clear();
    index_shards_.clear();
    segs_.clear();
}

size_t Server::kvmap_len() {
    std::lock_guard<std::mutex> lk(mu_);
    return store_->size();
}

size_t Server::purge() {
    std::lock_guard<std::mutex> lk(mu_);
    // Leases of host-mediated readers are NOT dropped here: a leased block leaves the map but
    // keeps its pool space until the reader's SYNC lets go of it, so a copy that is still
    // running never sees the space handed to a new writer (reference: intrusive_ptr keeps
    // in-flight blocks alive across purge, src/infinistore.cpp:1110-1116).
    const size_t n = store_->purge();
    for (auto& s : segs_) s->clear_index();
    index_incomplete_ = false;  // host map and device index are empty and in step again
    quarantine_.clear();  // the index is empty now: nothing can resolve these blocks any more
    return n;
}

ServerStats Server::stats() {
    std::lock_guard<std::mutex> lk(mu_);
    ServerStats s = stats_;
    s.connections = conns_.size();
    s.keys = store_->size();
    s.inflight = store_->inflight();
    s.pool_bytes = mm_.total_bytes();
    s.used_bytes = mm_.used_bytes();
    s.segments = segs_.size();
    s.evicted = store_->evicted();
    return s;
}

bool Server::erase_from_device_index(const std::vector<KVStore::Victim>& victims) {
    if (segs_.empty() || index_shards_.empty()) return true;
    // group the victims by the shard their fingerprint selects; each shard's table is erased
    // by a kernel on the GPU that holds it
    const uint32_t nshards = uint32_t(index_shards_.size());
    std::vector<std::vector<kernels::EraseRec>> per(nshards);
    for (auto& v : victims)
        per[kernels::index_shard_of(v.hash.h2, nshards)].push_back(
            kernels::EraseRec{v.hash.h1, v.hash.h2, v.block->addr()});
    if (erase_.size() < nshards) erase_.resize(nshards);
    bool ok = true;
    for (uint32_t sh = 0; sh < nshards && ok; ++sh) {
        std::vector<kernels::EraseRec>& recs = per[sh];
        if (recs.empty()) continue;
        const fabric::SegmentOwner& seg = *segs_[index_shards_[sh]];
        if (seg.info().kind != kSegDeviceIpc || !seg.info().index_slots) continue;
        DevGuard g(seg.info().device);
        EraseCtx& ec = erase_[sh];
        ec.device = seg.info().device;
        if (ec.cap < recs.size()) {
            if (ec.buf) cudaFree(ec.buf);
            ec.buf = nullptr;
            ec.cap = std::max<size_t>(4096, next_pow2(recs.size()));
            if (cudaMalloc(&ec.buf, ec.cap * sizeof(kernels::EraseRec)) != cudaSuccess) {
                ec.cap = 0;
                (void)cudaGetLastError();
                return false;
            }
        }
        kernels::EraseLaunch E;
        E.recs = static_cast<const kernels::EraseRec*>(ec.buf);
        E.n = uint32_t(recs.size());
        E.table = reinterpret_cast<kernels::IndexBucket*>(static_cast<uint8_t*>(seg.base()) +
                                                         seg.info().index_off);
        E.table_mask = kernels::index_bucket_mask(seg.info().index_slots);
        // The space may be handed out again only once no reader can resolve the old entries.
        // Own non-blocking stream: clients living in this process keep their kernels running.
        if (!ec.stream && cudaStreamCreateWithFlags(reinterpret_cast<cudaStream_t*>(&ec.stream),
                                                    cudaStreamNonBlocking) != cudaSuccess) {
            ec.stream = nullptr;
            (void)cudaGetLastError();
            return false;
        }
        cudaStream_t st = static_cast<cudaStream_t>(ec.stream);
        ok = cudaMemcpyAsync(ec.buf, recs.data(), recs.size() * sizeof(kernels::EraseRec),
                             cudaMemcpyHostToDevice, st) == cudaSuccess &&
             kernels::launch_index_erase(E, st) == cudaSuccess &&
             cudaStreamSynchronize(st) == cudaSuccess;
        if (!ok) LOG_ERROR("index erase failed: %s", cudaGetErrorString(cudaGetLastError()));
    }
    return ok;
}

// Shard 0's table plus the others, as the server's own process addresses them (load()).
void Server::fill_index_view(kernels::IndexBucket** table, uint64_t* mask,
                             kernels::IndexShards* shards) const {
    *table = nullptr;
    *mask = 0;
    uint32_t n = 0;
    for (uint32_t id : index_shards_) {
        const fabric::SegmentOwner& seg = *segs_[id];
        auto* t = reinterpret_cast<kernels::IndexBucket*>(static_cast<uint8_t*>(seg.base()) +
                                                         seg.info().index_off);
        const uint64_t m = kernels::index_bucket_mask(seg.info().index_slots);
        if (n == 0) {
            *table = t;
            *mask = m;
        } else {
            shards->table[n - 1] = t;
            shards->mask[n - 1] = m;
        }
        ++n;
    }
    shards->n = n;
}

bool Server::evict_some(size_t want, bool replica) {
    std::vector<KVStore::Victim> victims;
    const size_t freed = store_->evict(want, replica, victims);
    if (victims.empty()) return false;
    if (!erase_from_device_index(victims)) {
        // cannot prove the entries unreachable: keep the space reserved rather than risk a
        // reader copying a reused block (the blocks leak until the next purge)
        quarantine_.insert(quarantine_.end(), victims.begin(), victims.end());
        return false;
    }
    LOG_INFO("evicted %zu blocks (%zu KiB) from the %s", victims.size(), freed >> 10,
             replica ? "replicated region" : "pool");
    victims.clear();  // last references: the space returns to the pool
    return true;
}

std::vector<SegmentInfo> Server::segments() {
    std::lock_guard<std::mutex> lk(mu_);
    std::vector<SegmentInfo> v;
    for (auto& s : segs_) v.push_back(s->info());
    return v;
}

// ---------------------------------------------------------------- checkpoint / resume

namespace {
constexpr char kDumpMagic[8] = {'I', 'S', 'T', 'O', 'R', 'E', '0', '1'};

}  // namespace

long Server::dump(const std::string& path, std::string* err) {
    std::lock_guard<std::mutex> lk(mu_);
    FILE* f = std::fopen(path.c_str(), "wb");
    if (!f) {
        if (err) *err = "cannot open " + path + ": " + std::strerror(errno);
        return -1;
    }
    uint64_t count = 0;
    std::fwrite(kDumpMagic, 1, 8, f);
    std::fwrite(&count, 8, 1, f);  // patched at the end
    std::vector<uint8_t> buf;
    bool ok = true;
    store_->for_each_committed([&](const std::string& key, const Block& b) {
        if (!ok || b.seg >= segs_.size()) return;
        const fabric::SegmentOwner& seg = *segs_[b.seg];
        buf.resize(b.size);
        const uint8_t* src = static_cast<const uint8_t*>(seg.rw_base()) + b.offset;
        if (seg.info().kind == kSegHostShm) {
            std::memcpy(buf.data(), src, b.size);
        } else {
            DevGuard g(seg.rw_device());
            if (cudaMemcpy(buf.data(), src, b.size, cudaMemcpyDeviceToHost) != cudaSuccess) {
                (void)cudaGetLastError();
                ok = false;
                return;
            }
        }
        const uint32_t klen = uint32_t(key.size()), size = b.size;
        const uint8_t replicated = seg.info().kind == kSegReplica;
        ok = std::fwrite(&klen, 4, 1, f) == 1 && std::fwrite(key.data(), 1, klen, f) == klen &&
             std::fwrite(&size, 4, 1, f) == 1 && std::fwrite(&replicated, 1, 1, f) == 1 &&
             std::fwrite(buf.data(), 1, size, f) == size;
        ++count;
    });
    if (ok) {
        std::fseek(f, 8, SEEK_SET);
        ok = std::fwrite(&count, 8, 1, f) == 1;
    }
    std::fclose(f);
    if (!ok) {
        if (err) *err = "writing " + path + " failed";
        return -1;
    }
    LOG_INFO("checkpoint: %llu blocks written to %s", (unsigned long long)count, path.c_str());
    return long(count);
}

long Server::load(const std::string& path, std::string* err) {
    std::lock_guard<std::mutex> lk(mu_);
    FILE* f = std::fopen(path.c_str(), "rb");
    if (!f) {
        if (err) *err = "cannot open " + path + ": " + std::strerror(errno);
        return -1;
    }
    char magic[8];
    uint64_t count = 0;
    if (std::fread(magic, 1, 8, f) != 8 || std::memcmp(magic, kDumpMagic, 8) != 0 ||
        std::fread(&count, 8, 1, f) != 1) {
        std::fclose(f);
        if (err) *err = path + " is not a store checkpoint";
        return -1;
    }
    // pinned staging for the HBM path (the page mover reads it over PCIe)
    void* staging = nullptr;
    size_t staging_cap = 0;
    uint32_t* scratch = nullptr;
    long loaded = 0;
    bool ok = true;
    std::string key;
    std::vector<uint8_t> host_buf;
    for (uint64_t i = 0; i < count && ok; ++i) {
        uint32_t klen = 0, size = 0;
        uint8_t replicated = 0;
        if (std::fread(&klen, 4, 1, f) != 1 || klen > (1u << 20)) {
            ok = false;
            break;
        }
        key.resize(klen);
        if (std::fread(key.data(), 1, klen, f) != klen || std::fread(&size, 4, 1, f) != 1 ||
            std::fread(&replicated, 1, 1, f) != 1 || size == 0 || size > (1u << 30)) {
            ok = false;
            break;
        }
        std::vector<RemoteBlock> blocks;
        std::vector<std::string_view> keys{std::string_view(key)};
        const int hint = replicated ? kReplicaDevice : -1;
        int code = store_->reserve(keys, size, hint, 0, blocks);
        while (code == kOutOfMemory && !replicated && maybe_extend())
            code = store_->reserve(keys, size, hint, 0, blocks);
        if (code != kFinish) {
            if (err) *err = "pool exhausted while loading " + path;
            ok = false;
            break;
        }
        if (is_fake_block(blocks[0])) {  // key exists: keep the live copy, skip the bytes
            std::fseek(f, long(size), SEEK_CUR);
            continue;
        }
        const uint32_t segid = addr_seg(blocks[0].remote_addr);
        const fabric::SegmentOwner& seg = *segs_[segid];
        uint8_t* dst = static_cast<uint8_t*>(seg.rw_base()) + addr_off(blocks[0].remote_addr);
        if (seg.info().kind == kSegHostShm) {
            ok = std::fread(dst, 1, size, f) == size;
        } else {
            DevGuard g(seg.rw_device());
            if (staging_cap < size_t(size) + 256) {
                if (staging) cudaFreeHost(staging);
                staging_cap = std::max<size_t>(size_t(size) + 256, 4u << 20);
                if (cudaHostAlloc(&staging, staging_cap, cudaHostAllocMapped | cudaHostAllocPortable) !=
                    cudaSuccess) {
                    staging = nullptr;
                    staging_cap = 0;
                    ok = false;
                }
            }
            ok = ok && std::fread(staging, 1, size, f) == size;
            if (ok) {
            if (seg.info().kind == kSegReplica) {
                // every replica must receive the bytes: write through the multicast address
                dst = static_cast<uint8_t*>(seg.base()) + addr_off(blocks[0].remote_addr);
            }
            // the descriptor lives in the pinned (device-mapped) staging buffer too
            auto* descp = reinterpret_cast<kernels::CopyDesc*>(static_cast<uint8_t*>(staging) +
                                                               ((size_t(size) + 63) & ~size_t(63)));
            *descp = kernels::CopyDesc{reinterpret_cast<uint64_t>(staging), reinterpret_cast<uint64_t>(dst)};
            const KeyHash kh = hash_key(reinterpret_cast<const uint8_t*>(key.data()), key.size());
            kernels::IndexEntry rec{kh.h1, kh.h2, blocks[0].remote_addr, blocks[0].gen, size};
            kernels::CopyLaunch L;
            L.descs_host = descp;  // one block: the descriptor rides in the kernel parameters
            L.descs = descp;
            L.n = 1;
            L.bytes = size;
            L.align_or = size % 16 ? 1 : 0;
            L.multicast = seg.info().kind == kSegReplica && size % 16 == 0;
            void* rec_dev = nullptr;
            if (!index_shards_.empty()) {
                if (!scratch) {
                    cudaMalloc(reinterpret_cast<void**>(&scratch), 64);
                    cudaMemset(scratch, 0, 64);
                }
                cudaMalloc(&rec_dev, sizeof(rec));
                cudaMemcpy(rec_dev, &rec, sizeof(rec), cudaMemcpyHostToDevice);
                L.recs = static_cast<const kernels::IndexEntry*>(rec_dev);
                fill_index_view(&L.table, &L.table_mask, &L.shards);
                L.done = scratch;
            }
            const cudaError_t e = kernels::launch_kv_copy(L, nullptr);
            ok = e == cudaSuccess && cudaDeviceSynchronize() == cudaSuccess;
            if (rec_dev) cudaFree(rec_dev);
            }  // if (ok)
            if (!ok) (void)cudaGetLastError();
        }
        const uint64_t addr = blocks[0].remote_addr;
        if (!ok) {
            // the block was reserved for connection 0 and never committed: give it back
            std::vector<KVStore::Victim> victims;
            store_->drop_inflight(&addr, 1, 0, &victims);
            release_dropped(victims);
            break;
        }
        store_->commit(&addr, 1);
        ++loaded;
    }
    if (staging) cudaFreeHost(staging);
    if (scratch) cudaFree(scratch);
    std::fclose(f);
    if (!ok) {
        if (err && err->empty()) *err = "reading " + path + " failed";
        return -1;
    }
    LOG_INFO("checkpoint: %ld blocks loaded from %s", loaded, path.c_str());
    return loaded;
}

// ---------------------------------------------------------------- reactor

void Server::loop() {
    constexpr int kMaxEvents = 64;
    epoll_event evs[kMaxEvents];
    while (!stop_.load(std::memory_order_relaxed)) {
        const int n = epoll_wait(epoll_fd_, evs, kMaxEvents, 500);
        if (n < 0) {
            if (errno == EINTR) continue;
            LOG_ERROR("epoll_wait: %s", std::strerror(errno));
            break;
        }
        for (int i = 0; i < n; ++i) {
            const int fd = evs[i].data.fd;
            if (fd == wake_fd_) {
                uint64_t v;
                (void)!read(wake_fd_, &v, sizeof(v));
                continue;
            }
            if (fd == listen_fd_) {
                on_accept();
                continue;
            }
            std::lock_guard<std::mutex> lk(mu_);
            auto it = conns_.find(fd);
            if (it == conns_.end()) continue;
            Conn* c = it->second.get();
            if (evs[i].events & (EPOLLERR | EPOLLHUP)) {
                close_conn(c);
                continue;
            }
            if (evs[i].events & EPOLLOUT) on_writable(c);
            if (conns_.count(fd) && (evs[i].events & EPOLLIN)) on_readable(c);
        }
    }
}

void Server::on_accept() {
    for (;;) {
        sockaddr_in sa{};
        socklen_t sl = sizeof(sa);
        const int fd = accept4(listen_fd_, reinterpret_cast<sockaddr*>(&sa), &sl,
                               SOCK_NONBLOCK | SOCK_CLOEXEC);
        if (fd < 0) {
            if (errno != EAGAIN && errno != EWOULDBLOCK && errno != EINTR)
                LOG_WARN("accept: %s", std::strerror(errno));
            return;
        }
        int one = 1;
        setsockopt(fd, IPPROTO_TCP, TCP_NODELAY, &one, sizeof(one));
        auto c = std::make_unique<Conn>();
        c->fd = fd;
        char ip[INET_ADDRSTRLEN] = {0};
        inet_ntop(AF_INET, &sa.sin_addr, ip, sizeof(ip));
        c->addr = std::string(ip) + ":" + std::to_string(ntohs(sa.sin_port));
        epoll_event ev{};
        ev.events = EPOLLIN;
        ev.data.fd = fd;
        std::lock_guard<std::mutex> lk(mu_);
        c->id = next_conn_id_++;
        if (epoll_ctl(epoll_fd_, EPOLL_CTL_ADD, fd, &ev) != 0) {
            close(fd);
            continue;
        }
        LOG_DEBUG("connection %llu from %s", (unsigned long long)c->id, c->addr.c_str());
        stats_.accepted++;
        conns_[fd] = std::move(c);
    }
}

// Blocks a writer reserved but never committed.  Its kernel may already have claimed - or,
// with the in-band commit, even published - their ways of the device index, so the entries
// are erased before the space returns to the pool; if that cannot be proven the blocks are
// quarantined (space stays reserved until the next purge) rather than risk a device-path
// reader resolving the key to reused memory.
void Server::release_dropped(std::vector<KVStore::Victim>& victims) {
    if (victims.empty()) return;
    if (!erase_from_device_index(victims))
        quarantine_.insert(quarantine_.end(), victims.begin(), victims.end());
    victims.clear();
}

// A writer reports that `n` of its blocks found both index buckets full: those keys live in
// the host map only.  Sticky until the next purge; readers learn it from the exchange flags
// and from every SYNC reply, and resolve through the server from then on.
void Server::note_publish_failures(uint32_t n) {
    if (!index_incomplete_)
        LOG_WARN("device index overflow: %u block(s) not indexed on the GPU; device-side lookups "
                 "are disabled for clients until the next purge", n);
    index_incomplete_ = true;
    stats_.index_overflows += n;
}

void Server::close_conn(Conn* c) {
    std::vector<KVStore::Victim> victims;
    const size_t dropped = store_->drop_uncommitted(c->id, &victims);
    release_dropped(victims);
    if (dropped)
        LOG_WARN("connection %llu closed with %zu uncommitted blocks: released",
                 (unsigned long long)c->id, dropped);
    LOG_DEBUG("connection %llu closed", (unsigned long long)c->id);
    epoll_ctl(epoll_fd_, EPOLL_CTL_DEL, c->fd, nullptr);
    close(c->fd);
    conns_.erase(c->fd);  // destroys c (and its leases)
}

void Server::on_writable(Conn* c) {
    while (c->out_off < c->out.size()) {
        const ssize_t n =
            send(c->fd, c->out.data() + c->out_off, c->out.size() - c->out_off, MSG_NOSIGNAL);
        if (n > 0) {
            c->out_off += size_t(n);
        } else if (n < 0 && (errno == EAGAIN || errno == EWOULDBLOCK)) {
            break;
        } else if (n < 0 && errno == EINTR) {
            continue;
        } else {
            close_conn(c);
            return;
        }
    }
    const bool pending = c->out_off < c->out.size();
    if (!pending) {
        c->out.clear();
        c->out_off = 0;
        if (c->closing) {
            close_conn(c);
            return;
        }
    }
    if (pending != c->want_write) {
        epoll_event ev{};
        ev.events = EPOLLIN | (pending ? EPOLLOUT : 0);
        ev.data.fd = c->fd;
        epoll_ctl(epoll_fd_, EPOLL_CTL_MOD, c->fd, &ev);
        c->want_write = pending;
    }
}

void Server::reply(Conn* c, int32_t code, const void* payload, size_t len) {
    const size_t at = c->out.size();
    c->out.resize(at + sizeof(code) + len);
    std::memcpy(c->out.data() + at, &code, sizeof(code));
    if (len) std::memcpy(c->out.data() + at + sizeof(code), payload, len);
}

void Server::reply_blob(Conn* c, int32_t code, const void* blob, size_t len) {
    const size_t at = c->out.size();
    const uint32_t l32 = uint32_t(len);
    c->out.resize(at + sizeof(code) + sizeof(l32) + len);
    std::memcpy(c->out.data() + at, &code, sizeof(code));
    std::memcpy(c->out.data() + at + sizeof(code), &l32, sizeof(l32));
    if (len) std::memcpy(c->out.data() + at + sizeof(code) + sizeof(l32), blob, len);
}

// Stream parser: READ_HEADER (9 bytes) -> READ_BODY (body_size bytes) -> dispatch.
void Server::on_readable(Conn* c) {
    const int fd = c->fd;
    for (int budget = 0; budget < 256; ++budget) {
        if (c->closing) break;
        ssize_t n;
        if (c->state == Conn::kHeader) {
            n = recv(fd, c->hdr_buf + c->hdr_got, sizeof(Header) - c->hdr_got, 0);
        } else {
            n = recv(fd, c->body.data() + c->body_got, c->body.size() - c->body_got, 0);
        }
        if (n == 0) {
            close_conn(c);
            return;
        }
        if (n < 0) {
            if (errno == EAGAIN || errno == EWOULDBLOCK) break;
            if (errno == EINTR) continue;
            close_conn(c);
            return;
        }
        bool complete = false;
        if (c->state == Conn::kHeader) {
            c->hdr_got += size_t(n);
            if (c->hdr_got < sizeof(Header)) continue;
            std::memcpy(&c->hdr, c->hdr_buf, sizeof(Header));
            c->hdr_got = 0;
            if (c->hdr.magic != kMagic) {
                LOG_WARN("bad magic 0x%08x from %s: closing", c->hdr.magic, c->addr.c_str());
                stats_.bad_requests++;
                close_conn(c);
                return;
            }
            if (!op_known(c->hdr.op)) {
                LOG_WARN("unknown op 0x%02x from %s: 400 and close", (unsigned)(uint8_t)c->hdr.op,
                         c->addr.c_str());
                stats_.bad_requests++;
                reply(c, kInvalidReq);
                c->closing = true;
                break;
            }
            if (!op_has_body(c->hdr.op)) {
                // the reference client leaves body_size uninitialised for SYNC: ignore it
                c->body.clear();
                complete = true;
            } else if (c->hdr.body_size > kMaxBody) {
                LOG_WARN("body of %u bytes exceeds the %u byte cap: 400 and close",
                         c->hdr.body_size, kMaxBody);
                stats_.bad_requests++;
                reply(c, kInvalidReq);
                c->closing = true;
                break;
            } else if (c->hdr.body_size == 0) {
                c->body.clear();
                complete = true;
            } else {
                c->body.resize(c->hdr.body_size);
                c->body_got = 0;
                c->state = Conn::kBody;
            }
        } else {
            c->body_got += size_t(n);
            if (c->body_got == c->body.size()) {
                c->state = Conn::kHeader;
                complete = true;
            }
        }
        if (complete) {
            stats_.requests++;
            stats_.ops[uint8_t(c->hdr.op) & 127]++;
            const uint64_t d = drop_after_.load();
            if (d && drop_after_.fetch_sub(1) == 1) {  // fault injection
                close_conn(c);
                return;
            }
            if (delay_count_.load() && delay_count_.fetch_sub(1) >= 1)  // fault injection
                std::this_thread::sleep_for(std::chrono::milliseconds(delay_ms_.load()));
            if (!dispatch(c)) {
                c->closing = true;
                break;
            }
            if (c->out.size() - c->out_off > cfg_.max_pending_reply_bytes) {
                // the peer keeps sending requests but does not read the answers: do not
                // buffer without bound on its behalf
                LOG_WARN("conn %llu (%s): %zu MiB of unread replies: disconnected",
                         (unsigned long long)c->id, c->addr.c_str(),
                         (c->out.size() - c->out_off) >> 20);
                close_conn(c);
                return;
            }
        }
    }
    if (conns_.count(fd)) on_writable(c);  // flush replies (may close when `closing`)
}

bool Server::dispatch(Conn* c) {
    const auto t0 = std::chrono::steady_clock::now();
    int code = kInvalidReq;
    try {
        switch (c->hdr.op) {
            case kOpExchange: code = handle_exchange(c); break;
            case kOpPoolMap: code = handle_pool_map(c); break;
            case kOpAllocate: code = handle_allocate(c, false); break;
            case kOpLocalWrite: code = handle_allocate(c, true); break;
            case kOpReadLookup: code = handle_lookup(c, false); break;
            case kOpLocalRead: code = handle_lookup(c, true); break;
            case kOpCommit: code = handle_commit(c); break;
            case kOpStageCommit: code = handle_stage_commit(c); break;
            case kOpCheckExist: code = handle_check_exist(c); break;
            case kOpMatchLastIdx: code = handle_match(c); break;
            case kOpTouch: code = handle_touch(c); break;
            case kOpSync: {
                // Reply first, apply the staged commit right after: the reply leaves this
                // thread's hands before the map update, which the
                // client therefore does not wait for - and nobody can observe the gap, because
                // every later request of every connection is served by this same thread, after
                // the update.
                std::vector<uint64_t> apply;
                apply.swap(c->staged);
                c->leases.clear();  // the client's reads have completed
                // no server-side transfers exist in this design: the count is always 0
                const uint32_t remain = index_incomplete_ ? kSyncIndexIncomplete : 0u;
                uint8_t msg[8];
                const int32_t ok = kFinish;
                std::memcpy(msg, &ok, 4);
                std::memcpy(msg + 4, &remain, 4);
                size_t sent = 0;
                if (c->out_off >= c->out.size()) {  // nothing queued ahead of it: send it now
                    const ssize_t n = send(c->fd, msg, sizeof(msg), MSG_NOSIGNAL | MSG_DONTWAIT);
                    if (n > 0) sent = size_t(n);
                }
                if (sent < sizeof(msg)) {  // the rest (or all of it) takes the ordinary path
                    const size_t at = c->out.size();
                    c->out.resize(at + sizeof(msg) - sent);
                    std::memcpy(c->out.data() + at, msg + sent, sizeof(msg) - sent);
                }
                if (!apply.empty()) store_->commit(apply.data(), apply.size());
                code = kFinish;
                break;
            }
            default: break;
        }
    } catch (const fb::Malformed& e) {
        LOG_WARN("malformed %s request from %s: %s", op_name(c->hdr.op), c->addr.c_str(),
                 e.what());
        code = kInvalidReq;
        if (c->hdr.op != kOpCommit && c->hdr.op != kOpStageCommit) reply(c, kInvalidReq);
    } catch (const std::exception& e) {
        LOG_ERROR("%s request failed: %s", op_name(c->hdr.op), e.what());
        code = kInternalError;
        if (c->hdr.op != kOpCommit && c->hdr.op != kOpStageCommit) reply(c, kInternalError);
    }
    if (code >= 400) stats_.bad_requests++;
    const auto us = std::chrono::duration_cast<std::chrono::microseconds>(
                        std::chrono::steady_clock::now() - t0)
                        .count();
    stats_.timing[uint8_t(c->hdr.op) & 127].add(uint64_t(us < 0 ? 0 : us));
    LOG_DEBUG("%s from conn %llu -> %d in %lld us", op_name(c->hdr.op),
              (unsigned long long)c->id, code, (long long)us);
    // A malformed request leaves the stream position well defined (the body was consumed),
    // so the connection stays usable; only protocol-level violations close it.
    return true;
}

int Server::handle_exchange(Conn* c) {
    if (c->body.size() != sizeof(ConnInfo)) {
        reply(c, kInvalidReq);
        return kInvalidReq;
    }
    std::memcpy(&c->peer, c->body.data(), sizeof(ConnInfo));
    ConnInfo me{};
    me.qpn = uint32_t(getpid());
    me.psn = uint32_t(segs_.size());
    std::memcpy(me.gid, fabric::process_uuid(), 16);
    me.lid = uint16_t((fabric::cuda_available() ? 1 : 0) | (use_hbm_ ? 2 : 0) |
                      (cfg_.evict ? 4 : 0) | (index_incomplete_ ? 8 : 0));
    me.mtu = kFabricVersion;
    reply(c, kFinish, &me, sizeof(me));
    return kFinish;
}

int Server::handle_pool_map(Conn* c) {
    uint32_t first = 0;
    if (c->body.size() >= sizeof(first)) std::memcpy(&first, c->body.data(), sizeof(first));
    std::vector<uint8_t> blob(sizeof(uint32_t));
    uint32_t count = 0;
    for (size_t i = first; i < segs_.size(); ++i) {
        const SegmentInfo& info = segs_[i]->info();
        const size_t at = blob.size();
        blob.resize(at + sizeof(SegmentInfo));
        std::memcpy(blob.data() + at, &info, sizeof(SegmentInfo));
        ++count;
    }
    std::memcpy(blob.data(), &count, sizeof(count));
    reply_blob(c, kFinish, blob.data(), blob.size());
    return kFinish;
}

int Server::handle_allocate(Conn* c, bool local) {
    std::vector<std::string_view> keys;
    int32_t block_size = 0;
    int hint = -1;
    if (local) {
        LocalMetaRequest req = decode_local_meta(c->body.data(), c->body.size());
        block_size = req.block_size;
        keys.reserve(req.blocks.size());
        for (auto& b : req.blocks) keys.push_back(b.key);
        hint = -1;
    } else {
        RemoteMetaRequest req = decode_remote_meta(c->body.data(), c->body.size());
        block_size = req.block_size;
        keys = std::move(req.keys);
        hint = req.hint;
    }
    if (block_size <= 0 || keys.empty()) {
        reply(c, kInvalidReq);
        return kInvalidReq;
    }
    std::vector<RemoteBlock> blocks;
    int code = store_->reserve(keys, size_t(block_size), hint, c->id, blocks);
    while (code == kOutOfMemory && maybe_extend())
        code = store_->reserve(keys, size_t(block_size), hint, c->id, blocks);
    if (code == kOutOfMemory && cfg_.evict) {
        // a full cache makes room for new blocks: least recently used first
        const size_t granule = size_t(cfg_.minimal_allocate_size) << 10;
        const size_t need = keys.size() * ((size_t(block_size) + granule - 1) / granule * granule);
        const size_t want = std::max(need, size_t(double(mm_.total_bytes()) * cfg_.evict_ratio));
        for (int round = 0; round < 16 && code == kOutOfMemory; ++round) {
            if (!evict_some(want, hint == kReplicaDevice)) break;
            code = store_->reserve(keys, size_t(block_size), hint, c->id, blocks);
        }
    }
    if (code != kFinish) {
        LOG_WARN("allocate of %zu x %d bytes failed: pool exhausted (%zu/%zu MiB used)",
                 keys.size(), block_size, mm_.used_bytes() >> 20, mm_.total_bytes() >> 20);
        reply(c, code);
        return code;
    }
    if (cfg_.auto_increase && mm_.need_extend()) maybe_extend();
    for (const RemoteBlock& rb : blocks) stats_.dedup_skips += is_fake_block(rb);
    const size_t need = blocks.size() * sizeof(RemoteBlock) + 64;
    if (scratch_.size() < need) scratch_.resize((need + 7) & ~size_t(7));
    fb::Builder b(scratch_.data(), scratch_.size() & ~size_t(7));
    encode_allocate_response(b, blocks.data(), blocks.size());
    reply_blob(c, local ? kTaskAccepted : kFinish, b.data(), b.size());
    return kFinish;
}

int Server::handle_lookup(Conn* c, bool local) {
    std::vector<std::string_view> keys;
    int32_t block_size = 0;
    if (local) {
        LocalMetaRequest req = decode_local_meta(c->body.data(), c->body.size());
        block_size = req.block_size;
        keys.reserve(req.blocks.size());
        for (auto& b : req.blocks) keys.push_back(b.key);
    } else {
        RemoteMetaRequest req = decode_remote_meta(c->body.data(), c->body.size());
        block_size = req.block_size;
        keys = std::move(req.keys);
    }
    if (block_size <= 0 || keys.empty()) {
        reply(c, kInvalidReq);
        return kInvalidReq;
    }
    std::vector<RemoteBlock> blocks;
    const int code = store_->lookup(keys, size_t(block_size), blocks, &c->leases);
    if (code != kFinish) {
        if (code == kKeyNotFound) stats_.lookup_misses++;
        reply(c, code);  // explicit error reply (the reference's RDMA path stays silent)
        return code;
    }
    stats_.lookup_hits += keys.size();
    const size_t need = blocks.size() * sizeof(RemoteBlock) + 64;
    if (scratch_.size() < need) scratch_.resize((need + 7) & ~size_t(7));
    fb::Builder b(scratch_.data(), scratch_.size() & ~size_t(7));
    encode_allocate_response(b, blocks.data(), blocks.size());
    reply_blob(c, local ? kTaskAccepted : kFinish, b.data(), b.size());
    return kFinish;
}

int Server::handle_stage_commit(Conn* c) {
    RemoteMetaRequest req = decode_remote_meta(c->body.data(), c->body.size());
    if (req.block_size < 0) {  // the writer's kernels failed: nothing of it becomes visible
        // the staged blocks (plus any the client names) are released right away, device-index
        // entries included: the in-band commit may already have published some of them
        std::vector<KVStore::Victim> victims;
        store_->drop_inflight(c->staged.data(), c->staged.size(), c->id, &victims);
        store_->drop_inflight(req.remote_addrs.data(), req.remote_addrs.size(), c->id, &victims);
        release_dropped(victims);
        c->staged.clear();
        return kFinish;
    }
    if (c->staged.size() + req.remote_addrs.size() > (size_t(1) << 24)) {
        LOG_WARN("conn %llu stages too many commits: dropped", (unsigned long long)c->id);
        c->staged.clear();
        return kInvalidReq;
    }
    if (req.rkey) note_publish_failures(req.rkey);
    store_->warm(req.remote_addrs.data(), req.remote_addrs.size());
    c->staged.insert(c->staged.end(), req.remote_addrs.begin(), req.remote_addrs.end());
    return kFinish;  // no reply: applied by the next SYNC of this connection
}

int Server::handle_commit(Conn* c) {
    RemoteMetaRequest req = decode_remote_meta(c->body.data(), c->body.size());
    if (req.rkey) note_publish_failures(req.rkey);
    store_->commit(req.remote_addrs.data(), req.remote_addrs.size());
    return kFinish;  // no reply: ordered before the client's next SYNC on this connection
}

int Server::handle_check_exist(Conn* c) {
    const std::string_view key(reinterpret_cast<const char*>(c->body.data()), c->body.size());
    const int32_t v = store_->exists_committed(key) ? 0 : 1;
    reply(c, kFinish, &v, sizeof(v));
    return kFinish;
}

int Server::handle_touch(Conn* c) {
    std::vector<std::string_view> keys = decode_match_request(c->body.data(), c->body.size());
    const int32_t n = int32_t(store_->touch(keys));
    reply(c, kFinish, &n, sizeof(n));
    return kFinish;
}

int Server::handle_match(Conn* c) {
    std::vector<std::string_view> keys = decode_match_request(c->body.data(), c->body.size());
    const int32_t idx = store_->match_last_index(keys);
    reply(c, kFinish, &idx, sizeof(idx));
    return kFinish;
}

}  // namespace istore
