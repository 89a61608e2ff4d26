#include "client.h"

#include <arpa/inet.h>
#include <cuda_runtime_api.h>
#include <netdb.h>
#include <netinet/in.h>
#include <netinet/tcp.h>
#include <sys/socket.h>
#include <sys/time.h>
#include <sys/uio.h>
#include <unistd.h>

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

namespace {
bool send_all(int fd, const iovec* iov_in, int iovcnt) {
    iovec iov[4];
    for (int i = 0; i < iovcnt; ++i) iov[i] = iov_in[i];
    int first = 0;
    while (first < iovcnt) {
        msghdr mh{};
        mh.msg_iov = iov + first;
        mh.msg_iovlen = size_t(iovcnt - first);
        ssize_t n = sendmsg(fd, &mh, MSG_NOSIGNAL);
        if (n < 0) {
            if (errno == EINTR) continue;
            return false;
        }
        while (n > 0 && first < iovcnt) {
            if (size_t(n) >= iov[first].iov_len) {
                n -= ssize_t(iov[first].iov_len);
                ++first;
            } else {
                iov[first].iov_base = static_cast<uint8_t*>(iov[first].iov_base) + n;
                iov[first].iov_len -= size_t(n);
                n = 0;
            }
        }
        while (first < iovcnt && iov[first].iov_len == 0) ++first;
    }
    return true;
}

bool recv_all(int fd, void* buf, size_t len) {
    uint8_t* p = static_cast<uint8_t*>(buf);
    while (len) {
        const ssize_t n = recv(fd, p, len, 0);
        if (n == 0) return false;
        if (n < 0) {
            if (errno == EINTR) continue;
            return false;
        }
        p += n;
        len -= size_t(n);
    }
    return true;
}

}  // namespace

void PendingHashes::grow() {
    std::vector<Entry> old;
    old.swap(slots_);
    slots_.assign(old.empty() ? 1024 : old.size() * 2, Entry{});
    count_ = 0;
    for (auto& sl : old)
        if (sl.addr) map_put(sl.addr, sl.h);
}

void PendingHashes::map_put(uint64_t addr, const KeyHash& h) {
    if ((count_ + 1) * 2 > slots_.size()) grow();
    const size_t mask = slots_.size() - 1;
    size_t i = mix(addr) & mask;
    while (slots_[i].addr && slots_[i].addr != addr) i = (i + 1) & mask;
    if (!slots_[i].addr) ++count_;
    slots_[i].addr = addr;
    slots_[i].h = h;
}

bool PendingHashes::map_take(uint64_t addr, KeyHash* out) {
    if (slots_.empty() || count_ == 0) return false;
    const size_t mask = slots_.size() - 1;
    size_t i = mix(addr) & mask;
    while (slots_[i].addr != addr) {
        if (!slots_[i].addr) return false;
        i = (i + 1) & mask;
    }
    *out = slots_[i].h;
    // backward-shift deletion keeps probe sequences intact without tombstones
    size_t j = i;
    for (;;) {
        j = (j + 1) & mask;
        if (!slots_[j].addr) break;
        const size_t home = mix(slots_[j].addr) & mask;
        if ((i <= j) ? (home <= i || home > j) : (home <= i && home > j)) {
            slots_[i] = slots_[j];
            i = j;
        }
    }
    slots_[i].addr = 0;
    --count_;
    return true;
}

void PendingHashes::spill() {
    for (size_t i = head_; i < fifo_.size(); ++i) map_put(fifo_[i].addr, fifo_[i].h);
    fifo_.clear();
    head_ = 0;
}

bool PendingHashes::take(uint64_t addr, KeyHash* out) {
    if (head_ < fifo_.size()) {
        if (fifo_[head_].addr == addr) {  // in allocation order: the common case
            *out = fifo_[head_].h;
            if (++head_ == fifo_.size()) {
                fifo_.clear();
                head_ = 0;
            }
            return true;
        }
        spill();  // out of order: from here on look the blocks up by address
    }
    return map_take(addr, out);
}

struct Connection::Task {
    enum Kind { kAllocate, kWaitEvent, kStop } kind = kWaitEvent;
    // allocate
    std::vector<std::string> keys;
    int block_size = 0;
    std::function<void(std::vector<RemoteBlock>)> alloc_cb;
    // wait for device work, then commit + callback
    int device = -1;
    cudaEvent_t event = nullptr;
    int status = 0;
    bool commit = false;
    std::vector<uint64_t> commits;  // addresses written by exactly this task's launches
    std::function<void(int)> done_cb;

    // Complete with the launches of `res`: an event recorded behind them on their stream,
    // or, when there is no event, a wait for the whole stream now.
    void wait_for(const MoveResult& res) {
        DeviceGuard g(res.device);
        if (cudaEventCreateWithFlags(&event, cudaEventDisableTiming) == cudaSuccess &&
            cudaEventRecord(event, static_cast<cudaStream_t>(res.stream)) == cudaSuccess) {
            device = res.device;
            return;
        }
        if (event) cudaEventDestroy(event);
        event = nullptr;
        (void)cudaGetLastError();
        if (cudaStreamSynchronize(static_cast<cudaStream_t>(res.stream)) != cudaSuccess) status = -1;
    }
};

Connection::Connection() {}

Connection::~Connection() { close(); }

void Connection::fail(const std::string& msg) {
    last_error_ = msg;
    LOG_ERROR("%s", msg.c_str());
}

ClientStats Connection::stats() const { return stats_; }

// ---------------------------------------------------------------- control plane

int Connection::init_connection(const ClientConfig& cfg) {
    cfg_ = cfg;
    if (fd_ >= 0) return 0;
    addrinfo hints{};
    hints.ai_family = AF_INET;
    hints.ai_socktype = SOCK_STREAM;
    addrinfo* res = nullptr;
    const std::string port = std::to_string(cfg.service_port);
    if (getaddrinfo(cfg.host_addr.c_str(), port.c_str(), &hints, &res) != 0 || !res) {
        fail("cannot resolve " + cfg.host_addr);
        return -1;
    }
    int fd = -1;
    for (addrinfo* ai = res; ai; ai = ai->ai_next) {
        fd = socket(ai->ai_family, ai->ai_socktype | SOCK_CLOEXEC, ai->ai_protocol);
        if (fd < 0) continue;
        if (connect(fd, ai->ai_addr, ai->ai_addrlen) == 0) break;
        ::close(fd);
        fd = -1;
    }
    freeaddrinfo(res);
    if (fd < 0) {
        fail("cannot connect to " + cfg.host_addr + ":" + port + ": " + std::strerror(errno));
        return -1;
    }
    int one = 1;
    setsockopt(fd, IPPROTO_TCP, TCP_NODELAY, &one, sizeof(one));
    timeval tv{};
    tv.tv_sec = cfg.timeout_ms / 1000;
    tv.tv_usec = (cfg.timeout_ms % 1000) * 1000;
    setsockopt(fd, SOL_SOCKET, SO_RCVTIMEO, &tv, sizeof(tv));
    setsockopt(fd, SOL_SOCKET, SO_SNDTIMEO, &tv, sizeof(tv));
    fd_ = fd;

    ConnInfo me{};
    me.qpn = uint32_t(getpid());
    me.psn = cfg.device >= 0 ? uint32_t(cfg.device) : 0xffffffffu;
    std::memcpy(me.gid, fabric::process_uuid(), 16);
    me.lid = fabric::cuda_available() ? 1 : 0;
    me.mtu = kFabricVersion;
    int32_t code = 0;
    std::vector<uint8_t> payload;
    if (transact(kOpExchange, &me, sizeof(me), &code, &payload, sizeof(ConnInfo)) != 0 ||
        code != kFinish) {
        fail("fabric exchange with the server failed");
        close();
        return -1;
    }
    ConnInfo srv{};
    std::memcpy(&srv, payload.data(), sizeof(srv));
    if (srv.mtu != kFabricVersion) {
        fail("server speaks fabric protocol v" + std::to_string(srv.mtu));
        close();
        return -1;
    }
    server_cuda_ = srv.lid & 1;
    server_hbm_ = srv.lid & 2;
    server_evicts_ = srv.lid & 4;
    index_incomplete_.store((srv.lid & 8) != 0, std::memory_order_relaxed);
    std::memcpy(server_uuid_, srv.gid, 16);
    if (!worker_.joinable()) {
        stop_ = false;
        worker_ = std::thread([this] { worker(); });
    }
    return 0;
}

int Connection::setup_rdma(const ClientConfig&) {
    if (fd_ < 0) return -1;
    // The HBM pool is the fast path: look keys up on the GPU unless told otherwise.
    device_lookup_ = false;
    return refresh_pool_map();
}

void Connection::close() {
    if (worker_.joinable()) {
        {
            std::lock_guard<std::mutex> lk(q_mu_);
            stop_ = true;
            Task t;
            t.kind = Task::kStop;
            queue_.push_back(std::move(t));
        }
        q_cv_.notify_all();
        worker_.join();
    }
    {
        std::lock_guard<std::mutex> lk(mu_);
        ++session_;  // writers of this session must not touch the released blocks
        for (auto& kv : devs_) kv.second->wait_all();
        devs_.clear();
        host_maps_.clear();
        for (auto& kv : host_regs_)
            if (kv.second.registered) cudaHostUnregister(reinterpret_cast<void*>(kv.first));
        host_regs_.clear();
    }
    if (fd_ >= 0) {
        ::close(fd_);
        fd_ = -1;
    }
}

// One request/response exchange.  fixed_payload: bytes following the code on success, or
// kBlobPayload for "u32 length + blob".
int Connection::transact(char op, const void* body, size_t len, int32_t* code,
                         std::vector<uint8_t>* payload, size_t fixed_payload,
                         const std::vector<uint8_t>* prefix) {
    std::lock_guard<std::mutex> lk(sock_mu_);
    if (fd_ < 0) return -1;
    Header h{kMagic, op, uint32_t(len)};
    // `prefix`: already framed reply-less messages (COMMIT) that go out in the same segment
    iovec iov[3];
    int niov = 0;
    if (prefix && !prefix->empty())
        iov[niov++] = iovec{const_cast<uint8_t*>(prefix->data()), prefix->size()};
    iov[niov++] = iovec{&h, sizeof(h)};
    if (len) iov[niov++] = iovec{const_cast<void*>(body), len};
    // A transaction that breaks half way (send error, reply timeout, short reply) leaves the
    // byte stream in an unknown position: a late reply would be taken for the answer to the
    // NEXT request.  The connection is closed instead; later calls fail fast.
    auto broken = [&](const std::string& why) {
        fail(why);
        ::shutdown(fd_, SHUT_RDWR);
        ::close(fd_);
        fd_ = -1;
        return -1;
    };
    if (!send_all(fd_, iov, niov))
        return broken(std::string("send ") + op_name(op) + ": " + std::strerror(errno));
    stats_.ctrl_requests++;
    if (!recv_all(fd_, code, sizeof(*code)))
        return broken(std::string("no reply to ") + op_name(op) +
                      " (timeout or connection closed): connection dropped");
    if (payload) payload->clear();
    if (*code != kFinish && *code != kTaskAccepted) return 0;  // error replies carry no payload
    if (fixed_payload == kBlobPayload) {
        uint32_t n = 0;
        if (!recv_all(fd_, &n, sizeof(n)) || n > kMaxBody + 4096)
            return broken(std::string("short reply to ") + op_name(op));
        payload->resize(n);
        if (n && !recv_all(fd_, payload->data(), n))
            return broken(std::string("short reply to ") + op_name(op));
    } else if (fixed_payload) {
        payload->resize(fixed_payload);
        if (!recv_all(fd_, payload->data(), fixed_payload))
            return broken(std::string("short reply to ") + op_name(op));
    }
    return 0;
}

int Connection::send_raw(const void* framed, size_t len) {
    std::lock_guard<std::mutex> lk(sock_mu_);
    if (fd_ < 0) return -1;
    iovec iov[1] = {{const_cast<void*>(framed), len}};
    if (!send_all(fd_, iov, 1)) return -1;
    stats_.ctrl_requests++;
    return 0;
}

int Connection::send_only(char op, const void* body, size_t len) {
    std::lock_guard<std::mutex> lk(sock_mu_);
    if (fd_ < 0) return -1;
    Header h{kMagic, op, uint32_t(len)};
    iovec iov[2] = {{&h, sizeof(h)}, {const_cast<void*>(body), len}};
    if (!send_all(fd_, iov, len ? 2 : 1)) return -1;
    stats_.ctrl_requests++;
    return 0;
}

int Connection::refresh_pool_map() {
    const uint32_t first = uint32_t(segs_.size());
    int32_t code = 0;
    std::vector<uint8_t> blob;
    if (transact(kOpPoolMap, &first, sizeof(first), &code, &blob, kBlobPayload) != 0 ||
        code != kFinish || blob.size() < 4)
        return -1;
    uint32_t count = 0;
    std::memcpy(&count, blob.data(), 4);
    if (blob.size() != 4 + size_t(count) * sizeof(SegmentInfo)) return -1;
    for (uint32_t i = 0; i < count; ++i) {
        SegmentInfo s;
        std::memcpy(&s, blob.data() + 4 + size_t(i) * sizeof(SegmentInfo), sizeof(s));
        segs_.push_back(s);
    }
    return 0;
}

// The kernels resolve at most kMaxSegs segment bases; a pool that auto-increased beyond that
// is served through the control plane (authoritative anyway).
bool Connection::device_index_usable() {
    if (segs_.empty() || !segs_[0].index_slots) return false;
    // Some writer could not publish a block in the HBM index (both of the key's buckets were
    // full): that key is reachable through the server only, so every read of this connection
    // resolves through the server from now on instead of reporting a false miss.
    if (index_incomplete_.load(std::memory_order_relaxed)) return false;
    return segs_.size() <= size_t(kernels::LookupLaunch::kMaxSegs);
}

int Connection::check_exist(const std::string& key) {
    if (device_lookup_ && server_hbm_ && device_index_usable()) {
        const int r = match_via_device_index({std::string_view(key)}, true);
        if (r >= -1) return r == 0 ? 0 : 1;
    }
    int32_t code = 0;
    std::vector<uint8_t> p;
    if (transact(kOpCheckExist, key.data(), key.size(), &code, &p, sizeof(int32_t)) != 0 ||
        code != kFinish)
        return -1;
    int32_t v;
    std::memcpy(&v, p.data(), sizeof(v));
    return v;
}

int Connection::get_match_last_index(const std::vector<std::string_view>& keys) {
    if (keys.empty()) return -1;
    if (device_lookup_ && server_hbm_ && device_index_usable()) {
        const int r = match_via_device_index(keys, false);
        if (r >= -1) return r;
    }
    const std::vector<std::string_view>& kv = keys;
    std::vector<uint8_t> buf(remote_meta_bound(kv, 0));
    fb::Builder b(buf.data(), buf.size());
    encode_match_request(b, kv);
    int32_t code = 0;
    std::vector<uint8_t> p;
    if (transact(kOpMatchLastIdx, b.data(), b.size(), &code, &p, sizeof(int32_t)) != 0 ||
        code != kFinish)
        return -2;
    int32_t v;
    std::memcpy(&v, p.data(), sizeof(v));
    return v;
}

// A device-side miss on a path that makes no SYNC round trip: ask the server whether the HBM
// index is complete - if a writer overflowed it, the key may exist all the same, and from now
// on this connection resolves its reads through the server.
void Connection::refresh_index_state() {
    if (index_incomplete_.load(std::memory_order_relaxed)) return;
    int32_t code = 0;
    std::vector<uint8_t> p;
    if (transact(kOpSync, nullptr, 0, &code, &p, sizeof(uint32_t)) == 0 && code == kFinish &&
        p.size() == sizeof(uint32_t)) {
        uint32_t remain;
        std::memcpy(&remain, p.data(), sizeof(remain));
        if (remain & kSyncIndexIncomplete) index_incomplete_.store(true, std::memory_order_relaxed);
    }
}

int Connection::sync_local() {
    NvtxRange nvtx("istore.sync");
    // one sync at a time: a staged commit list and the SYNC that applies it belong together
    std::lock_guard<std::mutex> sync_lk(sync_mu_);
    {
        // Nothing to tell the server (no commits pending, no leases held by host-mediated
        // lookups): completion of the kernels is all there is to wait for.
        bool quiet;
        {
            std::lock_guard<std::mutex> lk(mu_);
            quiet = pending_commit_.empty() && !ctrl_dirty_;
        }
        bool async_idle;
        {
            std::lock_guard<std::mutex> lk(q_mu_);
            async_idle = inflight_async_ == 0;
        }
        if (quiet && async_idle) {
            const int drained = drain_devices();
            if (drained == -kKeyNotFound) refresh_index_state();
            return drained != 0 ? drained : 0;
        }
    }
    if (cfg_.posted_commit) {
        bool leases;
        {
            std::lock_guard<std::mutex> lk(mu_);
            leases = ctrl_dirty_;
        }
        if (!leases) {
            // Posted commit: wait for the kernels, then send the commit list one-way.  The
            // blocks are already visible to device-path readers (in-band commit); the server's
            // map follows when the message arrives - no round trip on the caller's path.
            std::vector<uint64_t> mine;
            {
                std::lock_guard<std::mutex> lk(mu_);
                mine.swap(pending_commit_);
            }
            bool device_error = false;
            const int drained = drain_devices(&device_error);
            if (device_error) {
                (void)discard_blocks(mine.data(), mine.size());
                return -1;
            }
            if (!mine.empty() && send_commit(mine.data(), mine.size()) != 0) return -1;
            if (drained == -kKeyNotFound) refresh_index_state();
            return drained;
        }
    }
    // The commit list is taken BEFORE waiting for the GPU, so it names only blocks whose
    // kernels the drain below covers, and it is shipped right away as a STAGED commit: the
    // server decodes it and pulls the block headers into its cache while this thread waits
    // for the kernels; the SYNC that follows the drain applies it.
    std::vector<uint64_t> addrs;
    {
        std::lock_guard<std::mutex> lk(mu_);
        addrs.swap(pending_commit_);
    }
    constexpr size_t kInline = 128 * 1024;  // addresses; larger lists use the chunked path
    auto frame_of = [&](char op, int32_t block_size, const uint64_t* a, size_t n) {
        std::vector<uint8_t> buf(align_up(n * 8 + 128, 8));
        fb::Builder b(buf.data(), buf.size());
        encode_remote_meta(b, {}, block_size, block_size >= 0 ? take_publish_failures() : 0, a, n, op);
        std::vector<uint8_t> framed(sizeof(Header) + b.size());
        Header ch{kMagic, op, uint32_t(b.size())};
        std::memcpy(framed.data(), &ch, sizeof(ch));
        std::memcpy(framed.data() + sizeof(ch), b.data(), b.size());
        return framed;
    };
    bool staged = false;
    if (!addrs.empty() && addrs.size() <= kInline) {
        const std::vector<uint8_t> f = frame_of(kOpStageCommit, 0, addrs.data(), addrs.size());
        if (send_raw(f.data(), f.size()) != 0) {
            fail("commit: send failed");
            return -1;
        }
        staged = true;
    }
    bool device_error = false;
    const int drained = drain_devices(&device_error);
    if (device_error) {
        // The data of these blocks may not have landed, while the in-band commit may already
        // have published some of them in the device index: the server releases them now,
        // index entries included (reservations it cannot match die with the connection).
        if (staged) {
            const std::vector<uint8_t> f = frame_of(kOpStageCommit, -1, nullptr, 0);
            (void)send_raw(f.data(), f.size());
        } else {
            (void)discard_blocks(addrs.data(), addrs.size());
        }
        return -1;
    }
    // A read that missed (drained < 0 without a device error) does not undo the writes of
    // the same window: their kernels completed, so their commits are applied all the same.
    std::vector<uint8_t> framed;  // reply-less messages that travel with the SYNC
    if (!staged && !addrs.empty() && send_commit(addrs.data(), addrs.size()) != 0) return -1;
    if (const uint32_t pf = take_publish_failures()) {
        // index insertions that failed are known only now (after the drain): an empty COMMIT
        // carries the count, ahead of the SYNC in the same segment
        std::vector<uint8_t> buf(256);
        fb::Builder b(buf.data(), buf.size());
        encode_remote_meta(b, {}, 0, pf, nullptr, 0, kOpCommit);
        framed.resize(sizeof(Header) + b.size());
        Header ch{kMagic, kOpCommit, uint32_t(b.size())};
        std::memcpy(framed.data(), &ch, sizeof(ch));
        std::memcpy(framed.data() + sizeof(ch), b.data(), b.size());
    }
    int32_t code = 0;
    std::vector<uint8_t> p;
    if (transact(kOpSync, nullptr, 0, &code, &p, sizeof(uint32_t), &framed) != 0 ||
        code != kFinish)
        return -1;
    {
        std::lock_guard<std::mutex> lk(mu_);
        ctrl_dirty_ = false;
    }
    if (drained != 0) return drained;
    uint32_t remain;
    std::memcpy(&remain, p.data(), sizeof(remain));
    if (remain & kSyncIndexIncomplete) index_incomplete_.store(true, std::memory_order_relaxed);
    return int(remain & ~kSyncIndexIncomplete);
}

int Connection::sync_rdma() {
    {  // async operations first: their completions append to the commit list
        std::unique_lock<std::mutex> lk(q_mu_);
        if (!idle_cv_.wait_for(lk, std::chrono::milliseconds(cfg_.timeout_ms),
                               [this] { return inflight_async_ == 0; })) {
            fail("sync: timed out waiting for asynchronous operations");
            return -1;
        }
    }
    const int r = sync_local();
    return r < 0 ? r : 0;
}

int Connection::send_commit(const uint64_t* addrs, size_t count) {
    // chunk so that one message stays far below the body cap
    constexpr size_t kChunk = 256 * 1024;
    for (size_t at = 0; at < count; at += kChunk) {
        const size_t n = std::min(kChunk, count - at);
        std::vector<uint8_t> buf(align_up(n * 8 + 128, 8));
        fb::Builder b(buf.data(), buf.size());
        // rkey (unused by COMMIT in the reference) reports index insertions that failed
        encode_remote_meta(b, {}, 0, take_publish_failures(), addrs + at, n, kOpCommit);
        if (send_only(kOpCommit, b.data(), b.size()) != 0) {
            fail("commit: send failed");
            return -1;
        }
    }
    return 0;
}

int Connection::discard_blocks(const uint64_t* addrs, size_t count) {
    constexpr size_t kChunk = 256 * 1024;
    for (size_t at = 0; at < count; at += kChunk) {
        const size_t n = std::min(kChunk, count - at);
        std::vector<uint8_t> buf(align_up(n * 8 + 128, 8));
        fb::Builder b(buf.data(), buf.size());
        encode_remote_meta(b, {}, -1, 0, addrs + at, n, kOpStageCommit);
        if (send_only(kOpStageCommit, b.data(), b.size()) != 0) return -1;
    }
    return 0;
}

uint32_t Connection::take_publish_failures() {
    std::lock_guard<std::mutex> lk(mu_);
    const uint32_t n = publish_failures_;
    publish_failures_ = 0;
    return n;
}

int Connection::flush_commits() {
    std::vector<uint64_t> addrs;
    {
        std::lock_guard<std::mutex> lk(mu_);
        addrs.swap(pending_commit_);
    }
    if (addrs.empty()) return 0;
    return send_commit(addrs.data(), addrs.size());
}

// One control-plane message holds at most kMaxBody bytes: large key lists are sent in chunks.
static std::vector<std::pair<size_t, size_t>> chunk_keys(const std::vector<std::string_view>& keys) {
    constexpr size_t kBudget = 3u << 20;
    std::vector<std::pair<size_t, size_t>> out;
    size_t begin = 0, bytes = 0;
    for (size_t i = 0; i < keys.size(); ++i) {
        const size_t need = keys[i].size() + 16;
        if (bytes + need > kBudget && i > begin) {
            out.emplace_back(begin, i);
            begin = i;
            bytes = 0;
        }
        bytes += need;
    }
    if (begin < keys.size()) out.emplace_back(begin, keys.size());
    return out;
}

int Connection::allocate(const std::vector<std::string_view>& keys, int block_size,
                         std::vector<RemoteBlock>& out, int hint) {
    out.clear();
    if (keys.empty() || block_size <= 0) return -1;
    out.reserve(keys.size());
    for (auto [b0, b1] : chunk_keys(keys)) {
        const std::vector<std::string_view> kv(keys.begin() + b0, keys.begin() + b1);
        std::vector<uint8_t> buf(remote_meta_bound(kv, 0));
        fb::Builder b(buf.data(), buf.size());
        encode_remote_meta(b, kv, block_size, 0, nullptr, 0, kOpAllocate,
                           hint == kHintDefault ? cfg_.pool_hint : hint);
        int32_t code = 0;
        std::vector<uint8_t> p;
        if (transact(kOpAllocate, b.data(), b.size(), &code, &p, kBlobPayload) != 0) return -1;
        if (code != kFinish) {
            // blocks reserved by earlier chunks stay reserved-uncommitted; the server releases
            // them when this connection closes
            fail("allocate: server returned " + std::to_string(code));
            out.clear();
            return -code;
        }
        std::vector<RemoteBlock> part;
        try {
            part = decode_allocate_response(p.data(), p.size());
        } catch (const std::exception& e) {
            fail(std::string("allocate: bad reply: ") + e.what());
            out.clear();
            return -1;
        }
        if (part.size() != kv.size()) {
            out.clear();
            return -1;
        }
        out.insert(out.end(), part.begin(), part.end());
    }
    if (server_hbm_) {  // remember fingerprints: the write kernel publishes them in-band
        std::lock_guard<std::mutex> lk(mu_);
        for (size_t i = 0; i < keys.size(); ++i) {
            if (is_fake_block(out[i])) continue;
            pending_hash_.put(out[i].remote_addr,
                              hash_key(reinterpret_cast<const uint8_t*>(keys[i].data()),
                                       keys[i].size()));
        }
    }
    return 0;
}

int Connection::touch(const std::vector<std::string_view>& keys) {
    if (keys.empty()) return 0;
    int total = 0;
    for (auto [b0, b1] : chunk_keys(keys)) {
        const std::vector<std::string_view> kv(keys.begin() + b0, keys.begin() + b1);
        std::vector<uint8_t> buf(remote_meta_bound(kv, 0));
        fb::Builder b(buf.data(), buf.size());
        encode_match_request(b, kv);
        int32_t code = 0;
        std::vector<uint8_t> p;
        if (transact(kOpTouch, b.data(), b.size(), &code, &p, sizeof(int32_t)) != 0 ||
            code != kFinish)
            return -1;
        int32_t v;
        std::memcpy(&v, p.data(), sizeof(v));
        total += v;
    }
    return total;
}

int Connection::lookup_blocks(char op, const std::vector<KeyOffset>& blocks, int block_size,
                              std::vector<RemoteBlock>& out) {
    {
        std::lock_guard<std::mutex> lk(mu_);
        ctrl_dirty_ = true;  // the server pins looked-up blocks until our next SYNC
    }
    int32_t code = 0;
    std::vector<uint8_t> p;
    if (op == kOpLocalRead || op == kOpLocalWrite) {
        std::vector<LocalBlock> lb(blocks.size());
        for (size_t i = 0; i < blocks.size(); ++i) lb[i] = LocalBlock{blocks[i].key, blocks[i].offset};
        std::vector<uint8_t> buf(local_meta_bound(lb));
        fb::Builder b(buf.data(), buf.size());
        encode_local_meta(b, std::max(default_device_, 0), std::string_view(), block_size, lb);
        if (transact(op, b.data(), b.size(), &code, &p, kBlobPayload) != 0) return -1;
    } else {
        std::vector<std::string_view> all;
        all.reserve(blocks.size());
        for (auto& kb : blocks) all.push_back(kb.key);
        const auto chunks = chunk_keys(all);
        if (chunks.size() > 1) {  // very large batch: one request per chunk
            out.clear();
            for (auto [b0, b1] : chunks) {
                const std::vector<std::string_view> kv(all.begin() + b0, all.begin() + b1);
                std::vector<uint8_t> buf(remote_meta_bound(kv, 0));
                fb::Builder b(buf.data(), buf.size());
                encode_remote_meta(b, kv, block_size, 0, nullptr, 0, op, cfg_.pool_hint);
                if (transact(op, b.data(), b.size(), &code, &p, kBlobPayload) != 0) return -1;
                if (code != kFinish && code != kTaskAccepted) {
                    last_error_ = std::string(op_name(op)) + ": server returned " + std::to_string(code);
                    return -code;
                }
                try {
                    auto part = decode_allocate_response(p.data(), p.size());
                    out.insert(out.end(), part.begin(), part.end());
                } catch (const std::exception& e) {
                    fail(std::string("bad reply: ") + e.what());
                    return -1;
                }
            }
            return out.size() == blocks.size() ? 0 : -1;
        }
        std::vector<uint8_t> buf(remote_meta_bound(all, 0));
        fb::Builder b(buf.data(), buf.size());
        encode_remote_meta(b, all, block_size, 0, nullptr, 0, op, cfg_.pool_hint);
        if (transact(op, b.data(), b.size(), &code, &p, kBlobPayload) != 0) return -1;
    }
    if (code != kFinish && code != kTaskAccepted) {
        last_error_ = std::string(op_name(op)) + ": server returned " + std::to_string(code);
        return -code;
    }
    try {
        out = decode_allocate_response(p.data(), p.size());
    } catch (const std::exception& e) {
        fail(std::string("bad reply: ") + e.what());
        return -1;
    }
    return out.size() == blocks.size() ? 0 : -1;
}

// ---------------------------------------------------------------- data plane

// ---------------------------------------------------------------- async API

void Connection::post(Task&& t) {
    {
        std::lock_guard<std::mutex> lk(q_mu_);
        queue_.push_back(std::move(t));
        ++inflight_async_;
    }
    q_cv_.notify_one();
}

void Connection::worker() {
    for (;;) {
        Task t;
        {
            std::unique_lock<std::mutex> lk(q_mu_);
            q_cv_.wait(lk, [this] { return !queue_.empty(); });
            t = std::move(queue_.front());
            queue_.pop_front();
        }
        if (t.kind == Task::kStop) return;
        if (t.kind == Task::kAllocate) {
            std::vector<RemoteBlock> out;
            std::vector<std::string_view> kv(t.keys.begin(), t.keys.end());
            if (allocate(kv, t.block_size, out) != 0) out.clear();
            if (t.alloc_cb) t.alloc_cb(std::move(out));
        } else {
            int status = t.status;
            if (t.event) {
                DeviceGuard g(t.device);
                if (cudaEventSynchronize(t.event) != cudaSuccess) status = -1;
                cudaEventDestroy(t.event);
            }
            if (t.commit && !t.commits.empty()) {
                if (status == 0) {
                    if (send_commit(t.commits.data(), t.commits.size()) != 0) status = -1;
                } else {
                    // this write's kernels failed: its blocks must never become visible
                    discard_blocks(t.commits.data(), t.commits.size());
                }
            }
            if (t.done_cb) t.done_cb(status);
        }
        {
            std::lock_guard<std::mutex> lk(q_mu_);
            --inflight_async_;
        }
        idle_cv_.notify_all();
    }
}

int Connection::allocate_async(const std::vector<std::string>& keys, int block_size,
                               std::function<void(std::vector<RemoteBlock>)> cb) {
    Task t;
    t.kind = Task::kAllocate;
    t.keys = keys;
    t.block_size = block_size;
    t.alloc_cb = std::move(cb);
    post(std::move(t));
    return 0;
}

int Connection::w_rdma_async(const std::vector<uint64_t>& offsets, int block_size,
                             const RemoteBlock* blocks, size_t nblocks, uint64_t base_ptr,
                             int device, uint64_t stream, std::function<void(int)> cb) {
    // The task owns the addresses of exactly the blocks this call wrote; its completion
    // commits those and no others (later writes of the connection may still be in flight on
    // other streams).  The event is recorded on the stream this call launched on.
    Task t;
    t.kind = Task::kWaitEvent;
    t.commit = true;
    MoveResult res;
    res.commits = &t.commits;
    const int r = w_rdma(offsets.data(), offsets.size(), 1, block_size, blocks, nblocks, base_ptr,
                         device, stream, &res);
    t.status = r;
    t.done_cb = std::move(cb);
    if (res.launched && res.device >= 0) t.wait_for(res);  // the commit waits for it
    post(std::move(t));
    return r;
}

int Connection::r_rdma_async(const std::vector<KeyOffset>& blocks, int block_size,
                             uint64_t base_ptr, int device, uint64_t stream,
                             std::function<void(int)> cb) {
    MoveResult res;
    const int r = r_rdma(blocks, block_size, base_ptr, device, stream, &res);
    Task t;
    t.kind = Task::kWaitEvent;
    t.status = r;
    t.done_cb = std::move(cb);
    if (r == 0 && res.launched && res.device >= 0) t.wait_for(res);
    post(std::move(t));
    return r;
}

}  // namespace istore
