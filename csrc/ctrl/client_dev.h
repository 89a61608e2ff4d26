// Private to the client's translation units (client.cpp: control plane, client_data.cpp: data
// plane, client_doorbell.cpp: latency mode): per-device state of a connection and small helpers.
#pragma once

#include <cuda_runtime_api.h>

#include <algorithm>
#include <atomic>
#include <chrono>
#include <cstring>
#include <memory>
#include <vector>

#include "../fabric/segment.h"
#include "../kernels/kernels.h"
#include "client.h"
#include "staging.h"

namespace istore {

inline constexpr size_t kBlobPayload = ~size_t(0);
inline constexpr size_t kRingBytes = 16u << 20;     // pinned, mapped staging ring per device
inline constexpr size_t kScratchBytes = 8u << 20;   // device scratch per device
inline constexpr size_t kZeroBytes = 2u << 20;      // self-cleaning zeroed counters per device
inline constexpr size_t kMaxBatch = 65536;          // blocks per kernel launch
// ring bytes one launch's piece tables may take (GatherSpec::rows.pieces): with a key batch's
// half of the ring, a launch's placements still never come round to each other
inline constexpr size_t kPieceRingBytes = kRingBytes / 4;
inline constexpr int kReaderSlots = 64;             // layered reads in flight per device

struct DeviceGuard {
    int prev = -1;
    explicit DeviceGuard(int dev) {
        if (cudaGetDevice(&prev) != cudaSuccess) prev = -1;
        if (dev >= 0 && dev != prev) cudaSetDevice(dev);
    }
    ~DeviceGuard() {
        if (prev >= 0) cudaSetDevice(prev);
    }
};

inline size_t align_up(size_t v, size_t a) { return (v + a - 1) & ~(a - 1); }

inline uint64_t now_ns() {
    return uint64_t(std::chrono::duration_cast<std::chrono::nanoseconds>(
                        std::chrono::steady_clock::now().time_since_epoch())
                        .count());
}

// A request line of the doorbell ring (kernels/kv_doorbell.cu): payload and checksum first,
// the word with the sequence number last - the worker accepts a line only when both match.
inline void doorbell_write_line(kernels::DoorbellReq* slot, uint64_t seq, uint32_t op,
                                const uint64_t (&q)[6]) {
    uint64_t line[8];
    line[0] = (seq << 2) | op;
    for (int i = 0; i < 6; ++i) line[1 + i] = q[i];
    uint64_t x = kernels::kDoorbellMagic;
    for (int i = 0; i < 7; ++i) x ^= line[i];
    line[7] = x;
    auto* dst = reinterpret_cast<volatile uint64_t*>(slot->q);
    for (int i = 1; i < 8; ++i) dst[i] = line[i];
    std::atomic_thread_fence(std::memory_order_release);
    dst[0] = line[0];
    std::atomic_thread_fence(std::memory_order_seq_cst);  // out of the store buffer now
}

// One launch's keys in the pinned ring, as the device reads them: packed the way the lookup
// kernels hash them (client.h: PackedKeys), with every block's destination offset.
struct StagedKeys {
    const uint8_t* bytes = nullptr;
    const uint32_t* off = nullptr;
    const uint32_t* len = nullptr;
    const uint64_t* dst = nullptr;
};

// Per-device data-plane state.
struct Connection::DevCtx {
    int device = -1;
    cudaStream_t stream = nullptr;
    std::vector<std::shared_ptr<fabric::Mapping>> maps;  // by segment id
    std::vector<uint8_t*> seg_ptr;  // maps[i]->dev_ptr, cached for the per-block hot loop
    std::vector<uint8_t> seg_remote;  // 1 when the segment is not in this device's own HBM
    std::vector<uint8_t*> seg_mc;     // NVLS replica segments: multicast base (writes)
    uint8_t* ring_h = nullptr;  // pinned + mapped: descriptors, publish records, key bytes
    uint8_t* ring_d = nullptr;
    uint8_t* scratch = nullptr;  // device memory: descriptors built by the lookup kernel
    uint8_t* zeros = nullptr;    // device memory kept zero between launches (counters/tickets)
    uint32_t* status_h = nullptr;
    uint32_t* status_d = nullptr;
    std::vector<cudaStream_t> busy;  // streams with launches since the last wait_all()
    bool dirty = false;
    // Layered reads (Connection::r_rdma_scatter with a reader): kReaderSlots slots of
    // kGatherMaxParts group flags, allocated and zeroed on the first such read; reader seq uses
    // slot seq % kReaderSlots (staging.h: ReaderSlots), whose event completes with its launches.
    uint32_t* group_flags = nullptr;
    ReaderSlots<cudaEvent_t, kReaderSlots> readers;
    cudaEvent_t reader_ev[kReaderSlots] = {};

    // Doorbell worker (ClientConfig::doorbell): request ring + control block in pinned,
    // device-mapped host memory; `posted` / `collected` are request numbers.
    struct Doorbell {
        kernels::DoorbellReq* ring_h = nullptr;
        kernels::DoorbellReq* ring_d = nullptr;
        kernels::DoorbellCtl* ctl_h = nullptr;
        kernels::DoorbellCtl* ctl_d = nullptr;
        cudaStream_t stream = nullptr;
        uint64_t posted = 0;     // last request written to the ring
        uint64_t collected = 0;  // statuses of requests <= collected have been taken
        uint32_t epoch = 0;      // launch counter
        bool running = false;    // a launch of `epoch` has not been seen to exit
        uint64_t next_serve = 1;  // first request the next launch serves
        size_t nsegs = 0;         // pool segments known when the running worker was launched
        uint32_t misses = 0, stale = 0, publish_failures = 0;  // since the last drain
    };
    std::unique_ptr<Doorbell> db;

    // Launch streams.  Back-to-back page-mover kernels of one connection are independent of
    // each other, but in a single stream the fixed head (launch, descriptor fetch) and tail
    // (store acks, fence, commit) of every kernel are exposed (bench/launch_overhead.py
    // measures them).  Round-robin over a few internal streams
    // lets the tail of one kernel overlap the body of the next.  Ordering: every launch
    // waits for the caller's stream (the pages are ready); reads / lookups additionally wait
    // for earlier writes of this connection; completion is established by sync().
    static constexpr int kMaxStreams = 8;
    cudaStream_t pool[kMaxStreams] = {nullptr};
    cudaEvent_t pool_ev[kMaxStreams] = {nullptr};
    uint64_t last_write[kMaxStreams] = {0};
    uint64_t joined[kMaxStreams] = {0};
    uint64_t write_epoch = 0;
    cudaEvent_t user_ev = nullptr;
    int nstreams = 0;
    int rr = 0;

    // Stream for the next launch.  nstreams == 0: the caller's stream itself (in-stream
    // semantics, CUDA-graph capturable).
    cudaStream_t pick(cudaStream_t user, bool is_write, int want_streams) {
        if (want_streams <= 0) return user ? user : stream;
        if (nstreams < want_streams) {
            for (int i = nstreams; i < want_streams && i < kMaxStreams; ++i) {
                cudaStreamCreateWithFlags(&pool[i], cudaStreamNonBlocking);
                cudaEventCreateWithFlags(&pool_ev[i], cudaEventDisableTiming);
            }
            nstreams = std::min(want_streams, int(kMaxStreams));
            if (!user_ev) cudaEventCreateWithFlags(&user_ev, cudaEventDisableTiming);
        }
        const int i = rr++ % nstreams;
        cudaStream_t s = pool[i];
        if (user) {  // run after whatever produced the pages
            cudaEventRecord(user_ev, user);
            cudaStreamWaitEvent(s, user_ev, 0);
        }
        if (is_write) {
            last_write[i] = ++write_epoch;
        } else if (joined[i] < write_epoch) {  // reads see this connection's earlier writes
            for (int w = 0; w < nstreams; ++w) {
                if (w == i || last_write[w] <= joined[i]) continue;
                cudaEventRecord(pool_ev[w], pool[w]);
                cudaStreamWaitEvent(s, pool_ev[w], 0);
            }
            joined[i] = write_epoch;
        }
        return s;
    }

    ~DevCtx() {
        DeviceGuard g(device);
        wait_all();
        if (db) {
            // the worker leaves on a STOP request (or by itself after its idle timeout)
            if (db->running && db->ring_h) {
                const uint64_t none[6] = {0, 0, 0, 0, 0, 0};
                const uint64_t seq = ++db->posted;
                doorbell_write_line(&db->ring_h[seq % kernels::kDoorbellMaxSlots], seq,
                                    kernels::kDoorbellStop, none);
            }
            if (db->stream) {
                cudaStreamSynchronize(db->stream);
                cudaStreamDestroy(db->stream);
            }
            if (db->ring_h) cudaFreeHost(db->ring_h);
            if (db->ctl_h) cudaFreeHost(db->ctl_h);
        }
        for (int i = 0; i < nstreams; ++i) {
            cudaStreamSynchronize(pool[i]);
            cudaStreamDestroy(pool[i]);
            cudaEventDestroy(pool_ev[i]);
        }
        if (user_ev) cudaEventDestroy(user_ev);
        for (cudaEvent_t ev; staging.take_free(&ev);) cudaEventDestroy(ev);
        for (cudaEvent_t ev : reader_ev)
            if (ev) cudaEventDestroy(ev);
        if (group_flags) cudaFree(group_flags);
        if (stream) {
            cudaStreamSynchronize(stream);
            cudaStreamDestroy(stream);
        }
        maps.clear();
        if (ring_h) cudaFreeHost(ring_h);
        if (status_h) cudaFreeHost(status_h);
        if (scratch) cudaFree(scratch);
        if (zeros) cudaFree(zeros);
    }

    // Completion of everything launched so far.  A blocking cudaStreamSynchronize sleeps on an
    // interrupt, whose wake-up is long next to a short transfer; short transfers are therefore
    // polled with cudaStreamQuery for a bounded time first.
    void wait_all() {
        DeviceGuard g(device);
        for (cudaStream_t s : busy) {
            bool done = false;
            const uint64_t t0 = now_ns();
            for (int spin = 0; spin < 4096; ++spin) {
                const cudaError_t q = cudaStreamQuery(s);
                if (q != cudaErrorNotReady) {  // finished, or failed: let synchronize report it
                    done = q == cudaSuccess;
                    break;
                }
                if ((spin & 15) == 15 && now_ns() - t0 > 60000) break;  // 60 us: not a short one
            }
            if (!done) cudaStreamSynchronize(s);
        }
        busy.clear();
        dirty = false;
        staging.retire_all();
        readers.retire_all();
    }
    cudaStream_t last = nullptr;  // stream of the most recent launch
    // Staging reuse (staging.h): one event per launch, recorded behind it on its stream.  A
    // launch leaves the FIFO at wait_all() or when its bytes come round, so the FIFO holds at
    // most one lap of launches; their events are recycled.
    enum { kRing, kScratch, kZeros, kRegions };
    StagingFifo<cudaEvent_t, kRegions> staging;
    uint64_t* drains = nullptr;  // ClientStats::drains of the connection
    void mark(cudaStream_t s) {
        dirty = true;
        last = s;
        cudaEvent_t ev;
        if (!staging.take_free(&ev)) {
            DeviceGuard g(device);
            cudaEventCreateWithFlags(&ev, cudaEventDisableTiming);
        }
        cudaEventRecord(ev, s);
        staging.push(ev);
        for (cudaStream_t b : busy)
            if (b == s) return;
        busy.push_back(s);
    }
    // Bump allocators.  Bytes come round again only after the launches that used them one lap
    // earlier have completed; launches that are still running on other bytes are not waited for.
    // zeros: every kernel returns the counters it was given to zero before it completes, so
    // waiting for those launches is also what makes the reused bytes zero again.
    size_t alloc(int region, size_t bytes, size_t size) {
        const uint64_t at = staging.place(region, bytes, size, [this](cudaEvent_t ev) {
            if (cudaEventQuery(ev) != cudaErrorNotReady) return;  // done, or failed: sync() reports it
            cudaEventSynchronize(ev);
            if (drains) ++*drains;
        });
        return size_t(at % size);
    }
    size_t ring_alloc(size_t bytes) { return alloc(kRing, align_up(bytes, 64), kRingBytes); }
    size_t scratch_alloc(size_t bytes) {
        return alloc(kScratch, align_up(bytes, 256), kScratchBytes);
    }
    size_t zeros_alloc(size_t bytes) { return alloc(kZeros, align_up(bytes, 256), kZeroBytes); }

    // Stage the keys and destination offsets of blocks[base, base + b.n) for one launch.
    // `packed` holds the call's keys in the staged layout already (b is then the whole call):
    // three memcpys instead of a pass over the keys.
    StagedKeys stage_keys(const std::vector<KeyOffset>& blocks, size_t base, const KeyBatch& b,
                          const PackedKeys* packed) {
        const size_t n = b.n;
        const size_t at_bytes = ring_alloc(b.key_bytes);
        const size_t at_off = ring_alloc(n * 4);
        const size_t at_len = ring_alloc(n * 4);
        const size_t at_dst = ring_alloc(n * 8);
        auto* off = reinterpret_cast<uint32_t*>(ring_h + at_off);
        auto* len = reinterpret_cast<uint32_t*>(ring_h + at_len);
        auto* dst = reinterpret_cast<uint64_t*>(ring_h + at_dst);
        if (packed) {
            std::memcpy(ring_h + at_bytes, packed->bytes, b.key_bytes);
            std::memcpy(off, packed->off, n * 4);
            std::memcpy(len, packed->len, n * 4);
        } else {
            // each key on an 8-byte boundary, zero padded to a multiple of 8
            size_t at = 0;
            for (size_t i = 0; i < n; ++i) {
                const std::string_view k = blocks[base + i].key;
                const size_t padded = align_up(k.size() ? k.size() : 1, 8);
                off[i] = uint32_t(at);
                len[i] = uint32_t(k.size());
                std::memcpy(ring_h + at_bytes + at, k.data(), k.size());
                std::memset(ring_h + at_bytes + at + k.size(), 0, padded - k.size());
                at += padded;
            }
        }
        for (size_t i = 0; i < n; ++i) dst[i] = blocks[base + i].offset;
        return StagedKeys{ring_d + at_bytes, reinterpret_cast<const uint32_t*>(ring_d + at_off),
                          reinterpret_cast<const uint32_t*>(ring_d + at_len),
                          reinterpret_cast<const uint64_t*>(ring_d + at_dst)};
    }
};

}  // namespace istore
