// Configuration structs shared by C++, the pybind layer and the Python kwargs/argparse
// surface.  Field names of the first block of each struct are the reference's
// (src/config.h:13-32); the second block is the NVLink fabric extension.
#pragma once

#include <cstddef>
#include <string>
#include <vector>

namespace istore {

struct ServerConfig {
    int service_port = 0;
    std::string log_level = "warning";
    std::string dev_name = "mlx5_1";  // accepted and ignored on the NVLink fabric
    size_t prealloc_size = 16;        // GB
    int ib_port = 1;                  // accepted and ignored
    std::string link_type = "IB";     // accepted and ignored
    int minimal_allocate_size = 64;   // KB (allocation granule)
    int num_stream = 1;               // deprecated in the reference; ignored
    bool auto_increase = false;

    // --- fabric extension
    std::string host = "0.0.0.0";          // listen address (the reference parses but ignores it)
    std::string pool_backend = "auto";     // auto | hbm | host
    std::vector<int> pool_devices;         // CUDA ordinals hosting pool segments (default {0})
    size_t extend_size = 10;               // GB added per auto-increase step
    size_t prealloc_bytes = 0;             // if non-zero overrides prealloc_size (tests)
    size_t index_slots = 0;                // device-index entries per segment (0 = auto)
    size_t replica_bytes = 0;              // NVLS-replicated region per GPU (0 = none)
    std::vector<int> replica_devices;      // GPUs holding a replica (default: all visible)
    bool evict = false;                    // full pool: evict least-recently-used blocks
                                           // instead of answering 507 (reference: never)
    double evict_ratio = 0.05;             // fraction of the pool freed per eviction round
    size_t max_pending_reply_bytes = 64u << 20;  // a client that pipelines requests without
                                           // reading its replies is disconnected beyond this
};

struct ClientConfig {
    int service_port = 0;
    std::string log_level = "warning";
    std::string dev_name = "mlx5_1";
    std::string host_addr;
    int ib_port = 1;
    std::string link_type = "IB";

    // --- fabric extension
    int device = -1;          // CUDA ordinal the client launches kernels on (-1: decide per tensor)
    int timeout_ms = 10000;   // per-request deadline on the control plane
    int pool_hint = -1;       // preferred pool segment device for allocations (-1 = any)
    // sync() and the server's host-side map.  false (default): sync() ends with a SYNC round
    // trip, so when it returns every client - also one that asks the SERVER - sees the writes.
    // true: the commit list is POSTED (one-way, like the reference's COMMIT SEND,
    // src/libinfinistore.cpp:362-395) and sync() returns once the kernels have finished; the
    // writes are already visible to every device-path reader (in-band commit in the HBM
    // index), server-mediated lookups of other connections follow within the TCP delivery
    // time.  Saves the control-plane round trip: the single-block write latency.
    bool posted_commit = false;
    // Latency mode: single blocks of <= 256 KB are served by a persistent worker CTA that
    // polls a request ring in pinned host memory (kernels/kv_doorbell.cu) - no launch, no
    // event, no stream poll per operation.  The worker leaves after doorbell_idle_us without
    // a request (a device-wide synchronise waits at most that long for it).
    bool doorbell = false;
    int doorbell_idle_us = 200;
};

}  // namespace istore
