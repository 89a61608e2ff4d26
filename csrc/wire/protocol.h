// Wire framing for the b200 KV store control plane.
//
// Behavioural parity with the reference framing (reference: src/protocol.h:36-71,85-93):
// a request is a 9-byte packed header {magic u32, op char, body_size u32} followed by
// `body_size` bytes; a reply is a 4-byte little-endian return code followed by an
// op-specific payload.  Opcodes and return codes keep the reference's values so that the
// control plane is recognisable on the wire.
//
// Differences by design (GPU-native data plane, no ibverbs message channel):
//   * the allocate / read-lookup / commit messages ('D','A','T'), which the reference
//     carries inside RDMA SEND messages, ride the same TCP connection here;
//   * 'P' (pool map) is new: it hands the client the list of pool segments (HBM IPC
//     handles or shm names) it must map before launching kv_write / kv_read kernels;
//   * 'U' (staged commit) is new: the writer ships its commit list BEFORE it waits for its
//     kernels; the server decodes it and warms the blocks meanwhile and applies it at the
//     next 'S' - the commit leaves the critical path of sync() without becoming visible early;
//   * variable-size reply payloads are prefixed with a u32 byte length.
#pragma once

#include <cstddef>
#include <cstdint>
#include <cstring>
#include <string>

namespace istore {

constexpr uint32_t kMagic = 0xdeadbeefu;

enum Op : char {
    kOpLocalRead = 'R',     // LocalMetaRequest  -> code [+ len + RdmaAllocateResponse]
    kOpLocalWrite = 'W',    // LocalMetaRequest  -> code [+ len + RdmaAllocateResponse]
    kOpSync = 'S',          // no body           -> code + u32 inflight
    kOpExchange = 'E',      // 30-byte conn info -> code + 30-byte conn info
    kOpAllocate = 'D',      // RemoteMetaRequest -> code + len + RdmaAllocateResponse
    kOpReadLookup = 'A',    // RemoteMetaRequest -> code + len + RdmaAllocateResponse
    kOpCommit = 'T',        // RemoteMetaRequest -> (no reply, ordered before next 'S')
    kOpCheckExist = 'C',    // raw key bytes     -> code + i32 (0 = exists & committed)
    kOpMatchLastIdx = 'M',  // GetMatchLastIndexRequest -> code + i32
    kOpPoolMap = 'P',       // u32 first_segment -> code + len + PoolMap blob
    kOpTouch = 'H',         // GetMatchLastIndexRequest (keys) -> code + i32 blocks refreshed:
                            // recency hint for stores that evict
    kOpStageCommit = 'U',   // RemoteMetaRequest -> (no reply) addresses to commit at the next 'S';
                            // block_size -1 discards what was staged
};

enum Code : int32_t {
    kFinish = 200,
    kTaskAccepted = 202,
    kInvalidReq = 400,
    kKeyNotFound = 404,
    kRetry = 408,
    kInternalError = 500,
    kSystemError = 503,
    kOutOfMemory = 507,
};

// Largest body / reply payload the reactor will buffer (reference: PROTOCOL_BUFFER_SIZE,
// src/protocol.h:65).  Unlike the reference, body_size is validated against this cap.
constexpr uint32_t kMaxBody = 4u << 20;

#pragma pack(push, 1)
struct Header {
    uint32_t magic;
    char op;
    uint32_t body_size;
};
// Same 30-byte layout as the reference's rdma_conn_info_t (src/protocol.h:85-91); on the
// NVLink fabric the fields carry process / device identity instead of QP numbers.
struct ConnInfo {
    uint32_t qpn;      // pid of the sender
    uint32_t psn;      // client: CUDA device ordinal (0xffffffff = none); server: #segments
    uint8_t gid[16];   // process uuid (same-process detection: no IPC open on own memory)
    uint16_t lid;      // fabric flags (bit0: CUDA available, bit1: HBM pool, bit2: evicts)
    uint32_t mtu;      // fabric protocol version
};
#pragma pack(pop)
static_assert(sizeof(Header) == 9, "header must be 9 bytes");
static_assert(sizeof(ConnInfo) == 30, "conn info must be 30 bytes");

constexpr uint32_t kFabricVersion = 2;  // 2: staged commits ('U')
// Bit 31 of the u32 that follows a SYNC reply's code (and bit 3 of ConnInfo::lid): some block
// could not be inserted into the HBM index, device-side lookups may miss keys that exist.
constexpr uint32_t kSyncIndexIncomplete = 1u << 31;

// 16-byte block locator returned by allocate / lookup.  numpy ABI: rkey:u4 @0,
// remote_addr:u8 @8, itemsize 16 (reference: src/pybind.cpp:47).  The 4 padding bytes of
// the reference struct carry the allocation generation here.
struct RemoteBlock {
    uint32_t rkey;         // segment id + 1 (0 only in the fake "already exists" block)
    uint32_t gen;          // allocation generation (commit tag)
    uint64_t remote_addr;  // (segment id + 1) << kSegShift | byte offset in the segment
};
static_assert(sizeof(RemoteBlock) == 16 && offsetof(RemoteBlock, remote_addr) == 8, "ABI");

constexpr int kSegShift = 44;
constexpr uint64_t kOffMask = (1ull << kSegShift) - 1;
inline uint64_t make_addr(uint32_t seg, uint64_t off) {
    return (uint64_t(seg + 1) << kSegShift) | off;
}
inline uint32_t addr_seg(uint64_t addr) { return uint32_t(addr >> kSegShift) - 1; }
inline uint64_t addr_off(uint64_t addr) { return addr & kOffMask; }
inline bool is_fake_block(const RemoteBlock& b) { return b.rkey == 0 && b.remote_addr == 0; }

const char* op_name(char op);
bool op_known(char op);
bool op_has_body(char op);

// Pool-map blob (reply to 'P'): u32 count, then `count` fixed-size records.
// kSegReplica: an NVLS-replicated region - one replica per GPU bound to a multicast object;
// writes go to the multicast address, reads to the local replica.  `handle` names the unix
// socket that hands out the VMM file descriptors (fabric/fdpass.h), `device` is -2.
enum SegKind : uint32_t { kSegHostShm = 0, kSegDeviceIpc = 1, kSegReplica = 2 };
constexpr int kReplicaDevice = -2;  // pool "device" / allocation hint of the replicated region
#pragma pack(push, 1)
struct SegmentInfo {
    uint32_t id;
    uint32_t kind;          // SegKind
    int32_t device;         // physical CUDA device ordinal of the pool (-1 for host)
    uint32_t granule;       // allocation granule in bytes
    uint64_t bytes;         // data bytes in the segment
    uint64_t index_off;     // byte offset of the device index table inside the mapping (0 = none)
    uint64_t index_slots;   // number of 32-byte index entries (power of two)
    uint64_t map_bytes;     // total bytes to map (data + index)
    uint8_t handle[64];     // cudaIpcMemHandle_t, or NUL-terminated shm name
    uint8_t owner[16];      // uuid of the owning process
    uint64_t owner_ptr;     // base pointer in the owner process (same-process shortcut)
};
#pragma pack(pop)

}  // namespace istore
