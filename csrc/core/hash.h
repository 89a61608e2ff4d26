// 64-bit keyed hash shared by host C++ and sm_90a device code.
//
// The store identifies a key by a 128-bit fingerprint (hash with two seeds).  The host
// kv map uses it as its hasher, the HBM-resident index stores it instead of key bytes,
// and the match_last_index / check_exist kernels recompute it on the GPU from the packed
// key bytes — so host and device MUST produce identical values.  The mixing step is a
// 64x64->128 multiply folded to 64 bits (the construction used by wyhash-style hashes).
//
// Device-side contract: `p` is 8-byte aligned and readable up to the next multiple of 8
// past `len` (the client packs keys that way), so the kernel uses aligned 64-bit loads.
#pragma once

#include <cstddef>
#include <cstdint>
#include <cstring>

#if defined(__CUDACC__)
#define IS_HD __host__ __device__ __forceinline__
#else
#define IS_HD inline
#endif

namespace istore {

constexpr uint64_t kHashSeed1 = 0x9e3779b97f4a7c15ull;
constexpr uint64_t kHashSeed2 = 0xc2b2ae3d27d4eb4full;

IS_HD uint64_t hash_mum(uint64_t a, uint64_t b) {
#if defined(__CUDA_ARCH__)
    return (a * b) ^ __umul64hi(a, b);
#else
    const __uint128_t r = (__uint128_t)a * b;
    return uint64_t(r) ^ uint64_t(r >> 64);
#endif
}

// little-endian value of the first n (1..8) bytes at p
IS_HD uint64_t hash_load(const uint8_t* p, size_t n) {
#if defined(__CUDA_ARCH__)
    const uint64_t v = *reinterpret_cast<const uint64_t*>(p);  // aligned + padded by contract
    return n >= 8 ? v : (v & ((uint64_t(1) << (8 * n)) - 1));
#else
    uint64_t v = 0;
    std::memcpy(&v, p, n < 8 ? n : 8);
    return v;
#endif
}

IS_HD uint64_t hash_bytes(const uint8_t* p, size_t len, uint64_t seed) {
    const uint64_t s0 = 0xa0761d6478bd642full, s1 = 0xe7037ed1a0b428dbull,
                   s2 = 0x8ebc6af09c88c6e3ull;
    uint64_t h = seed ^ hash_mum(seed ^ s0, s1 ^ uint64_t(len));
    size_t i = 0;
    for (; i + 16 <= len; i += 16)
        h = hash_mum(hash_load(p + i, 8) ^ s1, hash_load(p + i + 8, 8) ^ h);
    const size_t rem = len - i;
    uint64_t a = 0, b = 0;
    if (rem > 8) {
        a = hash_load(p + i, 8);
        b = hash_load(p + i + 8, rem - 8);
    } else if (rem > 0) {
        a = hash_load(p + i, rem);
    }
    h = hash_mum(a ^ s2, b ^ h ^ s1);
    return hash_mum(h ^ s0, uint64_t(len) ^ s2);
}

struct KeyHash {
    uint64_t h1;  // bucket selector and fingerprint; never 0 (0 marks an empty index way)
    uint64_t h2;  // verifier
};

IS_HD KeyHash hash_key(const uint8_t* p, size_t len) {
    KeyHash k;
    k.h1 = hash_bytes(p, len, kHashSeed1);
    k.h2 = hash_bytes(p, len, kHashSeed2);
    if (k.h1 == 0) k.h1 = 1;
    return k;
}

}  // namespace istore
