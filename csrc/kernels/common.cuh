// Device-side building blocks shared by the sm_90a kernels: vector / cache-hinted memory
// ops, system-scope acquire/release, mbarrier + 1-D bulk-async (TMA) copies, multimem.
// Inline PTX only; SASS mnemonics to look for are noted beside each wrapper.
#pragma once

#include <cuda_runtime.h>

#include <cstdint>

namespace istore::kernels::dev {

// ---------------------------------------------------------------- plain + hinted ld/st
__device__ __forceinline__ uint4 ld_v4(const void* p) {  // LDG.E.128
    uint4 r;
    asm volatile("ld.global.v4.u32 {%0,%1,%2,%3}, [%4];"
                 : "=r"(r.x), "=r"(r.y), "=r"(r.z), "=r"(r.w)
                 : "l"(p));
    return r;
}
// streaming read that does not pollute L1 (data is touched once)   LDG.E.NA.128
__device__ __forceinline__ uint4 ld_stream_v4(const void* p) {
    uint4 r;
    asm volatile("ld.global.L1::no_allocate.v4.u32 {%0,%1,%2,%3}, [%4];"
                 : "=r"(r.x), "=r"(r.y), "=r"(r.z), "=r"(r.w)
                 : "l"(p));
    return r;
}
__device__ __forceinline__ void st_v4(void* p, const uint4& v) {  // STG.E.128
    asm volatile("st.global.v4.u32 [%0], {%1,%2,%3,%4};" ::"l"(p), "r"(v.x), "r"(v.y), "r"(v.z),
                 "r"(v.w)
                 : "memory");
}
__device__ __forceinline__ void st_stream_v4(void* p, const uint4& v) {  // STG.E.NA.128
    asm volatile("st.global.L1::no_allocate.v4.u32 [%0], {%1,%2,%3,%4};" ::"l"(p), "r"(v.x),
                 "r"(v.y), "r"(v.z), "r"(v.w)
                 : "memory");
}
// ---------------------------------------------------------------- system-scope sync
__device__ __forceinline__ void fence_sys() { asm volatile("fence.acq_rel.sys;" ::: "memory"); }
__device__ __forceinline__ void fence_gpu() { asm volatile("fence.acq_rel.gpu;" ::: "memory"); }
// counter increment that releases this thread's earlier (fenced) work and acquires the
// other arrivers'; gpu scope: the counters live in this GPU's own memory
__device__ __forceinline__ uint32_t atom_add_acq_rel_gpu(uint32_t* p, uint32_t v) {
    uint32_t old;
    asm volatile("atom.acq_rel.gpu.global.add.u32 %0, [%1], %2;" : "=r"(old) : "l"(p), "r"(v) : "memory");
    return old;
}
__device__ __forceinline__ uint32_t ld_acquire_sys(const uint32_t* p) {  // LDG.E.STRONG.SYS
    uint32_t v;
    asm volatile("ld.acquire.sys.global.u32 %0, [%1];" : "=r"(v) : "l"(p) : "memory");
    return v;
}
__device__ __forceinline__ uint64_t ld_relaxed_sys_u64(const uint64_t* p) {
    uint64_t v;
    asm volatile("ld.relaxed.sys.global.u64 %0, [%1];" : "=l"(v) : "l"(p) : "memory");
    return v;
}
__device__ __forceinline__ void st_release_sys(uint32_t* p, uint32_t v) {  // STG.E.STRONG.SYS
    asm volatile("st.release.sys.global.u32 [%0], %1;" ::"l"(p), "r"(v) : "memory");
}
__device__ __forceinline__ void st_relaxed_sys_u64(uint64_t* p, uint64_t v) {
    asm volatile("st.relaxed.sys.global.u64 [%0], %1;" ::"l"(p), "l"(v) : "memory");
}
__device__ __forceinline__ uint64_t cas_relaxed_sys_u64(uint64_t* p, uint64_t cmp, uint64_t val) {
    uint64_t old;
    asm volatile("atom.relaxed.sys.global.cas.b64 %0, [%1], %2, %3;"
                 : "=l"(old)
                 : "l"(p), "l"(cmp), "l"(val)
                 : "memory");
    return old;
}

__device__ __forceinline__ uint64_t cas_relaxed_gpu_u64(uint64_t* p, uint64_t cmp, uint64_t val) {
    uint64_t old;
    asm volatile("atom.relaxed.gpu.global.cas.b64 %0, [%1], %2, %3;"
                 : "=l"(old)
                 : "l"(p), "l"(cmp), "l"(val)
                 : "memory");
    return old;
}

// ---------------------------------------------------------------- mbarrier + bulk async copy
__device__ __forceinline__ uint32_t smem_u32(const void* p) {
    return static_cast<uint32_t>(__cvta_generic_to_shared(p));
}
__device__ __forceinline__ void mbar_init(uint64_t* bar, uint32_t count) {  // SYNCS.EXCH.64
    asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count));
}
__device__ __forceinline__ void mbar_fence_init() {
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
}
__device__ __forceinline__ void mbar_arrive(uint64_t* bar) {  // SYNCS.ARRIVE
    asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(smem_u32(bar)) : "memory");
}
__device__ __forceinline__ void mbar_expect_tx(uint64_t* bar, uint32_t bytes) {  // SYNCS.ARRIVE.TRANS64
    asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)),
                 "r"(bytes)
                 : "memory");
}
// Waits for the phase with the given parity.  try_wait suspends the thread in hardware for a
// bounded time per attempt; a watchdog turns a lost completion (a bug) into a trap instead
// of a hung GPU.
__device__ __forceinline__ void mbar_wait(uint64_t* bar, uint32_t parity) {  // SYNCS.PHASECHK..TRYWAIT
    const uint32_t addr = smem_u32(bar);
    uint32_t done = 0;
    long long start = 0;
    for (uint32_t spins = 0;; ++spins) {
        asm volatile(
            "{\n\t"
            ".reg .pred p;\n\t"
            "mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n\t"
            "selp.u32 %0, 1, 0, p;\n\t"
            "}"
            : "=r"(done)
            : "r"(addr), "r"(parity)
            : "memory");
        if (done) return;
        if (spins == 64) start = clock64();
        if (spins > 64 && (spins & 1023) == 0 && clock64() - start > 8000000000ll) __trap();
    }
}
// global -> shared, completion signalled on an mbarrier                      UBLKCP.S.G
__device__ __forceinline__ void bulk_g2s(void* smem_dst, const void* gsrc, uint32_t bytes,
                                         uint64_t* bar) {
    asm volatile(
        "cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::
            "r"(smem_u32(smem_dst)),
        "l"(gsrc), "r"(bytes), "r"(smem_u32(bar))
        : "memory");
}
// shared -> global, tracked by the thread's bulk async-group                  UBLKCP.G.S
__device__ __forceinline__ void bulk_s2g(void* gdst, const void* smem_src, uint32_t bytes) {
    asm volatile("cp.async.bulk.global.shared::cta.bulk_group [%0], [%1], %2;" ::"l"(gdst),
                 "r"(smem_u32(smem_src)), "r"(bytes)
                 : "memory");
}
__device__ __forceinline__ void bulk_commit() {
    asm volatile("cp.async.bulk.commit_group;" ::: "memory");
}
template <int N>
__device__ __forceinline__ void bulk_wait_read() {  // source (smem) may be reused
    asm volatile("cp.async.bulk.wait_group.read %0;" ::"n"(N) : "memory");
}
template <int N>
__device__ __forceinline__ void bulk_wait() {  // writes complete
    asm volatile("cp.async.bulk.wait_group %0;" ::"n"(N) : "memory");
}
__device__ __forceinline__ void fence_proxy_async() {  // FENCE.VIEW.ASYNC
    asm volatile("fence.proxy.async;" ::: "memory");
}

// ---------------------------------------------------------------- NVLS multicast store
__device__ __forceinline__ void multimem_st_v4(void* mc_ptr, const uint4& v) {
    asm volatile("multimem.st.relaxed.sys.global.v4.f32 [%0], {%1,%2,%3,%4};" ::"l"(mc_ptr),
                 "r"(v.x), "r"(v.y), "r"(v.z), "r"(v.w)
                 : "memory");
}

}  // namespace istore::kernels::dev
