// sm_90a PTX wrappers: mbarrier, TMA (cp.async.bulk.tensor), clusters / DSMEM, wgmma.
// Hand-written for H100; no CUTLASS/CuTe on the hot path.
#pragma once
#include <cuda.h>
#include <cuda_fp16.h>
#include <cuda_runtime.h>
#include <stdint.h>
#include <stdio.h>

namespace b2 {

__device__ __forceinline__ uint32_t smem_u32(const void* p) {
    return static_cast<uint32_t>(__cvta_generic_to_shared(p));
}

__device__ __forceinline__ uint64_t globaltimer_ns() {
    uint64_t t;
    asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t));
    return t;
}

// ---------------------------------------------------------------- mbarrier
__device__ __forceinline__ void mbar_init(uint64_t* bar, uint32_t count) {
    asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count));
}
__device__ __forceinline__ void fence_mbar_init() {
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
}
__device__ __forceinline__ void mbar_expect_tx(uint64_t* bar, uint32_t bytes) {
    asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)),
                 "r"(bytes)
                 : "memory");
}
__device__ __forceinline__ void mbar_arrive(uint64_t* bar) {
    asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(smem_u32(bar)) : "memory");
}
__device__ __forceinline__ bool mbar_try_wait(uint64_t* bar, uint32_t parity) {
    uint32_t ok;
    asm volatile(
        "{\n\t"
        ".reg .pred P;\n\t"
        "mbarrier.try_wait.parity.shared::cta.b64 P, [%1], %2;\n\t"
        "selp.u32 %0, 1, 0, P;\n\t"
        "}\n"
        : "=r"(ok)
        : "r"(smem_u32(bar)), "r"(parity)
        : "memory");
    return ok != 0;
}
// Bounded wait: a protocol bug traps (sticky error, process keeps control) instead of hanging
// the GPU. 4 s is >1000x any legitimate wait in this library.  No printf here: a call inside a wgmma mainloop makes ptxas
// serialize the warpgroup MMAs.
#ifndef B2_WAIT_TIMEOUT_NS
#define B2_WAIT_TIMEOUT_NS 4000000000ull
#endif
__device__ __forceinline__ void mbar_wait(uint64_t* bar, uint32_t parity) {
    if (mbar_try_wait(bar, parity)) return;
    uint64_t t0 = 0;   // the timer is only consulted after 1024 failed (hardware-suspended) polls: ordinary waits never read it
    uint32_t spins = 0;
    while (!mbar_try_wait(bar, parity)) {
        if ((++spins & 0x3ff) == 0) {
            const uint64_t now = globaltimer_ns();
            if (t0 == 0) t0 = now;
            else if (now - t0 > B2_WAIT_TIMEOUT_NS) __trap();
        }
    }
}

// Arrive on a barrier in a peer CTA's shared memory (CTA pairs: "my warpgroups have finished reading this ring slot", so the
// peer's multicast may overwrite it).  Default semantics on purpose: what crosses the pair is the ORDER of async-proxy work
// (wgmma reads retired -> TMA may write), not generic-proxy data.
__device__ __forceinline__ void mbar_arrive_remote(uint32_t cluster_addr) {
    asm volatile("mbarrier.arrive.shared::cluster.b64 _, [%0];" ::"r"(cluster_addr) : "memory");
}

// smem writes by normal (generic-proxy) stores -> visible to async proxy (TMA / wgmma reads)
__device__ __forceinline__ void fence_proxy_async_smem() {
    asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
}

// ---------------------------------------------------------------- thread-block cluster / DSMEM
__device__ __forceinline__ void cluster_sync_all() {
    asm volatile("barrier.cluster.arrive.release.aligned;" ::: "memory");
    asm volatile("barrier.cluster.wait.acquire.aligned;" ::: "memory");
}
// split form: arrive early, wait later (e.g. "every CTA of the cluster has started" before the first DSMEM access)
__device__ __forceinline__ void cluster_arrive_relaxed() { asm volatile("barrier.cluster.arrive.relaxed.aligned;" ::: "memory"); }
__device__ __forceinline__ void cluster_wait() { asm volatile("barrier.cluster.wait.aligned;" ::: "memory"); }
__device__ __forceinline__ uint32_t cluster_ctarank() {
    uint32_t r;
    asm volatile("mov.u32 %0, %%cluster_ctarank;" : "=r"(r));
    return r;
}
// address of `local_smem_addr` inside CTA `rank` of this cluster (shared::cluster window)
__device__ __forceinline__ uint32_t dsmem_map(uint32_t local_smem_addr, uint32_t rank) {
    uint32_t r;
    asm volatile("mapa.shared::cluster.u32 %0, %1, %2;" : "=r"(r) : "r"(local_smem_addr), "r"(rank));
    return r;
}
__device__ __forceinline__ void dsmem_st_f2(uint32_t cluster_addr, float x, float y) {
    asm volatile("st.shared::cluster.v2.f32 [%0], {%1, %2};" ::"r"(cluster_addr), "f"(x), "f"(y) : "memory");
}
__device__ __forceinline__ float4 dsmem_ld_f4(uint32_t cluster_addr) {
    float4 v;
    asm volatile("ld.shared::cluster.v4.f32 {%0, %1, %2, %3}, [%4];"
                 : "=f"(v.x), "=f"(v.y), "=f"(v.z), "=f"(v.w)
                 : "r"(cluster_addr)
                 : "memory");
    return v;
}

// ---------------------------------------------------------------- TMA
__device__ __forceinline__ void tma_prefetch_desc(const CUtensorMap* m) {
    asm volatile("prefetch.tensormap [%0];" ::"l"(reinterpret_cast<uint64_t>(m)) : "memory");
}
__device__ __forceinline__ void tma_load_2d(void* smem_dst, const CUtensorMap* m, uint64_t* bar,
                                            int c0, int c1) {
    asm volatile(
        "cp.async.bulk.tensor.2d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%3, "
        "%4}], [%2];" ::"r"(smem_u32(smem_dst)),
        "l"(reinterpret_cast<uint64_t>(m)), "r"(smem_u32(bar)), "r"(c0), "r"(c1)
        : "memory");
}
__device__ __forceinline__ void tma_load_4d(void* smem_dst, const CUtensorMap* m, uint64_t* bar,
                                            int c0, int c1, int c2, int c3) {
    asm volatile(
        "cp.async.bulk.tensor.4d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%3, "
        "%4, %5, %6}], [%2];" ::"r"(smem_u32(smem_dst)),
        "l"(reinterpret_cast<uint64_t>(m)), "r"(smem_u32(bar)), "r"(c0), "r"(c1), "r"(c2), "r"(c3)
        : "memory");
}

// Shared -> global tensor store, tracked by the issuing thread's bulk async-groups; elements outside the tensor are not written.
// The writers of the source tile must have run fence_proxy_async_smem() (and synchronised with the issuing thread) first.
__device__ __forceinline__ void tma_store_4d(const CUtensorMap* m, const void* smem_src, int c0, int c1, int c2, int c3) {
    asm volatile("cp.async.bulk.tensor.4d.global.shared::cta.bulk_group [%0, {%2, %3, %4, %5}], [%1];" ::"l"(reinterpret_cast<uint64_t>(m)),
                 "r"(smem_u32(smem_src)), "r"(c0), "r"(c1), "r"(c2), "r"(c3)
                 : "memory");
}
__device__ __forceinline__ void bulk_commit_group() { asm volatile("cp.async.bulk.commit_group;" ::: "memory"); }
// at most N of this thread's committed stores still read their shared-memory source (the source may then be overwritten)
template <int N>
__device__ __forceinline__ void bulk_wait_group_read() { asm volatile("cp.async.bulk.wait_group.read %0;" ::"n"(N) : "memory"); }
// at most N of this thread's committed stores are still incomplete (their writes are not yet performed)
template <int N>
__device__ __forceinline__ void bulk_wait_group() { asm volatile("cp.async.bulk.wait_group %0;" ::"n"(N) : "memory"); }

// barrier over `count` threads (a multiple of 32) under id `id` (1..15; 0 is __syncthreads)
__device__ __forceinline__ void named_bar_sync(int id, int count) {
    asm volatile("bar.sync %0, %1;" ::"r"(id), "r"(count) : "memory");
}

// Multicast form (CTA pairs): the box lands at the same shared-memory offset in every CTA of `cta_mask` (cluster ranks),
// and each destination's mbarrier at `bar`'s offset receives the complete_tx of its bytes.
__device__ __forceinline__ void tma_load_2d_mc(void* smem_dst, const CUtensorMap* m, uint64_t* bar, int c0, int c1, uint16_t cta_mask) {
    asm volatile(
        "cp.async.bulk.tensor.2d.shared::cluster.global.mbarrier::complete_tx::bytes.multicast::cluster [%0], [%1, {%3, %4}], [%2], "
        "%5;" ::"r"(smem_u32(smem_dst)),
        "l"(reinterpret_cast<uint64_t>(m)), "r"(smem_u32(bar)), "r"(c0), "r"(c1), "h"(cta_mask)
        : "memory");
}

// ---------------------------------------------------------------- wgmma (warpgroup MMA, accumulators in registers)
// Every thread of the warpgroup executes these (.sync.aligned).
__device__ __forceinline__ void wgmma_fence() { asm volatile("wgmma.fence.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wgmma_commit() { asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory"); }
template <int N>
__device__ __forceinline__ void wgmma_wait() { asm volatile("wgmma.wait_group.sync.aligned %0;" ::"n"(N) : "memory"); }
// the compiler must not move accumulator reads/writes across an in-flight wgmma
template <int N>
__device__ __forceinline__ void wgmma_fence_regs(float (&d)[N]) {
#pragma unroll
    for (int i = 0; i < N; ++i) asm volatile("" : "+f"(d[i])::"memory");
}

// ---------------------------------------------------------------- descriptors
// K-major operand tile in smem, SWIZZLE_128B: rows of 64 fp16 (128 B), 8-row groups `sbo` bytes apart (1024 for a dense tile).
// Bit layout (sm_90 wgmma matrix descriptor): start[0,14) lbo[16,30) sbo[32,46) base_offset[49,52) layout[62,64) (1 = SWIZZLE_128B).
// The swizzle follows the shared-memory address bits, so tiles start on 1024-byte boundaries except where a caller shifts the
// start by whole 128-byte rows on purpose (tconv.cu).
__device__ __forceinline__ uint64_t make_kmajor_sw128_desc(uint32_t smem_addr, uint32_t sbo = 1024) {
    uint64_t d = 0;
    d |= (uint64_t)((smem_addr & 0x3ffff) >> 4);
    d |= (uint64_t)1 << 16;            // LBO (unused for swizzled K-major)
    d |= (uint64_t)(sbo >> 4) << 32;   // SBO: 8 rows * 128 B
    d |= (uint64_t)1 << 62;            // SWIZZLE_128B
    return d;
}

}  // namespace b2
