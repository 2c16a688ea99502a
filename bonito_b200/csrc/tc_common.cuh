// PTX wrappers shared by the Hopper tensor-core kernels (sm_90a): mbarriers, bulk copies, cluster / distributed-shared-memory
// helpers, wgmma descriptors and fences.
#pragma once

#include "common.cuh"

// One lane of a converged warp (elect.sync): unlike `lane == 0`, the compiler then knows the guarded code runs in a
// single thread and can issue bulk copies from uniform registers.
__device__ __forceinline__ bool elect_one_sync() {
    uint32_t pred;
    asm volatile(
        "{\n"
        ".reg .pred p;\n"
        "elect.sync _|p, 0xffffffff;\n"
        "selp.u32 %0, 1, 0, p;\n"
        "}\n"
        : "=r"(pred));
    return pred != 0;
}

// ---- mbarrier -----------------------------------------------------------------------------------
__device__ __forceinline__ void mbar_init(uint32_t bar, uint32_t count) {
    asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;\n" ::"r"(bar), "r"(count));
}
__device__ __forceinline__ void mbar_fence_init() {
    asm volatile("fence.mbarrier_init.release.cluster;\n" ::: "memory");
}
__device__ __forceinline__ void mbar_expect_tx(uint32_t bar, uint32_t bytes) {
    asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;\n" ::"r"(bar), "r"(bytes) : "memory");
}
__device__ __forceinline__ void mbar_arrive(uint32_t bar) {
    asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];\n" ::"r"(bar) : "memory");
}
// arrive on a barrier that lives in another CTA of the cluster (address from mapa), release at cluster scope
__device__ __forceinline__ void mbar_arrive_remote(uint32_t cluster_addr) {
    asm volatile("mbarrier.arrive.release.cluster.shared::cluster.b64 _, [%0];\n" ::"r"(cluster_addr) : "memory");
}
__device__ __forceinline__ void mbar_wait(uint32_t bar, uint32_t parity) {
    asm volatile(
        "{\n"
        ".reg .pred p;\n"
        "WAIT_LOOP:\n"
        "mbarrier.try_wait.parity.shared::cta.b64 p, [%0], %1;\n"
        "@p bra WAIT_DONE;\n"
        "bra WAIT_LOOP;\n"
        "WAIT_DONE:\n"
        "}\n" ::"r"(bar),
        "r"(parity)
        : "memory");
}
// wait with acquire semantics at cluster scope (the arrivals come from other CTAs)
__device__ __forceinline__ void mbar_wait_cluster(uint32_t bar, uint32_t parity) {
    asm volatile(
        "{\n"
        ".reg .pred p;\n"
        "WAITC_LOOP:\n"
        "mbarrier.try_wait.parity.acquire.cluster.shared::cta.b64 p, [%0], %1;\n"
        "@p bra WAITC_DONE;\n"
        "bra WAITC_LOOP;\n"
        "WAITC_DONE:\n"
        "}\n" ::"r"(bar),
        "r"(parity)
        : "memory");
}

// ---- cluster / DSMEM ----------------------------------------------------------------------------
__device__ __forceinline__ uint32_t cluster_ctarank() {
    uint32_t r;
    asm volatile("mov.u32 %0, %%cluster_ctarank;\n" : "=r"(r));
    return r;
}
__device__ __forceinline__ void cluster_sync_all() {
    asm volatile("barrier.cluster.arrive.release.aligned;\n" ::: "memory");
    asm volatile("barrier.cluster.wait.acquire.aligned;\n" ::: "memory");
}
__device__ __forceinline__ uint32_t mapa(uint32_t local_smem_addr, uint32_t cta_rank) {
    uint32_t r;
    asm volatile("mapa.shared::cluster.u32 %0, %1, %2;\n" : "=r"(r) : "r"(local_smem_addr), "r"(cta_rank));
    return r;
}
__device__ __forceinline__ void st_cluster_v4(uint32_t cluster_addr, uint4 v) {
    asm volatile("st.shared::cluster.v4.b32 [%0], {%1, %2, %3, %4};\n" ::"r"(cluster_addr), "r"(v.x), "r"(v.y),
                 "r"(v.z), "r"(v.w)
                 : "memory");
}
// asynchronous 16-byte store into the shared memory of a cluster peer; completes 16 tx-bytes on the peer's mbarrier
__device__ __forceinline__ void st_async_v4(uint32_t cluster_addr, uint4 v, uint32_t cluster_bar) {
    asm volatile("st.async.weak.shared::cluster.mbarrier::complete_tx::bytes.v4.b32 [%0], {%1, %2, %3, %4}, [%5];\n" ::
                     "r"(cluster_addr), "r"(v.x), "r"(v.y), "r"(v.z), "r"(v.w), "r"(cluster_bar)
                 : "memory");
}
// bulk copy own shared memory -> a peer's shared memory (TMA engine); completes `bytes` on the peer's mbarrier
__device__ __forceinline__ void bulk_copy_to_peer(uint32_t peer_dst, uint32_t local_src, uint32_t bytes, uint32_t peer_bar) {
    asm volatile("cp.async.bulk.shared::cluster.shared::cta.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];\n" ::
                     "r"(peer_dst), "r"(local_src), "r"(bytes), "r"(peer_bar)
                 : "memory");
}
// 2-D tensor copy global -> own shared memory (TMA engine) at element coordinates (c0 innermost, c1); elements outside
// the tensor are zero-filled and still count towards the `bytes` completed on the mbarrier
__device__ __forceinline__ void tma_load_2d(uint32_t dst, const void* tmap, int c0, int c1, uint32_t bar) {
    asm volatile(
        "cp.async.bulk.tensor.2d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%2, %3}], [%4];\n" ::"r"(dst),
        "l"(reinterpret_cast<uint64_t>(tmap)), "r"(c0), "r"(c1), "r"(bar)
        : "memory");
}
__device__ __forceinline__ void fence_proxy_async_smem() { asm volatile("fence.proxy.async.shared::cta;\n" ::: "memory"); }
// make generic-proxy writes (st.shared / st.shared::cluster) visible to the async proxy (wgmma / bulk-copy reads)
__device__ __forceinline__ void fence_proxy_async() { asm volatile("fence.proxy.async;\n" ::: "memory"); }

// ---- wgmma --------------------------------------------------------------------------------------
// Operand tiles are K-major WITHOUT swizzle: core matrices of 8 rows x 16 bytes (128 contiguous bytes); `lbo` = byte
// distance between core matrices adjacent along K, `sbo` = between adjacent 8-row groups along M / N.
__device__ __forceinline__ uint64_t wg_desc_noswz(uint32_t smem_addr, uint32_t lbo, uint32_t sbo) {
    uint64_t d = 0;
    d |= (uint64_t)((smem_addr & 0x3FFFF) >> 4);   // start address        bits [0,14)
    d |= (uint64_t)(lbo >> 4) << 16;               // leading byte offset  bits [16,30)
    d |= (uint64_t)(sbo >> 4) << 32;               // stride byte offset   bits [32,46)
    return d;                                      // layout type 0 (no swizzle) in bits [62,64)
}
// K-major tile with the 128-byte swizzle (what a TMA copy with CU_TENSOR_MAP_SWIZZLE_128B writes): rows of 128 bytes,
// 8-row atoms 1024 bytes apart (sbo), the atom 1024-byte aligned.  A k-step inside the row adds its byte offset to the
// start address.
__device__ __forceinline__ uint64_t wg_desc_sw128(uint32_t smem_addr) {
    uint64_t d = 0;
    d |= (uint64_t)((smem_addr & 0x3FFFF) >> 4);   // start address                     bits [0,14)
    d |= (uint64_t)1 << 16;                        // leading byte offset (unused: K-major swizzled)
    d |= (uint64_t)(1024 >> 4) << 32;              // stride byte offset                bits [32,46)
    d |= (uint64_t)1 << 62;                        // layout type 1: 128-byte swizzle   bits [62,64)
    return d;
}
__device__ __forceinline__ void wg_fence() { asm volatile("wgmma.fence.sync.aligned;\n" ::: "memory"); }
__device__ __forceinline__ void wg_commit() { asm volatile("wgmma.commit_group.sync.aligned;\n" ::: "memory"); }
template <int N>
__device__ __forceinline__ void wg_wait() {
    asm volatile("wgmma.wait_group.sync.aligned %0;\n" ::"n"(N) : "memory");
}
// keeps the compiler from moving accumulator reads / writes across the asynchronous wgmma (the constraint matches the
// register type, so no conversion moves land between the wgmma and its commit / wait)
template <int N>
__device__ __forceinline__ void wg_fence_regs(float (&d)[N]) {
#pragma unroll
    for (int i = 0; i < N; ++i) asm volatile("" : "+f"(d[i])::"memory");
}
template <int N>
__device__ __forceinline__ void wg_fence_regs(int (&d)[N]) {
#pragma unroll
    for (int i = 0; i < N; ++i) asm volatile("" : "+r"(d[i])::"memory");
}

#include "wgmma_ops.cuh"
