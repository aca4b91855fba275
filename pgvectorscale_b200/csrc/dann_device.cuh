// dann_device.cuh — device-side views and small helpers shared by the sm_90a kernels.
//
// HBM layout of one loaded index (all arrays row-major, 256-B aligned cudaMalloc regions):
//   codes   [n][cw]  u64   cw = words rounded up to even => every row is 16-B aligned so a
//                          lane group can fetch it with 128-bit loads; 96 B (1-bit@768) and
//                          192 B (2-bit@768) rows are whole 32-B sectors.
//   nbrs    [n][Rp]  u32   Rp = R rounded up to 8 (rows are whole 32-B sectors); the first
//                          0xFFFFFFFF ends the list                 (sbq/node.rs:261-285)
//   tids    [n]      u64   (block<<16)|offset, offset 0 = deleted   (scan.rs:231-234)
//   vectors [n][dim] f32   cosine rows normalised once at load      (sbq/storage.rs:304-328)
//   label_off[n+1] u32 / labels i16  CSR of sorted label sets       (labels/mod.rs:17-37)
//   mean[dim_index], m2[dim_index] f32, count                       (sbq/mod.rs:77-121)
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

#include "../../include/diskann_b200.h"

#define DANN_FULL 0xFFFFFFFFu

/* the kernel's dynamic shared memory window; static __shared__ variables are spelled DANN_STATIC_SMEM so that the CPU
 * SIMT emulator (tests/simt, -DDANN_SIMT_EMU) can give both a meaning without touching the CUDA build */
#ifdef DANN_SIMT_EMU
#define DANN_DYN_SMEM(name) extern unsigned char name[]
#define DANN_STATIC_SMEM static
#else
#define DANN_DYN_SMEM(name) extern __shared__ __align__(16) unsigned char name[]
#define DANN_STATIC_SMEM __shared__
#endif

// per-query internal status bits (retried by the host with a larger workspace)
#define DANN_ST_HEAP 1u
#define DANN_ST_HASH 2u
#define DANN_ST_VIS 4u
// the two-warp kernel's heap warp popped another node than the memory warp predicted (never retried: an internal error)
#define DANN_ST_INTERNAL 8u
// a deep scan (dann_make_deep_plan) suspended cleanly before a visit its workspace has no room for: the host grows the
// workspace in place and resumes the same step; no overflow happened and the saved state is valid
#define DANN_ST_GROW 16u

struct IndexView {
    uint32_t n, dim, dim_index, bits, words, cw, R, Rp;
    int32_t distance_type, has_labels;
    uint64_t count;
    const float *mean, *m2;
    const uint64_t *codes;
    const uint32_t *nbrs;
    const uint64_t *tids;
    const float *vectors;
    uint32_t start_default, n_start_labels;
    const int16_t *start_labels;
    const uint32_t *start_label_nodes;
    const uint32_t *label_off;
    const int16_t *labels;
};

// 128-bit read-only load that does not allocate in L1 (streaming gathers of SBQ codes).
#ifdef DANN_SIMT_EMU /* tests/simt: the same sources compiled by g++ for the CPU SIMT emulator (no PTX there) */
__device__ __forceinline__ ulonglong2 ldg_stream_u128(const void *p) { return *reinterpret_cast<const ulonglong2 *>(p); }
__device__ __forceinline__ uint32_t ldg_stream_u32(const void *p) { return *reinterpret_cast<const uint32_t *>(p); }
__device__ __forceinline__ float4 ldg_stream_f4(const void *p) { return *reinterpret_cast<const float4 *>(p); }
__device__ __forceinline__ float ldg_stream_f1(const void *p) { return *reinterpret_cast<const float *>(p); }
#else
__device__ __forceinline__ ulonglong2 ldg_stream_u128(const void *p) {
    ulonglong2 v;
    asm volatile("ld.global.nc.L1::no_allocate.v2.u64 {%0,%1}, [%2];"
                 : "=l"(v.x), "=l"(v.y)
                 : "l"(p));
    return v;
}
__device__ __forceinline__ uint32_t ldg_stream_u32(const void *p) {
    uint32_t v;
    asm volatile("ld.global.nc.L1::no_allocate.u32 %0, [%1];" : "=r"(v) : "l"(p));
    return v;
}
__device__ __forceinline__ float4 ldg_stream_f4(const void *p) {
    float4 v;
    asm volatile("ld.global.nc.L1::no_allocate.v4.f32 {%0,%1,%2,%3}, [%4];"
                 : "=f"(v.x), "=f"(v.y), "=f"(v.z), "=f"(v.w)
                 : "l"(p));
    return v;
}
__device__ __forceinline__ float ldg_stream_f1(const void *p) {
    float v;
    asm volatile("ld.global.nc.L1::no_allocate.f32 %0, [%1];" : "=f"(v) : "l"(p));
    return v;
}
#endif

// Hint: bring the 128-byte line holding p into L2 (no register, no dependency; a wrong guess costs one line of traffic).
__device__ __forceinline__ void prefetch_l2(const void *p) {
#ifdef DANN_SIMT_EMU
    (void)p;
#else
    asm volatile("prefetch.global.L2 [%0];" ::"l"(p));
#endif
}

// Asynchronous global -> shared copy of one 4- or 8-byte word (LDGSTS: no register, the issuing thread does not wait);
// dann_cp_async_wait_all() makes this thread's copies visible to it, a __syncwarp() after it to the rest of the warp.
template <typename W>
__device__ __forceinline__ void dann_cp_async(W *smem_dst, const W *gmem_src) {
    static_assert(sizeof(W) == 4 || sizeof(W) == 8, "cp.async word size");
#ifdef DANN_SIMT_EMU
    *smem_dst = *gmem_src;
#else
    const unsigned d = (unsigned)__cvta_generic_to_shared(smem_dst);
    if constexpr (sizeof(W) == 4) asm volatile("cp.async.ca.shared.global [%0], [%1], 4;" ::"r"(d), "l"(gmem_src) : "memory");
    else asm volatile("cp.async.ca.shared.global [%0], [%1], 8;" ::"r"(d), "l"(gmem_src) : "memory");
#endif
}
__device__ __forceinline__ void dann_cp_async_commit() {
#ifndef DANN_SIMT_EMU
    asm volatile("cp.async.commit_group;" ::: "memory");
#endif
}
__device__ __forceinline__ void dann_cp_async_wait_all() {
#ifndef DANN_SIMT_EMU
    asm volatile("cp.async.wait_all;" ::: "memory");
#endif
}

// f32::total_cmp key (core::f32::total_cmp): monotone signed-int image of the float.
__device__ __forceinline__ int32_t total_key(float f) {
    int32_t b = __float_as_int(f);
    b ^= (int32_t)(((uint32_t)(b >> 31)) >> 1);
    return b;
}
// same, biased so that unsigned compare gives the total order
__device__ __forceinline__ uint32_t total_ukey(float f) { return (uint32_t)total_key(f) ^ 0x80000000u; }
// the float whose total_ukey is k (the sign-dependent xor of total_key is its own inverse)
__device__ __forceinline__ float total_ukey_inverse(uint32_t k) {
    int32_t b = (int32_t)(k ^ 0x80000000u);
    b ^= (int32_t)(((uint32_t)(b >> 31)) >> 1);
    return __int_as_float(b);
}

// labels/mod.rs:124-142 LabelSetView::overlaps (two-pointer over two ascending i16 arrays)
__device__ __forceinline__ bool labels_overlap(const int16_t *a, uint32_t na, const int16_t *b,
                                               uint32_t nb) {
    uint32_t i = 0, j = 0;
    while (i < na && j < nb) {
        int16_t x = __ldg(a + i), y = __ldg(b + j);
        if (x == y) return true;
        if (x < y) i++;
        else j++;
    }
    return false;
}
