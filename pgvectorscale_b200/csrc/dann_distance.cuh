// dann_distance.cuh — the exact f32 distance of the reference's AVX2 path (distance/mod.rs:88-209,325-434,
// distance_x86.rs:21-36), one row per 8-lane group.  Used by the rerank kernels (dann_kernels.cuh) and by the
// plain-storage flavour of the beam search (dann_search.cuh).  No PTX beyond the streaming loads of dann_device.cuh,
// so the file also compiles for the CPU SIMT emulator.
#pragma once
#include "dann_device.cuh"

/* ------------------------------------------------------------------------------------ */
/* Exact distance with the reference's AVX2 summation order.                             */
/* distance_l2_simd_body! / inner_product_simd_body! (distance/mod.rs:325-434) with       */
/* S = Avx2: element e = 32*i + 8*k + j goes to accumulator k, lane j, steps i in order.  */
/* Here 8 GPU lanes share one row: lane m (0..7) owns the four accumulator slots          */
/* 4m..4m+3 (k = m/2, j = 4*(m%2)+t), i.e. one float4 per 32-element stride, so the 8      */
/* lanes read 128 contiguous bytes per step.  `y` is the query (shared memory).           */
/* Returns the finished distance on every lane of the 8-lane group.                      */
template <bool VEC4>
__device__ __forceinline__ float full_distance_group8(int type, const float *__restrict__ x,
                                                      const float *__restrict__ y, uint32_t n,
                                                      uint32_t m, unsigned gmask_base_lane) {
    float a0 = 0.0f, a1 = 0.0f, a2 = 0.0f, a3 = 0.0f;
    const uint32_t nfull = n >> 5;
    const bool l2 = type == DANN_L2;
    constexpr int UN = 8;
    for (uint32_t i0 = 0; i0 < nfull; i0 += UN) {
        float4 xv[UN];
#pragma unroll
        for (int u = 0; u < UN; u++) {
            uint32_t i = i0 + u;
            if (i < nfull) {
                const float *px = x + 32 * i + 4 * m;
                if (VEC4) xv[u] = ldg_stream_f4(px);
                else xv[u] = make_float4(ldg_stream_f1(px), ldg_stream_f1(px + 1), ldg_stream_f1(px + 2),
                                         ldg_stream_f1(px + 3));
            }
        }
#pragma unroll
        for (int u = 0; u < UN; u++) {
            uint32_t i = i0 + u;
            if (i < nfull) {
                const float *py = y + 32 * i + 4 * m;
                float4 yv = VEC4 ? *reinterpret_cast<const float4 *>(py) : make_float4(py[0], py[1], py[2], py[3]);
                if (l2) { /* accum = accum + ((x - y) * (x - y)) : separate sub, mul, add */
                    float d0 = __fsub_rn(xv[u].x, yv.x), d1 = __fsub_rn(xv[u].y, yv.y);
                    float d2 = __fsub_rn(xv[u].z, yv.z), d3 = __fsub_rn(xv[u].w, yv.w);
                    a0 = __fadd_rn(a0, __fmul_rn(d0, d0));
                    a1 = __fadd_rn(a1, __fmul_rn(d1, d1));
                    a2 = __fadd_rn(a2, __fmul_rn(d2, d2));
                    a3 = __fadd_rn(a3, __fmul_rn(d3, d3));
                } else { /* accum = fmadd(x, y, accum) */
                    a0 = __fmaf_rn(xv[u].x, yv.x, a0);
                    a1 = __fmaf_rn(xv[u].y, yv.y, a1);
                    a2 = __fmaf_rn(xv[u].z, yv.z, a2);
                    a3 = __fmaf_rn(xv[u].w, yv.w, a3);
                }
            }
        }
    }
    /* simdeez Avx2::horizontal_add_ps: ((a0+a4)+(a1+a5)) + ((a2+a6)+(a3+a7)); the pair of
     * lanes (2k, 2k+1) holds accumulator k: lane 2k has j=0..3, lane 2k+1 has j=4..7. */
    float v0 = __fadd_rn(a0, __shfl_xor_sync(DANN_FULL, a0, 1));
    float v1 = __fadd_rn(a1, __shfl_xor_sync(DANN_FULL, a1, 1));
    float v2 = __fadd_rn(a2, __shfl_xor_sync(DANN_FULL, a2, 1));
    float v3 = __fadd_rn(a3, __shfl_xor_sync(DANN_FULL, a3, 1));
    float h = __fadd_rn(__fadd_rn(v0, v1), __fadd_rn(v2, v3));
    float h0 = __shfl_sync(DANN_FULL, h, gmask_base_lane + 0);
    float h1 = __shfl_sync(DANN_FULL, h, gmask_base_lane + 2);
    float h2 = __shfl_sync(DANN_FULL, h, gmask_base_lane + 4);
    float h3 = __shfl_sync(DANN_FULL, h, gmask_base_lane + 6);
    float dist = __fadd_rn(__fadd_rn(__fadd_rn(h0, h1), h2), h3);
    /* scalar tail, in order (every lane of the group computes the same chain) */
    for (uint32_t i = nfull << 5; i < n; i++) {
        float xi = ldg_stream_f1(x + i), yi = y[i];
        if (l2) {
            float diff = __fsub_rn(xi, yi);
            dist = __fadd_rn(dist, __fmul_rn(diff, diff));
        } else {
            dist = __fadd_rn(dist, __fmul_rn(xi, yi));
        }
    }
    /* A NaN sum (inf + -inf; finite inputs reach it only in an inner product) carries the bits of the reference's x86
     * build: SSE's default NaN 0xFFC00000, sign-flipped by the inner product's `-dist`.  The GPU's float unit would
     * return its own canonical NaN (0x7FFFFFFF), so the constant is selected, not computed: any float operation on it
     * would canonicalise it again. */
    const bool nan = dist != dist;
    if (type == DANN_L2) return nan ? __int_as_float(0xFFC00000) : dist;  /* distance/mod.rs:88-104 (no sqrt) */
    if (type == DANN_IP) return nan ? __int_as_float(0x7FC00000) : -dist; /* :175-190 */
    float r = __fsub_rn(1.0f, dist);                  /* distance_x86.rs:34-36 (1.0 - ip).max(0.0): NaN -> +0.0 */
    return r > 0.0f ? r : 0.0f;
}

