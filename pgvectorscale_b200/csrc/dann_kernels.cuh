// dann_kernels.cuh — the non-graph kernels of the scan path (sm_90a):
//   prepare / prepare_plain : amrescan's vector preparation (cosine normalise + SBQ quantize)
//   sbq_distance     : stand-alone batched SBQ XOR+popcount gather (the roofline kernel)
//   full_distance    : exact f32 L2 / cosine / inner product, AVX2 summation order
//   rerank           : get_full_distance_for_resort + the sliding rerank window, a batch at a time
//   scan_distance / scan_finish : the same for the streaming scan, the rows of one or more amgettuple calls per step
//   scan_distance_many / scan_finish_many : one amgettuple of each of many scans per launch
//   normalize_rows / pad_rows / check_unique : index load helpers
// Reference paths are relative to pgvectorscale/src/access_method/.
// Every f32 operation that decides a result is spelled with an explicit-rounding
// intrinsic (__fadd_rn, __fmul_rn, __fmaf_rn, __fdiv_rn, __fsqrt_rn): nvcc never
// contracts or reorders those, so the arithmetic is the reference's op for op.
#pragma once
#include <math_constants.h>

#include "dann_device.cuh"
#include "dann_distance.cuh"
#include "dann_heap.cuh"
#include "dann_search_common.cuh"

/* f32::NAN (0x7fc00000): the "no distance" value of padded / unrescored rows */
#define DANN_NAN_F __int_as_float(0x7fc00000)

/* ------------------------------------------------------------------------------------ */
/* preprocess_cosine (distance/mod.rs:225-253): norm = sequential f32 sum of v*v;        */
/* returns the divisor (sqrt(norm)) or 0 when the vector is left untouched.              */
__device__ __forceinline__ float cosine_divisor_from_norm(float norm, uint32_t len) {
    const float eps = 1.1920929e-07f; /* f32::EPSILON */
    float adj = __fmul_rn(eps, (float)len);
    if (norm < eps) return 0.0f;
    if (norm >= __fsub_rn(1.0f, adj) && norm <= __fadd_rn(1.0f, adj)) return 0.0f;
    return __fsqrt_rn(norm);
}

/* amrescan's two cosine divisors of query row `src` (pg_vector.rs:125-157): `dfull` for the full copy of `dim` values,
 * `dindex` for the copy truncated to `dim_index`; 0 leaves a copy untouched, and always does when !cosine.  Block-wide. */
__device__ __forceinline__ void query_cosine_divisors(const float *src, uint32_t dim, uint32_t dim_index, bool cosine,
                                                      float &dfull, float &dindex) {
    DANN_STATIC_SMEM float s_div[2];
    if (cosine) {
        /* Iterator::sum over v*v in index order: a sequential dependent chain; two warps
         * run the two chains (full copy / truncated copy) side by side. */
        if (threadIdx.x == 0 || threadIdx.x == 32) {
            const uint32_t len = threadIdx.x == 0 ? dim : dim_index;
            float norm = 0.0f;
            for (uint32_t i = 0; i < len; i++) {
                float v = src[i];
                norm = __fadd_rn(norm, __fmul_rn(v, v));
            }
            s_div[threadIdx.x >> 5] = cosine_divisor_from_norm(norm, len);
        }
    } else if (threadIdx.x == 0) {
        s_div[0] = 0.0f;
        s_div[1] = 0.0f;
    }
    __syncthreads();
    dfull = s_div[0];
    dindex = s_div[1];
}

/* SbqQuantizer::quantize, one dimension (sbq/quantize.rs:52-102): number of leading ones */
__device__ __forceinline__ uint32_t sbq_count_ones(float v, float mean, float m2, float count_f,
                                                   uint32_t bits) {
    if (bits == 1) return v > mean ? 1u : 0u;
    float variance = __fdiv_rn(m2, count_f);
    float std_dev = __fsqrt_rn(variance);
    float z = __fdiv_rn(__fsub_rn(v, mean), std_dev);
    float ranges = (float)(bits + 1);
    float index = __fdiv_rn(__fadd_rn(z, 2.0f), __fdiv_rn(4.0f, ranges));
    if (index < 1.0f) return 0u;
    float fl = floorf(index); /* `index.floor() as usize`: saturating, NaN -> 0 */
    uint32_t as_u;
    if (!(fl == fl)) as_u = 0u;
    else if (fl >= 4294967040.0f) as_u = 0xFFFFFFFFu;
    else if (fl <= 0.0f) as_u = 0u;
    else as_u = (uint32_t)fl;
    return as_u < bits ? as_u : bits;
}

/* One CTA per query.  q_full_out [B][dim] (optional), q_codes_out [B][cw].
 * labels/mod.rs:209-238 (from_scan_key_data) -> pg_vector.rs:125-157 (create_inner: the
 * index copy is truncated to dim_index, each copy normalised on its own) ->
 * sbq/mod.rs:145-148 (quantize the index copy). */
__global__ void __launch_bounds__(128) dann_prepare_kernel(IndexView ix, const float *queries, int B,
                                                           float *q_full_out, uint64_t *q_codes_out) {
    DANN_DYN_SMEM(dann_smem);
    float *qi = reinterpret_cast<float *>(dann_smem); /* [dim_index] normalised index copy */
    const int q = blockIdx.x;
    const float *src = queries + (size_t)q * ix.dim;
    float dfull, dindex;
    query_cosine_divisors(src, ix.dim, ix.dim_index, ix.distance_type == DANN_COSINE, dfull, dindex);
    for (uint32_t i = threadIdx.x; i < ix.dim; i += blockDim.x) {
        float v = src[i];
        if (q_full_out) q_full_out[(size_t)q * ix.dim + i] = dfull != 0.0f ? __fdiv_rn(v, dfull) : v;
        if (i < ix.dim_index) qi[i] = dindex != 0.0f ? __fdiv_rn(v, dindex) : v;
    }
    __syncthreads();
    const float count_f = __ull2float_rn(ix.count); /* `self.count as f32` */
    for (uint32_t w = threadIdx.x; w < ix.cw; w += blockDim.x) {
        uint64_t word = 0;
        if (w < ix.words) {
            for (uint32_t b = 0; b < 64; b++) {
                uint32_t p = w * 64 + b;
                uint32_t i = p / ix.bits, j = p - i * ix.bits;
                if (i >= ix.dim_index) break;
                uint32_t ones = sbq_count_ones(qi[i], ix.mean[i], ix.bits > 1 ? ix.m2[i] : 0.0f,
                                               count_f, ix.bits);
                if (j < ones) word |= 1ull << b;
            }
        }
        q_codes_out[(size_t)q * ix.cw + w] = word;
    }
}

/* Plain storage layout: amrescan's vector preparation without a quantizer (pg_vector.rs:125-157): the full copy and
 * the copy truncated to dim_index, each cosine-normalised on its own.  One CTA per query. */
__global__ void __launch_bounds__(128) dann_prepare_plain_kernel(uint32_t dim, uint32_t dim_index, int cosine,
                                                                 const float *queries, float *q_full_out,
                                                                 float *q_index_out) {
    const int q = blockIdx.x;
    const float *src = queries + (size_t)q * dim;
    float dfull, dindex;
    query_cosine_divisors(src, dim, dim_index, cosine != 0, dfull, dindex);
    for (uint32_t i = threadIdx.x; i < dim; i += blockDim.x) {
        float v = src[i];
        q_full_out[(size_t)q * dim + i] = dfull != 0.0f ? __fdiv_rn(v, dfull) : v;
        if (i < dim_index) q_index_out[(size_t)q * dim_index + i] = dindex != 0.0f ? __fdiv_rn(v, dindex) : v;
    }
}

/* Plain storage layout, after the rerank kernel: every comparison of the beam search was a full-distance comparison
 * (plain/storage.rs:238,288), so d_full = candidates + reranked rows and d_quantized = 0.  Only launched when the
 * rerank ran (num_dimensions_to_index < num_dimensions, scan.rs:392-403). */
__global__ void dann_plain_stats_kernel(dann_query_stats *stats, int B, const QueryParam *qp = nullptr) {
    const int q = blockIdx.x * blockDim.x + threadIdx.x;
    if (q >= B) return;
    if (qp && qp[q].rescore == 0u) return; /* a query that reranks nothing keeps its search counters */
    dann_query_stats st = stats[q];
    st.d_full = st.candidates + st.d_full; /* the rerank kernel left the number of reranked rows here */
    st.d_quantized = 0;
    stats[q] = st;
}

/* ------------------------------------------------------------------------------------ */
/* Stand-alone SBQ distance: out[i] = popcount(code[pair_node[i]] ^ qcode[pair_q[i]])     */
/* (distance_xor_optimized, distance/mod.rs:265-323).  G lanes share one code row with    */
/* 128-bit no-allocate loads; UNR pairs are in flight per lane group.                     */
template <int NCH, int UNR>
__global__ void __launch_bounds__(512) dann_sbq_distance_kernel(const uint64_t *__restrict__ codes,
                                                                uint32_t cw,
                                                                const uint64_t *__restrict__ qcodes,
                                                                const uint32_t *__restrict__ pair_q,
                                                                const uint32_t *__restrict__ pair_node,
                                                                size_t npairs, uint32_t *__restrict__ out,
                                                                uint32_t G, uint32_t Gshift) {
    const uint32_t lane = threadIdx.x & 31, gl = lane & (G - 1);
    const uint32_t nchunks = cw >> 1;
    const size_t groups_per_block = blockDim.x >> Gshift;
    const size_t gid = (size_t)blockIdx.x * groups_per_block + (threadIdx.x >> Gshift);
    const size_t ngroups = (size_t)gridDim.x * groups_per_block;
    for (size_t p0 = gid * UNR; p0 < npairs; p0 += ngroups * UNR) {
        uint32_t nq[UNR], nn[UNR];
#pragma unroll
        for (int u = 0; u < UNR; u++) {
            size_t p = p0 + u;
            bool ok = p < npairs;
            nq[u] = ok ? ldg_stream_u32(pair_q + p) : 0u;
            nn[u] = ok ? ldg_stream_u32(pair_node + p) : 0u;
        }
        ulonglong2 v[UNR][NCH];
#pragma unroll
        for (int u = 0; u < UNR; u++) {
            const ulonglong2 *row = reinterpret_cast<const ulonglong2 *>(codes + (size_t)nn[u] * cw);
#pragma unroll
            for (int i = 0; i < NCH; i++) {
                uint32_t c = gl + i * G;
                v[u][i] = (c < nchunks && p0 + u < npairs) ? ldg_stream_u128(row + c) : make_ulonglong2(0, 0);
            }
        }
#pragma unroll
        for (int u = 0; u < UNR; u++) {
            const ulonglong2 *qrow = reinterpret_cast<const ulonglong2 *>(qcodes + (size_t)nq[u] * cw);
            uint32_t s = 0;
#pragma unroll
            for (int i = 0; i < NCH; i++) {
                uint32_t c = gl + i * G;
                if (c < nchunks) {
                    ulonglong2 qv = __ldg(qrow + c);
                    s += __popcll(v[u][i].x ^ qv.x) + __popcll(v[u][i].y ^ qv.y);
                }
            }
            for (uint32_t o = G >> 1; o > 0; o >>= 1) s += __shfl_xor_sync(DANN_FULL, s, o);
            if (gl == 0 && p0 + u < npairs) out[p0 + u] = s;
        }
    }
}

/* ---- 1-D TMA bulk copy (cp.async.bulk) of one query row into shared memory ---------- */
#ifndef DANN_SIMT_EMU
__device__ __forceinline__ uint32_t smem_u32(const void *p) {
    return (uint32_t)__cvta_generic_to_shared(p);
}
__device__ __forceinline__ void mbar_init(uint64_t *bar, uint32_t count) {
    asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count));
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
}
__device__ __forceinline__ void tma_load_1d(void *dst, const void *src, uint32_t bytes, uint64_t *bar) {
    asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes)
                 : "memory");
    asm volatile(
        "cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(
            smem_u32(dst)),
        "l"(src), "r"(bytes), "r"(smem_u32(bar))
        : "memory");
}
__device__ __forceinline__ void mbar_wait(uint64_t *bar, uint32_t phase) {
    asm volatile(
        "{\n"
        ".reg .pred p;\n"
        "WAIT_%=:\n"
        "mbarrier.try_wait.parity.shared::cta.b64 p, [%0], %1;\n"
        "@p bra DONE_%=;\n"
        "bra WAIT_%=;\n"
        "DONE_%=:\n"
        "}\n" ::"r"(smem_u32(bar)),
        "r"(phase)
        : "memory");
}

#endif /* !DANN_SIMT_EMU */

/* Stage query row `src` [n floats] into shared `dst`: TMA bulk copy when the row is a
 * multiple of 16 B and 16-B aligned, plain loads otherwise.  Block-wide. */
__device__ __forceinline__ void stage_query_row(float *dst, const float *src, uint32_t n, uint64_t *bar) {
#ifndef DANN_SIMT_EMU
    const bool tma_ok = (n & 3u) == 0 && ((reinterpret_cast<uintptr_t>(src) & 15u) == 0);
    if (tma_ok) {
        if (threadIdx.x == 0) mbar_init(bar, 1);
        __syncthreads();
        if (threadIdx.x == 0) tma_load_1d(dst, src, n * 4u, bar);
        mbar_wait(bar, 0);
    } else
#else
    (void)bar; /* no TMA under the CPU emulator: the plain-copy branch below */
#endif
    {
        for (uint32_t i = threadIdx.x; i < n; i += blockDim.x) dst[i] = src[i];
        __syncthreads();
    }
}

/* out[i] = distance_fn(vectors[nodes[i]], qs) for i in [begin, end), begin <= end, with the query row `qs` already
 * staged in shared memory: 8 lanes per row, 128-bit loads when dim is a multiple of 4.  DANN_INVALID_NODE reads row 0
 * and gives DANN_NAN_F.  Block-wide. */
__device__ __forceinline__ void full_distances(const IndexView &ix, const float *qs, const uint32_t *nodes,
                                               uint32_t begin, uint32_t end, float *out) {
    const uint32_t lane = threadIdx.x & 31, mm = lane & 7, gbase = lane & 24;
    const uint32_t group = threadIdx.x >> 3, ngroups = blockDim.x >> 3;
    const bool vec4 = (ix.dim & 3u) == 0;
    const uint32_t rounds = (end - begin + ngroups - 1) / ngroups;
    for (uint32_t r = 0; r < rounds; r++) {
        const uint32_t it = begin + r * ngroups + group;
        const uint32_t node = it < end ? nodes[it] : DANN_INVALID_NODE;
        const float *x = ix.vectors + (size_t)(node == DANN_INVALID_NODE ? 0 : node) * ix.dim;
        const float d = vec4 ? full_distance_group8<true>(ix.distance_type, x, qs, ix.dim, mm, gbase)
                             : full_distance_group8<false>(ix.distance_type, x, qs, ix.dim, mm, gbase);
        if (mm == 0 && it < end) out[it] = node == DANN_INVALID_NODE ? DANN_NAN_F : d;
    }
}

/* out[b*m+i] = distance_fn(vectors[nodes[b*m+i]], q_full[b]) ; one CTA per query */
__global__ void __launch_bounds__(128) dann_full_distance_kernel(IndexView ix, const float *q_full,
                                                                 const uint32_t *nodes, int m, float *out) {
    DANN_DYN_SMEM(dann_smem);
    float *qs = reinterpret_cast<float *>(dann_smem);
    DANN_STATIC_SMEM uint64_t bar;
    const int q = blockIdx.x;
    stage_query_row(qs, q_full + (size_t)q * ix.dim, ix.dim, &bar);
    full_distances(ix, qs, nodes + (size_t)q * m, 0, (uint32_t)m, out + (size_t)q * m);
}

/* ------------------------------------------------------------------------------------ */
/* next_with_resort (scan.rs:244-305) for the first k rows of one query per CTA:          */
/*   phase 1  get_full_distance_for_resort (sbq/storage.rs:304-328) of every streamed     */
/*            node — 8 lanes per 3-KB row, 128-bit loads, query row staged by TMA;        */
/*   phase 2  the sliding window: a BinaryHeap<ResortData> (min on total_cmp distance,    */
/*            scan.rs:111-117) filled to `rescore`, pop one, refill one, ...              */
/* rescore == 0 bypasses phase 1 and returns the stream order (scan.rs:251-253).          */
struct RerankArgs {
    IndexView ix;
    const float *q_full;        /* [B][dim] */
    const uint32_t *stream;     /* [B][c_target] */
    const uint32_t *stream_len; /* [B] */
    uint32_t c_target, k, rescore;
    uint64_t *out_tid;          /* [B][k] */
    float *out_dist;            /* [B][k] or NULL */
    uint32_t *out_node;         /* [B][k] or NULL */
    uint32_t *out_count;        /* [B] or NULL */
    dann_query_stats *stats;    /* [B] or NULL : d_full is filled here */
    /* per-query k, rescore and c_target (NULL = the three above apply to every query).  When set, c_target and k above
     * are the row strides of the stream and the outputs, the batch maxima, and query q's rows past its own k are
     * filled like the rows past its count.  Kept last. */
    const QueryParam *qp = nullptr;
};

__global__ void __launch_bounds__(128) dann_rerank_kernel(const RerankArgs a) {
    DANN_DYN_SMEM(dann_smem);
    const IndexView &ix = a.ix;
    float *qs = reinterpret_cast<float *>(dann_smem);                    /* [dim rounded to 4] */
    const uint32_t dim4 = (ix.dim + 3u) & ~3u;
    const int q = blockIdx.x;
    /* this query's k, rescore and stream length: its CTA lays out shared memory for its own sizes */
    const uint32_t rescore = a.qp ? a.qp[q].rescore : a.rescore;
    const uint32_t ctq = a.qp ? a.qp[q].c_target : a.c_target;
    float *ds = qs + dim4;                                              /* [ctq] */
    uint64_t *hp = reinterpret_cast<uint64_t *>(ds + ((ctq + 1u) & ~1u)); /* [rescore] */
    DANN_STATIC_SMEM uint64_t bar;
    const uint32_t sl = a.stream_len[q];
    const uint32_t *st = a.stream + (size_t)q * a.c_target;
    uint64_t *otid = a.out_tid + (size_t)q * a.k;

    if (rescore == 0) {
        const uint32_t kq = a.qp ? a.qp[q].k : a.k;
        const uint32_t rows = sl < kq ? sl : kq;
        for (uint32_t i = threadIdx.x; i < a.k; i += blockDim.x) {
            bool ok = i < rows;
            uint32_t node = ok ? st[i] : DANN_INVALID_NODE;
            otid[i] = ok ? ix.tids[node] : DANN_INVALID_TID;
            if (a.out_dist) a.out_dist[(size_t)q * a.k + i] = DANN_NAN_F;
            if (a.out_node) a.out_node[(size_t)q * a.k + i] = node;
        }
        if (threadIdx.x == 0 && a.out_count) a.out_count[q] = rows;
        return;
    }

    stage_query_row(qs, a.q_full + (size_t)q * ix.dim, ix.dim, &bar);
    full_distances(ix, qs, st, 0, sl, ds);
    __syncthreads();
    if (threadIdx.x == 0) {
        using H = RustHeap<uint64_t, 32>;
        ArrayStore<uint64_t> store{hp};
        /* read again rather than held across the distance phase (which would cost a spill) */
        const uint32_t kq = a.qp ? a.qp[q].k : a.k, window = a.qp ? a.qp[q].rescore : a.rescore;
        uint32_t len = 0, si = 0, rows = 0;
        for (; rows < kq; rows++) {
            while (len < window && si < sl) { /* refill: resort_buffer.push(ResortData{..}) */
                H::push(store, len, ((uint64_t)total_ukey(ds[si]) << 32) | si);
                si++;
            }
            if (len == 0) break;
            uint64_t e = H::pop(store, len);
            uint32_t idx = (uint32_t)e, node = st[idx];
            otid[rows] = ix.tids[node];
            if (a.out_dist) a.out_dist[(size_t)q * a.k + rows] = ds[idx];
            if (a.out_node) a.out_node[(size_t)q * a.k + rows] = node;
        }
        if (a.out_count) a.out_count[q] = rows;
        if (a.stats) a.stats[q].d_full = si; /* full_distance_comparisons, scan.rs:258 */
        for (uint32_t i = rows; i < a.k; i++) {
            otid[i] = DANN_INVALID_TID;
            if (a.out_dist) a.out_dist[(size_t)q * a.k + i] = DANN_NAN_F;
            if (a.out_node) a.out_node[(size_t)q * a.k + i] = DANN_INVALID_NODE;
        }
    }
}

/* ------------------------------------------------------------------------------------ */
/* Index load: cosine rows are normalised ONCE with preprocess_cosine's arithmetic        */
/* (sequential sum per row).  Each warp takes 32 rows: coalesced 128-B row segments go     */
/* through a padded shared tile so that every lane runs the sequential chain of one row.  */
__global__ void __launch_bounds__(256) dann_normalize_rows_kernel(float *vectors, uint32_t n, uint32_t dim) {
    DANN_STATIC_SMEM float tile[8][32][33];
    DANN_STATIC_SMEM float divs[8][32];
    const uint32_t lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const uint32_t nblocks32 = (n + 31) / 32;
    for (uint32_t blk = blockIdx.x * 8 + warp; blk < nblocks32; blk += gridDim.x * 8) {
        const uint32_t row0 = blk * 32;
        float norm = 0.0f;
        for (uint32_t c0 = 0; c0 < dim; c0 += 32) {
            for (uint32_t r = 0; r < 32; r++) {
                uint32_t row = row0 + r, col = c0 + lane;
                tile[warp][r][lane] = (row < n && col < dim) ? vectors[(size_t)row * dim + col] : 0.0f;
            }
            __syncwarp();
            uint32_t lim = dim - c0 < 32 ? dim - c0 : 32;
            for (uint32_t j = 0; j < lim; j++) {
                float v = tile[warp][lane][j];
                norm = __fadd_rn(norm, __fmul_rn(v, v));
            }
            __syncwarp();
        }
        divs[warp][lane] = cosine_divisor_from_norm(norm, dim);
        __syncwarp();
        for (uint32_t r = 0; r < 32; r++) {
            uint32_t row = row0 + r;
            float dv = divs[warp][r];
            if (row < n && dv != 0.0f)
                for (uint32_t col = lane; col < dim; col += 32) {
                    size_t o = (size_t)row * dim + col;
                    vectors[o] = __fdiv_rn(vectors[o], dv);
                }
        }
        __syncwarp();
    }
}

/* dst[n][dst_w] <- src[n][src_w] padded with `fill` (u32 rows: neighbour lists; u64: codes) */
template <typename Tp>
__global__ void dann_pad_rows_kernel(Tp *dst, const Tp *src, size_t n, uint32_t src_w, uint32_t dst_w,
                                     Tp fill) {
    size_t total = n * dst_w;
    for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < total;
         i += (size_t)gridDim.x * blockDim.x) {
        size_t r = i / dst_w;
        uint32_t c = (uint32_t)(i - r * dst_w);
        dst[i] = c < src_w ? src[r * src_w + c] : fill;
    }
}

/* Index load: does any neighbour list repeat an id?  (The reference's builder never produces
 * one — add_neighbors dedupes through a HashSet, graph/mod.rs:212-266 — but the scan must not
 * depend on that: when a list does, the search kernel stages the list 32 ids at a time so the
 * FIRST occurrence is the one that inserts.)  One warp per row, lists up to 64 ids. */
__global__ void dann_check_unique_kernel(const uint32_t *nbrs, uint32_t n, uint32_t R, uint32_t Rp,
                                         uint32_t *flag) {
    const uint32_t lane = threadIdx.x & 31;
    const uint32_t warps = (gridDim.x * blockDim.x) >> 5;
    for (uint32_t row = (blockIdx.x * blockDim.x + threadIdx.x) >> 5; row < n; row += warps) {
        const uint32_t *r = nbrs + (size_t)row * Rp;
        uint32_t n0 = lane < R ? r[lane] : DANN_INVALID_NODE;
        uint32_t n1 = lane + 32 < R ? r[lane + 32] : DANN_INVALID_NODE;
        bool v0, v1;
        neighbour_cut(n0, n1, (int)lane, v0, v1);
        if (!v0) n0 = DANN_INVALID_NODE;
        if (!v1) n1 = DANN_INVALID_NODE;
        const unsigned mm0 = __match_any_sync(DANN_FULL, n0), mm1 = __match_any_sync(DANN_FULL, n1);
        bool dup = (v0 && __popc(mm0) > 1) || (v1 && __popc(mm1) > 1);
        for (int k = 0; k < 32; k++) {
            uint32_t x = __shfl_sync(DANN_FULL, n1, k);
            dup |= v0 && x != DANN_INVALID_NODE && x == n0;
        }
        if (__any_sync(DANN_FULL, dup) && lane == 0) atomicOr(flag, 1u);
    }
}

/* ------------------------------------------------------------------------------------ */
/* Streaming scan (dann_scan_gettuple, dann_scan_fetch): one step of next_with_resort (scan.rs:244-305) yields the rows of
 * one or more consecutive amgettuple calls, with one host synchronisation.  The search launch, dann_scan_distance_kernel
 * (exact distances of the rows the search appended) and dann_scan_finish_kernel (the window step) are enqueued back to
 * back; the two kernels read the search's outcome (rows produced, overflow bits) from device memory, and the last one
 * gathers everything the host needs into one ScanStepOut and one ScanRow per row.  A search that overflowed its
 * workspace leaves the window alone.  The rerank window lives in HBM between calls: win[] is the
 * BinaryHeap<ResortData> array, entries (total_cmp key of the exact distance << 32) | node. */
struct ScanWindow {
    uint32_t len, d_full;
};
/* one row of a step, with the scan's counters after the amgettuple call that would have returned it */
struct ScanRow {
    uint64_t tid;
    uint32_t node;
    float dist;
    uint32_t end;                /* the stream index its refill ended at */
    uint32_t d_full;             /* the window's full-distance comparisons after its refill */
    uint32_t visits, candidates; /* the search's counters */
};
struct ScanStepOut {
    uint32_t overflow, slen;
    uint32_t nrows, pad;     /* rows produced: fewer than asked only at end of scan */
    dann_query_stats stats;  /* the search's counters at the end of the step */
    ScanWindow win;
};
#define DANN_SCAN_WIN_MAX 1000u /* the largest window: rescore <= 1000 */

/* Exact distances of the rows a scan's search appended in [begin, begin + span) (none when it overflowed), into out[].
 * qs: the dynamic window, [dim rounded up to 4].  Block-wide. */
__device__ __forceinline__ void scan_distance_step(const IndexView &ix, float *qs, uint64_t *bar, const float *q_full,
                                                   const uint32_t *stream, const uint32_t *slen_p,
                                                   const uint32_t *overflow_p, uint32_t begin, uint32_t span, float *out) {
    if (*overflow_p) return;
    const uint32_t slen = *slen_p;
    if (slen <= begin) return;
    const uint32_t end = slen - begin > span ? begin + span : slen;
    stage_query_row(qs, q_full, ix.dim, bar);
    full_distances(ix, qs, stream, begin, end, out);
}

/* CTA b: rows [skip + b * span, skip + (b + 1) * span) of the step; the host sizes the grid from the rows the search
 * may append, and CTAs past the rows it did append exit */
__global__ void __launch_bounds__(128) dann_scan_distance_kernel(IndexView ix, const float *q_full, const uint32_t *stream,
                                                                 const uint32_t *slen_p, const uint32_t *overflow_p,
                                                                 uint32_t skip, uint32_t span, float *out) {
    DANN_DYN_SMEM(dann_smem);
    float *qs = reinterpret_cast<float *>(dann_smem);
    DANN_STATIC_SMEM uint64_t bar;
    scan_distance_step(ix, qs, &bar, q_full, stream, slen_p, overflow_p, skip + blockIdx.x * span, span, out);
}

/* One amgettuple step of many scans (dann_scan_gettuple_many, and the first step of a sharded scan): the arguments
 * dann_scan_distance_kernel and dann_scan_finish_kernel take, per scan.  `view` picks the scan's index in the launch's
 * table of IndexViews, so one launch can carry scans of several indexes on one device. */
struct ScanDistanceDesc {
    const float *q_full;
    const uint32_t *stream, *slen_p, *overflow_p;
    float *out;
    uint32_t skip, view;
};
struct ScanFinishDesc {
    ScanWindow *w;
    uint64_t *win;
    const uint32_t *stream;
    const float *dist;
    const uint32_t *slen_p;     /* NULL: the scan did not search this step */
    const uint32_t *overflow_p; /* NULL: the scan did not search this step */
    const dann_query_stats *stats_p;
    uint32_t rescore, skip, slen_fixed, view;
};

/* CTA b: the exact distances of scan d[b], which searched with rescore > 0, on its index views[d[b].view] */
__global__ void __launch_bounds__(128) dann_scan_distance_many_kernel(const IndexView *views, const ScanDistanceDesc *d) {
    DANN_DYN_SMEM(dann_smem);
    float *qs = reinterpret_cast<float *>(dann_smem);
    DANN_STATIC_SMEM uint64_t bar;
    const ScanDistanceDesc &e = d[blockIdx.x];
    scan_distance_step(views[e.view], qs, &bar, e.q_full, e.stream, e.slen_p, e.overflow_p, e.skip, 0xFFFFFFFFu, e.out);
}

/* The window step of one scan, on one thread: for each of up to nrows rows, next_with_resort's refill (push stream rows
 * until the window holds `rescore`, or the rows the search appended run out), then one pop; with rescore == 0 the rows
 * in stream order.  rows[r] gets row r's node, distance, refill end and d_full (scan_row_fill adds its tid and
 * counters); *out gathers the step (overflow bits, rows appended and produced, final counters, the window).  win is the
 * window's heap array: in HBM, or a shared-memory copy of it. */
__device__ __forceinline__ void scan_finish_step(ScanWindow *w, uint64_t *win, uint32_t rescore, const uint32_t *stream,
                                                 const float *dist, uint32_t skip, const uint32_t *slen_p, uint32_t slen_fixed,
                                                 const uint32_t *overflow_p, const dann_query_stats *stats_p, uint32_t nrows,
                                                 ScanStepOut *out, ScanRow *rows) {
    ScanStepOut o;
    o.overflow = overflow_p ? *overflow_p : 0u;
    o.slen = slen_p ? *slen_p : slen_fixed; /* no search this call: nothing new beyond `skip` */
    o.nrows = 0;
    o.pad = 0;
    o.stats = *stats_p;
    o.win = *w;
    if (o.overflow) { /* the host regrows the workspace and replays: the window must not move */
        *out = o;
        return;
    }
    uint32_t pos = skip;
    if (rescore == 0) { /* resort_buffer.capacity() == 0: the stream order is the result (scan.rs:251-253) */
        for (; o.nrows < nrows && pos < o.slen; o.nrows++, pos++) {
            ScanRow &x = rows[o.nrows];
            x.node = stream[pos];
            x.dist = DANN_NAN_F;
            x.end = pos + 1;
            x.d_full = o.win.d_full;
        }
        *out = o;
        return;
    }
    using H = RustHeap<uint64_t, 32>;
    ArrayStore<uint64_t> store{win};
    uint32_t len = o.win.len, dfull = o.win.d_full;
    for (; o.nrows < nrows; o.nrows++) {
        for (; len < rescore && pos < o.slen; pos++) { /* full_distance_comparisons += 1; resort_buffer.push(..) */
            H::push(store, len, ((uint64_t)total_ukey(dist[pos]) << 32) | stream[pos]);
            dfull++;
        }
        if (len == 0) break;
        const uint64_t e = H::pop(store, len);
        ScanRow &x = rows[o.nrows];
        x.node = (uint32_t)e;
        x.dist = total_ukey_inverse((uint32_t)(e >> 32));
        x.end = pos;
        x.d_full = dfull;
    }
    w->len = o.win.len = len;
    w->d_full = o.win.d_full = dfull;
    *out = o;
}

/* Row r's tid and counters.  Its refill asked for the stream up to index skip + first + r (first = the rows the step's
 * first refill asked for).  If it got them all, the call that returns it would have stopped its search right after
 * appending the last of them: the counters at that row (snap; a one-row step passes NULL, its search stopped there).
 * If the stream ended during that refill or before it, or the step did not search, that call's search ran dry: the
 * step's final counters st. */
__device__ __forceinline__ void scan_row_fill(const IndexView &ix, ScanRow &x, uint32_t r, uint32_t first, uint32_t skip,
                                              bool searched, const uint2 *snap, const dann_query_stats &st) {
    x.tid = ix.tids[x.node];
    if (searched && snap && x.end == skip + first + r) {
        const uint2 c = snap[x.end - 1];
        x.visits = c.x;
        x.candidates = c.y;
    } else {
        x.visits = st.visits;
        x.candidates = st.candidates;
    }
}

/* One step of one scan (dann_scan_gettuple: nrows = 1; dann_scan_fetch): the window step on thread 0, then every row's
 * tid and counters across the CTA.  A step of several rows stages the window (at most DANN_SCAN_WIN_MAX entries) in
 * shared memory for its pushes and pops and writes it back once. */
__global__ void __launch_bounds__(128) dann_scan_finish_kernel(IndexView ix, ScanWindow *w, uint64_t *win, uint32_t rescore,
                                                               const uint32_t *stream, const float *dist, const uint2 *snap,
                                                               uint32_t skip, const uint32_t *slen_p, uint32_t slen_fixed,
                                                               const uint32_t *overflow_p, const dann_query_stats *stats_p,
                                                               uint32_t nrows, ScanStepOut *out, ScanRow *rows) {
    DANN_STATIC_SMEM uint64_t win_sm[DANN_SCAN_WIN_MAX];
    const uint32_t len0 = w->len;
    const bool stage = nrows > 1 && rescore > 0 && !(overflow_p && *overflow_p);
    if (stage)
        for (uint32_t i = threadIdx.x; i < len0; i += blockDim.x) win_sm[i] = win[i];
    __syncthreads(); /* every thread has read the window before thread 0 moves it */
    if (threadIdx.x == 0)
        scan_finish_step(w, stage ? win_sm : win, rescore, stream, dist, skip, slen_p, slen_fixed, overflow_p, stats_p, nrows,
                         out, rows);
    __syncthreads();
    const ScanStepOut &o = *out;
    if (stage)
        for (uint32_t i = threadIdx.x; i < o.win.len; i += blockDim.x) win[i] = win_sm[i];
    const uint32_t first = rescore == 0 ? 1u : (len0 < rescore ? rescore - len0 : 0u);
    for (uint32_t r = threadIdx.x; r < o.nrows; r += blockDim.x)
        scan_row_fill(ix, rows[r], r, first, skip, slen_p != nullptr, snap, o.stats);
}

/* thread i: the one-row window step of scan d[i] on its index views[d[i].view], its outcome into out[i] and rows[i] (one
 * copy brings every scan's back) */
__global__ void __launch_bounds__(128) dann_scan_finish_many_kernel(const IndexView *views, const ScanFinishDesc *d,
                                                                    uint32_t n, ScanStepOut *out, ScanRow *rows) {
    const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const ScanFinishDesc f = d[i];
    scan_finish_step(f.w, f.win, f.rescore, f.stream, f.dist, f.skip, f.slen_p, f.slen_fixed, f.overflow_p, f.stats_p, 1u,
                     out + i, rows + i);
    if (out[i].nrows) scan_row_fill(views[f.view], rows[i], 0u, 1u, f.skip, f.slen_p != nullptr, nullptr, out[i].stats);
}
