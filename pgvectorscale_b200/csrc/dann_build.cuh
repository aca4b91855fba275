// dann_build.cuh — GPU batch Vamana construction over SBQ codes (SURVEY.md §8f row 1).
//
// NOT part of the scan hot path: this is the first "next" row of the scope table, built from the
// hot path's own kernels.  The reference builds its graph serially (graph/mod.rs:637-737: search
// the current graph for the new node with quantized distances, alpha-prune the visited set,
// add back-pointers and prune on overflow).  A batch of nodes is inserted here at once, the way
// parallel DiskANN builders do:
//   1. greedy_search_for_build (graph/mod.rs:285-327) for every node of the batch with the beam
//      search kernel in build mode (query code = the node's own SBQ code, result = visited list);
//   2. prune_neighbors (graph/mod.rs:392-488) per node: a warp-cooperative restatement of the
//      two-round alpha prune over Hamming distances (sbq/mod.rs:178-190 node-to-node distances);
//   3. update_back_pointer (graph/mod.rs:720-737): the (neighbour <- node) edges of the batch are
//      sorted by destination, appended, and lists that outgrow the slack are pruned again.
// The result is a valid diskann graph but not the reference's serial one (insertion is batched),
// so it is used for fixtures/benchmarks; scan parity is always checked oracle-vs-GPU on the SAME
// graph.
#pragma once
#include "dann_device.cuh"

/* labels/mod.rs:84-111 LabelSet::contains_intersection: is (a ∩ b) ⊆ c ?  (sorted i16 arrays) */
__device__ __forceinline__ bool labels_contains_intersection(const int16_t *c, uint32_t nc, const int16_t *a, uint32_t na,
                                                             const int16_t *b, uint32_t nb) {
    uint32_t i = 0, j = 0, k = 0;
    while (i < na && j < nb) {
        int16_t x = __ldg(a + i), y = __ldg(b + j);
        if (x == y) {
            while (k < nc && __ldg(c + k) < x) k++;
            if (k == nc || __ldg(c + k) > x) return false;
            i++;
            j++;
        } else if (x < y) {
            i++;
        } else {
            j++;
        }
    }
    return true;
}

#define DANN_BUILD_CMAX 128u /* candidates considered by one prune */
#define DANN_BUILD_SLACK 64u /* neighbour slots per node while building (the reference keeps up to ceil(1.3 R), unbounded by slots) */

/* candidate key: (distance << 32) | node id ; sorted ascending = reference's candidates.sort() up to
 * the tie-break among equal distances (id order here, ip_distance order there) */

__device__ __forceinline__ void build_bitonic_sort128(uint64_t *k, int lane) {
    for (uint32_t size = 2; size <= DANN_BUILD_CMAX; size <<= 1) {
        for (uint32_t stride = size >> 1; stride > 0; stride >>= 1) {
            for (uint32_t t = lane; t < DANN_BUILD_CMAX; t += 32) {
                uint32_t u = t ^ stride;
                if (u > t) {
                    uint64_t a = k[t], b = k[u];
                    bool up = (t & size) == 0;
                    if ((a > b) == up) {
                        k[t] = b;
                        k[u] = a;
                    }
                }
            }
            __syncwarp();
        }
    }
}

/* prune_neighbors (graph/mod.rs:392-488) for point `p`: ck[0..C) sorted candidate keys (no duplicates,
 * p itself excluded).  cc = staging for candidate codes [C][cws] (cws odd stride), mf[C] factors.
 * Writes up to R (id, dist) pairs; returns the count. */
__device__ __forceinline__ uint32_t build_prune_warp(const uint64_t *__restrict__ codes, uint32_t cw, uint32_t cws,
                                                     uint32_t p, const uint64_t *ck, float *mf, uint64_t *cc,
                                                     uint32_t C, uint32_t R, float max_alpha, uint32_t *out_id,
                                                     uint16_t *out_d, int lane, const uint32_t *label_off = nullptr,
                                                     const int16_t *labels = nullptr) {
    const int16_t *pl = nullptr;
    uint32_t npl = 0;
    if (label_off) {
        uint32_t o0 = __ldg(label_off + p);
        pl = labels + o0;
        npl = __ldg(label_off + p + 1) - o0;
    }
    for (uint32_t c = 0; c < C; c++) {
        const uint64_t *row = codes + (size_t)(uint32_t)ck[c] * cw;
        for (uint32_t w = lane; w < cw; w += 32) cc[c * cws + w] = __ldg(row + w);
    }
    for (uint32_t c = lane; c < C; c += 32) mf[c] = 0.0f;
    __syncwarp();
    uint32_t nres = 0;
    float alpha = 1.0f;
    while (alpha <= max_alpha && nres < R) {
        for (uint32_t i = 0; i < C && nres < R; i++) {
            if (mf[i] > alpha) continue;
            __syncwarp();
            if (lane == 0) {
                mf[i] = 3.0e38f; /* don't consider again */
                out_id[nres] = (uint32_t)ck[i];
                out_d[nres] = (uint16_t)(ck[i] >> 32);
            }
            nres++;
            const uint32_t idi = (uint32_t)ck[i];
            const uint64_t *ci = cc + i * cws;
            const int16_t *il = nullptr;
            uint32_t nil = 0;
            if (label_off) {
                uint32_t o0 = __ldg(label_off + idi);
                il = labels + o0;
                nil = __ldg(label_off + idi + 1) - o0;
            }
            for (uint32_t j = i + 1 + lane; j < C; j += 32) {
                float f = mf[j];
                if (f > max_alpha) continue; /* completely excluded already */
                if (label_off) { /* does the kept neighbour carry every label the candidate shares with the point? */
                    const uint32_t idj0 = (uint32_t)ck[j];
                    uint32_t o0 = __ldg(label_off + idj0);
                    if (!labels_contains_intersection(il, nil, labels + o0, __ldg(label_off + idj0 + 1) - o0, pl, npl)) continue;
                }
                const uint64_t *cj = cc + j * cws;
                uint32_t dij = 0;
                for (uint32_t w = 0; w < cw; w++) dij += __popcll(ci[w] ^ cj[w]);
                const uint32_t dpj = (uint32_t)(ck[j] >> 32), idj = (uint32_t)ck[j];
                float factor; /* DistanceWithTieBreak::get_factor, neighbor_with_distance.rs:55-65 */
                if (dij == 0) {
                    if (dpj == 0) {
                        float tp = (float)(idj > p ? idj - p : p - idj), te = (float)(idj > idi ? idj - idi : idi - idj);
                        factor = tp / te;
                    } else {
                        factor = 3.0e38f;
                    }
                } else {
                    factor = (float)dpj / (float)dij;
                }
                mf[j] = f > factor ? f : factor;
            }
            __syncwarp();
        }
        alpha *= 1.2f;
    }
    __syncwarp();
    return nres;
}

struct BuildArgs {
    const uint64_t *codes;
    uint32_t cw, cws, n;
    uint32_t *nbrs;       /* [n][SLACK] */
    uint16_t *nbr_dist;   /* [n][SLACK] */
    uint8_t *deg;         /* [n] */
    uint32_t R;           /* num_neighbors */
    uint32_t limit;       /* max_neighbors_during_build = ceil(1.3 R) (meta_page.rs:24,253-255), at most the 64 slots */
    float max_alpha;
    uint32_t per_warp_smem;
    const uint32_t *label_off; /* NULL: unlabeled index */
    const int16_t *labels;
};

__device__ __forceinline__ void build_smem(unsigned char *base, uint32_t cws, uint64_t *&ck, uint64_t *&cc, float *&mf,
                                           uint32_t *&oid, uint16_t *&od) {
    ck = reinterpret_cast<uint64_t *>(base);
    cc = ck + DANN_BUILD_CMAX;
    mf = reinterpret_cast<float *>(cc + (size_t)DANN_BUILD_CMAX * cws);
    oid = reinterpret_cast<uint32_t *>(mf + DANN_BUILD_CMAX);
    od = reinterpret_cast<uint16_t *>(oid + DANN_BUILD_SLACK);
}

__device__ __forceinline__ void build_write_list(const BuildArgs &a, uint32_t p, const uint32_t *oid, const uint16_t *od,
                                                 uint32_t cnt, int lane) {
    uint32_t *row = a.nbrs + (size_t)p * DANN_BUILD_SLACK;
    uint16_t *drow = a.nbr_dist + (size_t)p * DANN_BUILD_SLACK;
    for (uint32_t t = lane; t < DANN_BUILD_SLACK; t += 32) {
        row[t] = t < cnt ? oid[t] : DANN_INVALID_NODE;
        drow[t] = t < cnt ? od[t] : (uint16_t)0;
    }
    if (lane == 0) a.deg[p] = (uint8_t)cnt;
}

/* step 2: forward edges of the batch nodes [lo, lo+m) from their visited lists; also emits the
 * back-link triples key = (dst << 32) | (dist << 16), val = src into [m][SLACK] slots (~0 = unused) */
__global__ void __launch_bounds__(256) dann_build_prune_kernel(BuildArgs a, uint32_t lo, uint32_t m,
                                                               const uint64_t *vis, const uint32_t *vis_len,
                                                               uint32_t vis_cap, uint64_t *trip_key, uint32_t *trip_val) {
    DANN_DYN_SMEM(dann_smem);
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, W = blockDim.x >> 5;
    uint64_t *ck, *cc;
    float *mf;
    uint32_t *oid;
    uint16_t *od;
    build_smem(dann_smem + (size_t)warp * a.per_warp_smem, a.cws, ck, cc, mf, oid, od);
    for (uint32_t b = blockIdx.x * W + warp; b < m; b += gridDim.x * W) {
        const uint32_t p = lo + b;
        /* add_neighbors (graph/mod.rs:212-266): candidates = current neighbours of p (from the filtered pass of a
         * labeled insert) + the visited set, without duplicates and without p itself */
        const uint32_t deg = a.deg[p];
        uint32_t nv = vis_len[b];
        if (nv > DANN_BUILD_CMAX - deg) nv = DANN_BUILD_CMAX - deg; /* the visited list is sorted: keep the closest */
        const uint32_t *row = a.nbrs + (size_t)p * DANN_BUILD_SLACK;
        const uint16_t *drow = a.nbr_dist + (size_t)p * DANN_BUILD_SLACK;
        for (uint32_t c = lane; c < DANN_BUILD_CMAX; c += 32) {
            uint64_t k = ~0ull;
            if (c < deg) k = ((uint64_t)drow[c] << 32) | row[c];
            else if (c < deg + nv) k = vis[(size_t)b * vis_cap + (c - deg)];
            if ((uint32_t)k == p) k = ~0ull; /* prevent self-loops */
            ck[c] = k;
        }
        __syncwarp();
        build_bitonic_sort128(ck, lane);
        /* equal keys are adjacent after the sort: drop repeats, compact */
        uint32_t C = 0;
        for (uint32_t c0 = 0; c0 < DANN_BUILD_CMAX; c0 += 32) {
            const uint32_t c = c0 + lane;
            const uint64_t k = ck[c];
            const bool keep = k != ~0ull && (c == 0 || ck[c - 1] != k);
            const unsigned mk = __ballot_sync(DANN_FULL, keep);
            __syncwarp();
            if (keep) ck[C + __popc(mk & ((1u << lane) - 1u))] = k;
            C += __popc(mk);
            __syncwarp();
        }
        uint32_t cnt;
        /* a forward list keeps every candidate the 64 slots hold until a back-link or finalize prunes it - NOT the
         * reference's max_neighbors_during_build = ceil(1.3 R) that back-links overflow at (a.limit): a new node keeps
         * more out-edges while its batch mates cannot see it yet.  Equal at R >= 50 (min(64, 65)); DESIGN.md 6b */
        if (C <= DANN_BUILD_SLACK) {
            for (uint32_t t = lane; t < C; t += 32) {
                oid[t] = (uint32_t)ck[t];
                od[t] = (uint16_t)(ck[t] >> 32);
            }
            cnt = C;
            __syncwarp();
        } else {
            cnt = build_prune_warp(a.codes, a.cw, a.cws, p, ck, mf, cc, C, a.R, a.max_alpha, oid, od, lane, a.label_off, a.labels);
        }
        build_write_list(a, p, oid, od, cnt, lane);
        for (uint32_t t = lane; t < DANN_BUILD_SLACK; t += 32) {
            size_t o = (size_t)b * DANN_BUILD_SLACK + t;
            trip_key[o] = t < cnt ? (((uint64_t)oid[t] << 32) | ((uint64_t)od[t] << 16)) : ~0ull;
            trip_val[o] = p;
        }
        __syncwarp();
    }
}

/* segment heads of the sorted triples: first entry of every destination */
__global__ void dann_build_heads_kernel(const uint64_t *key, size_t total, uint32_t *heads, uint32_t *nheads) {
    for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (size_t)gridDim.x * blockDim.x) {
        uint64_t k = key[i];
        if (k == ~0ull) continue;
        if (i == 0 || (uint32_t)(key[i - 1] >> 32) != (uint32_t)(k >> 32)) heads[atomicAdd(nheads, 1u)] = (uint32_t)i;
    }
}

/* step 3: back-pointers.  One warp per destination node: append the (closest 64) new sources; a list
 * that would outgrow max_neighbors_during_build is pruned back to R (graph/mod.rs:212-266 add_neighbors) */
__global__ void __launch_bounds__(256) dann_build_backlink_kernel(BuildArgs a, const uint64_t *key, const uint32_t *val,
                                                                  size_t total, const uint32_t *heads, uint32_t nheads) {
    DANN_DYN_SMEM(dann_smem);
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, W = blockDim.x >> 5;
    uint64_t *ck, *cc;
    float *mf;
    uint32_t *oid;
    uint16_t *od;
    build_smem(dann_smem + (size_t)warp * a.per_warp_smem, a.cws, ck, cc, mf, oid, od);
    for (uint32_t h = blockIdx.x * W + warp; h < nheads; h += gridDim.x * W) {
        const size_t s = heads[h];
        const uint32_t q = (uint32_t)(key[s] >> 32);
        const uint32_t deg = a.deg[q];
        /* additions: up to 64 entries of this destination, already sorted by distance */
        uint32_t nadd = 0;
        for (uint32_t t0 = 0; t0 < DANN_BUILD_SLACK; t0 += 32) {
            size_t i = s + t0 + lane;
            bool ok = i < total && key[i] != ~0ull && (uint32_t)(key[i] >> 32) == q;
            unsigned mk = __ballot_sync(DANN_FULL, ok);
            if (ok) ck[deg + t0 + lane] = (((key[i] >> 16) & 0xFFFFull) << 32) | val[i];
            nadd += __popc(mk);
            if (mk != DANN_FULL) break;
        }
        const uint32_t *row = a.nbrs + (size_t)q * DANN_BUILD_SLACK;
        const uint16_t *drow = a.nbr_dist + (size_t)q * DANN_BUILD_SLACK;
        for (uint32_t t = lane; t < deg; t += 32) ck[t] = ((uint64_t)drow[t] << 32) | row[t];
        __syncwarp();
        const uint32_t tot = deg + nadd;
        if (tot <= a.limit && !a.label_off) { /* room left and no repeats possible: plain append */
            uint32_t *wrow = a.nbrs + (size_t)q * DANN_BUILD_SLACK;
            uint16_t *wdrow = a.nbr_dist + (size_t)q * DANN_BUILD_SLACK;
            for (uint32_t t = deg + lane; t < tot; t += 32) {
                wrow[t] = (uint32_t)ck[t];
                wdrow[t] = (uint16_t)(ck[t] >> 32);
            }
            if (lane == 0) a.deg[q] = (uint8_t)tot;
        } else {
            for (uint32_t t = tot + lane; t < DANN_BUILD_CMAX; t += 32) ck[t] = ~0ull;
            __syncwarp();
            build_bitonic_sort128(ck, lane);
            /* a source may already be a neighbour (second pass of a labeled insert): equal keys are adjacent */
            uint32_t C = 0;
            for (uint32_t c0 = 0; c0 < DANN_BUILD_CMAX; c0 += 32) {
                const uint32_t c = c0 + lane;
                const uint64_t k = ck[c];
                const bool keep = k != ~0ull && (c == 0 || ck[c - 1] != k);
                const unsigned mk = __ballot_sync(DANN_FULL, keep);
                __syncwarp();
                if (keep) ck[C + __popc(mk & ((1u << lane) - 1u))] = k;
                C += __popc(mk);
                __syncwarp();
            }
            uint32_t cnt;
            if (C <= a.limit) {
                for (uint32_t t = lane; t < C; t += 32) {
                    oid[t] = (uint32_t)ck[t];
                    od[t] = (uint16_t)(ck[t] >> 32);
                }
                cnt = C;
                __syncwarp();
            } else {
                cnt = build_prune_warp(a.codes, a.cw, a.cws, q, ck, mf, cc, C, a.R, a.max_alpha, oid, od, lane, a.label_off, a.labels);
            }
            build_write_list(a, q, oid, od, cnt, lane);
        }
        __syncwarp();
    }
}

/* finalize_index_build (build.rs:905-960): lists longer than R are pruned to R */
__global__ void __launch_bounds__(256) dann_build_finalize_kernel(BuildArgs a) {
    DANN_DYN_SMEM(dann_smem);
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, W = blockDim.x >> 5;
    uint64_t *ck, *cc;
    float *mf;
    uint32_t *oid;
    uint16_t *od;
    build_smem(dann_smem + (size_t)warp * a.per_warp_smem, a.cws, ck, cc, mf, oid, od);
    for (uint32_t p = blockIdx.x * W + warp; p < a.n; p += gridDim.x * W) {
        const uint32_t deg = a.deg[p];
        if (deg <= a.R) continue;
        const uint32_t *row = a.nbrs + (size_t)p * DANN_BUILD_SLACK;
        const uint16_t *drow = a.nbr_dist + (size_t)p * DANN_BUILD_SLACK;
        for (uint32_t t = lane; t < DANN_BUILD_CMAX; t += 32) ck[t] = t < deg ? (((uint64_t)drow[t] << 32) | row[t]) : ~0ull;
        __syncwarp();
        build_bitonic_sort128(ck, lane);
        const uint32_t cnt = build_prune_warp(a.codes, a.cw, a.cws, p, ck, mf, cc, deg, a.R, a.max_alpha, oid, od, lane, a.label_off, a.labels);
        build_write_list(a, p, oid, od, cnt, lane);
        __syncwarp();
    }
}

/* ---- in-edge rescue (DANN_BUILD_RESCUE=1, not part of the reference's algorithm) --------------------------------
 * Batched insertion can leave a node without any in-edge (every list that pointed at it was pruned while the node's
 * batch mates - which it never saw - crowded the same destinations; tie-heavy data makes this common).  Such a node is
 * invisible to every scan.  After finalize, a few rounds of: mark nodes that have an in-edge; every other node asks its
 * nearest out-neighbour for a slot - a free one if the list is shorter than R, else one of the farthest (at most R/2
 * per list and round).  A displaced neighbour that loses its last in-edge is picked up by the next round. */
__global__ void dann_build_mark_indegree_kernel(const uint32_t *nbrs, const uint8_t *deg, uint32_t n, uint32_t *indeg) {
    for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < (size_t)n * DANN_BUILD_SLACK;
         i += (size_t)gridDim.x * blockDim.x) {
        const uint32_t p = (uint32_t)(i / DANN_BUILD_SLACK), t = (uint32_t)(i % DANN_BUILD_SLACK);
        if (t < deg[p]) {
            const uint32_t x = nbrs[i];
            if (x < n && x != p) atomicAdd(indeg + x, 1u);
        }
    }
}

__global__ void dann_build_rescue_kernel(uint32_t *nbrs, const uint8_t *deg, uint32_t n, uint32_t R, uint32_t *indeg,
                                         uint32_t *claim, uint32_t *rescued) {
    for (uint32_t p = blockIdx.x * blockDim.x + threadIdx.x; p < n; p += gridDim.x * blockDim.x) {
        if (p == 0 || indeg[p]) continue; /* node 0 is the entry point */
        const uint32_t *row = nbrs + (size_t)p * DANN_BUILD_SLACK;
        const uint32_t dp = deg[p];
        bool done = false;
        /* pass A: a FREE slot in the list of any out-neighbour (nearest first), the entry point as a last resort */
        for (uint32_t t = 0; t <= dp && !done; t++) {
            const uint32_t q = t < dp ? row[t] : 0u;
            if (q >= n || q == p) continue;
            const uint32_t dq = deg[q];
            if (dq >= R) continue;
            const uint32_t c = atomicAdd(claim + q, 1u);
            if (dq + c >= R) continue; /* lost the race for the last free slot */
            nbrs[(size_t)q * DANN_BUILD_SLACK + dq + c] = p;
            done = true;
        }
        /* pass B: take the place of an entry of a full list that has another in-edge to spare (farthest first): the
         * swap is a compare-and-swap on the slot, the victim's spare in-edge is reserved with an atomic decrement */
        for (uint32_t t = 0; t < dp && !done; t++) {
            const uint32_t q = row[t];
            if (q >= n || q == p || deg[q] < R) continue;
            uint32_t *qrow = nbrs + (size_t)q * DANN_BUILD_SLACK;
            for (uint32_t sl = R; sl-- > R / 2 && !done;) {
                const uint32_t x = qrow[sl];
                if (x >= n || x == p) continue;
                const uint32_t had = atomicSub(indeg + x, 1u);
                if (had >= 2 && atomicCAS(qrow + sl, x, p) == x) done = true;
                else atomicAdd(indeg + x, 1u); /* not spare after all (or the slot changed): give it back */
            }
        }
        if (done) atomicAdd(rescued, 1u);
    }
}

__global__ void dann_build_rescue_degrees_kernel(uint8_t *deg, const uint32_t *claim, uint32_t n, uint32_t R) {
    for (uint32_t q = blockIdx.x * blockDim.x + threadIdx.x; q < n; q += gridDim.x * blockDim.x) {
        const uint32_t c = claim[q];
        if (!c) continue;
        const uint32_t d = deg[q] + c;
        deg[q] = (uint8_t)(d < R ? d : R);
    }
}

