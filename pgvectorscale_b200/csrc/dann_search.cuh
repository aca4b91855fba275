// dann_search.cuh — persistent warp-per-query StreamingDiskANN beam search (sm_90a).
//
// Replaces, for one query per warp (reference paths relative to
// pgvectorscale/src/access_method/):
//   Graph::greedy_search_streaming_init      graph/mod.rs:331-354
//   ListSearchResult::{new,prepare_insert,insert_neighbor,visit_closest,consume}
//                                            graph/mod.rs:97-185
//   Graph::greedy_search_iterate             graph/mod.rs:357-385
//   SbqSpeedupStorage::visit_lsn_internal    sbq/storage.rs:125-190 (Disk arm)
//   create_lsn_for_start_node / return_lsn   sbq/storage.rs:365-414
//   distance_xor_optimized                   distance/mod.rs:265-323
//   TSVResponseIterator::next                scan.rs:210-242 (deleted-tuple skip)
//
// Work split inside a warp
//   * all lanes: neighbour-list fetch, dedupe (match_any + a CAS hash set in HBM),
//     label overlap, SBQ code gathers (G lanes per code row, 128-bit no-allocate loads),
//     XOR+popcount with shfl reduction, visited-list shifting.
//   * lane 0: the candidate heap — an exact clone of Rust's BinaryHeap (dann_heap.cuh),
//     because Hamming ties pop in heap order and that order decides returned row ids.
//
// State placement
//   shared : visited list (sorted, (dist<<32)|node), first `hs` heap entries, 64-entry
//            staging list for one neighbour list.
//   HBM    : per-warp workspace — inserted-set, seq->node table, heap tail beyond `hs`.
//            The inserted-set is a bitmap over node ids (one atomicOr per neighbour, cleared
//            by replaying the list of inserted ids) when the index is small enough for
//            one bitmap per resident warp, else an open-addressing CAS hash set.
//   The heap entry packs (dist, seq) in 4 bytes whenever it can (Ent32x21 / Ent32x16), else 8.
//
// Per visit the dependent memory round trips are: seq->node (L2) -> neighbour list (HBM,
// overlapped with the pop's sift-down and the visited-list insert) -> inserted-set atomics
// (L2, both 32-id chunks in flight together) -> SBQ code gather (HBM, every staged row in
// flight at once).  Heap pushes: lanes test in parallel which new elements stay at their
// leaf ("inert": parent <= elem, which later pushes cannot undo because a slot's value only
// decreases during pushes) and write those directly; the rest are sifted one at a time, in
// order, by the warp-cooperative sift-up of dann_heap.cuh (one lane per tree level).
#pragma once
#include "dann_search_common.cuh"
#include "dann_distance.cuh"
#include "dann_heap.cuh"

/* PLAIN = 1: the plain storage layout.  Keys are total_ukey(f32 distance) (Ent64 entries), every comparison is a
 * full-distance comparison (counted as d_full), there is no label filter (plain/storage.rs:260). */
template <typename T, int NCH, int PLAIN = 0>
struct SearchWarp {
    using E = typename T::E;
    using H = RustHeap<E, T::KSHIFT>;
    /* code rows gathered per lane group before reducing (16-B loads in flight = RPI*NCH):
     * with G=4 lanes per 192-B row, 8 x 8 rows = all 64 staged rows in one round */
    static constexpr int RPI = NCH <= 3 ? 8 : (NCH == 4 ? 4 : 2);

    const SearchArgs &a;
    const int lane;
    /* per-warp storage */
    uint64_t *vis;
    uint32_t *list, *dl;
    uint32_t *hash, *bitmap, *ins, *cnode;
    SplitStore<E> heap;
    float *qrow; /* PLAIN: this query's index slice in shared memory */
    /* query */
    ulonglong2 qc[NCH];
    QueryLabels key;
    /* warp-uniform state */
    uint32_t heap_len, vis_head, vis_len, ncand, nins, listn;
    uint32_t visits, dq, status;

    __device__ __forceinline__ SearchWarp(const SearchArgs &a_, int lane_) : a(a_), lane(lane_) {}

    /* ---- stage: dedupe + label filter of up to 64 neighbour ids (two per lane: list slots
     * `lane` and `lane+32`), appended to the staging list in list order.
     * sbq/storage.rs:149-172. */
    __device__ __forceinline__ void stage(uint32_t n0, bool v0, uint32_t n1, bool v1, bool apply_filter) {
        if (__ballot_sync(DANN_FULL, v0 || v1) == 0) return;
        /* a node listed twice within a chunk: only its first occurrence may insert.  (A node
         * repeated ACROSS the two chunks is handled by the caller: it stages the chunks one
         * at a time unless the index was checked to have duplicate-free lists.) */
        unsigned m0 = __match_any_sync(DANN_FULL, n0);
        unsigned m1 = __match_any_sync(DANN_FULL, n1);
        const bool f0 = v0 && ((__ffs(m0) - 1) == lane);
        const bool f1 = v1 && ((__ffs(m1) - 1) == lane);
        bool new0 = false, new1 = false;
        if (a.bitmap_words) {
            uint32_t o0 = 0xFFFFFFFFu, o1 = 0xFFFFFFFFu;
            const uint32_t b0 = 1u << (n0 & 31), b1 = 1u << (n1 & 31);
            if (f0) o0 = atomicOr(bitmap + (n0 >> 5), b0);
            if (f1) o1 = atomicOr(bitmap + (n1 >> 5), b1);
            new0 = f0 && !(o0 & b0);
            new1 = f1 && !(o1 & b1);
        } else {
            if (f0) new0 = hash_insert(hash, a.hash_cap, n0);
            __syncwarp();
            if (f1) new1 = hash_insert(hash, a.hash_cap, n1);
        }
        const unsigned lt = (1u << lane) - 1u;
        const unsigned nm0 = __ballot_sync(DANN_FULL, new0), nm1 = __ballot_sync(DANN_FULL, new1);
        const uint32_t c0 = __popc(nm0), c1 = __popc(nm1);
        if (a.bitmap_words) {
            if (nins + c0 + c1 > a.ins_cap) {
                /* undo this round's bits so that the replay below leaves the bitmap all zero */
                if (new0) atomicAnd(bitmap + (n0 >> 5), ~(1u << (n0 & 31)));
                if (new1) atomicAnd(bitmap + (n1 >> 5), ~(1u << (n1 & 31)));
                status |= DANN_ST_HASH;
                return;
            }
            if (new0) ins[nins + __popc(nm0 & lt)] = n0;
            if (new1) ins[nins + c0 + __popc(nm1 & lt)] = n1;
            nins += c0 + c1;
        } else {
            nins += c0 + c1;
            if (nins * 2 > a.hash_cap) {
                status |= DANN_ST_HASH;
                return;
            }
        }
        bool p0 = new0, p1 = new1;
        if (apply_filter) {
            if (new0) p0 = node_passes_filter(a.ix, key, n0);
            if (new1) p1 = node_passes_filter(a.ix, key, n1);
        }
        const unsigned pm0 = __ballot_sync(DANN_FULL, p0), pm1 = __ballot_sync(DANN_FULL, p1);
        const uint32_t t0 = __popc(pm0), t1 = __popc(pm1);
        if (t0 + t1 == 0) return;
        if (ncand + listn + t0 + t1 > a.cand_cap) {
            status |= DANN_ST_HEAP;
            return;
        }
        if (p0) {
            uint32_t pos = listn + __popc(pm0 & lt);
            list[pos] = n0;
            cnode[ncand + pos] = n0;
        }
        if (p1) {
            uint32_t pos = listn + t0 + __popc(pm1 & lt);
            list[pos] = n1;
            cnode[ncand + pos] = n1;
        }
        listn += t0 + t1;
        __syncwarp();
    }

    /* BinaryHeap::push x tn, in list order.  A new element whose parent already holds a key
     * <= its own stays at its leaf whatever the earlier pushes of this batch do (a slot's key
     * never increases during pushes, and sift_up only reads ancestors), so those "inert"
     * elements are written in parallel; the others go through the warp-cooperative sift-up one
     * at a time, in order. */
    template <typename Store>
    __device__ __forceinline__ void push_batch(Store &st, const uint32_t tn) {
        for (uint32_t base = 0; base < tn; base += 32) {
            const uint32_t r = base + lane;
            const bool have = r < tn;
            const uint32_t dmine = have ? dl[r] : 0u;
            bool inert = false;
            if (have) {
                const uint32_t pos = heap_len + r;
                if (pos > 0) {
                    const uint32_t parent = (pos - 1) >> 1;
                    if (parent < heap_len + base) { /* parent is settled (old, or from an earlier round) */
                        inert = H::key(st.get(parent)) <= dmine;
                        if (inert) st.set(pos, T::make(dmine, ncand + r));
                    }
                }
            }
            unsigned act = __ballot_sync(DANN_FULL, have && !inert);
            __syncwarp();
            const uint32_t pos0 = heap_len + base, seq0 = ncand + base;
            while (act) { /* warp-uniform loop: one cooperative sift-up per remaining element */
                const int b = __ffs(act) - 1;
                act &= act - 1;
                const uint32_t d = __shfl_sync(DANN_FULL, dmine, b);
                H::sift_up_warp(st, pos0 + (uint32_t)b, T::make(d, seq0 + (uint32_t)b), lane);
            }
        }
    }

    /* ---- flush: SBQ distance of every staged node (distance/mod.rs:265-323) and the
     * ordered heap pushes (insert_neighbor, graph/mod.rs:144-147) */
    __device__ __forceinline__ void flush() {
        const uint32_t tn = listn;
        if (tn == 0 || status) {
            listn = 0;
            return;
        }
        if constexpr (PLAIN == 1) {
            /* PlainDistanceMeasure::calculate_distance (plain/mod.rs:22-32): distance_fn(query.to_index_slice(),
             * node.vector), 8 lanes per row, the AVX2 summation order of dann_distance.cuh; the heap key is the
             * total order image of the f32 (-0.0 folded into +0.0: DistanceWithTieBreak treats them as equal,
             * graph/neighbor_with_distance.rs:31-43) */
            const uint32_t mm = lane & 7, gbase = lane & 24, grp8 = lane >> 3;
            const bool vec4 = (a.plain_dim & 3u) == 0;
            for (uint32_t b = 0; b < tn; b += 4) {
                const uint32_t r = b + grp8;
                const uint32_t node = r < tn ? list[r] : 0u;
                const float *x = a.plain_vectors + (size_t)node * a.plain_dim;
                const float d = vec4 ? full_distance_group8<true>(a.ix.distance_type, x, qrow, a.plain_dim, mm, gbase)
                                     : full_distance_group8<false>(a.ix.distance_type, x, qrow, a.plain_dim, mm, gbase);
                if (mm == 0 && r < tn) dl[r] = total_ukey(__fadd_rn(d, 0.0f));
            }
            __syncwarp();
            push_batch(heap, tn);
            heap_len += tn;
            ncand += tn;
            dq += tn;
            listn = 0;
            return;
        }
        const uint32_t G = a.G, gl = lane & (G - 1), grp = lane >> a.Gshift, RP = 32u >> a.Gshift;
        const uint32_t nchunks = a.ix.cw >> 1;
        for (uint32_t b = 0; b < tn; b += RP * RPI) {
            ulonglong2 v[RPI][NCH];
#pragma unroll
            for (int u = 0; u < RPI; u++) {
                uint32_t r = b + u * RP + grp;
                uint32_t node = r < tn ? list[r] : 0u;
                const ulonglong2 *row =
                    reinterpret_cast<const ulonglong2 *>(a.ix.codes + (size_t)node * a.ix.cw);
#pragma unroll
                for (int i = 0; i < NCH; i++) {
                    uint32_t c = gl + i * G;
                    v[u][i] = (r < tn && c < nchunks) ? ldg_stream_u128(row + c) : qc[i];
                }
            }
#pragma unroll
            for (int u = 0; u < RPI; u++) {
                uint32_t s = 0;
#pragma unroll
                for (int i = 0; i < NCH; i++)
                    s += __popcll(v[u][i].x ^ qc[i].x) + __popcll(v[u][i].y ^ qc[i].y);
                for (uint32_t o = G >> 1; o > 0; o >>= 1) s += __shfl_xor_sync(DANN_FULL, s, o);
                uint32_t r = b + u * RP + grp;
                if (gl == 0 && r < tn) dl[r] = s;
            }
        }
        __syncwarp();
        /* BinaryHeap::push x tn, in list order (fast path: everything in shared memory) */
        if (heap_len + tn <= heap.hs) {
            ArrayStore<E> sm{heap.sm};
            push_batch(sm, tn);
        } else {
            push_batch(heap, tn);
        }
        heap_len += tn;
        ncand += tn;
        dq += tn;
        listn = 0;
    }

    /* ---- expand one visited node: sbq/storage.rs:135-190.  n0/n1 = list slots lane, lane+32
     * (already loaded by the caller so that the HBM latency overlaps the heap pop). */
    __device__ __forceinline__ void expand(uint32_t v, uint32_t n0, uint32_t n1) {
        for (uint32_t base = 0; base < a.ix.R && !status; base += 64) {
            if (base) fetch_neighbours(a.ix, v, base, lane, n0, n1);
            bool v0, v1;
            const bool ends = neighbour_cut(n0, n1, lane, v0, v1);
            if (a.lists_unique) {
                stage(n0, v0, n1, v1, key.filter);
            } else { /* a list may repeat an id: keep strict list order across the two chunks */
                stage(n0, v0, DANN_INVALID_NODE, false, key.filter);
                if (!status) stage(n1, v1, DANN_INVALID_NODE, false, key.filter);
            }
            flush();
            if (ends) break;
        }
    }

    /* ---- visited.insert(partition_point(x < c), c) : graph/mod.rs:166-168 */
    __device__ __forceinline__ void visited_insert(uint32_t d, uint32_t node) {
        if (vis_head + vis_len + 1 > a.vcap) { /* slide the window back to offset 0 */
            if (vis_len + 1 > a.vcap) {
                status |= DANN_ST_VIS;
                return;
            }
            for (uint32_t i0 = 0; i0 < vis_len; i0 += 32) {
                uint32_t i = i0 + lane;
                uint64_t e = 0;
                if (i < vis_len) e = vis[vis_head + i];
                __syncwarp();
                if (i < vis_len) vis[i] = e;
                __syncwarp();
            }
            vis_head = 0;
        }
        uint64_t *w = vis + vis_head;
        uint32_t idx = 0;
        for (uint32_t i0 = 0; i0 < vis_len; i0 += 32) {
            uint32_t i = i0 + lane;
            bool lt = i < vis_len && (uint32_t)(w[i] >> 32) < d;
            idx += __popc(__ballot_sync(DANN_FULL, lt));
        }
        for (int hi = (int)vis_len; hi > (int)idx; hi -= 32) {
            int i = hi - 1 - lane;
            uint64_t e = 0;
            bool act = i >= (int)idx;
            if (act) e = w[i];
            __syncwarp();
            if (act) w[i + 1] = e;
            __syncwarp();
        }
        if (lane == 0) w[idx] = ((uint64_t)d << 32) | node;
        vis_len++;
        __syncwarp();
    }

    __device__ __forceinline__ void run(uint32_t q) {
        const IndexView &ix = a.ix;
        heap_len = vis_head = vis_len = ncand = nins = listn = 0;
        visits = dq = status = 0;
        uint32_t scount = 0;
        const bool resumed = a.saved && a.saved->valid;
        if (resumed) { /* pick the suspended ListSearchResult up where the last amgettuple left it */
            heap_len = a.saved->heap_len;
            vis_len = a.saved->vis_len;
            ncand = a.saved->ncand;
            nins = a.saved->nins;
            visits = a.saved->visits;
            dq = a.saved->dq;
            const E *hsrc = reinterpret_cast<const E *>(a.saved_heap_sm);
            const uint32_t hn = heap_len < heap.hs ? heap_len : heap.hs;
            for (uint32_t i = lane; i < hn; i += 32) heap.sm[i] = hsrc[i];
            for (uint32_t i = lane; i < vis_len; i += 32) vis[i] = a.saved_vis[i];
            __syncwarp();
        }
        if constexpr (PLAIN == 1) { /* the query's index slice, read by every distance of this scan */
            const float *src = a.q_index + (size_t)q * a.plain_dim;
            for (uint32_t i = lane; i < a.plain_dim; i += 32) qrow[i] = src[i];
            __syncwarp();
        }
        /* query code chunks this lane compares against (SbqSearchDistanceMeasure, sbq/mod.rs:139-159) */
        if constexpr (PLAIN == 0) {
            const uint32_t gl = lane & (a.G - 1), nchunks = ix.cw >> 1;
            const ulonglong2 *qrow = reinterpret_cast<const ulonglong2 *>(a.q_codes + (size_t)q * ix.cw);
#pragma unroll
            for (int i = 0; i < NCH; i++) {
                uint32_t c = gl + i * a.G;
                qc[i] = c < nchunks ? qrow[c] : make_ulonglong2(0, 0);
            }
        }
        if (!a.bitmap_words && !resumed) hash_set_clear(hash, a.hash_cap, lane);
        key = query_labels(a, q);
        /* greedy_search_streaming_init + ListSearchResult::new (graph/mod.rs:97-124,331-354) */
        if (ix.start_default != DANN_INVALID_NODE && !resumed) {
            if (a.q_label_off) {
                for (uint32_t b = 0; b < key.n && !status; b += 32) {
                    uint32_t n;
                    const bool valid = label_start_node(ix, key, b + lane, n);
                    /* start nodes are not label-checked (storage.rs:365-391) */
                    stage(n, valid, DANN_INVALID_NODE, false, false);
                    flush();
                }
            } else {
                stage(lane == 0 ? ix.start_default : DANN_INVALID_NODE, lane == 0, DANN_INVALID_NODE, false, false);
                flush();
            }
        }

        bool done = false;
        while (!done && !status) { /* TSVResponseIterator::next, scan.rs:210-242 */
            /* greedy_search_iterate: while let Some(idx) = visit_closest(L) */
            while (true) {
                E head = 0;
                int go = 0;
                if (lane == 0 && heap_len > 0) { /* visit_closest, graph/mod.rs:153-170 */
                    head = heap.get(0);
                    go = 1;
                    if (vis_len > a.L) {
                        uint64_t at = vis[vis_head + a.L - 1];
                        if (H::key(head) >= (uint32_t)(at >> 32)) go = 0;
                    }
                }
                go = __shfl_sync(DANN_FULL, go, 0);
                if (!go) break;
                head = __shfl_sync(DANN_FULL, head, 0);
                /* the popped element IS the current root: fetch its node id and neighbour list
                 * first, then let the sift-down and the visited insert run under that latency */
                const uint32_t d = H::key(head);
                const uint32_t node = __ldcg(cnode + T::seq(head));
                uint32_t n0, n1;
                fetch_neighbours(ix, node, 0, lane, n0, n1);
                if (heap_len <= heap.hs) {
                    ArrayStore<E> sm{heap.sm};
                    H::pop_warp(sm, heap_len, lane);
                } else {
                    H::pop_warp(heap, heap_len, lane);
                }
                visited_insert(d, node);
                if (status) break;
                visits++;
                expand(node, n0, n1);
                if (status) break;
            }
            if (status) break;
            if (vis_len == 0) break; /* consume() -> None */
            uint64_t e = vis[vis_head]; /* visited.remove(0), graph/mod.rs:174-184 */
            __syncwarp();
            vis_head++;
            vis_len--;
            const uint32_t node = (uint32_t)e;
            const uint64_t tid = __ldg(ix.tids + node); /* return_lsn, sbq/storage.rs:404-414 */
            if ((tid & 0xFFFFull) == 0) continue;       /* InvalidOffsetNumber: deleted tuple, scan.rs:231-234 */
            if (lane == 0) a.stream[(size_t)q * a.c_target + scount] = node;
            scount++;
            if (scount == a.c_target) done = true;
        }
        if (a.saved) { /* suspend: the inserted-set and the heap tail stay where they are */
            __syncwarp();
            E *hdst = reinterpret_cast<E *>(a.saved_heap_sm);
            const uint32_t hn = heap_len < heap.hs ? heap_len : heap.hs;
            for (uint32_t i = lane; i < hn; i += 32) hdst[i] = heap.sm[i];
            for (uint32_t i = lane; i < vis_len; i += 32) a.saved_vis[i] = vis[vis_head + i];
            if (lane == 0) {
                SavedScan sv;
                sv.valid = status ? 0u : 1u;
                sv.heap_len = heap_len;
                sv.vis_len = vis_len;
                sv.ncand = ncand;
                sv.nins = nins;
                sv.visits = visits;
                sv.dq = dq;
                sv.exhausted = (!done && !status) ? 1u : 0u; /* next() returned None */
                *a.saved = sv;
            }
        } else if (a.bitmap_words) { /* bitmap flavour: clear exactly the bits this query set */
            __syncwarp();
            for (uint32_t i = lane; i < nins; i += 32) bitmap[ins[i] >> 5] = 0u;
            __threadfence_block();
        }
        write_query_stats(a, q, lane, scount, visits, dq, PLAIN == 1, status);
    }
};

template <typename T, int NCH, int PLAIN = 0>
__global__ void __launch_bounds__(384, 1) dann_search_kernel(const SearchArgs a) {
    using E = typename T::E;
    DANN_DYN_SMEM(dann_smem);
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, W = blockDim.x >> 5;
    const uint32_t slot = blockIdx.x * W + warp;
    unsigned char *base = dann_smem + (size_t)warp * a.per_warp_smem;
    SearchWarp<T, NCH, PLAIN> w(a, lane);
    w.vis = reinterpret_cast<uint64_t *>(base);
    E *hsm = reinterpret_cast<E *>(base + (size_t)a.vcap * 8);
    w.list = reinterpret_cast<uint32_t *>(base + (size_t)a.vcap * 8 + (size_t)a.hs * sizeof(E));
    w.dl = w.list + DANN_LIST_CAP;
    w.qrow = reinterpret_cast<float *>(w.dl + DANN_LIST_CAP); /* PLAIN only: [plain_dim rounded up to 4] */
    w.hash = a.hash + (size_t)slot * a.hash_cap;
    w.bitmap = a.bitmap + (size_t)slot * a.bitmap_words;
    w.ins = a.ins_list + (size_t)slot * a.ins_cap;
    w.cnode = a.cand_node + (size_t)slot * a.cand_cap;
    w.heap.sm = hsm;
    w.heap.gl = reinterpret_cast<E *>(a.heap_tail) + (size_t)slot * a.cand_cap;
    w.heap.hs = a.hs;
    serve_queries(a, lane, w);
}
