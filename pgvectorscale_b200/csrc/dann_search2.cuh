// dann_search2.cuh — two-warp StreamingDiskANN beam search (sm_90a): one MEMORY/CONTROL warp and one
// HEAP warp per query, so that the HBM/L2 round trips of visit i+1 run under the heap pushes of
// visit i.  The memory warp drives the scan (visit_closest's stop test, the visited list, consume, the
// deleted-tuple skip, the stream output, neighbour fetch, dedupe, label filter, SBQ distances); the heap
// warp is a pure BinaryHeap engine (pop, ordered pushes) that reports the root the next pop will leave.  Same algorithm, same results and counters as dann_search.cuh (the single-warp
// kernel, kept for R > 64 and as the cross-check in tests); see that file for the reference map.
//
// Why the split is exact.  The reference's loop is pop -> expand -> push* -> pop ... .  The
// node popped next is the heap root after the pushes.  A pushed element reaches the root iff
// its key is STRICTLY below the root's at that moment (sift_up moves only while
// `elem < parent`, dann_heap.cuh), so after a batch of pushes the root is
//     the FIRST element of the batch that attains the batch minimum, if that minimum is
//     strictly below the root the heap had before the batch;  otherwise that old root.
// "The root the heap has before the batch" is the root after the pop, which is
//     c = (key(heap[2]) <= key(heap[1])) ? heap[2] : heap[1]   (right child on ties), or the
//     displaced last element if its key is strictly below key(c)
// — three loads, available BEFORE the pop's sift-down runs.  So the memory warp can start
// fetching the neighbour list, the inserted-set bits and the SBQ codes of visit i+1 while the
// heap warp is still pushing the batch of visit i.  The prediction is certain, not speculative;
// the memory warp therefore also evaluates the stop test itself and only expands nodes the reference
// would visit.  The heap warp still checks every prediction against the node it actually pops and
// reports DANN_ST_INTERNAL on a mismatch.
//
// Hand-off: double-buffered (list, dist) pages and control words in shared memory, one named
// barrier (bar.sync id, 64) per visit.
#pragma once
#include "dann_search_common.cuh"
#include "dann_heap.cuh"

struct PairCtl {
    uint32_t q;             /* query id for this round, 0xFFFFFFFF = no more work */
    uint32_t status_a;      /* overflow bits raised by the memory warp */
    uint32_t tn[2];         /* entries in list page p */
    uint32_t seq0[2];       /* candidate sequence number of entry 0 of page p */
    uint32_t expect[2];     /* node whose expansion page p holds (INVALID for start pages) */
    uint32_t root_valid[2]; /* heap root as it will be just before page p's successor is pushed */
    uint32_t root_key[2];
    uint32_t root_seq[2];
    uint32_t cmd[2];        /* memory warp -> heap warp: 0 = scan over, 1 = pop then push page p, 2 = push page p (start nodes) */
    uint32_t status_b;      /* heap warp's cross-check failures */
    uint32_t pad_;          /* keeps sizeof a multiple of 8: the push queue behind it holds 8-byte entries */
};

static_assert(sizeof(PairCtl) % 8 == 0, "PairCtl must keep 8-byte alignment for what follows it");

__device__ __forceinline__ void pair_sync(uint32_t id) {
#ifdef DANN_SIMT_EMU
    simt::named_barrier(id, 64);
#else
    /* bar.sync is the ALIGNED barrier: every thread of a warp must arrive together.  Lanes that left a divergent
     * branch may not have reconverged yet (compute-sanitizer synccheck: "divergent thread(s) in block"), so converge
     * the warp first. */
    __syncwarp();
    asm volatile("bar.sync %0, 64;" ::"r"(id) : "memory");
#endif
}

template <typename T, int NCH>
struct PairSearch {
    using E = typename T::E;
    using H = RustHeap<E, T::KSHIFT>;
    /* rows gathered per lane group per round: 6 x 8 = 48 rows (G=4) covers a typical 50-id list at once */
    static constexpr int RPI = NCH <= 2 ? 8 : (NCH == 3 ? 6 : (NCH == 4 ? 4 : 2));

    const SearchArgs &a;
    const int lane;
    const uint32_t bar;
    uint64_t *vis;
    uint32_t *listp, *dlp; /* [2][64] */
    PairCtl *ctl;
    E *cqe;         /* [32] compacted active pushes: entry */
    uint32_t *cqp;  /* [32]                          : 1-based slot */
    uint32_t *hash, *bitmap, *ins, *cnode;
    SplitStore<E> heap;

    __device__ __forceinline__ PairSearch(const SearchArgs &a_, int lane_, uint32_t bar_)
        : a(a_), lane(lane_), bar(bar_) {}

    /* ================================ memory warp ====================================== */
    ulonglong2 qc[NCH];
    const int16_t *ql;
    uint32_t nql, ncand, nins, listn, status;
    uint32_t vis_head, vis_len; /* the visited list belongs to the controller (memory) warp */
    bool filter;

    __device__ __forceinline__ bool node_passes_filter(uint32_t n) {
        if (!a.ix.has_labels) return false;
        uint32_t o0 = __ldg(a.ix.label_off + n), o1 = __ldg(a.ix.label_off + n + 1);
        return labels_overlap(ql, nql, a.ix.labels + o0, o1 - o0);
    }

    /* dedupe + label filter of up to 64 ids, appended to page `list` (see SearchWarp::stage) */
    __device__ __forceinline__ void stage(uint32_t *list, uint32_t n0, bool v0, uint32_t n1, bool v1,
                                          bool apply_filter, bool known_unique = false) {
        if (__ballot_sync(DANN_FULL, v0 || v1) == 0) return;
        bool f0, f1;
        if (known_unique) {
            /* the index was checked at load to have no repeated id within a neighbour list (lists_unique): the
             * intra-list dedupe - two MATCH.ANY on the path between the list's arrival and the inserted-set
             * atomics - has nothing to find */
            f0 = v0;
            f1 = v1;
        } else {
            unsigned m0 = __match_any_sync(DANN_FULL, n0);
            unsigned m1 = __match_any_sync(DANN_FULL, n1);
            f0 = v0 && ((__ffs(m0) - 1) == lane);
            f1 = v1 && ((__ffs(m1) - 1) == lane);
        }
        if (known_unique) {
            /* the SBQ code rows are needed one L2 round trip from now (after the inserted-set answers): start pulling
             * them into L2 already; rows of ids that turn out to be known are the only wasted traffic */
            const size_t rowbytes = (size_t)a.ix.cw * 8;
            const unsigned char *cb = reinterpret_cast<const unsigned char *>(a.ix.codes);
            if (f0) {
                prefetch_l2(cb + (size_t)n0 * rowbytes);
                if (rowbytes > 128) prefetch_l2(cb + (size_t)n0 * rowbytes + 128);
            }
            if (f1) {
                prefetch_l2(cb + (size_t)n1 * rowbytes);
                if (rowbytes > 128) prefetch_l2(cb + (size_t)n1 * rowbytes + 128);
            }
        }
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
            if (new0) p0 = node_passes_filter(n0);
            if (new1) p1 = node_passes_filter(n1);
        }
        const unsigned pm0 = __ballot_sync(DANN_FULL, p0), pm1 = __ballot_sync(DANN_FULL, p1);
        const uint32_t t0 = __popc(pm0), t1 = __popc(pm1);
        if (t0 + t1 == 0) return;
        if (ncand + listn + t0 + t1 + 1 > a.cand_cap) { /* 1-based heap slots: the last one is cand_cap-1 */
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

    /* SBQ distances of page `list` -> `dl` (distance/mod.rs:265-323).  EXACT: every lane's NCH
     * chunk slots exist (cw/2 == NCH*G), so the per-chunk bounds test disappears.
     * One round = RPI row slots per lane group: all 16-byte loads first, then XOR + popcount + group reduction. */
    template <bool EXACT>
    __device__ __forceinline__ void distances_impl(const uint32_t *list, uint32_t *dl, uint32_t tn) {
        const uint32_t G = a.G, gl = lane & (G - 1), grp = lane >> a.Gshift, RP = 32u >> a.Gshift;
        const uint32_t nchunks = a.ix.cw >> 1;
        const size_t rowbytes = (size_t)a.ix.cw * 8;
        const unsigned char *cbase = reinterpret_cast<const unsigned char *>(a.ix.codes) + (size_t)gl * 16;
        const uint32_t cstep = G * 16;
        for (uint32_t b = 0; b < tn; b += RP * RPI) {
            ulonglong2 v[RPI][NCH];
#pragma unroll
            for (int u = 0; u < RPI; u++) {
                const uint32_t r = b + u * RP + grp;
                const bool live = r < tn;
                const unsigned char *row = cbase + (size_t)(live ? list[r] : 0u) * rowbytes;
#pragma unroll
                for (int i = 0; i < NCH; i++) {
                    const bool ok = live && (EXACT || gl + i * G < nchunks);
                    v[u][i] = ok ? ldg_stream_u128(row + i * cstep) : qc[i];
                }
            }
#pragma unroll
            for (int u = 0; u < RPI; u++) {
                uint32_t s = 0;
#pragma unroll
                for (int i = 0; i < NCH; i++)
                    s += __popcll(v[u][i].x ^ qc[i].x) + __popcll(v[u][i].y ^ qc[i].y);
                for (uint32_t o = G >> 1; o > 0; o >>= 1) s += __shfl_xor_sync(DANN_FULL, s, o);
                const uint32_t r = b + u * RP + grp;
                if (gl == 0 && r < tn) dl[r] = s;
            }
        }
        __syncwarp();
    }
    __device__ __forceinline__ void distances(const uint32_t *list, uint32_t *dl, uint32_t tn) {
        if ((a.ix.cw >> 1) == (uint32_t)NCH * a.G) distances_impl<true>(list, dl, tn);
        else distances_impl<false>(list, dl, tn);
    }

    __device__ __forceinline__ void run_memory(uint32_t q) {
        const IndexView &ix = a.ix;
        ncand = nins = status = 0;
        {
            const uint32_t gl = lane & (a.G - 1), nchunks = ix.cw >> 1;
            const ulonglong2 *qrow = reinterpret_cast<const ulonglong2 *>(a.q_codes + (size_t)q * ix.cw);
#pragma unroll
            for (int i = 0; i < NCH; i++) {
                uint32_t c = gl + i * a.G;
                qc[i] = c < nchunks ? qrow[c] : make_ulonglong2(0, 0);
            }
        }
        if (!a.bitmap_words) {
            uint4 ff = make_uint4(DANN_INVALID_NODE, DANN_INVALID_NODE, DANN_INVALID_NODE, DANN_INVALID_NODE);
            uint4 *h4 = reinterpret_cast<uint4 *>(hash);
            for (uint32_t i = lane; i < a.hash_cap / 4; i += 32) h4[i] = ff;
            __threadfence_block();
            __syncwarp();
        }
        ql = nullptr;
        nql = 0;
        filter = false;
        uint32_t nstart_pages = 1;
        const bool have_graph = ix.start_default != DANN_INVALID_NODE;
        if (a.q_label_off) {
            int32_t o0 = a.q_label_off[q], o1 = a.q_label_off[q + 1];
            ql = a.q_labels + o0;
            nql = (uint32_t)(o1 - o0);
            filter = nql > 0;
            nstart_pages = nql ? (nql + 63) / 64 : 1;
        }
        vis_head = vis_len = 0;
        uint32_t visits = 0, scount = 0, k = 0;
        /* ---- start nodes (graph/mod.rs:97-124, start_nodes.rs:39-48): 64 per page, never label-checked */
        for (; k < nstart_pages; k++) {
            const uint32_t p = k & 1;
            uint32_t *list = listp + p * DANN_LIST_CAP, *dl = dlp + p * DANN_LIST_CAP;
            listn = 0;
            if (have_graph && !status) {
                if (a.q_label_off) {
                    uint32_t n[2];
                    bool v[2];
#pragma unroll
                    for (int h = 0; h < 2; h++) {
                        uint32_t i = k * 64 + h * 32 + lane;
                        n[h] = DANN_INVALID_NODE;
                        v[h] = false;
                        if (i < nql) {
                            int16_t lab = __ldg(ql + i);
                            uint32_t lo = 0, hi = ix.n_start_labels;
                            while (lo < hi) {
                                uint32_t mid = (lo + hi) >> 1;
                                if (__ldg(ix.start_labels + mid) < lab) lo = mid + 1;
                                else hi = mid;
                            }
                            if (lo < ix.n_start_labels && __ldg(ix.start_labels + lo) == lab) {
                                n[h] = __ldg(ix.start_label_nodes + lo);
                                v[h] = true;
                            }
                        }
                    }
                    /* two start nodes may coincide across the halves: keep list order */
                    stage(list, n[0], v[0], DANN_INVALID_NODE, false, false);
                    if (!status) stage(list, n[1], v[1], DANN_INVALID_NODE, false, false);
                } else {
                    stage(list, lane == 0 ? ix.start_default : DANN_INVALID_NODE, lane == 0, DANN_INVALID_NODE, false,
                          false);
                }
            }
            if (status) listn = 0;
            distances(list, dl, listn);
            if (lane == 0) {
                ctl->tn[p] = listn;
                ctl->seq0[p] = ncand;
                ctl->expect[p] = DANN_INVALID_NODE;
                ctl->cmd[p] = 2u;
            }
            ncand += listn;
            pair_sync(bar); /* page p handed over; the heap warp has published root[p] */
        }
        /* ---- TSVResponseIterator::next (scan.rs:210-242) driven from here: this warp knows the next
         * root of the heap (node and key) as soon as the previous page's distances exist */
        for (;; k++) {
            const uint32_t p = k & 1, pp = (k - 1) & 1;
            const uint32_t *pl = listp + pp * DANN_LIST_CAP, *pd = dlp + pp * DANN_LIST_CAP;
            const uint32_t ptn = ctl->tn[pp];
            uint32_t d0 = lane < ptn ? pd[lane] : 0xFFFFFFFFu;
            uint32_t d1 = lane + 32 < ptn ? pd[lane + 32] : 0xFFFFFFFFu;
            uint32_t m = min(d0, d1);
            for (int o = 16; o > 0; o >>= 1) m = min(m, __shfl_xor_sync(DANN_FULL, m, o));
            uint32_t node = DANN_INVALID_NODE, key = 0;
            const bool rv = ctl->root_valid[pp] != 0;
            if (ptn && (!rv || m < ctl->root_key[pp])) { /* first element of the batch attaining a strictly smaller minimum */
                unsigned e0 = __ballot_sync(DANN_FULL, d0 == m), e1 = __ballot_sync(DANN_FULL, d1 == m);
                uint32_t idx = e0 ? (uint32_t)(__ffs(e0) - 1) : 32u + (uint32_t)(__ffs(e1) - 1);
                node = pl[idx];
                key = m;
            } else if (rv) { /* the root the pop left behind stays on top */
                node = cnode[ctl->root_seq[pp]];
                key = ctl->root_key[pp];
            }
            const bool have = node != DANN_INVALID_NODE;
            bool visit = false;
            while (!status) {
                /* visit_closest (graph/mod.rs:153-170): candidates empty -> None; strictly more than L
                 * visited and head >= visited[L-1] -> None; else pop */
                if (have && !(vis_len > a.L && key >= (uint32_t)(vis[vis_head + a.L - 1] >> 32))) {
                    visit = true;
                    break;
                }
                if (a.build_mode) { /* greedy_search_for_build: one-shot search, the visited set is the result */
                    const uint32_t nv = vis_len < a.vis_out_cap ? vis_len : a.vis_out_cap;
                    for (uint32_t i = lane; i < nv; i += 32) a.vis_out[(size_t)q * a.vis_out_cap + i] = vis[vis_head + i];
                    if (lane == 0) a.vis_out_len[q] = nv;
                    break;
                }
                if (vis_len == 0) break;        /* consume() -> None */
                const uint64_t e = vis[vis_head]; /* visited.remove(0), graph/mod.rs:174-184 */
                __syncwarp();
                vis_head++;
                vis_len--;
                const uint32_t cn = (uint32_t)e;
                const uint64_t tid = __ldg(ix.tids + cn); /* return_lsn, sbq/storage.rs:404-414 */
                if ((tid & 0xFFFFull) == 0) continue;     /* InvalidOffsetNumber: deleted tuple, scan.rs:231-234 */
                if (lane == 0) a.stream[(size_t)q * a.c_target + scount] = cn;
                scount++;
                if (scount == a.c_target) break;
            }
            if (!visit) { /* the scan is over (enough rows, stream exhausted, or a workspace overflow) */
                if (lane == 0) ctl->cmd[p] = 0u;
                pair_sync(bar);
                break;
            }
            /* sbq/storage.rs:135-190: expand `node`; its neighbour list is fetched first so that the
             * visited-list insert runs under that latency */
            const uint32_t *row = ix.nbrs + (size_t)node * ix.Rp;
            uint32_t n0 = (uint32_t)lane < ix.R ? ldg_stream_u32(row + lane) : DANN_INVALID_NODE;
            uint32_t n1 = (uint32_t)lane + 32 < ix.R ? ldg_stream_u32(row + 32 + lane) : DANN_INVALID_NODE;
            visited_insert(key, node);
            visits++;
            uint32_t *list = listp + p * DANN_LIST_CAP, *dl = dlp + p * DANN_LIST_CAP;
            listn = 0;
            if (!status) {
                const unsigned i0 = __ballot_sync(DANN_FULL, n0 == DANN_INVALID_NODE);
                const unsigned i1 = __ballot_sync(DANN_FULL, n1 == DANN_INVALID_NODE);
                const uint32_t cut0 = i0 ? (uint32_t)(__ffs(i0) - 1) : 32u;
                const uint32_t cut1 = i0 ? 0u : (i1 ? (uint32_t)(__ffs(i1) - 1) : 32u);
                const bool v0 = (uint32_t)lane < cut0, v1 = (uint32_t)lane < cut1;
                if (a.lists_unique) {
                    stage(list, n0, v0, n1, v1, filter, true);
                } else {
                    stage(list, n0, v0, DANN_INVALID_NODE, false, filter);
                    if (!status) stage(list, n1, v1, DANN_INVALID_NODE, false, filter);
                }
            }
            if (status) listn = 0;
            distances(list, dl, listn);
            if (lane == 0) {
                ctl->tn[p] = listn;
                ctl->seq0[p] = ncand;
                ctl->expect[p] = node;
                ctl->cmd[p] = 1u; /* pop (it will be `node`) and push this page */
            }
            ncand += listn;
            pair_sync(bar);
        }
        status |= ctl->status_b;
        /* bitmap flavour: clear exactly the bits this query set */
        if (a.bitmap_words) {
            __syncwarp();
            uint32_t i = lane;
            for (; i + 7 * 32 < nins; i += 8 * 32) { /* 8 independent loads in flight per lane */
                uint32_t w[8];
#pragma unroll
                for (int u = 0; u < 8; u++) w[u] = ins[i + u * 32];
#pragma unroll
                for (int u = 0; u < 8; u++) bitmap[w[u] >> 5] = 0u;
            }
            for (; i < nins; i += 32) bitmap[ins[i] >> 5] = 0u;
            __threadfence_block();
        }
        write_query_stats(a, q, lane, scount, visits, ncand, false, status); /* every staged candidate was pushed */
    }

    /* ================================= heap warp ======================================= */
    uint32_t heap_len, hk;

    /* BinaryHeap::push x tn in list order (insert_neighbor, graph/mod.rs:144-147); 1-based slots.
     * Inert elements (parent key <= own key: they stay at their leaf whatever earlier pushes of
     * the batch do) are written in parallel; the others are compacted into a small queue and
     * replayed in order through the cooperative sift-up, the next one prefetched meanwhile. */
    template <bool PSM, typename Store>
    __device__ __forceinline__ void push_batch(Store &st, const uint32_t *dl, uint32_t tn, uint32_t seq0) {
        const unsigned lt = (1u << lane) - 1u;
        for (uint32_t base = 0; base < tn; base += 32) {
            const uint32_t r = base + lane;
            const bool have = r < tn;
            const uint32_t dmine = have ? dl[r] : 0u;
            const uint32_t slot = heap_len + r + 1;
            const E mine = T::make(dmine, seq0 + r);
            bool inert = false;
            if (have && slot > 1) {
                const uint32_t parent = slot >> 1;
                if (parent <= heap_len + base) { /* parent is settled (old, or from an earlier round) */
                    inert = H::key(PSM ? st.get_sm(parent) : st.get(parent)) <= dmine;
                    if (inert) st.set(slot, mine);
                }
            }
            const unsigned act = __ballot_sync(DANN_FULL, have && !inert);
            const uint32_t nact = __popc(act);
            if (have && !inert) {
                const uint32_t k = __popc(act & lt);
                cqe[k] = mine;
                cqp[k] = slot;
            }
            __syncwarp();
            if (nact == 0) continue;
            E e = cqe[0];
            uint32_t sp = cqp[0];
            for (uint32_t i = 0; i < nact; i++) {
                const uint32_t nx = i + 1 < nact ? i + 1 : i;
                const E en = cqe[nx]; /* next element fetched before this one's dependent chain */
                const uint32_t sn = cqp[nx];
                H::template sift_up_warp1<PSM>(st, sp, e, lane);
                e = en;
                sp = sn;
            }
        }
    }

    __device__ __forceinline__ void push_page(uint32_t p) {
        const uint32_t tn = ctl->tn[p], seq0 = ctl->seq0[p];
        const uint32_t *dl = dlp + p * DANN_LIST_CAP;
        if (tn == 0) return;
        if (heap_len + tn < heap.hs) { /* everything in shared memory */
            ArrayStore<E> sm{heap.sm};
            push_batch<true>(sm, dl, tn, seq0);
        } else if (heap_len + tn < 2 * heap.hs) { /* leaves spill to HBM, every parent still in shared memory */
            push_batch<true>(heap, dl, tn, seq0);
        } else {
            push_batch<false>(heap, dl, tn, seq0);
        }
        heap_len += tn;
    }

    __device__ __forceinline__ void visited_insert(uint32_t d, uint32_t node) {
        if (vis_head + vis_len + 1 > a.vcap) {
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

    /* publish the heap root as it stands before page k is pushed, and meet the memory warp */
    __device__ __forceinline__ void handoff(bool rv, E root) {
        const uint32_t p = hk & 1;
        if (lane == 0) {
            ctl->root_valid[p] = rv ? 1u : 0u;
            ctl->root_key[p] = H::key(root);
            ctl->root_seq[p] = T::seq(root);
        }
        pair_sync(bar);
        hk++;
    }

    __device__ __forceinline__ void run_heap(uint32_t q) {
        heap_len = hk = 0;
        uint32_t nstart_pages = 1;
        if (a.q_label_off) {
            uint32_t nql_ = (uint32_t)(a.q_label_off[q + 1] - a.q_label_off[q]);
            nstart_pages = nql_ ? (nql_ + 63) / 64 : 1;
        }
        for (uint32_t k = 0;; k++) {
            const uint32_t p = k & 1;
            E head = 0, pub = 0;
            int pv = 0;
            if (lane == 0 && heap_len > 0) {
                head = heap.get(1);
                if (k < nstart_pages) { /* a start page is pushed without a pop: the root is the root */
                    pub = head;
                    pv = 1;
                } else if (heap_len > 1) { /* root of the heap once the coming pop is done (header comment) */
                    const uint32_t m = heap_len - 1;
                    const E last = heap.get(heap_len);
                    E c = last;
                    if (m >= 2) {
                        c = heap.get(2);
                        if (m >= 3) {
                            E cr = heap.get(3);
                            if (H::key(cr) <= H::key(c)) c = cr;
                        }
                    }
                    pub = (m >= 2 && H::key(last) < H::key(c)) ? last : c;
                    pv = 1;
                }
            }
            head = __shfl_sync(DANN_FULL, head, 0);
            pub = __shfl_sync(DANN_FULL, pub, 0);
            pv = __shfl_sync(DANN_FULL, pv, 0);
            handoff(pv != 0, pub);
            const uint32_t cmd = ctl->cmd[p];
            if (cmd == 0) break;
            uint32_t node_chk = DANN_INVALID_NODE;
            if (cmd == 1) { /* candidates.pop(): the memory warp already knows which node this is */
                if (heap_len == 0) {
                    if (lane == 0) ctl->status_b = DANN_ST_INTERNAL;
                    continue;
                }
                node_chk = __ldcg(cnode + T::seq(head)); /* cross-check, read under the pop */
                if (heap_len < heap.hs) {
                    ArrayStore<E> sm{heap.sm};
                    H::pop_warp1(sm, heap_len, lane);
                } else {
                    H::pop_warp1(heap, heap_len, lane);
                }
            }
            push_page(p);
            if (cmd == 1 && node_chk != ctl->expect[p] && lane == 0) ctl->status_b = DANN_ST_INTERNAL;
        }
    }
};

template <typename T, int NCH>
__global__ void __launch_bounds__(448, 1) dann_search2_kernel(const SearchArgs a) {
    using E = typename T::E;
    DANN_DYN_SMEM(dann_smem);
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, pair = warp >> 1, role = warp & 1;
    const int P = blockDim.x >> 6;
    const uint32_t slot = blockIdx.x * P + pair;
    unsigned char *base = dann_smem + (size_t)pair * a.per_warp_smem;
    PairSearch<T, NCH> w(a, lane, 1u + (uint32_t)pair);
    w.vis = reinterpret_cast<uint64_t *>(base);
    E *hsm = reinterpret_cast<E *>(base + (size_t)a.vcap * 8);
    w.listp = reinterpret_cast<uint32_t *>(base + (size_t)a.vcap * 8 + (size_t)a.hs * sizeof(E));
    w.dlp = w.listp + 2 * DANN_LIST_CAP;
    w.ctl = reinterpret_cast<PairCtl *>(w.dlp + 2 * DANN_LIST_CAP);
    w.cqp = reinterpret_cast<uint32_t *>(w.ctl + 1);
    w.cqe = reinterpret_cast<E *>(w.cqp + 32);
    w.hash = a.hash + (size_t)slot * a.hash_cap;
    w.bitmap = a.bitmap + (size_t)slot * a.bitmap_words;
    w.ins = a.ins_list + (size_t)slot * a.ins_cap;
    w.cnode = a.cand_node + (size_t)slot * a.cand_cap;
    w.heap.sm = hsm;
    w.heap.gl = reinterpret_cast<E *>(a.heap_tail) + (size_t)slot * a.cand_cap;
    w.heap.hs = a.hs;
    for (;;) {
        if (role == 0 && lane == 0) {
            uint32_t qi = atomicAdd(a.counter, 1u);
            w.ctl->q = qi < a.nq ? (a.qlist ? a.qlist[qi] : qi) : 0xFFFFFFFFu;
            w.ctl->status_a = 0;
            w.ctl->status_b = 0;
        }
        pair_sync(w.bar);
        const uint32_t q = w.ctl->q;
        if (q == 0xFFFFFFFFu) break;
        if (role == 0) w.run_memory(q);
        else w.run_heap(q);
        pair_sync(w.bar); /* both warps are done with this query's shared state */
    }
}
