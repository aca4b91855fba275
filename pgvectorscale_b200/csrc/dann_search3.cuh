// dann_search3.cuh — "lean" persistent warp-per-query StreamingDiskANN beam search (sm_90a), sized for FULL
// occupancy: up to 32 resident queries per SM (one warp each, <= 64 registers per thread, a few KB of shared
// memory per query) instead of the 7 two-warp slots of dann_search2.cuh.  Same algorithm, same results and
// counters as dann_search.cuh (see that file for the reference map; paths below are relative to
// pgvectorscale/src/access_method/):
//   ListSearchResult::{new,prepare_insert,insert_neighbor,visit_closest,consume}   graph/mod.rs:97-185
//   Graph::greedy_search_iterate                                                   graph/mod.rs:357-385
//   SbqSpeedupStorage::visit_lsn_internal (Disk arm)                               sbq/storage.rs:125-190
//   distance_xor_optimized                                                         distance/mod.rs:265-323
//   TSVResponseIterator::next (deleted-tuple skip)                                 scan.rs:210-242
//
// The search of one query is a dependent chain (pop -> neighbour row -> inserted-set -> code rows -> pushes -> pop);
// one warp cannot make it shorter than its memory round trips, so throughput = resident queries / chain latency.
// This kernel therefore minimises (a) the per-query footprint and (b) the instructions per visit:
//   * heap entries carry their own node reference (node id under the bitmap inserted-set, hash slot under the
//     hash inserted-set): no seq -> node table, no store per candidate, no inserted-id list;
//   * BinaryHeap::push x page: inert elements written by all lanes at once, the rest through a warp-cooperative
//     sift-up (one load, one ballot, one store whatever the rise height);
//   * BinaryHeap::pop's sift_down_to_bottom four levels per memory round trip: 30 lanes fetch the hole's
//     2+4+8+16 descendants at once, one ballot decides every sibling pair ("right child on ties"), the path is
//     walked on that mask in registers and the winners store themselves into their parents;
//   * visited list = ring buffer of heap entries (4 bytes each at 768-d), 32-ary partition_point, the shorter
//     side is shifted; consume() is a head increment;
//   * the bitmap inserted-set is cleared with one streaming memset per query (n/8 bytes) instead of replaying a list.
// Everything is an exact restatement of the sequential algorithm: Rust's BinaryHeap decides which of several equal
// Hamming distances pops first, and that decides returned row ids (dann_heap.cuh).
//
// Shared memory per query slot: visited ring [vcap] E, heap slots [hs] E (1-based, slot 0 unused), page of node ids
// [64] u32, page of entries [64] E, staging area of the pushes [160] E.  HBM per slot: heap tail [cand_cap] E, inserted-set (bitmap n/8 bytes, or
// hash_cap u32).
#pragma once
#include "dann_search_common.cuh"
#include "dann_heap.cuh"

/* staged slots of one page of pushes: tn leaves + (tn/2 + 1) + (tn/4 + 1) + ... <= 2 tn + 32 */
#define DANN_STG_CAP (2u * DANN_LIST_CAP + 32u)

template <typename T, int NCH>
struct LeanWarp {
    using E = typename T::E;
    using H = RustHeap<E, T::KSHIFT>;
    static constexpr E KM = (E(1) << T::KSHIFT) - E(1);
    /* a 4-byte entry under the hash inserted-set carries the node's hash slot (21 bits) */
    static constexpr bool SMALL = sizeof(E) == 4;

    const SearchArgs &a;
    const int lane;
    E *vis;         /* ring [a.vcap] */
    uint32_t *list; /* [64] node ids of the page being expanded */
    E *ent;         /* [64] payload, then (key | payload) of the page */
    E *stg;         /* [DANN_STG_CAP] heap slots staged for the pushes of one page */
    bool stg_async; /* the ancestors of the page about to be pushed are already on their way into stg (cp.async) */
    uint32_t *hash, *bitmap;
    SplitStore<E> heap; /* 1-based: Rust's data[i] is slot i + 1 */
    ulonglong2 *qcode; /* [NCH * G] 16-byte chunks of the query's SBQ code, zero past the code's end */
    uint32_t *rootnode; /* hash flavour: node id of the heap's root as the last pop left it (filled by cp.async) */
    QueryLabels key;
    bool slotpay;
    uint32_t heap_len, vis_head, vis_len, nset, listn, visits, dq, status;

    __device__ __forceinline__ LeanWarp(const SearchArgs &a_, int lane_) : a(a_), lane(lane_) {}

    __device__ __forceinline__ uint32_t node_of(E e) const {
        const uint32_t p = T::seq(e);
        return slotpay ? __ldcg(hash + p) : p;
    }

    /* prepare_insert = HashSet::insert (graph/mod.rs:126-128) of up to 64 neighbour ids (list slots `lane` and
     * `lane + 32`): dedupe within the list, then against `inserted` (sbq/storage.rs:149-163).  The atomics are only
     * ISSUED here - one atomicOr per id under the bitmap flavour, the first compare-and-swap probe of each id under
     * the hash flavour (open addressing, linear probing, any table size: multiplicative hash scaled to [0, cap)) -
     * and their answers are first read in stage_tail, so whatever the caller runs in between overlaps the L2/HBM
     * round trip. */
    struct Probe {
        uint32_t o0, o1; /* what the atomics returned */
        uint32_t h0, h1; /* hash flavour: the slots probed */
        bool f0, f1;     /* this lane's id takes part (valid and first occurrence) */
    };
    __device__ __forceinline__ Probe stage_probe(uint32_t n0, bool v0, uint32_t n1, bool v1, bool unique) {
        Probe pr;
        pr.f0 = v0;
        pr.f1 = v1;
        if (!unique) { /* a node listed twice within a chunk: only its first occurrence may insert */
            const unsigned m0 = __match_any_sync(DANN_FULL, n0);
            const unsigned m1 = __match_any_sync(DANN_FULL, n1);
            pr.f0 = v0 && ((__ffs(m0) - 1) == lane);
            pr.f1 = v1 && ((__ffs(m1) - 1) == lane);
        }
        pr.o0 = pr.o1 = 0xFFFFFFFFu;
        pr.h0 = pr.h1 = 0;
        if (a.bitmap_words) {
            if (pr.f0) pr.o0 = atomicOr(bitmap + (n0 >> 5), 1u << (n0 & 31));
            if (pr.f1) pr.o1 = atomicOr(bitmap + (n1 >> 5), 1u << (n1 & 31));
        } else {
            pr.h0 = __umulhi(n0 * 2654435761u, a.hash_cap);
            pr.h1 = __umulhi(n1 * 2654435761u, a.hash_cap);
            if (pr.f0) pr.o0 = atomicCAS(hash + pr.h0, DANN_INVALID_NODE, n0);
            if (pr.f1) pr.o1 = atomicCAS(hash + pr.h1, DANN_INVALID_NODE, n1);
        }
        return pr;
    }

    /* the atomics' answers (hash flavour: further probes for the ids that collided), then the label filter of the new
     * ids (sbq/storage.rs:165-172) and their compaction into the page, in list order */
    __device__ __forceinline__ void stage_tail(const Probe &pr, uint32_t n0, uint32_t n1, bool apply_filter) {
        bool new0, new1;
        uint32_t s0 = n0, s1 = n1; /* payload: the node id, or its hash slot */
        if (a.bitmap_words) {
            new0 = pr.f0 && !(pr.o0 & (1u << (n0 & 31)));
            new1 = pr.f1 && !(pr.o1 & (1u << (n1 & 31)));
        } else {
            const uint32_t cap = a.hash_cap;
            uint32_t h0 = pr.h0, h1 = pr.h1, o0 = pr.o0, o1 = pr.o1;
            bool p0 = pr.f0, p1 = pr.f1;
            new0 = new1 = false;
            for (uint32_t probe = 0; probe < cap; probe++) {
                if (p0) {
                    if (o0 == DANN_INVALID_NODE || o0 == n0) {
                        new0 = o0 == DANN_INVALID_NODE;
                        p0 = false;
                    } else {
                        h0 = h0 + 1 == cap ? 0u : h0 + 1;
                    }
                }
                if (p1) {
                    if (o1 == DANN_INVALID_NODE || o1 == n1) {
                        new1 = o1 == DANN_INVALID_NODE;
                        p1 = false;
                    } else {
                        h1 = h1 + 1 == cap ? 0u : h1 + 1;
                    }
                }
                if (!(p0 || p1)) break;
                if (p0) o0 = atomicCAS(hash + h0, DANN_INVALID_NODE, n0);
                if (p1) o1 = atomicCAS(hash + h1, DANN_INVALID_NODE, n1);
            }
            __syncwarp();
            if (slotpay) {
                s0 = h0;
                s1 = h1;
            }
            nset += __popc(__ballot_sync(DANN_FULL, new0)) + __popc(__ballot_sync(DANN_FULL, new1));
            if ((uint64_t)nset * 3u > (uint64_t)a.hash_cap * 2u) { /* load factor bound 2/3 */
                status |= DANN_ST_HASH;
                return;
            }
        }
        bool p0 = new0, p1 = new1;
        if (apply_filter) {
            if (new0) p0 = node_passes_filter(a.ix, key, n0);
            if (new1) p1 = node_passes_filter(a.ix, key, n1);
        }
        const unsigned lt = (1u << lane) - 1u;
        const unsigned pm0 = __ballot_sync(DANN_FULL, p0), pm1 = __ballot_sync(DANN_FULL, p1);
        const uint32_t t0 = __popc(pm0), t1 = __popc(pm1);
        if (t0 + t1 == 0) return;
        if (heap_len + listn + t0 + t1 + 1 > a.cand_cap) { /* 1-based heap slots: the last one is cand_cap - 1 */
            status |= DANN_ST_HEAP;
            return;
        }
        if (p0) {
            const uint32_t pos = listn + __popc(pm0 & lt);
            list[pos] = n0;
            ent[pos] = (E)s0;
        }
        if (p1) {
            const uint32_t pos = listn + t0 + __popc(pm1 & lt);
            list[pos] = n1;
            ent[pos] = (E)s1;
        }
        listn += t0 + t1;
        __syncwarp();
    }

    __device__ __forceinline__ void stage(uint32_t n0, bool v0, uint32_t n1, bool v1, bool apply_filter, bool unique) {
        if (__ballot_sync(DANN_FULL, v0 || v1) == 0) return;
        const Probe pr = stage_probe(n0, v0, n1, v1, unique);
        stage_tail(pr, n0, n1, apply_filter);
    }

    /* SBQ distance of every node of the page (distance/mod.rs:265-323): G lanes per code row, 128-bit no-allocate
     * loads, two row slots per lane group in flight, XOR + popcount + shuffle reduction; ent[r] becomes the entry.
     * EXACT: every lane's NCH chunk slots exist (cw / 2 == NCH * G, e.g. 768-d x 2 bits with G = 4), so the loads
     * need no bounds test and row slots past the end of the page simply read row 0. */
    template <bool EXACT>
    __device__ __forceinline__ void load_slot(ulonglong2 (&v)[NCH], uint32_t r, uint32_t tn, const ulonglong2 *qs) const {
        const bool live = r < tn;
        const ulonglong2 *row =
            reinterpret_cast<const ulonglong2 *>(a.ix.codes + (size_t)(live ? list[r] : 0u) * a.ix.cw) + (lane & (a.G - 1));
#pragma unroll
        for (int i = 0; i < NCH; i++) {
            if (EXACT) v[i] = ldg_stream_u128(row + i * a.G);
            else v[i] = (live && (lane & (a.G - 1)) + i * a.G < (a.ix.cw >> 1)) ? ldg_stream_u128(row + i * a.G) : qs[i * a.G];
        }
    }
    __device__ __forceinline__ void eat_slot(const ulonglong2 (&v)[NCH], uint32_t r, uint32_t tn, const ulonglong2 *qs) {
        uint32_t s = 0;
#pragma unroll
        for (int i = 0; i < NCH; i++) {
            const ulonglong2 qv = qs[i * a.G];
            s += __popcll(v[i].x ^ qv.x) + __popcll(v[i].y ^ qv.y);
        }
#pragma unroll
        for (int o = 16; o > 0; o >>= 1)
            if ((uint32_t)o < a.G) s += __shfl_xor_sync(DANN_FULL, s, o); /* warp-uniform */
        if ((lane & (a.G - 1)) == 0 && r < tn) ent[r] = T::make(s, T::seq(ent[r]));
    }
    /* A rolling pipeline of depth two over the page's row slots (one slot = one row per lane group, 32 / G rows per
     * warp): slot s + 2 is requested as soon as slot s has been reduced, so after the first (HBM) wait every later
     * slot - already on its way into L2 by the prefetch - arrives under the reduction of the slot before it. */
    template <bool EXACT>
    __device__ __forceinline__ void distances_t(uint32_t tn) {
        const uint32_t G = a.G, grp = lane >> a.Gshift, RP = 32u >> a.Gshift;
        const ulonglong2 *qs = qcode + (lane & (G - 1)); /* this lane's chunks of the query code: qs[i * G] */
        if (tn > 2 * RP) { /* rows of the later slots: pull them into L2 now, their loads then cost an L2 hit */
            const size_t rowbytes = (size_t)a.ix.cw * 8;
            const unsigned char *cb = reinterpret_cast<const unsigned char *>(a.ix.codes);
            for (uint32_t r = 2 * RP + lane; r < tn; r += 32) {
                const unsigned char *rowp = cb + (size_t)list[r] * rowbytes;
                prefetch_l2(rowp);
                if (rowbytes > 128) prefetch_l2(rowp + 128);
            }
        }
        ulonglong2 va[NCH], vb[NCH];
        load_slot<EXACT>(va, grp, tn, qs);
        load_slot<EXACT>(vb, RP + grp, tn, qs);
#pragma unroll 1
        for (uint32_t b = 0; b < tn; b += 2 * RP) {
            eat_slot(va, b + grp, tn, qs);
            load_slot<EXACT>(va, b + 2 * RP + grp, tn, qs);
            eat_slot(vb, b + RP + grp, tn, qs);
            load_slot<EXACT>(vb, b + 3 * RP + grp, tn, qs);
        }
        __syncwarp();
    }
    __device__ __forceinline__ void distances(uint32_t tn) {
        if (a.ix.cw == 2u * NCH * a.G) distances_t<true>(tn);
        else distances_t<false>(tn);
    }

    /* Σ_{t<h} (x >> t) */
    static __device__ __forceinline__ uint32_t shift_sum(uint32_t x, uint32_t h) {
        return 2u * x - (uint32_t)__popc(x) - 2u * (x >> h) + (uint32_t)__popc(x >> h);
    }

    /* BinaryHeap::push x tn in page order (insert_neighbor, graph/mod.rs:144-147) for a page whose leaves s0..s1 lie on
     * ONE heap level.  Elements that are inert (parent key <= own key: they stay at their leaf whatever earlier pushes
     * of the page do, because a slot's key never increases during pushes) are written by all lanes at once; the others
     * go through a warp-cooperative sift-up one at a time, in page order: lane j owns the path slot at height j, loads
     * its parent, one ballot finds where std's loop would break, the passed ancestors move one level down and the
     * element lands - one load, one ballot, one store whatever the rise height.  (A register-resident root-ward path -
     * ballot + shuffle per push, no memory on the chain - was measured slower at 7 and at 28 resident warps
     * per SM, and is gone.)
     * Slots in the HBM tail: every slot the pushes can touch - the leaves and, per height h, the ancestors
     * (s0 >> h)..(s1 >> h), about 2 tn + log n slots - is staged in shared memory with ONE round trip (all loads
     * issued together), the sift-ups run at shared-memory latency, and the staged slots go back in one pass; without
     * this every non-inert push of a deep heap waits for its own L2/HBM round trip (measured: 9 of the 30 us per visit
     * at 28 resident warps per SM).  Heights >= hcut have all their slots below hs, i.e. in the shared-memory top
     * already; the staging area sits in the same shared-memory array (behind the page), so a lane addresses its slot
     * as sm[B + slot] with a per-lane base B chosen once per page - no branch in the loop.
     * Requires tn <= heap_len (every ancestor is an old slot) and tn <= DANN_LIST_CAP.  eoff: where the (sub-)page
     * starts in ent[]. */
    /* Called as soon as the page length is known (before the distance stage): starts the copy of the page's ancestor
     * slots from the HBM tail into the staging area with cp.async - no registers, nothing waits - so that the round
     * trip runs under the code-row gather instead of in front of the pushes.  Single-level pages only (a page that
     * crosses a power of two is staged synchronously by its two sub-pages).  heap_len must not change until the push. */
    __device__ __forceinline__ void stage_ancestors_async(uint32_t tn) {
        stg_async = false;
        if (tn == 0 || tn > heap_len) return;
        const uint32_t s0 = heap_len + 1, s1 = heap_len + tn;
        if (s0 < (0x80000000u >> __clz(s1))) return;
        uint32_t hcut = 0;
        while ((s1 >> hcut) >= heap.hs) hcut++;
        for (uint32_t h = 1, off = tn; h < hcut; h++) { /* off(h) = sum of the counts of the heights below */
            const uint32_t lo = s0 >> h, cnt = (s1 >> h) - lo + 1u;
            for (uint32_t i = lane; i < cnt; i += 32) {
                const uint32_t slot = lo + i;
                if (slot < heap.hs) stg[off + i] = heap.sm[slot];
                else dann_cp_async(stg + off + i, heap.gl + slot);
            }
            off += cnt;
        }
        dann_cp_async_commit();
        stg_async = true;
    }

    __device__ __forceinline__ void push_page_staged(uint32_t tn, uint32_t eoff) {
        const E *pg = ent + eoff; /* this (sub-)page's entries */
        E *const sm = heap.sm;
        const uint32_t s0 = heap_len + 1, s1 = heap_len + tn;
        uint32_t hcut = 0;
        while ((s1 >> hcut) >= heap.hs) hcut++;
        /* staged index of slot x at height h: off(h) + x - (s0 >> h), off(h) = sum over t < h of the per-height counts */
        const uint32_t SB = (uint32_t)(stg - sm);
        const uint32_t hj = (uint32_t)lane, hp = lane < 31 ? (uint32_t)lane + 1u : 31u; /* lane 31 has no slot */
        const uint32_t B0 = hj < hcut ? SB + shift_sum(s1, hj) - shift_sum(s0, hj) + hj - (s0 >> hj) : 0u;
        const uint32_t B1 = hp < hcut ? SB + shift_sum(s1, hp) - shift_sum(s0, hp) + hp - (s0 >> hp) : 0u;
        const uint32_t Bpar = hcut > 1 ? SB + tn - (s0 >> 1) : 0u; /* height 1 (off(1) = tn), the same for every lane */
        const uint32_t Bleaf = hcut > 0 ? SB - s0 : 0u;
        if (stg_async) { /* started by stage_ancestors_async for exactly this page */
            dann_cp_async_wait_all();
            stg_async = false;
        } else {
            for (uint32_t h = 1, off = tn; h < hcut; h++) { /* stage the ancestors: independent loads, one round trip */
                const uint32_t lo = s0 >> h, cnt = (s1 >> h) - lo + 1u;
                for (uint32_t i = lane; i < cnt; i += 32) stg[off + i] = heap.get(lo + i);
                off += cnt;
            }
        }
        __syncwarp();
        for (uint32_t base = 0; base < tn; base += 32) {
            const uint32_t r = base + lane;
            const bool have = r < tn;
            const E mine = have ? pg[r] : E(0);
            const uint32_t slot = s0 + r;
            bool inert = false;
            if (have) {
                inert = sm[Bpar + (slot >> 1)] <= (mine | KM);
                if (inert) sm[Bleaf + slot] = mine;
            }
            unsigned act = __ballot_sync(DANN_FULL, have && !inert);
            __syncwarp();
            while (act) { /* warp-uniform: one cooperative sift-up per remaining element, in page order */
                const int b = __ffs(act) - 1;
                act &= act - 1;
                const E elem = pg[base + b];
                const uint32_t pp = s0 + base + (uint32_t)b;
                const uint32_t ast = pp >> lane, ald = ast >> 1;
                E av = 0;
                if (ald) av = sm[B1 + ald];
                const unsigned above = __ballot_sync(DANN_FULL, av > (elem | KM)); /* av = 0 above the root */
                const unsigned tm = above & ~(above + 1u); /* trailing ones: the ancestors the element passes */
                const unsigned wm = tm | (tm + 1u);        /* lanes 0..rise write */
                if ((wm >> lane) & 1u) sm[B0 + ast] = ((tm >> lane) & 1u) ? av : elem;
                __syncwarp();
            }
        }
        for (uint32_t h = 0, off = 0; h < hcut; h++) { /* staged slots back to the heap */
            const uint32_t lo = s0 >> h, cnt = (s1 >> h) - lo + 1u;
            for (uint32_t i = lane; i < cnt; i += 32) heap.set(lo + i, stg[off + i]);
            off += cnt;
        }
        __syncwarp();
        heap_len += tn;
    }

    __device__ __forceinline__ void push_page(uint32_t tn) {
        if (tn <= heap_len) {
            const uint32_t s0 = heap_len + 1, s1 = heap_len + tn;
            /* leaves on two heap levels (the page crosses a power of two): one sub-page per level */
            const uint32_t top = 0x80000000u >> __clz(s1); /* first slot of s1's level */
            if (s0 < top) {
                const uint32_t first = top - s0;
                push_page_staged(first, 0);
                push_page_staged(tn - first, first);
            } else {
                push_page_staged(tn, 0);
            }
            return;
        }
        /* the first pages of a scan: ancestors of a new slot may belong to the page itself */
        for (uint32_t i = 0; i < tn; i++) {
            heap_len++;
            H::template sift_up_warp1<false>(heap, heap_len, ent[i], lane);
        }
    }

    /* BinaryHeap::pop: the last element replaces the root, sift_down_to_bottom(0) walks the hole to the bottom taking
     * `child += (data[child] <= data[child+1])` (the right child on ties), then sift_up.  Four levels per round: lane
     * map 0-1 / 2-5 / 6-13 / 14-29 = the hole's children / grandchildren / ..., one ballot over all sibling pairs.
     * heap_len > 0; the caller has already read the root. */
    __device__ __forceinline__ void pop() {
        __syncwarp(); /* every lane has read the root (the caller's peek) before any lane overwrites slot 1 */
        if (!(a.hv_flags & DANN_HV_POP)) { /* lane 0 walks the hole down, one level per shared-memory round trip */
            H::pop_warp1(heap, heap_len, lane);
            return;
        }
        heap_len--;
        if (heap_len == 0) return;
        const uint32_t end = heap_len;
        const E item = heap.get(end + 1);
        const int lvl = lane < 2 ? 1 : lane < 6 ? 2 : lane < 14 ? 3 : lane < 30 ? 4 : 0;
        const uint32_t off = (uint32_t)lane - ((1u << lvl) - 2u);
        uint32_t p = 1;
        E lastv = 0;      /* what the walk moved into the final hole's parent */
        bool moved = false;
        while (2u * p + 1u <= end) {
            const uint32_t s = (p << lvl) + off;
            const bool ok = lvl != 0 && s <= end;
            E v = 0;
            if (ok) v = heap.get(s);
            const E vr = __shfl_down_sync(DANN_FULL, v, 1);
            const unsigned m = __ballot_sync(DANN_FULL, vr <= (v | KM)); /* data[child] <= data[child+1] */
            unsigned win = 0;
            uint32_t cur = p, idx = 0, lastlane = 0;
#pragma unroll
            for (int l = 1; l <= 4; l++) {
                const uint32_t c = 2u * cur;
                const uint32_t left = (1u << l) - 2u + 2u * idx;
                if (c + 1u <= end) {
                    const uint32_t r = (m >> left) & 1u;
                    lastlane = left + r;
                    win |= 1u << lastlane;
                    cur = c + r;
                    idx = 2u * idx + r;
                } else {
                    if (c == end) { /* a single child at the bottom is moved up without a comparison */
                        lastlane = left;
                        win |= 1u << left;
                        cur = c;
                    }
                    break;
                }
            }
            if ((win >> lane) & 1u) heap.set(s >> 1, v);
            lastv = __shfl_sync(DANN_FULL, v, (int)lastlane); /* the deepest winner of this round */
            moved = true;
            p = cur;
        }
        if (2u * p == end) { /* round boundary fell on the single-child step */
            const E c = heap.get(end);
            if (lane == 0) heap.set(p, c);
            lastv = c;
            moved = true;
            p = end;
        }
        /* sift_up(0, p) of the displaced element: it moves only while it is STRICTLY below its parent, and the parent of
         * the hole is the entry the walk just moved up - known without a load.  A former leaf is rarely smaller than
         * that, so the ancestor fetch of the generic sift-up (an L2/HBM round trip for a deep heap) is usually saved. */
        if (moved && !((item | KM) < (lastv & ~KM))) {
            if (lane == 0) heap.set(p, item);
            __syncwarp();
            return;
        }
        __syncwarp();
        H::template sift_up_warp1<false>(heap, p, item, lane);
    }

    __device__ __forceinline__ uint32_t vix(uint32_t i) const {
        const uint32_t x = vis_head + i;
        return x >= a.vcap ? x - a.vcap : x;
    }

    /* visited.insert(partition_point(|x| x < c), c): graph/mod.rs:166-168 */
    __device__ __forceinline__ void visited_insert(E e) {
        if (vis_len + 1 > a.vcap) {
            status |= DANN_ST_VIS;
            return;
        }
        const E eh = e & ~KM; /* x < eh  <=>  key(x) < key(e) */
        /* 32-ary search: one probe per lane at the end of its stride finds the boundary stride, then count inside it */
        const uint32_t stride = (vis_len + 31u) >> 5;
        const uint32_t s0 = (uint32_t)lane * stride;
        const uint32_t pe = s0 + stride < vis_len ? s0 + stride : vis_len;
        const bool whole = s0 < vis_len && vis[vix(pe - 1)] < eh;
        const uint32_t c = __popc(__ballot_sync(DANN_FULL, whole));
        uint32_t idx = c * stride < vis_len ? c * stride : vis_len;
        const uint32_t b0 = idx, b1 = b0 + stride < vis_len ? b0 + stride : vis_len;
        for (uint32_t i0 = b0; i0 < b1; i0 += 32) {
            const uint32_t i = i0 + lane;
            const bool lt = i < b1 && vis[vix(i)] < eh;
            idx += __popc(__ballot_sync(DANN_FULL, lt));
        }
        if (idx * 2 < vis_len) { /* fewer elements in front: open the gap by moving them one slot towards the head */
            vis_head = vis_head ? vis_head - 1 : a.vcap - 1;
            for (uint32_t i0 = 0; i0 < idx; i0 += 32) {
                const uint32_t i = i0 + lane;
                const bool act = i < idx;
                E t = 0;
                if (act) t = vis[vix(i + 1)];
                __syncwarp();
                if (act) vis[vix(i)] = t;
                __syncwarp();
            }
        } else {
            for (int hi = (int)vis_len; hi > (int)idx; hi -= 32) {
                const int i = hi - 1 - lane;
                const bool act = i >= (int)idx;
                E t = 0;
                if (act) t = vis[vix((uint32_t)i)];
                __syncwarp();
                if (act) vis[vix((uint32_t)i + 1)] = t;
                __syncwarp();
            }
        }
        if (lane == 0) vis[vix(idx)] = e;
        vis_len++;
        __syncwarp();
    }

    /* One visit (graph/mod.rs:166-168,370-383 + sbq/storage.rs:135-190): pop the root `head`, insert it into the
     * visited list, expand its neighbour list n0/n1 (list slots lane, lane + 32; R <= 64; loaded by the caller one
     * phase ahead).  The inserted-set atomics are issued first and the heap / visited-list work - which does not
     * depend on them - runs under their round trip.  Leaves the page (ids + entries with distances) staged: the
     * caller pushes it.  Returns the page length. */
    __device__ __forceinline__ uint32_t visit(E head, uint32_t n0, uint32_t n1) {
        bool v0, v1;
        neighbour_cut(n0, n1, lane, v0, v1);
        if (a.lists_unique) {
            const Probe pr = stage_probe(n0, v0, n1, v1, true);
            pop();
            root_node_async();
            visited_insert(head);
            if (status) return 0;
            stage_tail(pr, n0, n1, key.filter);
        } else {
            pop();
            root_node_async();
            visited_insert(head);
            if (status) return 0;
            /* a list may repeat an id: keep strict list order across the two chunks */
            stage(n0, v0, DANN_INVALID_NODE, false, key.filter, false);
            if (!status) stage(n1, v1, DANN_INVALID_NODE, false, key.filter, false);
        }
        const uint32_t tn = listn;
        listn = 0;
        if (tn == 0 || status) return 0;
        stage_ancestors_async(tn); /* the pushes' ancestor slots travel while the code rows are gathered */
        distances(tn);
        dq += tn;
        return tn;
    }

    /* start nodes: page -> distances -> pushes at once */
    __device__ __forceinline__ void flush() {
        const uint32_t tn = listn;
        listn = 0;
        if (tn == 0 || status) return;
        distances(tn);
        push_page(tn);
        dq += tn;
    }

    /* visit_closest's test (graph/mod.rs:153-170) for a candidate root */
    __device__ __forceinline__ bool may_visit(E head) const {
        if (vis_len > a.L) {
            const E at = vis[vix(a.L - 1)];
            if ((head | KM) >= (at | KM)) return false; /* head >= node_at_pos */
        }
        return true;
    }

    /* Hash flavour: a 4-byte entry names its node through its hash slot.  The root the pop leaves behind is the likeliest
     * next visit (about two visits in three), so its node id is fetched right after the pop, asynchronously into shared
     * memory, and root_after_page finds it there instead of paying a dependent HBM load in front of the neighbour row.
     * The PTX ISA orders two cp.async only through a wait, and the previous visit's copy to the same word may still be
     * in flight: neither root_after_page (the page minimum became the root) nor push_page_staged (no staged ancestors)
     * waited for it.  So it is waited for first; it landed a whole visit ago, the wait costs nothing. */
    __device__ __forceinline__ void root_node_async() {
        if (slotpay && heap_len > 0) {
            dann_cp_async_wait_all();
            if (lane == 0) dann_cp_async(rootnode, hash + T::seq(heap.get_sm(1)));
            dann_cp_async_commit();
        }
    }

    /* The entry the heap's root will hold once the staged page (tn entries in ent[]) has been pushed, and its node.  A
     * pushed element reaches the root iff its key is STRICTLY below the root's at that moment (sift_up moves only while
     * elem < parent), so the root after the page is the FIRST entry attaining the page minimum if that minimum is
     * strictly below the current root's key (or the heap is empty), else the current root.  Exact, not speculative:
     * it lets the next visit's neighbour row be fetched while the pushes run.  false = the heap stays empty. */
    __device__ __forceinline__ bool root_after_page(uint32_t tn, E *out, uint32_t *node) {
        E best = ~E(0);
        for (uint32_t r = lane; r < tn; r += 32) {
            const E c = (ent[r] & ~KM) | (E)r; /* key, then page position: the minimum is the first of the ties */
            best = c < best ? c : best;
        }
        if constexpr (SMALL) {
            best = __reduce_min_sync(DANN_FULL, best);
        } else {
            for (int o = 16; o > 0; o >>= 1) {
                const E t = __shfl_xor_sync(DANN_FULL, best, o);
                best = t < best ? t : best;
            }
        }
        const uint32_t idx = (uint32_t)(best & E(63));
        if (heap_len == 0) {
            if (tn == 0) return false;
            *out = ent[idx];
            *node = list[idx];
            return true;
        }
        const E root = heap.get_sm(1);
        if (tn != 0 && (best | KM) < (root & ~KM)) {
            *out = ent[idx];
            *node = list[idx];
        } else {
            *out = root;
            if (slotpay) {
                dann_cp_async_wait_all(); /* lane 0's copy of the root's node id (root_node_async) */
                __syncwarp();
                *node = *rootnode;
            } else {
                *node = T::seq(root);
            }
        }
        return true;
    }

    __device__ __forceinline__ void run(uint32_t q) {
        const IndexView &ix = a.ix;
        heap_len = vis_head = vis_len = nset = listn = 0;
        stg_async = false;
        visits = dq = status = 0;
        uint32_t scount = 0;
        slotpay = SMALL && a.bitmap_words == 0;
        { /* the query's SBQ code (SbqSearchDistanceMeasure, sbq/mod.rs:139-159) into shared memory: lane group member gl
           * compares chunks gl, gl + G, ... of every row against the same chunks of the query */
            const uint32_t nchunks = ix.cw >> 1, padded = (uint32_t)NCH * a.G;
            const ulonglong2 *qrow = reinterpret_cast<const ulonglong2 *>(a.q_codes + (size_t)q * ix.cw);
            for (uint32_t c = lane; c < padded; c += 32) qcode[c] = c < nchunks ? qrow[c] : make_ulonglong2(0, 0);
            __syncwarp();
        }
        if (!a.bitmap_words) hash_set_clear(hash, a.hash_cap, lane);
        key = query_labels(a, q);
        /* greedy_search_streaming_init + ListSearchResult::new (graph/mod.rs:97-124,331-354) */
        if (ix.start_default != DANN_INVALID_NODE) {
            if (a.q_label_off) {
                for (uint32_t b = 0; b < key.n && !status; b += 32) {
                    uint32_t n;
                    const bool valid = label_start_node(ix, key, b + lane, n);
                    /* start nodes are not label-checked (storage.rs:365-391); two labels may share a start node */
                    stage(n, valid, DANN_INVALID_NODE, false, false, false);
                    flush();
                }
            } else {
                stage(lane == 0 ? ix.start_default : DANN_INVALID_NODE, lane == 0, DANN_INVALID_NODE, false, false, true);
                flush();
            }
        }

        bool done = false;
        bool pend = false; /* n0 / n1 = the neighbour row of the current root `head`, requested ahead of its visit */
        uint32_t n0 = DANN_INVALID_NODE, n1 = DANN_INVALID_NODE;
        E head = 0;
        while (!done && !status) { /* TSVResponseIterator::next, scan.rs:210-242 */
            /* greedy_search_iterate: while let Some(idx) = visit_closest(L) */
            while (heap_len > 0) {
                if (!pend) head = heap.get_sm(1);
                if (!may_visit(head)) break; /* a requested row stays valid: nothing touches the heap until the visit */
                if (!pend) fetch_neighbours(ix, node_of(head), 0, lane, n0, n1); /* the popped element IS the current root */
                pend = false;
                visits++;
                const uint32_t tn = visit(head, n0, n1);
                if (status) break;
                /* the next visit is decided before this page is pushed - now, or after the consume()s that make
                 * room in the visited list - and its neighbour row is in flight while the pushes run */
                uint32_t nnode = 0;
                pend = root_after_page(tn, &head, &nnode);
                if (pend) fetch_neighbours(ix, nnode, 0, lane, n0, n1);
                if (tn) push_page(tn);
            }
            if (status) break;
            if (vis_len == 0) break; /* consume() -> None */
            const E e = vis[vis_head]; /* visited.remove(0), graph/mod.rs:174-184 */
            __syncwarp();
            vis_head = vix(1);
            vis_len--;
            const uint32_t node = node_of(e);
            const uint64_t tid = __ldg(ix.tids + node); /* return_lsn, sbq/storage.rs:404-414 */
            if ((tid & 0xFFFFull) == 0) continue;       /* InvalidOffsetNumber: deleted tuple, scan.rs:231-234 */
            if (lane == 0) a.stream[(size_t)q * a.c_target + scount] = node;
            scount++;
            if (scount == a.c_target) done = true;
        }
        if (slotpay) dann_cp_async_wait_all(); /* no copy of this query's root node id outlives it */
        if (a.bitmap_words) { /* leave the bitmap all zero for the slot's next query */
            __syncwarp();
            const uint4 z = make_uint4(0, 0, 0, 0);
            uint4 *b4 = reinterpret_cast<uint4 *>(bitmap);
            for (uint32_t i = lane; i < a.bitmap_words / 4; i += 32) b4[i] = z;
            __threadfence_block();
        }
        write_query_stats(a, q, lane, scount, visits, dq, false, status);
    }
};

/* MAXW = resident query slots (warps) per SM this instantiation is compiled for: 32 -> 64 registers per thread. */
template <typename T, int NCH, int MAXW>
__global__ void __launch_bounds__(MAXW * 32, 1) dann_search3_kernel(const SearchArgs a) {
    using E = typename T::E;
    DANN_DYN_SMEM(dann_smem);
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, W = blockDim.x >> 5;
    const uint32_t slot = blockIdx.x * W + warp;
    unsigned char *base = dann_smem + (size_t)warp * a.per_warp_smem;
    LeanWarp<T, NCH> w(a, lane);
    w.vis = reinterpret_cast<E *>(base);
    w.heap.sm = reinterpret_cast<E *>(base + (size_t)a.vcap * sizeof(E));
    w.ent = w.heap.sm + a.hs;
    w.stg = w.ent + DANN_LIST_CAP;
    w.list = reinterpret_cast<uint32_t *>(w.stg + DANN_STG_CAP);
    w.qcode = reinterpret_cast<ulonglong2 *>(base + a.per_warp_smem - (size_t)NCH * a.G * 16u); /* 16-byte aligned tail */
    w.rootnode = reinterpret_cast<uint32_t *>(w.qcode) - 4; /* the plan leaves 16 bytes in front of the query code */
    w.hash = a.hash + (size_t)slot * a.hash_cap;
    w.bitmap = a.bitmap + (size_t)slot * a.bitmap_words;
    w.heap.gl = reinterpret_cast<E *>(a.heap_tail) + (size_t)slot * a.cand_cap;
    w.heap.hs = a.hs;
    serve_queries(a, lane, w);
}
