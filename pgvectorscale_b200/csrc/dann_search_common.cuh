// dann_search_common.cuh — what the three beam-search kernels share: their arguments, the heap entry layouts and the
// steps of the reference algorithm that none of them tunes.
//   dann_search.cuh   single warp per query: the resumable scan, the plain layout, R > 64
//   dann_search2.cuh  two warps per query: batches of at most 7 queries per SM, the GPU builder
//   dann_search3.cuh  the lean warp-per-query kernel: every larger batch
// Reference paths below are relative to pgvectorscale/src/access_method/.
#pragma once
#include "dann_device.cuh"

/* what a suspended scan keeps besides its HBM workspace (heap tail, inserted-set, seq->node table) */
struct SavedScan {
    uint32_t valid, heap_len, vis_len, ncand, nins, visits, dq, exhausted;
};

/* Index- and plan-derived fields are filled by search_args_for_plan (dann_plan.h); each launch adds its request, its
 * buffers and its mode.  Everything it leaves alone is null or zero. */
struct SearchArgs {
    IndexView ix{};
    const uint64_t *q_codes = nullptr;    /* [B][cw] */
    const int16_t *q_labels = nullptr;    /* CSR values, sorted+dedup per query */
    const int32_t *q_label_off = nullptr; /* [B+1]; NULL => no scan key (labels None) */
    const uint32_t *qlist = nullptr;      /* optional [nq] query ids (retry pass) */
    uint32_t nq = 0;
    uint32_t L = 0, c_target = 0;
    uint32_t *stream = nullptr;           /* [B][c_target] node ids in consume order */
    uint32_t *stream_len = nullptr;       /* [B] */
    dann_query_stats *stats = nullptr;    /* [B] */
    uint32_t *overflow = nullptr;         /* OR of status bits over all queries of this launch */
    uint32_t *counter = nullptr;          /* work-queue head */
    uint32_t *hash = nullptr;             /* [slots][hash_cap] (bitmap_words == 0) */
    uint32_t hash_cap = 0;                /* power of two */
    uint32_t *bitmap = nullptr;           /* [slots][bitmap_words], all zero between queries */
    uint32_t bitmap_words = 0;            /* 0 => use the hash set */
    uint32_t *ins_list = nullptr;         /* [slots][ins_cap] inserted ids (bitmap mode: replayed to clear) */
    uint32_t ins_cap = 0;
    uint32_t *cand_node = nullptr;        /* [slots][cand_cap] */
    uint32_t cand_cap = 0;
    void *heap_tail = nullptr;            /* [slots][cand_cap] entries E (indices >= hs used) */
    uint32_t hs = 0, vcap = 0;
    uint32_t G = 0, Gshift = 0;           /* lanes per code row (power of two) */
    uint32_t lists_unique = 0;            /* no neighbour list repeats an id (checked at index load) */
    uint32_t per_warp_smem = 0;
    /* resumable scan (dann_scan_gettuple): single query, single warp; the per-scan workspace is not
     * shared with other queries, so the state below survives between launches */
    struct SavedScan *saved = nullptr; /* NULL = one-shot */
    void *saved_heap_sm = nullptr;     /* [hs] copy of the shared-memory part of the heap */
    uint64_t *saved_vis = nullptr;     /* [vcap] */
    /* build mode (dann_build.cuh): the scan stops when visit_closest first returns None and the
     * visited list (graph/mod.rs:285-327 greedy_search_for_build) is written out instead of a stream */
    uint32_t build_mode = 0;
    uint64_t *vis_out = nullptr;      /* [B][vis_out_cap] (dist << 32) | node, ascending */
    uint32_t *vis_out_len = nullptr;  /* [B] */
    uint32_t vis_out_cap = 0;
    /* engine switches read from DANN_HV_FLAGS (default: all on).  Bit 2 (DANN_HV_POP): the lean kernel's pop walks
     * the hole down four heap levels per memory round trip (off: lane 0 walks it level by level).  Kept last: the
     * offsets of the fields above are unchanged. */
    uint32_t hv_flags = 0;
    /* plain storage layout (SearchWarp<.., PLAIN=1> only; storage.rs:144-169, plain/storage.rs:223-299): the beam
     * search compares the query's index slice with the f32 vector each node stores.  Kept after everything else. */
    const float *plain_vectors = nullptr; /* [n][plain_dim] */
    const float *q_index = nullptr;       /* [B][plain_dim] prepared (truncated, cosine-normalised) queries */
    uint32_t plain_dim = 0;               /* num_dimensions_to_index */
};
#define DANN_HV_POP 2u

#define DANN_LIST_CAP 64u

/* Heap entry layouts: (distance << SEQ_BITS) | candidate sequence number.  Only the distance takes part in
 * comparisons.  Ent32x21: 11-bit distances (codes of up to 2047 bits, e.g. 768-d x 2 bits = 1536) and up
 * to 2M candidates per query in 4 bytes; Ent32x16: 16-bit distances, up to 65536 candidates; Ent64: anything. */
struct Ent32x21 {
    using E = uint32_t;
    static constexpr int KSHIFT = 21;
    static __device__ __forceinline__ uint32_t make(uint32_t d, uint32_t seq) { return (d << 21) | seq; }
    static __device__ __forceinline__ uint32_t seq(uint32_t e) { return e & 0x1FFFFFu; }
};
struct Ent32x16 {
    using E = uint32_t;
    static constexpr int KSHIFT = 16;
    static __device__ __forceinline__ uint32_t make(uint32_t d, uint32_t seq) { return (d << 16) | seq; }
    static __device__ __forceinline__ uint32_t seq(uint32_t e) { return e & 0xFFFFu; }
};
struct Ent64 {
    using E = uint64_t;
    static constexpr int KSHIFT = 32;
    static __device__ __forceinline__ uint64_t make(uint32_t d, uint32_t seq) { return ((uint64_t)d << 32) | seq; }
    static __device__ __forceinline__ uint32_t seq(uint64_t e) { return (uint32_t)e; }
};

/* The persistent kernels' work queue: the warp takes the next query of the launch (or of the retry list qlist) until
 * none is left. */
template <typename Warp>
__device__ __forceinline__ void serve_queries(const SearchArgs &a, int lane, Warp &w) {
    for (;;) {
        uint32_t qi = 0;
        if (lane == 0) qi = atomicAdd(a.counter, 1u);
        qi = __shfl_sync(DANN_FULL, qi, 0);
        if (qi >= a.nq) break;
        w.run(a.qlist ? a.qlist[qi] : qi);
    }
}

/* the query's scan key: its labels, sorted and deduplicated (none when the launch has no q_label_off: labels None) */
struct QueryLabels {
    const int16_t *l;
    uint32_t n;
    bool filter; /* has_label_filter, scan.rs:189 */
};
__device__ __forceinline__ QueryLabels query_labels(const SearchArgs &a, uint32_t q) {
    QueryLabels k{nullptr, 0u, false};
    if (a.q_label_off) {
        const int32_t o0 = a.q_label_off[q], o1 = a.q_label_off[q + 1];
        k.l = a.q_labels + o0;
        k.n = (uint32_t)(o1 - o0);
        k.filter = k.n > 0;
    }
    return k;
}

/* StartNodes::get_for_node(Some(labels)), start_nodes.rs:39-48: the start node of the query's i-th label, by binary
 * search in the index's sorted start labels.  false (n = INVALID) when i >= k.n or the label has no start node. */
__device__ __forceinline__ bool label_start_node(const IndexView &ix, const QueryLabels &k, uint32_t i, uint32_t &n) {
    n = DANN_INVALID_NODE;
    if (i >= k.n) return false;
    const int16_t lab = __ldg(k.l + i);
    uint32_t lo = 0, hi = ix.n_start_labels;
    while (lo < hi) {
        const uint32_t mid = (lo + hi) >> 1;
        if (__ldg(ix.start_labels + mid) < lab) lo = mid + 1;
        else hi = mid;
    }
    if (lo < ix.n_start_labels && __ldg(ix.start_labels + lo) == lab) {
        n = __ldg(ix.start_label_nodes + lo);
        return true;
    }
    return false;
}

/* labels.overlaps(node_neighbor.get_labels()), sbq/storage.rs:165-172 */
__device__ __forceinline__ bool node_passes_filter(const IndexView &ix, const QueryLabels &k, uint32_t n) {
    if (!ix.has_labels) return false;
    const uint32_t o0 = __ldg(ix.label_off + n), o1 = __ldg(ix.label_off + n + 1);
    return labels_overlap(k.l, k.n, ix.labels + o0, o1 - o0);
}

/* inserted = HashSet::new(), hash-set flavour: every slot empty (the bitmap flavour is left all zero by the slot's
 * previous query) */
__device__ __forceinline__ void hash_set_clear(uint32_t *hash, uint32_t hash_cap, int lane) {
    const uint4 ff = make_uint4(DANN_INVALID_NODE, DANN_INVALID_NODE, DANN_INVALID_NODE, DANN_INVALID_NODE);
    uint4 *h4 = reinterpret_cast<uint4 *>(hash);
    for (uint32_t i = lane; i < hash_cap / 4; i += 32) h4[i] = ff;
    __threadfence_block();
    __syncwarp();
}

/* prepare_insert = HashSet::insert (graph/mod.rs:126-128), hash-set flavour of the single-warp and two-warp kernels:
 * open addressing over a power-of-two table, linear probing.  true = n was not in the set yet. */
__device__ __forceinline__ bool hash_insert(uint32_t *hash, uint32_t hash_cap, uint32_t n) {
    const uint32_t mask = hash_cap - 1;
    uint32_t h = (n * 2654435761u) >> (32 - __popc(mask));
    for (uint32_t probe = 0; probe <= mask; probe++) {
        const uint32_t old = atomicCAS(hash + h, DANN_INVALID_NODE, n);
        if (old == DANN_INVALID_NODE) return true;
        if (old == n) return false;
        h = (h + 1) & mask;
    }
    return false;
}

/* list slots base + lane and base + 32 + lane of node's neighbour row; INVALID past R */
__device__ __forceinline__ void fetch_neighbours(const IndexView &ix, uint32_t node, uint32_t base, int lane, uint32_t &n0,
                                                 uint32_t &n1) {
    const uint32_t *row = ix.nbrs + (size_t)node * ix.Rp + base;
    n0 = base + (uint32_t)lane < ix.R ? ldg_stream_u32(row + lane) : DANN_INVALID_NODE;
    n1 = base + 32u + (uint32_t)lane < ix.R ? ldg_stream_u32(row + 32 + lane) : DANN_INVALID_NODE;
}

/* iter_neighbors stops at the first InvalidBlockNumber slot (sbq/node.rs:261-285): v0 / v1 = list slot lane / lane + 32
 * (of n0 / n1) lies before it.  Returns whether the list ends within these 64 slots. */
__device__ __forceinline__ bool neighbour_cut(uint32_t n0, uint32_t n1, int lane, bool &v0, bool &v1) {
    const unsigned i0 = __ballot_sync(DANN_FULL, n0 == DANN_INVALID_NODE);
    const unsigned i1 = __ballot_sync(DANN_FULL, n1 == DANN_INVALID_NODE);
    const uint32_t cut0 = i0 ? (uint32_t)(__ffs(i0) - 1) : 32u;
    const uint32_t cut1 = i0 ? 0u : (i1 ? (uint32_t)(__ffs(i1) - 1) : 32u);
    v0 = (uint32_t)lane < cut0;
    v1 = (uint32_t)lane < cut1;
    return (i0 | i1) != 0;
}

/* The query's stream length, its counters and status bits, and the launch's OR of status bits (the host reruns the
 * queries that overflowed).  dq = distances computed: full-precision ones when `full` (record_full_distance_comparison,
 * plain/storage.rs:238,288), else quantized. */
__device__ __forceinline__ void write_query_stats(const SearchArgs &a, uint32_t q, int lane, uint32_t scount, uint32_t visits,
                                                  uint32_t dq, bool full, uint32_t status) {
    if (lane == 0) {
        a.stream_len[q] = scount;
        dann_query_stats st;
        st.visits = visits;
        st.d_quantized = full ? 0u : dq;
        st.candidates = dq;
        st.d_full = full ? dq : 0u;
        st.stream_len = scount;
        st.status = status;
        a.stats[q] = st;
        if (status) atomicOr(a.overflow, status);
    }
    __syncwarp();
}
