/*
 * oracle.h — CPU oracle for the pgvectorscale StreamingDiskANN index-scan path.
 *
 * TEST INFRASTRUCTURE ONLY.  Nothing under pgvectorscale_b200/ may include, link
 * or call this.  Only tests/, __graft_entry__.smoke() and bench.py's cpu_baseline /
 * `--impl reference` legs use it, and only as the checker / the timed CPU baseline.
 *
 * It is a line-for-line restatement (in C++17) of the reference's Rust scan path;
 * every function cites the reference file:line it follows (paths relative to
 * pgvectorscale/src/access_method/).
 *
 * PARITY PIN STATUS (see DESIGN.md "Oracle"):
 *   - label overlap truth tables, 3-vector L2/IP KATs, rescore KAT, quantizer
 *     edge cases: pinned against the reference's own tests (restated in tests/).
 *   - tie order (Rust std BinaryHeap sift rules) and the intra-register order of
 *     simdeez's horizontal_add_ps are third-party code that is NOT vendored in
 *     the reference repository and was not executed (no rustc/cargo): for those two
 *     items the oracle says "parity unpinned" — it clones the published std
 *     algorithm (Rust 1.7x–1.8x alloc::collections::binary_heap) and the
 *     simdeez 1.0.x AVX2 hadd sequence, each isolated in one function.
 */
#ifndef PGVS_ORACLE_H
#define PGVS_ORACLE_H

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define ORC_INVALID_NODE 0xFFFFFFFFu /* InvalidBlockNumber sentinel, sbq/node.rs:261-273 */

enum { ORC_COSINE = 0, ORC_L2 = 1, ORC_IP = 2 }; /* distance/mod.rs:11-15 */

/* Flat index snapshot (same logical content as the product's dann_snapshot_desc). */
typedef struct {
    uint32_t n;            /* nodes */
    uint32_t dim;          /* full vector dimensions (heap column) */
    uint32_t dim_index;    /* num_dimensions_to_index (<= dim), pg_vector.rs:143-148 */
    uint32_t bits;         /* SBQ bits per dimension, meta_page.rs:312-323 */
    uint32_t words;        /* u64 words per code = ceil(dim_index*bits/64), quantize.rs:38-46 */
    uint32_t R;            /* num_neighbors, meta_page.rs:284-294 */
    int32_t distance_type; /* ORC_COSINE / ORC_L2 / ORC_IP */
    int32_t has_labels;    /* meta_page has_labels */
    uint64_t count;        /* SbqMeans.count */
    const float *mean;     /* [dim_index] */
    const float *m2;       /* [dim_index] (unused for bits==1) */
    const uint64_t *codes; /* [n*words] */
    const uint32_t *nbrs;  /* [n*R], ORC_INVALID_NODE terminates a list */
    const uint64_t *heap_tid; /* [n] (block<<16)|offset ; offset==0 => deleted (vacuum.rs) */
    const float *vectors;  /* [n*dim] raw heap vectors (NOT normalised) */
    uint32_t start_default; /* ORC_INVALID_NODE => no start nodes (empty graph) */
    uint32_t n_start_labels;
    const int16_t *start_labels;      /* ascending, start_nodes.rs BTreeMap order */
    const uint32_t *start_label_nodes;
    const uint32_t *label_off; /* [n+1] CSR into labels, only if has_labels */
    const int16_t *labels;     /* sorted+dedup per node */
    /* storage_layout (storage.rs:144-169).  ORC_STORAGE_PLAIN: the node holds the f32 vector it was built
     * from (truncated to dim_index, cosine-normalised at insert, plain/node.rs:17-22) and the beam search
     * compares the query against it directly (plain/storage.rs:223-299); no label filters. */
    int32_t storage_type;        /* ORC_STORAGE_SBQ (0) / ORC_STORAGE_PLAIN (1) */
    const float *index_vectors;  /* [n*dim_index], plain storage only */
} orc_snapshot;

enum { ORC_STORAGE_SBQ = 0, ORC_STORAGE_PLAIN = 1 };

typedef struct {
    uint64_t visits;      /* stats.visits           (stats.rs record_visit)   */
    uint64_t d_quantized; /* quantized distance comparisons                   */
    uint64_t candidates;  /* stats.candidate        (graph/mod.rs:145)        */
    uint64_t d_full;      /* full_distance_comparisons (scan.rs:258)          */
    uint64_t stream_len;  /* number of non-deleted items consumed from the LSR */
} orc_stats;

/* ---- leaf arithmetic ------------------------------------------------- */
/* distance/mod.rs:265-323 */
uint64_t orc_hamming(const uint64_t *a, const uint64_t *b, uint32_t words);
/* distance/mod.rs:88-104,175-209,325-434 + distance_x86.rs:21-36 ; scalar emulation of the
 * AVX2 4x8-lane order.  type: ORC_COSINE => max(0,1-dot), ORC_L2 => sum sq, ORC_IP => -dot */
float orc_distance(int type, const float *x, const float *y, uint32_t n);
/* same arithmetic written with real AVX2/FMA intrinsics (what the CPU baseline times) */
float orc_distance_avx2(int type, const float *x, const float *y, uint32_t n);
/* distance/mod.rs:107-117,212-223 (the *_unoptimized scalar forms) */
float orc_distance_unoptimized(int type, const float *x, const float *y, uint32_t n);
/* distance/mod.rs:225-253 */
void orc_preprocess_cosine(float *v, uint32_t n);
/* sbq/quantize.rs:104-148 ; vectors are [n*dim] already truncated to dim and (cosine) normalised */
void orc_train(const float *vectors, uint32_t n, uint32_t dim, uint32_t bits, float *mean,
               float *m2, uint64_t *count);
/* sbq/quantize.rs:52-102 */
void orc_quantize(const float *v, uint32_t dim, uint32_t bits, const float *mean,
                  const float *m2, uint64_t count, uint64_t *out_words);
uint32_t orc_code_words(uint32_t dim, uint32_t bits); /* quantize.rs:38-46 */
/* labels/mod.rs:124-142 */
int orc_labels_overlap(const int16_t *a, uint32_t na, const int16_t *b, uint32_t nb);
/* labels/mod.rs:84-111 */
int orc_labels_contains_intersection(const int16_t *self, uint32_t ns, const int16_t *a,
                                     uint32_t na, const int16_t *b, uint32_t nb);
/* labels/mod.rs:30-37 : sort_unstable + dedup, returns new length */
uint32_t orc_labels_normalize(int16_t *labels, uint32_t n);

/* ---- Rust std BinaryHeap clone, exposed for unit tests ---------------- */
/* Runs a script over a max-heap of (key,payload) ordered by key with the std sift rules.
 * ops[i] >= 0: push(key=ops[i], payload=i) ; ops[i] == -1: pop -> appended to out_payload.
 * Returns number of pops written. */
uint32_t orc_binary_heap_script(const int64_t *ops, uint32_t nops, int64_t *out_payload);

/* ---- scan: amrescan + amgettuple*max_rows (scan.rs:336-405) ------------ */
/* query: [dim] raw (NULL => SQL NULL query, labels/mod.rs:214-216)
 * labels/nlabels: nlabels < 0 => no scan key (None); >= 0 => Some(sorted-dedup(labels))
 * Writes up to max_rows results in amgettuple order; returns rows produced.
 * out_stream (optional, capacity stream_cap): node ids in LSR consume order (non-deleted). */
uint32_t orc_scan(const orc_snapshot *s, const float *query, const int16_t *labels,
                  int32_t nlabels, uint32_t search_list_size, uint32_t rescore,
                  uint32_t max_rows, uint64_t *out_tid, uint32_t *out_node, float *out_dist,
                  uint32_t *out_stream, uint32_t stream_cap, orc_stats *out_stats);

/* Batch of independent scans, one per query, `threads` host threads (0 => hardware). */
void orc_scan_batch(const orc_snapshot *s, const float *queries, const int16_t *labels,
                    const int32_t *label_off /* [B+1] or NULL */, uint32_t B,
                    uint32_t search_list_size, uint32_t rescore, uint32_t k, uint64_t *out_tid,
                    float *out_dist, uint32_t *out_count, orc_stats *out_stats, uint32_t threads);

/* ---- serial Vamana build restating graph/mod.rs:212-266,285-327,392-533,637-737 ------
 * Inputs: codes/labels for n nodes in insertion (heap-scan) order. Output nbrs [n*R].
 * index pointer of node i is modelled as i (ip_distance = |i-j|, util/mod.rs:165-170). */
void orc_build(uint32_t n, uint32_t words, const uint64_t *codes, uint32_t R,
               uint32_t search_list_size, double max_alpha, int32_t has_labels,
               const uint32_t *label_off, const int16_t *labels, uint32_t *out_nbrs,
               uint32_t *out_start_default, int16_t *out_start_labels,
               uint32_t *out_start_label_nodes, uint32_t *out_n_start_labels,
               uint32_t start_label_cap);

/* ---- model of the product's batched builder (dann_build_graph) --------------------------
 * The SAME prune / add_neighbors / search_for_build as orc_build, run under the batch schedule:
 * node 0 first, then batches of min(max(1, lo/16), max_batch, n - lo) nodes; every search of a
 * batch sees the graph as it stood before the batch, then the forward lists are written, then
 * the back-links of the whole batch are added per destination in (distance, source) order.  A
 * labeled batch runs twice (filtered, then unfiltered; the second pass merges with the first).
 * Each way the GPU builder departs from the reference is one switch; all zero and
 * max_batch == 1 is the reference's serial build (== orc_build). */
typedef struct {
    uint32_t scan_ties;     /* 1: the build search orders equal distances as a scan does (tie-break 0,
                             *    neighbor_with_distance.rs:31-43) instead of by |id - p| (:45-49) */
    uint32_t order_by_id;   /* 1: prune candidates are ordered by (distance, id) instead of the stable sort by
                             *    DistanceWithTieBreak, and a list that went through a merge is stored in that order */
    uint32_t visited_cap;   /* N > 0: only the first N entries of the distance-ordered visited list are handed over */
    uint32_t cand_cap;      /* N > 0: a forward prune sees its current neighbours + the closest N - deg visited nodes */
    uint32_t back_src_cap;  /* N > 0: a destination takes at most the N closest new sources of one batch */
    uint32_t slots;         /* N > 0: lists have N storage slots: back-links overflow at min(N, ceil(1.3 R)) */
    uint32_t fwd_keep_slots; /* 1: a forward list is pruned only when it outgrows `slots`, not ceil(1.3 R) */
} orc_build_switches;

/* how often each branch ran (indices into out_counts[ORC_BC_N]) */
enum {
    ORC_BC_FWD_KEPT = 0,     /* forward list written unpruned */
    ORC_BC_FWD_PRUNED,       /* forward list pruned to R */
    ORC_BC_FWD_MERGED,       /* forward pass that started from a non-empty list (second pass of a labeled insert) */
    ORC_BC_BACK_APPENDED,    /* back-links appended, no merge */
    ORC_BC_BACK_MERGED,      /* back-links merged and stored in candidate order, no prune */
    ORC_BC_BACK_PRUNED,      /* back-link overflow: pruned to R */
    ORC_BC_BACK_SRC_CUT,     /* destination with more than back_src_cap new sources in one batch */
    ORC_BC_BACK_REPEAT,      /* a new source that was already a neighbour of its destination */
    ORC_BC_FINAL_PRUNED,     /* finalize: list longer than R pruned */
    ORC_BC_VISITED_CUT,      /* visited list longer than visited_cap */
    ORC_BC_CAND_CUT,         /* visited nodes dropped by cand_cap */
    ORC_BC_EMPTY_SEARCH,     /* a search that visited nothing (no start node for any label of the point) */
    ORC_BC_ROUND2_KEPT,      /* prune: a neighbour accepted in the second alpha round */
    ORC_BC_TIE_FACTOR,       /* prune: the |id - p| / |id - kept| factor of two zero distances */
    ORC_BC_ZERO_OCCLUDED,    /* prune: zero distance to the kept neighbour, non-zero to the point */
    ORC_BC_LABEL_SKIP,       /* prune: occlusion skipped by contains_intersection */
    ORC_BC_N
};

void orc_build_batched(uint32_t n, uint32_t words, const uint64_t *codes, uint32_t R,
                       uint32_t search_list_size, double max_alpha, int32_t has_labels,
                       const uint32_t *label_off, const int16_t *labels, uint32_t max_batch /* 0 = unbounded */,
                       const orc_build_switches *sw, uint32_t *out_nbrs /* [n * out_stride], INVALID-padded */,
                       uint32_t out_stride /* >= R */, uint64_t *out_counts /* [ORC_BC_N] or NULL */);

#ifdef __cplusplus
}
#endif
#endif
