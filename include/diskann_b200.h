/*
 * diskann_b200.h — C ABI of the H100-native StreamingDiskANN index-scan engine.
 *
 * This is the drop-in boundary for pgvectorscale's `diskann` index *scan* path: the
 * Rust/pgrx access-method callbacks stay host code and call these entry points where
 * they used to run `TSVScanState::initialize` and `TSVResponseIterator::next_with_resort`.
 * Reference citations are relative to pgvectorscale/src/access_method/.
 *
 *   reference interface                              replaced by
 *   ------------------------------------------------ -----------------------------------
 *   ambeginscan            scan.rs:309-333           dann_scan_begin
 *   amrescan               scan.rs:336-367           dann_scan_rescan
 *     TSVScanState::initialize      scan.rs:57-88
 *     LabeledVector::from_scan_key_data labels/mod.rs:209-238
 *     Graph::greedy_search_streaming_init graph/mod.rs:331-354
 *   amgettuple             scan.rs:370-436           dann_scan_gettuple (dann_scan_fetch: n calls' rows in one step)
 *     TSVResponseIterator::next_with_resort scan.rs:244-305
 *     Graph::greedy_search_iterate  graph/mod.rs:357-385
 *     SbqSpeedupStorage::visit_lsn  sbq/storage.rs:125-190
 *     get_full_distance_for_resort  sbq/storage.rs:304-328
 *   amendscan              scan.rs:439-476           dann_scan_end (+ dann_scan_stats)
 *   MetaPage::fetch / SbqMeans::load (index -> RAM)  dann_index_load (index -> HBM)
 *   PlainStorage::load_for_search plain/storage.rs   dann_index_load_plain
 *   distance_xor_optimized distance/mod.rs:265-323   dann_sbq_distance (micro-kernel)
 *   distance_l2 / _cosine / _inner_product :88-209   dann_full_distance (micro-kernel)
 *   SbqQuantizer::quantize sbq/quantize.rs:52-102    dann_prepare_queries
 *
 * Conventions: every function returns DANN_OK (0) or a negative dann_status; nothing
 * throws, longjmps or aborts (the Rust shim turns a non-zero code into pgrx::error!).
 * dann_last_error() gives a thread-local message.  Host pointers are borrowed for the
 * duration of the call only.  A dann_index is immutable after load and may be shared
 * by host threads (calls on one index are serialised internally); a dann_scan is
 * single-threaded, like a Postgres backend.
 */
#ifndef DISKANN_B200_H
#define DISKANN_B200_H

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define DANN_INVALID_NODE 0xFFFFFFFFu          /* InvalidBlockNumber, sbq/node.rs:261-273 */
#define DANN_INVALID_TID 0xFFFFFFFFFFFFFFFFull /* "no row" in batch outputs */

typedef enum {
    DANN_OK = 0,
    DANN_ERR_INVALID_ARG = -1,
    DANN_ERR_CUDA = -2,      /* sticky: the handle is poisoned */
    DANN_ERR_NO_DEVICE = -3, /* no CUDA device / driver: there is NO CPU fallback */
    DANN_ERR_OOM = -4,
    DANN_ERR_CAPACITY = -5,  /* per-query state outgrew the largest workspace we may allocate */
    DANN_ERR_STATE = -6,
    DANN_ERR_FORMAT = -7     /* dann_pg_*: the relation file is not what the reader can vouch for; nothing is guessed */
} dann_status;

typedef enum { DANN_COSINE = 0, DANN_L2 = 1, DANN_IP = 2 } dann_distance; /* distance/mod.rs:11-15 */

/* Flat snapshot of one diskann index (host memory, row-major). See
 * pgvectorscale_b200/snapshot.py for the field-by-field provenance. */
typedef struct {
    uint32_t n;             /* nodes */
    uint32_t dim;           /* heap vector dimensions */
    uint32_t dim_index;     /* num_dimensions_to_index, pg_vector.rs:143-148 */
    uint32_t bits;          /* SBQ bits per dimension, meta_page.rs:312-323 */
    uint32_t words;         /* u64 per code = ceil(dim_index*bits/64), quantize.rs:38-46 */
    uint32_t R;             /* num_neighbors, meta_page.rs:284-294 */
    int32_t distance_type;  /* dann_distance */
    int32_t has_labels;
    uint64_t count;         /* SbqMeans.count */
    const float *mean;      /* [dim_index] */
    const float *m2;        /* [dim_index], may be NULL when bits == 1 */
    const uint64_t *codes;  /* [n*words] */
    const uint32_t *nbrs;   /* [n*R], list ends at first DANN_INVALID_NODE */
    const uint64_t *heap_tid; /* [n] (block<<16)|offset, offset 0 = deleted */
    const float *vectors;   /* [n*dim] raw heap vectors */
    uint32_t start_default; /* DANN_INVALID_NODE = empty graph */
    uint32_t n_start_labels;
    const int16_t *start_labels;       /* ascending */
    const uint32_t *start_label_nodes;
    const uint32_t *label_off;         /* [n+1] if has_labels */
    const int16_t *labels;             /* sorted, dedup per node */
} dann_snapshot_desc;

/* Per-query counters: the ones the reference logs at amendscan (scan.rs:461-472). */
typedef struct {
    uint32_t visits;      /* visits=      */
    uint32_t d_quantized; /* d_quantized= */
    uint32_t candidates;  /* candidate=   */
    uint32_t d_full;      /* d_full=      */
    uint32_t stream_len;  /* non-deleted items consumed from the ListSearchResult */
    uint32_t status;      /* 0 ok; internal overflow bits are retried and never surface */
} dann_query_stats;

typedef struct dann_index dann_index;
typedef struct dann_scan dann_scan;

const char *dann_last_error(void);
int dann_device_count(void);

/* ---- index lifetime ----------------------------------------------------------- */
/* Copies the snapshot into HBM of `device` (vectors cosine-normalised once, with the
 * reference's preprocess_cosine arithmetic, distance/mod.rs:225-253). */
int dann_index_load(const dann_snapshot_desc *snap, int device, dann_index **out);
/* storage_layout = plain (storage.rs:144-169; PlainStorage, plain/storage.rs:223-307): every node carries the f32
 * vector it was indexed with - index_vectors [n*dim_index], i.e. truncated to num_dimensions_to_index and, for cosine,
 * normalised after truncation (pg_vector.rs:143-155) - and the beam search compares the query with it directly; the
 * snapshot's SBQ fields (bits, words, count, mean, m2, codes) are ignored.  As in the reference (build.rs:264-290)
 * inner product, label filters and more than 2000 indexed dimensions are rejected.  Scans rerank from `vectors` only
 * when dim_index < dim (scan.rs:392-403), otherwise rows come back in beam-search order with dist = NaN.
 * Verified bit-exact against the oracle on the GPU (tests/test_zz_plain_gpu.py) and under CPU emulation of the kernel. */
int dann_index_load_plain(const dann_snapshot_desc *snap, const float *index_vectors, int device, dann_index **out);
void dann_index_free(dann_index *ix);
/* `vectors` may be NULL in the snapshot (see dann_index_set_vectors); scans then need rescore == 0.
 * Bytes of HBM held by the index arrays (codes, nbrs, tids, vectors, labels, means): */
uint64_t dann_index_hbm_bytes(const dann_index *ix);

/* ---- scan operator: one row at a time, amgettuple order ------------------------ */
int dann_scan_begin(dann_index *ix, dann_scan **out);
/* query: [dim] raw floats, NULL = SQL NULL order-by argument (zero vector, no labels,
 * labels/mod.rs:214-216). nlabels < 0 = no scan key; >= 0 = `labels && ARRAY[...]`
 * (sorted+dedup is done here, labels/mod.rs:30-37). search_list_size / rescore are the
 * GUCs diskann.query_search_list_size / diskann.query_rescore (guc.rs:3-4). */
int dann_scan_rescan(dann_scan *sc, const float *query, const int16_t *labels, int nlabels,
                     int search_list_size, int rescore);
/* How far a scan may stream: to the end of the index, as the reference's next_with_resort does, with exactly its rows,
 * dist bits and dann_scan_stats after every call.  The only condition is device memory for the search state: a
 * failed allocation returns DANN_ERR_OOM.  The suspended search's workspace is planned for rescore + 64 streamed rows
 * (for more when the first dann_scan_fetch after the rescan asks for more);
 * a scan that runs past it (a selective post-filter, or no LIMIT) has its workspace rebuilt twice as large and the
 * stream replayed from row 0 - invisible to the caller except in time.  Where that planned workspace can grow no
 * further (eight doublings in one call, or a visited list past shared memory, or 2^30 candidates) the scan enters the
 * deep mode once: its search is rebuilt with 8-byte heap entries, an inserted-set bitmap over every node id (n / 8
 * bytes) and the visited list in HBM, and replayed one last time.  From then on it suspends before a visit that
 * might not fit, grows its buffers in place (at least twice as large, the live state copied on the device) and
 * resumes the same step: no row is generated twice.  dann_scan_rescan returns the scan to the planned workspace and
 * frees the deep buffers, as dann_scan_end does.  The batch entry points keep their bounds.
 * One amgettuple: resumes the scan's suspended search (its state lives in HBM between calls), pulls
 * exactly the rows TSVResponseIterator::next_with_resort would (scan.rs:244-305), pops one.
 * Returns 1 and fills the outputs for the next row, 0 at end of scan, <0 on error.
 * dist is the exact rerank distance (NaN when rescore == 0). Any output may be NULL. */
int dann_scan_gettuple(dann_scan *sc, uint32_t *block, uint16_t *offset, uint32_t *node_id,
                       float *dist);
/* The next rows of a scan in one GPU step: exactly what max_rows consecutive dann_scan_gettuple calls return.
 * Returns r = rows produced (0..max_rows; r < max_rows only at end of scan) or < 0.  block/offset/node_id/dist are
 * [max_rows] (each may be NULL); row_stats[i] (may be NULL) = dann_scan_stats after the (i+1)-th of those calls.
 * Afterwards the scan is in the state those max_rows calls leave: dann_scan_stats == row_stats[r-1] when r == max_rows,
 * and when r < max_rows the counters of the call that found the end of scan (its search may have run on past the last
 * row).  The next dann_scan_gettuple / dann_scan_fetch / dann_scan_gettuple_many continues the same stream, and the
 * three may be interleaved at any call.  Rows, dist bits and counters never differ from the single calls'; the one
 * thing that may is dann_scan_workspace: the eight replay regrows before the deep mode are counted per call, so a fetch
 * may enter the deep mode at a different row than single calls would.  The search, the exact distances and the window
 * step run once for all the rows (a fixed number of kernel launches, whatever max_rows), and the rows come back in one
 * copy and one synchronisation; growing the workspace adds attempts, as in dann_scan_gettuple.
 * Arguments are checked as dann_scan_gettuple checks them; in addition max_rows outside 1..65536 returns
 * DANN_ERR_INVALID_ARG before anything runs.  A failed fetch fails as a failed dann_scan_gettuple does. */
int dann_scan_fetch(dann_scan *sc, int max_rows, uint32_t *block, uint16_t *offset, uint32_t *node_id,
                    float *dist, dann_query_stats *row_stats);
/* n amgettuple calls, one per scan, all on the same index: out_rc[i] = 1 (row), 0 (end of scan) or a negative status
 * for that scan alone; block/offset/node_id/dist are [n] arrays, each may be NULL.
 * Every scan gets exactly the row, dist bits and dann_scan_stats the same sequence of dann_scan_gettuple calls would
 * give it; the scans may differ in query, key, search_list_size and rescore, and a scan may switch between the two
 * entry points at any call.  Many suspended searches resume in one kernel launch (one warp each, with the scan's own
 * plan and workspace), so the backends of a serving process share the GPU instead of queueing behind each other.
 * Returns DANN_OK, or before anything runs: DANN_ERR_INVALID_ARG for n outside 1..65536, a NULL scans / out_rc / scan,
 * scans of different indexes or a scan listed twice, DANN_ERR_STATE for a scan that has not been rescanned.  A scan
 * whose buffers cannot be allocated gets DANN_ERR_OOM in out_rc and leaves the others unaffected; a scan that must grow
 * its workspace (by replay or, in the deep mode, in place) does so alone and rejoins the next round.  Any other failure returns an error only while no scan has taken
 * its step; once one has, it goes to out_rc of the scans it hit, and the rows of the others stand.  dann_last_error()
 * describes the last failure of the call, which need not be scan i's. */
int dann_scan_gettuple_many(dann_scan *const *scans, int n, int32_t *out_rc, uint32_t *block, uint16_t *offset,
                            uint32_t *node_id, float *dist);
int dann_scan_stats(dann_scan *sc, dann_query_stats *out);
/* What a scan holds: its mode, how it got there since the last dann_scan_rescan, and the device memory it keeps. */
typedef struct {
    uint32_t mode;         /* 0 = the planned workspace, 1 = deep (see dann_scan_gettuple) */
    uint32_t regrows;      /* replay regrows */
    uint32_t growths;      /* in-place growths of the deep mode */
    uint32_t reserved;     /* 0 */
    uint64_t device_bytes; /* bytes of device memory held by the scan */
} dann_scan_workspace_info;
int dann_scan_workspace(dann_scan *sc, dann_scan_workspace_info *out);
void dann_scan_end(dann_scan *sc);

/* ---- entry points that take DEVICE buffers (dann_search_batch_device, dann_prepare_queries, dann_sbq_distance,
 * dann_full_distance, dann_index_set_vectors_device): `stream` is the CUDA stream the call runs on and the order in
 * which the caller's buffers must be ready.  stream == NULL: the call runs on the index's own non-blocking stream,
 * after everything the caller has already submitted to the legacy default stream (the order a default-stream kernel
 * or a plain cudaMemcpy would have had); buffers produced on OTHER non-blocking streams need that stream passed here,
 * or a synchronisation by the caller.  Outputs are complete when the call returns. */

/* ---- batch: B independent scans, first k rows of each ---------------------------- */
/* Host buffers; H2D/D2H copies are part of the call (this is the end-to-end path).
 * labels/label_off: CSR of each query's scan-key labels, label_off == NULL = no key.
 * out_tid [B*k] (block<<16|offset, DANN_INVALID_TID past out_count[b]), out_dist [B*k],
 * out_count [B] rows produced, out_stats [B] (each may be NULL except out_tid).
 * rescore + k is bounded by the rerank kernel's shared memory (about 45 000 rows at 768 dimensions):
 * larger requests return DANN_ERR_INVALID_ARG (the streaming scan operator is not bound by the rerank window). */
int dann_search_batch(dann_index *ix, const float *queries, const int16_t *labels,
                      const int32_t *label_off, int B, int k, int search_list_size,
                      int rescore, uint64_t *out_tid, float *out_dist, uint32_t *out_count,
                      dann_query_stats *out_stats);
/* Same with every buffer already resident in HBM of the index's device; work is
 * enqueued on `stream` (a cudaStream_t; NULL = the index's own stream, see the note on device buffers above) and
 * the call returns after the stream has drained (it must read back a 4-byte overflow flag). Query labels
 * must already be sorted+dedup per query. */
int dann_search_batch_device(dann_index *ix, const float *d_queries, const int16_t *d_labels,
                             const int32_t *d_label_off, int B, int k, int search_list_size,
                             int rescore, uint64_t *d_out_tid, float *d_out_dist,
                             uint32_t *d_out_count, dann_query_stats *d_out_stats,
                             void *stream);

/* ---- batch whose queries differ in k, search_list_size, rescore and key ---------------------------------------
 * One query's request.  `params` is a host array [B] for the host entry points and a device array for _device. */
typedef struct {
    int32_t k;                /* rows wanted, >= 1 */
    int32_t search_list_size; /* 1..10000, guc.rs:11-26 */
    int32_t rescore;          /* 0..1000,  guc.rs:28-43 */
    int32_t keyed;            /* 0 = no scan key (labels None); 1 = labels[label_off[b] .. label_off[b+1]) */
} dann_query_params;
/* B independent scans in one launch of each kernel, each with its own parameters.
 * - Output: rows are [B][kmax] with kmax the largest params[b].k; query b's rows start at b * kmax.  Past out_count[b]
 *   (at most params[b].k) a row holds DANN_INVALID_TID and NaN.
 * - Per query: query b gets exactly what a dann_search_batch of that query alone returns with its own k,
 *   search_list_size, rescore and key - tids, distance bits, out_count and every dann_query_stats field - whatever it
 *   is batched with, and through any workspace-growth reruns.
 * - Keys: keyed = 0 is no key, and its label_off range must be empty.  keyed = 1 with an empty range is
 *   `labels && ARRAY[]`, which returns no rows.  label_off may be NULL only when no query is keyed.  The host entry
 *   point sorts and deduplicates each key, as dann_search_batch does; the device entry point needs sorted keys.
 * - Checks, all before anything runs (DANN_ERR_INVALID_ARG, the message names the query; the handle stays usable):
 *   B < 1, a NULL params, a value out of range, keyed not 0 or 1, a non-monotone label_off, a keyed query without
 *   label_off, a query whose own k and rescore exceed the rerank kernel's shared memory (the dann_search_batch rule).
 * - Plain layout: a keyed query is refused, and a query's rescore counts as 0 when dim == dim_index.
 * The plan is made for the batch's largest search_list_size and stream, and for a key if any query has one.
 * dann_search_batch_mixed_device reads params (and label_off) back to check them, then runs as
 * dann_search_batch_device does. */
int dann_search_batch_mixed(dann_index *ix, const float *queries, const int16_t *labels, const int32_t *label_off,
                            const dann_query_params *params, int B, uint64_t *out_tid, float *out_dist,
                            uint32_t *out_count, dann_query_stats *out_stats);
int dann_search_batch_mixed_device(dann_index *ix, const float *d_queries, const int16_t *d_labels,
                                   const int32_t *d_label_off, const dann_query_params *d_params, int B,
                                   uint64_t *d_out_tid, float *d_out_dist, uint32_t *d_out_count,
                                   dann_query_stats *d_out_stats, void *stream);

/* ---- stand-alone kernels (roofline metric + per-kernel parity tests), device buffers -- */
/* amrescan's vector preparation: cosine-normalise + SBQ-quantize B queries.
 * d_q_full [B*dim] (may be NULL), d_q_codes [B*dann_code_stride(ix)]. */
int dann_prepare_queries(dann_index *ix, const float *d_queries, int B, float *d_q_full,
                         uint64_t *d_q_codes, void *stream);
uint32_t dann_code_stride(const dann_index *ix); /* u64 per code row in HBM (words rounded up to even) */
/* SBQ distance: out[i] = popcount(code[pair_node[i]] ^ qcode[pair_q[i]]). */
int dann_sbq_distance(dann_index *ix, const uint64_t *d_qcodes, const uint32_t *d_pair_q,
                      const uint32_t *d_pair_node, size_t npairs, uint32_t *d_out, void *stream);
/* Exact rerank distance: out[b*m+i] = distance_fn(vectors[nodes[b*m+i]], q_full[b]);
 * nodes == DANN_INVALID_NODE are skipped (out = NaN). */
int dann_full_distance(dann_index *ix, const float *d_q_full, const uint32_t *d_nodes, int B,
                       int m, float *d_out, void *stream);

/* ---- index construction (SURVEY.md §8f row 1; NOT the scan hot path) -----------------------------
 * GPU batch Vamana over SBQ codes built from the scan kernels: greedy_search_for_build
 * (graph/mod.rs:285-327) + prune_neighbors (:392-488) + back-pointers (:212-266,720-737), nodes
 * inserted in batches.  The index must have been loaded with R == 64 neighbour slots per node
 * (contents ignored) and start_default == 0; `vectors` may be NULL at load and supplied later.  A labeled
 * index (has_labels, with start_labels/start_label_nodes = the first node carrying each label) is built
 * the reference's way: a label-filtered insertion pass from the label start nodes, then the unfiltered
 * one (graph/mod.rs:637-660), with the label-aware prune (:445-455).  On return every list holds
 * <= num_neighbors ids.  The graph is a valid diskann graph but not the reference's serial insertion
 * order, so it serves bulk builds, fixtures and benchmarks. */
typedef struct {
    uint32_t batches;
    float search_ms, prune_ms, sort_ms, backlink_ms, total_ms;
    double avg_degree;
} dann_build_stats;
int dann_build_graph(dann_index *ix, int num_neighbors, int search_list_size, float max_alpha, uint32_t max_batch,
                     dann_build_stats *out);
/* Copy the neighbour lists back to the host: out [n][R] with R = the snapshot's R. */
int dann_index_download_nbrs(dann_index *ix, uint32_t *out);
/* Supply (or replace) the heap vectors of an index loaded with vectors == NULL; [n][dim] host floats. */
int dann_index_set_vectors(dann_index *ix, const float *vectors);
/* The same with the rows already in HBM on the index's device: d_vectors [n][dim] is BORROWED - the index reads it in
 * place (no second copy: 50M x 768-d rows are 153.6 GB of the 180) and, for cosine, normalises it in place once like
 * dann_index_load does; the caller keeps it allocated until dann_index_free. */
int dann_index_set_vectors_device(dann_index *ix, float *d_vectors);

/* ---- query-batch data parallelism over replicated indexes (SURVEY.md §8b / §8e) ------------------------------
 * One host process, one full replica of the index per GPU.  dann_group_search_batch cuts the batch into contiguous
 * slices (the first devices take the remainder), every device runs the whole hot path on its slice concurrently,
 * and each device's result copy lands directly in the caller's arrays at its slice's offset: rows come back in
 * query order, identical to a single-device dann_search_batch.  The graph is never sharded (every hop would cross
 * NVLink).  Separate PROCESSES per GPU (torchrun) gather with one NCCL collective instead: pgvectorscale_b200/group.py.
 * devices == NULL means devices 0..ndev-1.  Host pointers, borrowed for the call. */
typedef struct dann_group dann_group;
int dann_group_create(const dann_snapshot_desc *snap, int ndev, const int *devices, dann_group **out);
int dann_group_size(const dann_group *g);
dann_index *dann_group_replica(dann_group *g, int i); /* replica i (e.g. to attach vectors or read timings); NULL if out of range */
int dann_group_search_batch(dann_group *g, const float *queries, const int16_t *labels, const int32_t *label_offsets,
                            int B, int k, int search_list_size, int rescore, uint64_t *out_tid, float *out_dist,
                            uint32_t *out_count, dann_query_stats *out_stats);
/* dann_search_batch_mixed over the replicas: params is sliced with the queries, rows are [B][kmax] of the whole batch,
 * and the whole batch is checked before any replica runs. */
int dann_group_search_batch_mixed(dann_group *g, const float *queries, const int16_t *labels, const int32_t *label_off,
                                  const dann_query_params *params, int B, uint64_t *out_tid, float *out_dist,
                                  uint32_t *out_count, dann_query_stats *out_stats);
void dann_group_free(dann_group *g);

/* ---- a table split into shards: one independent index per shard, one merged top-k per query -------------------
 * Shard i is an ordinary diskann index over a disjoint set of the table's rows (its own graph, SBQ means and start
 * nodes), loaded on devices[i] (NULL: device i); several shards may share a device.  1..256 shards, which must agree
 * on dim, dim_index, distance_type and has_labels (else DANN_ERR_INVALID_ARG); they may differ in n (0 included),
 * bits, means and R.  A failed load frees the shards loaded so far.  Plain-layout shards are not supported.
 *
 * dann_shards_search_batch runs every shard's host-buffer batch on all B queries (one worker thread per distinct
 * device, that device's shards in shard order: each shard's rows, distance bits and counters are what a private
 * dann_search_batch on it gives), then merges them on the device of shard 0.  The merge is a k-way merge of the
 * shards' lists by their heads: k times, among the shards whose list of count_s[b] rows is not used up, take the head
 * with the smallest (f32::total_cmp key of its distance, shard index) and advance that shard.  A shard's rows
 * therefore appear as a prefix of its own list, in its own order; one shard gives exactly dann_search_batch's rows.
 * out_tid / out_dist / out_shard [B*k] (DANN_INVALID_TID, NaN and -1 past out_count[b]), out_count [B] =
 * min(k, sum of the shards' counts), out_stats [nshards*B] shard-major (query b of shard s at s*B + b); any may be
 * NULL except out_tid.  rescore == 0 is DANN_ERR_INVALID_ARG (rows would carry no distance to merge on); a shard's own
 * failure fails the call as "shard i: ...".  One call at a time per handle. */
typedef struct dann_shards dann_shards;
int dann_shards_create(const dann_snapshot_desc *const *shards, int nshards, const int *devices, dann_shards **out);
int dann_shards_count(const dann_shards *g);
dann_index *dann_shards_index(dann_shards *g, int i); /* borrowed: build a shard's graph / attach its rows in place; NULL if out of range */
int dann_shards_search_batch(dann_shards *g, const float *queries, const int16_t *labels, const int32_t *label_off,
                             int B, int k, int search_list_size, int rescore,
                             uint64_t *out_tid, float *out_dist, int32_t *out_shard, uint32_t *out_count,
                             dann_query_stats *out_stats);
void dann_shards_free(dann_shards *g);

/* ---- streaming scan of a sharded table: amrescan, then amgettuple one row at a time over every shard -------------
 * The scan operator of a sharded table, for a post-filter that is not a label key or a query without LIMIT: the batch's
 * merge rule applied to unbounded streams.  A sharded scan holds one dann_scan per shard.
 * - dann_shards_scan_rescan runs dann_scan_rescan on every shard with the same query, key, search_list_size and
 *   rescore, and validates its arguments the way dann_scan_rescan does.  rescore == 0 is DANN_ERR_INVALID_ARG (rows
 *   would carry no distance to merge on).  The shards of one device are prepared together and waited for with one
 *   synchronisation per device.
 * - dann_shards_scan_gettuple returns the head with the smallest (f32::total_cmp key of its distance, shard index)
 *   among the shards whose scan has not ended, then advances that shard.  The first call after a rescan steps every
 *   shard once to get its head: the shards of one device take that step together in one many-scan round (see
 *   dann_scan_gettuple_many), all devices at the same time.  Every later call steps exactly one shard, the one whose
 *   head the previous call returned, with an ordinary dann_scan_gettuple.  A shard whose step returns end of scan drops
 *   out; the merged scan ends (0) when every shard has.  node_id is local to its shard, *shard says which shard (any
 *   output pointer may be NULL).  Returns 1 (row), 0 (end of scan) or < 0.
 * - Consequences: after any call, shard s has taken exactly as many amgettuple steps as this rule implies, and
 *   dann_shards_scan_stats(out[s]) equals dann_scan_stats of a private scan of shard s after that many
 *   dann_scan_gettuple calls (out has nshards entries).  For any k that dann_shards_search_batch accepts, the first k
 *   rows of a sharded scan are exactly the batch's k rows: tid, distance bits and shard.
 * - A shard's own failure fails the call as "shard i: ...".  A gettuple that fails, or a rescan that fails after its
 *   arguments were checked, leaves the sharded scan unusable until the next successful rescan (DANN_ERR_STATE).
 * - Threads: a sharded scan is single-threaded, like a dann_scan.  The handle serialises dann_shards_search_batch calls
 *   only; every step of a scan or of a batch on a shard holds that shard's index lock (a first step or a rescan holds
 *   the locks of several shards, taken in ascending shard order), so different sharded scans of one handle and
 *   dann_shards_search_batch may be driven from different threads at once.  End every sharded scan before
 *   dann_shards_free. */
typedef struct dann_shards_scan dann_shards_scan;
int dann_shards_scan_begin(dann_shards *g, dann_shards_scan **out);
int dann_shards_scan_rescan(dann_shards_scan *sc, const float *query, const int16_t *labels, int nlabels,
                            int search_list_size, int rescore);
int dann_shards_scan_gettuple(dann_shards_scan *sc, uint32_t *block, uint16_t *offset, uint32_t *node_id, float *dist,
                              int32_t *shard);
int dann_shards_scan_stats(dann_shards_scan *sc, dann_query_stats *out /* [nshards] */);
void dann_shards_scan_end(dann_shards_scan *sc);

/* ---- reading an index RELATION FILE (SURVEY.md §8f row 2; pgvectorscale_b200/csrc/dann_pgreader.h) -------------------
 * Host-only, no GPU involved.  Replaces, for an external loader (the sidecar after a CHECKPOINT, an offline exporter):
 *   ReadablePage::read / get_type / get_item_unchecked   util/page.rs:254-290   dann_pg_relation_open / _info
 *   TsvPageOpaqueData::read_from_page / verify            util/page.rs:59-97     (every page is checked the same way)
 *   ChainItemReader::read                                 util/chain.rs:125-183  dann_pg_read_chain
 *   MetaPage::fetch: magic + version of MetaPageHeader    meta_page.rs:386-419   dann_pg_relation_info.meta_*
 *   ArchivedSbqNode accessors + SbqMeans::load            sbq/node.rs:236-330, sbq/mod.rs:88-122   dann_pg_extract_sbq
 *   ArchivedPlainNode accessors                           plain/node.rs:15-120   dann_pg_extract_plain
 *   TableSlot::from_index_heap_pointer + PgVector::from_datum  util/table_slot.rs:13-53, pg_vector.rs:125-199   dann_pg_heap_fetch_vectors
 * The MetaPage BODY is an rkyv archive of a repr(Rust) struct whose field order cannot be pinned offline: the caller
 * supplies its scalars (dann_pg_meta; a Rust host fills them from MetaPage's getters) and the reader cross-checks them
 * against the node items; the node items' own field order is inferred and verified, never assumed (see the header of
 * dann_pgreader.h).  Anything unexpected is DANN_ERR_FORMAT with a message, not a best effort.
 * Staleness: a snapshot is valid for exactly the `fingerprint` it was extracted under - a hash over every page's
 * (block, pd_lsn, pd_checksum, pd_lower, pd_upper); every WAL-logged change of a page moves its pd_lsn. */
typedef struct dann_pg_relation dann_pg_relation;
typedef struct {
    uint32_t nblocks;
    uint32_t pages_by_type[9]; /* PageType histogram, util/page.rs:28-38 (5 = SbqNode, 7 = SbqMeans, 8 = Meta) */
    uint32_t new_pages;        /* all-zero pages (PageIsNew) */
    uint32_t foreign_pages;    /* pages that fail the extension's page checks */
    uint32_t meta_magic;       /* 768756476 when block 0 is a Meta page whose header item parses, else 0 */
    uint32_t meta_version;     /* TSV_VERSION (3 in the reference at hand) */
    uint64_t node_items;       /* LP_NORMAL line pointers on SbqNode pages */
    uint64_t max_lsn;
    uint64_t fingerprint;
} dann_pg_relation_info;
/* path = the relation's first segment file (base/<db>/<relfilenode>); "<path>.1", ".2", ... are picked up */
int dann_pg_relation_open(const char *path, dann_pg_relation **out);
void dann_pg_relation_close(dann_pg_relation *rel);
int dann_pg_relation_stat(const dann_pg_relation *rel, dann_pg_relation_info *out);
/* Reassembles the chained item that starts at (block, offset): *len = its size; copies min(*len, cap) bytes into buf
 * (buf may be NULL with cap == 0 to ask for the size).  page_type < 0 = do not check the pages' PageType. */
int dann_pg_read_chain(const dann_pg_relation *rel, uint32_t block, uint16_t offset, int page_type, void *buf, size_t cap,
                       size_t *len);
typedef struct { /* MetaPage scalars (meta_page.rs:212-282) and the pointers it holds */
    uint32_t num_dimensions, num_dimensions_to_index, bq_bits, num_neighbors;
    int32_t distance_type; /* dann_distance */
    int32_t has_labels;
    uint32_t start_block;  /* start_nodes.default_node; DANN_INVALID_NODE (InvalidBlockNumber) = empty graph */
    uint16_t start_offset;
    uint32_t n_start_labels; /* start_nodes.labeled_nodes */
    const int16_t *start_labels;
    const uint32_t *start_label_block;
    const uint16_t *start_label_offset;
    uint32_t means_block;  /* quantizer_metadata; DANN_INVALID_NODE = the quantizer uses no means */
    uint16_t means_offset;
} dann_pg_meta;
typedef struct { /* owned by the library until dann_pg_snapshot_free */
    dann_snapshot_desc snap;   /* ready for dann_index_load (dann_index_load_plain with index_vectors below) except
                                  vectors == NULL: heap rows live in the TABLE; fetch heap_tid[i] in order and attach
                                  them with dann_index_set_vectors */
    const float *index_vectors; /* plain layout: [n * dim_index] the vector each node stores (plain/node.rs:17-22); else NULL */
    const uint64_t *index_tid; /* [n] (block<<16)|offset of node i inside the index relation, ascending: the
                                  IndexPointer -> dense node id map */
    uint64_t fingerprint;      /* of the relation as extracted */
    uint32_t layout[4];        /* which 8-byte cell of the archived root held: heap pointer, code (or f32 vector),
                                  neighbour vector, fourth vector */
    void *self;                /* the library's owner object (dann_pg_snapshot_free) */
} dann_pg_snapshot;
/* storage_layout = memory_optimized: SbqNode pages (sbq/node.rs:26-42) + the SbqMeans chain */
int dann_pg_extract_sbq(const dann_pg_relation *rel, const dann_pg_meta *meta, dann_pg_snapshot **out);
/* storage_layout = plain: Node pages (plain/node.rs:15-22); bq_bits, has_labels and the means pointer of `meta` are ignored */
int dann_pg_extract_plain(const dann_pg_relation *rel, const dann_pg_meta *meta, dann_pg_snapshot **out);
void dann_pg_snapshot_free(dann_pg_snapshot *s);

/* The heap rows of a snapshot: the vector column of the TABLE's relation file(s), read the way the rerank reads it
 * (sbq/storage.rs:304-328 -> util/table_slot.rs:13-53 -> pg_vector.rs:125-199: tuple by TID, detoast, f32[dim]).
 * Postgres' documented heap / varlena / TOAST formats and pgvector's value layout only (no rkyv).  `heap` and `toast`
 * are opened with dann_pg_relation_open on the table's and its TOAST table's files (toast may be NULL when every value
 * is inline).  The caller describes the attributes IN FRONT of the vector column (pg_attribute.attlen: > 0 fixed, -1
 * varlena; attalign 'c' 's' 'i' 'd').  Rows that are gone - heap_tid offset 0, dead or unused line pointer, NULL value -
 * come back as zeros and are counted in *n_missing; HOT redirects are followed; there is no visibility test (the
 * index names the tuples, the executor re-checks each row).  Compressed values are refused (the type is STORAGE external). */
typedef struct {
    uint32_t natts_before;  /* attributes in front of the vector column */
    const int16_t *attlen;  /* [natts_before] */
    const char *attalign;   /* [natts_before] */
    uint32_t dim;           /* vector(dim) */
    char vector_align;      /* 0 = 'i' (what CREATE TYPE vector declares) */
} dann_pg_heap_layout;
int dann_pg_heap_fetch_vectors(const dann_pg_relation *heap, const dann_pg_relation *toast, const dann_pg_heap_layout *layout,
                               const uint64_t *heap_tid, uint32_t n, float *out, uint32_t *n_missing);

/* How the last batch search of this index was planned (diagnostics for benchmarks and profiles). */
typedef struct {
    uint32_t kernel;         /* 1 = single-warp, 2 = two-warp (round 1), 3 = lean warp-per-query (dann_search3.cuh) */
    uint32_t slots_per_sm;   /* resident queries per SM */
    uint32_t grid;           /* CTAs (one per SM) */
    uint32_t heap_smem;      /* heap entries kept in shared memory per query */
    uint32_t visited_cap, cand_cap;
    uint32_t entry_bytes;    /* 4 or 8 */
    uint32_t bitmap;         /* 1 = bitmap inserted-set, 0 = hash set */
    uint64_t slot_hbm_bytes; /* per-slot HBM workspace (heap tail + inserted-set [+ side tables]) */
    uint32_t smem_per_slot;
    uint32_t retries;        /* workspace-growth reruns of the last call */
} dann_search_plan_info;
int dann_last_search_plan(dann_index *ix, dann_search_plan_info *out);

/* ---- query coalescing (SURVEY.md §8f row 4: multi-process serving, the in-process half) ----------------------
 * Postgres is process-per-connection with amcanparallel = false (mod.rs:63): one scan per backend at a time, while
 * the engine's throughput comes from batches.  A coalescer owns a dispatcher thread; any number of host threads (one
 * per connected backend in a sidecar that holds the HBM-resident index) call dann_coalescer_search with ONE query and
 * block; the search requests that arrive within max_wait_us of the first one (at most max_batch, whatever their k,
 * search_list_size, rescore and key) become one dann_search_batch_mixed call.  Each caller receives exactly the rows,
 * distances and counters a private dann_search_batch of its query returns.  nlabels < 0 = no scan key.  A request the
 * index would refuse (a value out of range, a rescore past the rerank window) is refused at once, for its caller alone.
 * The socket / shared-memory transport between backends and the sidecar is not part of this library. */
typedef struct dann_coalescer dann_coalescer;
int dann_coalescer_create(dann_index *ix, int max_batch, int max_wait_us, dann_coalescer **out);
int dann_coalescer_search(dann_coalescer *c, const float *query, const int16_t *labels, int nlabels, int k,
                          int search_list_size, int rescore, uint64_t *out_tid, float *out_dist,
                          uint32_t *out_count, dann_query_stats *out_stats);
/* One amgettuple of `sc`, a scan of the coalescer's index: blocks and returns exactly what dann_scan_gettuple would
 * (1 row, 0 end of scan, < 0 error).  The gettuple calls that arrive within max_wait_us of each other (at most
 * max_batch, any search_list_size / rescore / key) become one dann_scan_gettuple_many; search and gettuple calls never
 * share one.  A scan stays single-threaded: at most one call on it at a time; a second call on a scan that already
 * has one in the same dispatch is refused alone (DANN_ERR_INVALID_ARG) and the other callers are unaffected.  The
 * message of a failed call is that of its own scan. */
int dann_coalescer_gettuple(dann_coalescer *c, dann_scan *sc, uint32_t *block, uint16_t *offset, uint32_t *node_id,
                            float *dist);
/* batches / queries / largest_batch count the dispatches of both kinds: one dann_search_batch or one
 * dann_scan_gettuple_many is one batch, each search or gettuple request one query. */
int dann_coalescer_stats(dann_coalescer *c, uint64_t *batches, uint64_t *queries, uint64_t *largest_batch);
void dann_coalescer_destroy(dann_coalescer *c); /* drains what is queued, then stops; destroy before dann_index_free */

/* Number of this library's kernel launches since load (bench.py "gpu_launches"). */
uint64_t dann_kernel_launches(const dann_index *ix);

/* ---- device-timed leg of the last batch call (CUDA events on the launch stream) ---- */
typedef struct {
    float prepare_ms, search_ms, rerank_ms, resort_ms, total_ms;
    uint32_t retries; /* workspace-growth retries of the search kernel */
} dann_batch_timing;
int dann_last_batch_timing(dann_index *ix, dann_batch_timing *out);

#ifdef __cplusplus
}
#endif
#endif
