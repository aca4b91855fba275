// diskann_b200.cu — C ABI (include/diskann_b200.h) over the sm_90a kernels.
//
// There is NO CPU fallback anywhere in this file: without a CUDA device every entry
// point that computes returns DANN_ERR_NO_DEVICE.  The CPU oracle under oracle/ is
// test infrastructure and is never linked or called from here.
#include <cuda_runtime.h>

#include <algorithm>
#include <atomic>
#include <cmath>
#include <cstdarg>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <functional>
#include <mutex>
#include <new>
#include <string>
#include <vector>

#include "dann_device.cuh"
#include "dann_kernels.cuh"
#include "dann_search.cuh"
#include "dann_search2.cuh"
#include "dann_search3.cuh"
#include "dann_build.cuh"
#include "dann_shards.cuh"
#include "dann_plan.h"

#include <cub/device/device_radix_sort.cuh>

/* ------------------------------------------------------------------------------------ */
#define DANN_SMEM_SLACK 128u /* bytes behind every dynamic shared-memory window (see launch_prepare) */

/* The static __shared__ bytes of `kernel`: they come off the shared memory a launch of it may take.  The CPU emulator
 * (tests/simt) keeps static shared variables outside the simulated window, so there they take none. */
template <typename K>
static cudaError_t static_smem_bytes(K kernel, size_t *bytes) {
#ifdef DANN_SIMT_EMU
    (void)kernel;
    *bytes = 0;
    return cudaSuccess;
#else
    cudaFuncAttributes fa;
    const cudaError_t e = cudaFuncGetAttributes(&fa, kernel);
    *bytes = e == cudaSuccess ? fa.sharedSizeBytes : 0;
    return e;
#endif
}

/* A launch gets at most 48 KB of shared memory, the kernel's static __shared__ included, unless its kernel has opted in
 * to more.  (A 12256-d query row fills a 48 KB window exactly; with the few static bytes of the staging kernels, such as
 * the mbarrier of stage_query_row, it needs the opt-in.) */
template <typename K>
static cudaError_t allow_dynamic_smem(K kernel, size_t bytes) {
    size_t fixed = 0;
    const cudaError_t e = static_smem_bytes(kernel, &fixed);
    if (e != cudaSuccess || bytes + fixed <= 48 * 1024) return e;
    return cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)bytes);
}

/* dynamic shared memory of one dann_rerank_kernel CTA (its layout is in dann_kernels.cuh): the query row, one f32 per
 * streamed row rounded up to an even count, the rescore window of 8-byte entries, 16 bytes, DANN_SMEM_SLACK */
static size_t rerank_smem_bytes(uint32_t dim, uint32_t c_target, uint32_t rescore) {
    return (size_t)((dim + 3u) & ~3u) * 4 + (size_t)((c_target + 1u) & ~1u) * 4 + (size_t)rescore * 8 + 16 + DANN_SMEM_SLACK;
}

/* LabelSet::from(Vec): sort_unstable + dedup (labels/mod.rs:30-37) of [first, last), appended to `out` */
static void append_label_set(std::vector<int16_t> &out, const int16_t *first, const int16_t *last) {
    const size_t s0 = out.size();
    out.insert(out.end(), first, last);
    std::sort(out.begin() + s0, out.end());
    out.erase(std::unique(out.begin() + s0, out.end()), out.end());
}

static thread_local std::string g_err;

static int fail(int code, const char *fmt, ...) {
    char buf[512];
    va_list ap;
    va_start(ap, fmt);
    vsnprintf(buf, sizeof buf, fmt, ap);
    va_end(ap);
    try {
        g_err = buf;
    } catch (...) { /* out of memory while recording the message: the code still goes back */
    }
    return code;
}

extern "C" const char *dann_last_error(void) { return g_err.c_str(); }

/* Nothing may propagate out of an extern "C" entry point into the Rust / pgrx caller: every int-returning entry
 * point is a function-try-block that ends with this handler (std::bad_alloc from a host-side vector -> DANN_ERR_OOM). */
#define DANN_CATCH                                                                               \
    catch (const std::bad_alloc &) { return fail(DANN_ERR_OOM, "host allocation failed"); }      \
    catch (...) { return fail(DANN_ERR_STATE, "unexpected C++ exception in the host code"); }

extern "C" int dann_device_count(void) try {
    int n = 0;
    if (cudaGetDeviceCount(&n) != cudaSuccess) {
        cudaGetLastError();
        return 0;
    }
    return n;
} DANN_CATCH

#define CK(call)                                                                               \
    do {                                                                                       \
        cudaError_t e_ = (call);                                                               \
        if (e_ != cudaSuccess) {                                                               \
            if (ix) ix->poisoned = (e_ != cudaErrorMemoryAllocation);                          \
            cudaGetLastError();                                                                \
            return fail(e_ == cudaErrorMemoryAllocation ? DANN_ERR_OOM : DANN_ERR_CUDA,        \
                        "%s:%d %s: %s", __FILE__, __LINE__, #call, cudaGetErrorString(e_));    \
        }                                                                                      \
    } while (0)

/* The stream a call that takes DEVICE buffers from its caller runs on.  A caller that names a stream gets exactly that
 * (its buffers must be ready in that stream's order).  A caller that passes NULL gets the index's own
 * cudaStreamNonBlocking stream - which is ordered behind NOTHING the caller did, so the library first makes it wait for
 * everything already submitted to the legacy default stream: what a default-stream kernel or a plain cudaMemcpy of the
 * caller's would have been ordered after.  (Found in round 2: the fixture quantized rows that torch was still
 * generating on its default stream; until e0113f2 the index load's blocking cudaMemcpy calls had been the accidental
 * barrier.  Work a caller runs on other non-blocking streams needs that stream passed in, or a synchronisation.) */
struct dann_index;
static cudaError_t order_after_default_stream(dann_index *ix, cudaStream_t st);
struct DevBuf {
    void *p = nullptr;
    size_t cap = 0;
    bool fresh = false; /* set when reserve() had to allocate new (uninitialised) memory */
    cudaError_t reserve(size_t bytes) {
        fresh = false;
        if (bytes <= cap) return cudaSuccess;
        fresh = true;
        if (p) cudaFree(p);
        p = nullptr;
        cap = 0;
        size_t want = bytes + bytes / 4 + 256;
        cudaError_t e = cudaMalloc(&p, want);
        if (e == cudaSuccess) cap = want;
        return e;
    }
    /* reserve() that keeps bytes [from, to) of the old contents: copied device to device on `st`, which is then
     * synchronised, before the old allocation goes */
    cudaError_t grow_keep(size_t bytes, size_t from, size_t to, cudaStream_t st) {
        if (bytes <= cap) return cudaSuccess;
        void *q = nullptr;
        const size_t want = bytes + bytes / 4 + 256;
        cudaError_t e = cudaMalloc(&q, want);
        if (e != cudaSuccess) return e;
        if (to > from) e = cudaMemcpyAsync((char *)q + from, (const char *)p + from, to - from, cudaMemcpyDeviceToDevice, st);
        if (e == cudaSuccess) e = cudaStreamSynchronize(st);
        if (e != cudaSuccess) {
            cudaFree(q);
            return e;
        }
        if (p) cudaFree(p);
        p = q;
        cap = want;
        return cudaSuccess;
    }
    void release() {
        if (p) cudaFree(p);
        p = nullptr;
        cap = 0;
    }
    template <typename T>
    T *as() const { return reinterpret_cast<T *>(p); }
};

struct dann_index {
    int device = 0;
    IndexView v{};
    std::vector<void *> owned;
    uint64_t hbm_bytes = 0;
    cudaStream_t stream = nullptr;
    std::mutex mu;
    int sm_count = 0;
    size_t smem_optin = 0;
    size_t rerank_smem_max = 0; /* dynamic shared memory a dann_rerank_kernel launch may take: smem_optin less its static */
    std::atomic<uint64_t> launches{0}; /* bumped by entry points that do not take `mu` too */
    bool poisoned = false;
    /* per-warp-slot search workspace */
    DevBuf ws_hash, ws_cand, ws_heap, ws_bitmap, ws_ins;
    /* per-batch scratch */
    DevBuf sc_qfull, sc_qcodes, sc_stream, sc_stream_len, sc_stats, sc_qlist, sc_ctl, sc_node;
    /* staging for the host-buffer entry point */
    DevBuf st_queries, st_labels, st_label_off, st_tid, st_dist, st_count, st_stats;
    DevBuf sc_qparams; /* a mixed batch's QueryParam per query */
    dann_batch_timing timing{};
    dann_search_plan_info last_plan{};
    cudaEvent_t ev[5] = {nullptr, nullptr, nullptr, nullptr, nullptr};
    cudaEvent_t ev_order = nullptr; /* see DANN_DEVICE_INPUT_STREAM */
    uint32_t G = 1, Gshift = 0, NCH = 1;
    uint32_t lists_unique = 0;
    /* plain storage layout (experimental): nodes carry their f32 index vector, no SBQ codes */
    bool plain = false;
    const float *index_vectors = nullptr; /* [n][dim_index] in HBM */
    DevBuf sc_qindex;
    /* dann_scan_gettuple_many: one round's per-scan launch arguments and descriptors, then its ScanStepOut and ScanRow
     * arrays */
    DevBuf sc_many;
};


static cudaError_t order_after_default_stream(dann_index *ix, cudaStream_t st) {
    cudaError_t e = cudaEventRecord(ix->ev_order, cudaStreamLegacy);
    if (e == cudaSuccess) e = cudaStreamWaitEvent(st, ix->ev_order, 0);
    return e;
}
#define DANN_DEVICE_INPUT_STREAM(st, stream)                         \
    cudaStream_t st = (stream) ? (cudaStream_t)(stream) : ix->stream; \
    if (!(stream)) CK(order_after_default_stream(ix, st))

struct dann_scan {
    dann_index *ix = nullptr;
    std::vector<float> query;
    std::vector<int16_t> labels;
    int nlabels = -1;
    int L = 100, rescore = 50;
    bool active = false;
    /* suspended search state in HBM (see SavedScan / dann_search_common.cuh) */
    DevBuf d_qindex; /* plain layout: the prepared index slice */
    DevBuf d_step;   /* one step's ScanStepOut, then its ScanRow records */
    DevBuf d_snap;   /* a multi-row step's counters at each stream row (SearchArgs::row_counters) */
    DevBuf d_query, d_qfull, d_qcodes, d_labels, d_label_off, d_saved, d_heap_sm, d_vis, d_heap_tail, d_cnode, d_set,
        d_ins, d_stream, d_slen, d_stats, d_dist, d_win, d_winst, d_ctl;
    std::vector<unsigned char> h_step; /* the step's ScanStepOut and records, copied back */
    SearchPlan plan{};
    uint32_t grow = 1;
    bool deep = false;      /* plan is the deep plan (dann_make_deep_plan): the workspace grows in place */
    uint32_t regrows = 0;   /* replay regrows since the rescan */
    uint32_t growths = 0;   /* in-place growths since the rescan */
    uint32_t plan_rows = 0; /* streamed rows the workspace is planned for (times grow): rescore + 64, or a first fetch's */
    uint32_t streamed = 0;  /* rows taken off the approximate stream so far */
    uint32_t win_len = 0;   /* rows sitting in the rerank window */
    bool exhausted = false; /* next() returned None */
    dann_query_stats stats{};
};

/* ------------------------------------------------------------------------------------ */
template <typename Tp>
static cudaError_t upload(dann_index *ix, const Tp *host, size_t count, Tp **out) {
    void *p = nullptr;
    size_t bytes = std::max<size_t>(count * sizeof(Tp), 16);
    cudaError_t e = cudaMalloc(&p, bytes);
    if (e != cudaSuccess) return e;
    ix->owned.push_back(p);
    ix->hbm_bytes += bytes;
    /* Every copy of the index goes through ix->stream, the cudaStreamNonBlocking stream its kernels run on.  A plain
     * cudaMemcpy from pageable memory runs on the legacy stream and may return once the data is STAGED, before the DMA
     * has landed; a kernel on a non-blocking stream is not ordered behind it and can read the stale destination
     * (found in round 2: dann_pad_rows_kernel padded rows of whatever the buffer held before - garbage neighbour ids,
     * wrong rows or an illegal access, depending on the process's allocation history). */
    if (host && count) e = cudaMemcpyAsync(p, host, count * sizeof(Tp), cudaMemcpyHostToDevice, ix->stream);
    else e = cudaMemsetAsync(p, 0, bytes, ix->stream);
    if (e == cudaSuccess) e = cudaStreamSynchronize(ix->stream); /* the caller's buffer is borrowed for the call only */
    *out = reinterpret_cast<Tp *>(p);
    return e;
}

/* rows of width src_w -> device rows of width dst_w (padded with `fill`), in row chunks so
 * the temporary never exceeds ~256 MB */
template <typename Tp>
static cudaError_t upload_padded(dann_index *ix, const Tp *host, size_t n, uint32_t src_w, uint32_t dst_w,
                                 Tp fill, Tp **out) {
    void *p = nullptr;
    size_t bytes = std::max<size_t>(n * dst_w * sizeof(Tp), 16);
    cudaError_t e = cudaMalloc(&p, bytes);
    if (e != cudaSuccess) return e;
    ix->owned.push_back(p);
    ix->hbm_bytes += bytes;
    *out = reinterpret_cast<Tp *>(p);
    if (n == 0) return cudaSuccess;
    if (src_w == dst_w) {
        e = cudaMemcpyAsync(p, host, n * src_w * sizeof(Tp), cudaMemcpyHostToDevice, ix->stream);
        return e == cudaSuccess ? cudaStreamSynchronize(ix->stream) : e;
    }
    size_t chunk = std::max<size_t>(1, (256ull << 20) / (src_w * sizeof(Tp)));
    void *tmp = nullptr;
    e = cudaMalloc(&tmp, std::min(chunk, n) * src_w * sizeof(Tp));
    if (e != cudaSuccess) return e;
    for (size_t r0 = 0; r0 < n && e == cudaSuccess; r0 += chunk) {
        size_t rows = std::min(chunk, n - r0);
        e = cudaMemcpyAsync(tmp, host + r0 * src_w, rows * src_w * sizeof(Tp), cudaMemcpyHostToDevice, ix->stream);
        if (e != cudaSuccess) break; /* same stream as the kernel below: ordered */
        dann_pad_rows_kernel<Tp><<<1024, 256, 0, ix->stream>>>(reinterpret_cast<Tp *>(p) + r0 * dst_w,
                                                             reinterpret_cast<Tp *>(tmp), rows, src_w,
                                                             dst_w, fill);
        ix->launches++;
        e = cudaStreamSynchronize(ix->stream);
    }
    cudaFree(tmp);
    return e;
}

extern "C" void dann_index_free(dann_index *ix) {
    if (!ix) return;
    cudaSetDevice(ix->device);
    for (void *p : ix->owned) cudaFree(p);
    DevBuf *bufs[] = {&ix->ws_hash, &ix->ws_cand, &ix->ws_heap, &ix->ws_bitmap, &ix->ws_ins, &ix->sc_qfull, &ix->sc_qcodes,
                      &ix->sc_stream, &ix->sc_stream_len, &ix->sc_stats, &ix->sc_qlist, &ix->sc_ctl,
                      &ix->sc_node, &ix->sc_qindex, &ix->st_queries, &ix->st_labels, &ix->st_label_off, &ix->st_tid,
                      &ix->st_dist, &ix->st_count, &ix->st_stats, &ix->sc_many, &ix->sc_qparams};
    for (DevBuf *b : bufs) b->release();
    for (auto &e : ix->ev)
        if (e) cudaEventDestroy(e);
    if (ix->ev_order) cudaEventDestroy(ix->ev_order);
    if (ix->stream) cudaStreamDestroy(ix->stream);
    cudaGetLastError();
    delete ix;
}

/* Everything the kernels index with comes from the snapshot: reject ids and offsets that would send a
 * gather out of bounds here, on the host, before anything is copied (the reference gets the same guarantee
 * from Postgres' page/item bounds checks, util/page.rs:254-290). */
static int validate_snapshot(const dann_snapshot_desc *s, uint32_t *words_out, bool plain) {
    if (s->dim == 0 || s->dim_index == 0 || s->dim_index > s->dim || s->R == 0 || (!plain && s->bits == 0))
        return fail(DANN_ERR_INVALID_ARG, "bad snapshot geometry");
    uint32_t words = 0;
    if (!plain) {
        uint64_t nb = (uint64_t)s->dim_index * s->bits;
        words = (uint32_t)(nb % 64 == 0 ? nb / 64 : nb / 64 + 1); /* quantize.rs:38-46 */
        if (words != s->words) return fail(DANN_ERR_INVALID_ARG, "words=%u but dim_index*bits needs %u", s->words, words);
    }
    *words_out = words;
    if (s->distance_type < DANN_COSINE || s->distance_type > DANN_IP)
        return fail(DANN_ERR_INVALID_ARG, "unknown distance type %d", s->distance_type);
    if (s->n == DANN_INVALID_NODE) return fail(DANN_ERR_INVALID_ARG, "n collides with the invalid-node sentinel");
    if (plain) { /* build.rs:264-290: what CREATE INDEX rejects for storage_layout = plain */
        if (s->distance_type == DANN_IP) return fail(DANN_ERR_INVALID_ARG, "inner product distance is not supported with plain storage");
        if (s->has_labels) return fail(DANN_ERR_INVALID_ARG, "labeled filtering is not supported with plain storage");
        if (s->dim_index > 2000) return fail(DANN_ERR_INVALID_ARG, "too many dimensions to index with plain storage (max is 2000)");
        if (s->n && (!s->nbrs || !s->heap_tid)) return fail(DANN_ERR_INVALID_ARG, "snapshot arrays missing");
    } else {
        if (s->n && (!s->codes || !s->nbrs || !s->heap_tid || !s->mean))
            return fail(DANN_ERR_INVALID_ARG, "snapshot arrays missing");
        if (s->bits > 1 && s->n && !s->m2) return fail(DANN_ERR_INVALID_ARG, "m2 is required when bits > 1 (sbq/quantize.rs:73-101)");
    }
    if (s->has_labels && s->n && (!s->label_off || (s->label_off[s->n] && !s->labels)))
        return fail(DANN_ERR_INVALID_ARG, "has_labels set but label arrays missing");
    if (s->start_default != DANN_INVALID_NODE && s->start_default >= s->n)
        return fail(DANN_ERR_INVALID_ARG, "start_default out of range");
    if (s->n_start_labels && s->start_labels && s->start_label_nodes) {
        for (uint32_t i = 0; i < s->n_start_labels; i++) {
            if (s->start_label_nodes[i] >= s->n) return fail(DANN_ERR_INVALID_ARG, "start node of label %d out of range", (int)s->start_labels[i]);
            if (i && s->start_labels[i] <= s->start_labels[i - 1]) return fail(DANN_ERR_INVALID_ARG, "start_labels must be strictly ascending");
        }
    }
    for (size_t r = 0; r < s->n; r++) { /* a list ends at its first invalid id (sbq/node.rs:260-273) */
        const uint32_t *row = s->nbrs + r * s->R;
        for (uint32_t j = 0; j < s->R && row[j] != DANN_INVALID_NODE; j++)
            if (row[j] >= s->n) return fail(DANN_ERR_INVALID_ARG, "neighbour %u of node %zu is %u, outside the index (n=%u)", j, r, row[j], s->n);
    }
    if (s->has_labels && s->n) {
        if (s->label_off[0] != 0) return fail(DANN_ERR_INVALID_ARG, "label_off[0] must be 0");
        for (size_t r = 0; r < s->n; r++)
            if (s->label_off[r + 1] < s->label_off[r]) return fail(DANN_ERR_INVALID_ARG, "label_off is not monotone at node %zu", r);
    }
    return DANN_OK;
}

/* Cosine heap rows are normalised once, where they arrive: the rerank reads the heap vector through
 * PgVector::from_datum -> preprocess_cosine (sbq/storage.rs:304-328, pg_vector.rs:153-155), whose result only depends on
 * the row.  d holds the index's n rows of dim values. */
static int normalize_rows(dann_index *ix, float *d) {
    const IndexView &v = ix->v;
    if (v.distance_type != DANN_COSINE) return DANN_OK;
    int blocks = std::min<long long>((v.n + 255) / 256, (long long)ix->sm_count * 8);
    dann_normalize_rows_kernel<<<std::max(blocks, 1), 256, 0, ix->stream>>>(d, v.n, v.dim);
    ix->launches++;
    CK(cudaGetLastError());
    CK(cudaStreamSynchronize(ix->stream));
    return DANN_OK;
}

static int index_load_impl(const dann_snapshot_desc *s, const float *index_vectors, int device, dann_index **out) {
    dann_index *ix = nullptr;
    if (!s || !out) return fail(DANN_ERR_INVALID_ARG, "dann_index_load: NULL argument");
    *out = nullptr;
    const bool plain = index_vectors != nullptr;
    uint32_t words = 0;
    int vrc = validate_snapshot(s, &words, plain);
    if (vrc) return vrc;
    int ndev = dann_device_count();
    if (ndev <= 0) return fail(DANN_ERR_NO_DEVICE, "no CUDA device visible (this library has no CPU path)");
    if (device < 0 || device >= ndev) return fail(DANN_ERR_INVALID_ARG, "device %d out of range (%d devices)", device, ndev);

    ix = new (std::nothrow) dann_index();
    if (!ix) return fail(DANN_ERR_OOM, "host allocation failed");
    ix->device = device;
    struct Guard {
        dann_index *&p;
        bool keep = false;
        ~Guard() {
            if (!keep && p) {
                dann_index_free(p);
                p = nullptr;
            }
        }
    } guard{ix};

    CK(cudaSetDevice(device));
    cudaDeviceProp prop;
    CK(cudaGetDeviceProperties(&prop, device));
    ix->sm_count = prop.multiProcessorCount;
    ix->smem_optin = prop.sharedMemPerBlockOptin;
    size_t rerank_static = 0;
    CK(static_smem_bytes(dann_rerank_kernel, &rerank_static));
    ix->rerank_smem_max = ix->smem_optin > rerank_static ? ix->smem_optin - rerank_static : 0;
    CK(cudaStreamCreateWithFlags(&ix->stream, cudaStreamNonBlocking));
    for (auto &e : ix->ev) CK(cudaEventCreate(&e));
    CK(cudaEventCreateWithFlags(&ix->ev_order, cudaEventDisableTiming));

    IndexView &v = ix->v;
    v.n = s->n;
    v.dim = s->dim;
    v.dim_index = s->dim_index;
    v.bits = s->bits;
    v.words = words;
    v.cw = (words + 1u) & ~1u;
    v.R = s->R;
    v.Rp = (s->R + 7u) & ~7u;
    v.distance_type = s->distance_type;
    v.has_labels = s->has_labels ? 1 : 0;
    v.count = s->count;
    v.start_default = s->n ? s->start_default : DANN_INVALID_NODE;
    v.n_start_labels = s->start_labels && s->start_label_nodes ? s->n_start_labels : 0;
    if (!plain && pick_code_mapping(v.cw, &ix->G, &ix->Gshift, &ix->NCH) != 0)
        return fail(DANN_ERR_INVALID_ARG, "SBQ code of %u words is wider than this build supports", words);
    ix->plain = plain;

    float *mean = nullptr, *m2 = nullptr, *vectors = nullptr;
    uint64_t *codes = nullptr, *tids = nullptr;
    uint32_t *nbrs = nullptr, *sln = nullptr, *loff = nullptr;
    int16_t *sl = nullptr, *labs = nullptr;
    if (plain) { /* nodes carry their f32 index vector instead of an SBQ code (plain/node.rs:17-22) */
        float *iv = nullptr;
        CK(upload(ix, index_vectors, (size_t)s->n * s->dim_index, &iv));
        ix->index_vectors = iv;
    } else {
        CK(upload(ix, s->mean, (size_t)s->dim_index, &mean));
        CK(upload(ix, s->bits > 1 ? s->m2 : nullptr, (size_t)s->dim_index, &m2));
        CK(upload_padded<uint64_t>(ix, s->codes, s->n, words, v.cw, 0ull, &codes));
    }
    CK(upload_padded<uint32_t>(ix, s->nbrs, s->n, v.R, v.Rp, DANN_INVALID_NODE, &nbrs));
    CK(upload(ix, s->heap_tid, (size_t)s->n, &tids));
    if (s->vectors) CK(upload(ix, s->vectors, (size_t)s->n * s->dim, &vectors)); /* NULL: supplied later (dann_index_set_vectors) */
    CK(upload(ix, v.n_start_labels ? s->start_labels : nullptr, (size_t)v.n_start_labels, &sl));
    CK(upload(ix, v.n_start_labels ? s->start_label_nodes : nullptr, (size_t)v.n_start_labels, &sln));
    if (v.has_labels && s->n) {
        CK(upload(ix, s->label_off, (size_t)s->n + 1, &loff));
        CK(upload(ix, s->labels, (size_t)s->label_off[s->n], &labs));
    } else {
        v.has_labels = 0;
    }
    v.mean = mean;
    v.m2 = m2;
    v.codes = codes;
    v.nbrs = nbrs;
    v.tids = tids;
    v.vectors = vectors;
    v.start_labels = sl;
    v.start_label_nodes = sln;
    v.label_off = loff;
    v.labels = labs;
    if (s->n && s->R <= 64) {
        uint32_t *flag = nullptr;
        CK(cudaMalloc(&flag, 4));
        ix->owned.push_back(flag);
        CK(cudaMemsetAsync(flag, 0, 4, ix->stream));
        dann_check_unique_kernel<<<ix->sm_count * 8, 256, 0, ix->stream>>>(nbrs, s->n, v.R, v.Rp, flag);
        ix->launches++;
        uint32_t h = 1;
        CK(cudaMemcpyAsync(&h, flag, 4, cudaMemcpyDeviceToHost, ix->stream));
        CK(cudaStreamSynchronize(ix->stream));
        ix->lists_unique = h == 0;
    }
    if (s->n && vectors) {
        int rc = normalize_rows(ix, vectors);
        if (rc) return rc;
    }
    guard.keep = true;
    *out = ix;
    return DANN_OK;
}

extern "C" int dann_index_load(const dann_snapshot_desc *s, int device, dann_index **out) try {
    return index_load_impl(s, nullptr, device, out);
} DANN_CATCH

extern "C" int dann_index_load_plain(const dann_snapshot_desc *s, const float *index_vectors, int device, dann_index **out) try {
    if (!index_vectors && s && s->n) return fail(DANN_ERR_INVALID_ARG, "dann_index_load_plain: NULL index_vectors");
    /* Bit-exact against the oracle under the CPU SIMT emulator, not yet run on hardware: opt-in until it has been. */
    static const float dummy = 0.0f;
    return index_load_impl(s, index_vectors ? index_vectors : &dummy, device, out);
} DANN_CATCH

extern "C" uint64_t dann_index_hbm_bytes(const dann_index *ix) { return ix ? ix->hbm_bytes : 0; }
extern "C" uint64_t dann_kernel_launches(const dann_index *ix) { return ix ? ix->launches.load() : 0; }
extern "C" uint32_t dann_code_stride(const dann_index *ix) { return ix ? ix->v.cw : 0; }

extern "C" int dann_last_search_plan(dann_index *ix, dann_search_plan_info *out) try {
    if (!ix || !out) return fail(DANN_ERR_INVALID_ARG, "dann_last_search_plan: NULL argument");
    std::lock_guard<std::mutex> lk(ix->mu);
    *out = ix->last_plan;
    return DANN_OK;
} DANN_CATCH

extern "C" int dann_last_batch_timing(dann_index *ix, dann_batch_timing *out) try {
    if (!ix || !out) return fail(DANN_ERR_INVALID_ARG, "NULL argument");
    *out = ix->timing;
    return DANN_OK;
} DANN_CATCH

/* ------------------------------------------------------------------------------------ */
static int check_live(dann_index *ix) {
    if (!ix) return fail(DANN_ERR_INVALID_ARG, "NULL index");
    if (ix->poisoned) return fail(DANN_ERR_CUDA, "index handle is poisoned by an earlier CUDA error");
    cudaError_t e = cudaSetDevice(ix->device);
    if (e != cudaSuccess) {
        cudaGetLastError();
        return fail(DANN_ERR_CUDA, "cudaSetDevice(%d): %s", ix->device, cudaGetErrorString(e));
    }
    return DANN_OK;
}

/* amrescan's vector preparation of B queries: q_full [B][dim], plus the SBQ codes q_codes [B][cw], or for a plain index
 * the normalised index copy q_index [B][dim_index] */
static int launch_prepare(dann_index *ix, const float *d_queries, int B, float *d_q_full, uint64_t *d_q_codes,
                          float *d_q_index, cudaStream_t st) {
    const IndexView &v = ix->v;
    if (ix->plain) {
        dann_prepare_plain_kernel<<<B, 128, 0, st>>>(v.dim, v.dim_index, v.distance_type == DANN_COSINE, d_queries,
                                                    d_q_full, d_q_index);
    } else {
        /* DANN_SMEM_SLACK: ptxas may turn neighbouring shared-memory loads of a loop into one 16-byte load issued BEFORE
         * the loop's bounds test (compute-sanitizer caught dann_prepare_kernel reading 16 bytes past a 28-byte window; on
         * hardware that is a fault whenever it crosses the CTA's allocation), so no dynamic window ends where its data ends */
        size_t smem = (size_t)((v.dim_index + 3u) & ~3u) * sizeof(float) + DANN_SMEM_SLACK;
        CK(allow_dynamic_smem(dann_prepare_kernel, smem));
        dann_prepare_kernel<<<B, 128, smem, st>>>(v, d_queries, B, d_q_full, d_q_codes);
    }
    ix->launches++;
    CK(cudaGetLastError());
    return DANN_OK;
}

extern "C" int dann_prepare_queries(dann_index *ix, const float *d_queries, int B, float *d_q_full,
                                    uint64_t *d_q_codes, void *stream) try {
    int rc = check_live(ix);
    if (rc) return rc;
    if (!d_queries || !d_q_codes || B <= 0) return fail(DANN_ERR_INVALID_ARG, "dann_prepare_queries: bad argument");
    if (ix->plain) return fail(DANN_ERR_STATE, "dann_prepare_queries: a plain-storage index has no quantizer");
    std::lock_guard<std::mutex> lk(ix->mu);
    DANN_DEVICE_INPUT_STREAM(st, stream);
    rc = launch_prepare(ix, d_queries, B, d_q_full, d_q_codes, nullptr, st);
    if (rc) return rc;
    CK(cudaStreamSynchronize(st));
    return DANN_OK;
} DANN_CATCH

template <int NCH, int UNR>
static void launch_sbq_u(dann_index *ix, const uint64_t *q, const uint32_t *pq, const uint32_t *pn, size_t np,
                         uint32_t *out, cudaStream_t st) {
    const int threads = (int)env_u32("DANN_SBQ_THREADS", 256);
    /* one full wave of resident CTAs (grid-stride loop inside): no partial last wave */
    int occ = 0;
    if (cudaOccupancyMaxActiveBlocksPerMultiprocessor(&occ, dann_sbq_distance_kernel<NCH, UNR>, threads, 0) != cudaSuccess || occ < 1)
        occ = 4;
    int blocks = ix->sm_count * (int)env_u32("DANN_SBQ_BLOCKS_PER_SM", (uint32_t)occ);
    dann_sbq_distance_kernel<NCH, UNR><<<blocks, threads, 0, st>>>(ix->v.codes, ix->v.cw, q, pq, pn, np, out, ix->G,
                                                                  ix->Gshift);
}

template <int NCH>
static void launch_sbq(dann_index *ix, const uint64_t *q, const uint32_t *pq, const uint32_t *pn, size_t np,
                       uint32_t *out, cudaStream_t st) {
    /* pairs in flight per lane group.  More pairs per thread cost registers (192-B codes: UNR=1/2/4/8 -> 32/38/77/128)
     * and so resident warps.  Measured on an H100 SXM (700 W, tools/bench_sbq.py, 1M rows of 192-B codes,
     * profiles/h100_tuning_ab.json): UNR=4 2.49 TB/s, UNR=2 2.46, UNR=1 2.28 - the 128-register UNR=8 is not the default. */
    constexpr int UNR = NCH <= 3 ? 4 : NCH <= 4 ? 2 : 1;
    if (NCH <= 3) {
        switch (env_u32("DANN_SBQ_UNR", UNR)) {
            case 1: return launch_sbq_u<NCH, 1>(ix, q, pq, pn, np, out, st);
            case 2: return launch_sbq_u<NCH, 2>(ix, q, pq, pn, np, out, st);
            case 4: return launch_sbq_u<NCH, 4>(ix, q, pq, pn, np, out, st);
            case 8: return launch_sbq_u<NCH, 8>(ix, q, pq, pn, np, out, st);
            default: break;
        }
    }
    launch_sbq_u<NCH, UNR>(ix, q, pq, pn, np, out, st);
}

extern "C" int dann_sbq_distance(dann_index *ix, const uint64_t *d_qcodes, const uint32_t *d_pair_q,
                                 const uint32_t *d_pair_node, size_t npairs, uint32_t *d_out, void *stream) try {
    int rc = check_live(ix);
    if (rc) return rc;
    if (!d_qcodes || !d_pair_q || !d_pair_node || !d_out) return fail(DANN_ERR_INVALID_ARG, "dann_sbq_distance: NULL buffer");
    if (ix->plain) return fail(DANN_ERR_STATE, "dann_sbq_distance: a plain-storage index has no SBQ codes");
    if (npairs == 0) return DANN_OK;
    DANN_DEVICE_INPUT_STREAM(st, stream);
    switch (ix->NCH) {
        case 1: launch_sbq<1>(ix, d_qcodes, d_pair_q, d_pair_node, npairs, d_out, st); break;
        case 2: launch_sbq<2>(ix, d_qcodes, d_pair_q, d_pair_node, npairs, d_out, st); break;
        case 3: launch_sbq<3>(ix, d_qcodes, d_pair_q, d_pair_node, npairs, d_out, st); break;
        case 4: launch_sbq<4>(ix, d_qcodes, d_pair_q, d_pair_node, npairs, d_out, st); break;
        default: launch_sbq<8>(ix, d_qcodes, d_pair_q, d_pair_node, npairs, d_out, st); break;
    }
    ix->launches++;
    CK(cudaGetLastError());
    if (!stream) CK(cudaStreamSynchronize(st));
    return DANN_OK;
} DANN_CATCH

extern "C" int dann_full_distance(dann_index *ix, const float *d_q_full, const uint32_t *d_nodes, int B, int m,
                                  float *d_out, void *stream) try {
    int rc = check_live(ix);
    if (rc) return rc;
    if (!d_q_full || !d_nodes || !d_out || B <= 0 || m <= 0) return fail(DANN_ERR_INVALID_ARG, "dann_full_distance: bad argument");
    DANN_DEVICE_INPUT_STREAM(st, stream);
    size_t smem = (size_t)((ix->v.dim + 3u) & ~3u) * sizeof(float) + DANN_SMEM_SLACK;
    CK(allow_dynamic_smem(dann_full_distance_kernel, smem));
    dann_full_distance_kernel<<<B, 128, smem, st>>>(ix->v, d_q_full, d_nodes, m, d_out);
    ix->launches++;
    CK(cudaGetLastError());
    if (!stream) CK(cudaStreamSynchronize(st));
    return DANN_OK;
} DANN_CATCH

/* ------------------------------------------------------------------------------------ */
/* search kernel dispatch                                                                */
typedef void (*search_fn)(const SearchArgs);
template <typename T, int DEEP = 0>
static search_fn pick_search(uint32_t nch) {
    switch (nch) {
        case 1: return dann_search_kernel<T, 1, 0, DEEP>;
        case 2: return dann_search_kernel<T, 2, 0, DEEP>;
        case 3: return dann_search_kernel<T, 3, 0, DEEP>;
        case 4: return dann_search_kernel<T, 4, 0, DEEP>;
        default: return dann_search_kernel<T, 8, 0, DEEP>;
    }
}
template <typename T>
static search_fn pick_search2(uint32_t nch) {
    switch (nch) {
        case 1: return dann_search2_kernel<T, 1>;
        case 2: return dann_search2_kernel<T, 2>;
        case 3: return dann_search2_kernel<T, 3>;
        case 4: return dann_search2_kernel<T, 4>;
        default: return dann_search2_kernel<T, 8>;
    }
}
static search_fn pick_kernel(bool pairs, int entry, uint32_t nch, bool plain = false, bool deep = false) {
    if (deep) return plain ? dann_search_kernel<Ent64, 1, 1, 1> : pick_search<Ent64, 1>(nch); /* the deep plan: Ent64 */
    if (plain) return dann_search_kernel<Ent64, 1, 1>;
    if (pairs) return entry == 0 ? pick_search2<Ent32x21>(nch) : entry == 1 ? pick_search2<Ent32x16>(nch) : pick_search2<Ent64>(nch);
    return entry == 0 ? pick_search<Ent32x21>(nch) : entry == 1 ? pick_search<Ent32x16>(nch) : pick_search<Ent64>(nch);
}

/* dann_scan_search_many_kernel: the instantiations pick_kernel(false, ...) offers the streaming scan */
typedef void (*scan_many_fn)(const SearchArgs *, uint32_t);
template <typename T, int DEEP = 0>
static scan_many_fn pick_scan_many_t(uint32_t nch) {
    switch (nch) {
        case 1: return dann_scan_search_many_kernel<T, 1, 0, DEEP>;
        case 2: return dann_scan_search_many_kernel<T, 2, 0, DEEP>;
        case 3: return dann_scan_search_many_kernel<T, 3, 0, DEEP>;
        case 4: return dann_scan_search_many_kernel<T, 4, 0, DEEP>;
        default: return dann_scan_search_many_kernel<T, 8, 0, DEEP>;
    }
}
static scan_many_fn pick_scan_many(int entry, uint32_t nch, bool plain, bool deep) {
    if (deep) return plain ? dann_scan_search_many_kernel<Ent64, 1, 1, 1> : pick_scan_many_t<Ent64, 1>(nch);
    if (plain) return dann_scan_search_many_kernel<Ent64, 1, 1>;
    return entry == 0 ? pick_scan_many_t<Ent32x21>(nch) : entry == 1 ? pick_scan_many_t<Ent32x16>(nch) : pick_scan_many_t<Ent64>(nch);
}

template <typename T, int MAXW>
static search_fn pick_lean_t(uint32_t nch) {
    switch (nch) {
        case 1: return dann_search3_kernel<T, 1, MAXW>;
        case 2: return dann_search3_kernel<T, 2, MAXW>;
        default: return dann_search3_kernel<T, 3, MAXW>; /* the plan offers the lean kernel up to 96 16-byte chunks */
    }
}
/* dann_search3.cuh: 4-byte (key11 | node-or-hash-slot21) or 8-byte (key32 | node32) entries; 32 or 16 resident warps */
static search_fn pick_lean(int entry, uint32_t nch, int maxw) {
    if (maxw <= 16) return entry == 0 ? pick_lean_t<Ent32x21, 16>(nch) : pick_lean_t<Ent64, 16>(nch);
    return entry == 0 ? pick_lean_t<Ent32x21, 32>(nch) : pick_lean_t<Ent64, 32>(nch);
}

static int make_plan(dann_index *ix, uint32_t nq, uint32_t L, uint32_t c_target, uint32_t grow, bool keyed,
                     SearchPlan *p, bool force_single = false, bool allow_lean = false) {
    PlanInputs in;
    in.n = ix->v.n;
    in.R = ix->v.R;
    in.words = ix->v.words;
    in.smem_optin = ix->smem_optin;
    in.sm_count = ix->sm_count;
    in.plain_dim = ix->plain ? ix->v.dim_index : 0;
    in.allow_lean = allow_lean;
    in.ws_budget = 0;
    char err[256];
    int rc = dann_make_plan(in, nq, L, c_target, grow, keyed, p, force_single, err, sizeof err);
    if (rc) return fail(rc, "%s", err);
    if (p->lean) {
        /* the lean plan takes as many query slots as the batch fills; only when that needs more HBM than the
         * workspaces already hold is free memory looked at (cudaMemGetInfo costs about half a millisecond - more than
         * a small batch's other host work) and the slot count cut to what fits: free HBM now plus what the
         * workspaces hold, less a reserve for the batch scratch that is sized after the plan */
        const uint64_t slots = (uint64_t)p->grid * p->W;
        const uint64_t need_heap = slots * p->cand_cap * (uint64_t)p->esize;
        const uint64_t need_set = slots * (p->bitmap_words ? (uint64_t)p->bitmap_words * 4u : (uint64_t)p->hash_cap * 4u);
        const uint64_t held_set = p->bitmap_words ? ix->ws_bitmap.cap : ix->ws_hash.cap;
        if (need_heap > ix->ws_heap.cap || need_set > held_set) {
            size_t fr = 0, tot = 0;
            if (cudaMemGetInfo(&fr, &tot) == cudaSuccess) {
                const uint64_t held = (uint64_t)ix->ws_hash.cap + ix->ws_heap.cap + ix->ws_bitmap.cap + ix->ws_cand.cap + ix->ws_ins.cap;
                const uint64_t reserve = 768ull << 20;
                const uint64_t avail = (uint64_t)fr + held;
                in.ws_budget = avail > reserve ? avail - reserve : 1;
                /* DevBuf::reserve over-allocates by a quarter: plan against 4/5 of the budget */
                in.ws_budget = in.ws_budget / 5 * 4;
                rc = dann_make_plan(in, nq, L, c_target, grow, keyed, p, force_single, err, sizeof err);
                if (rc) return fail(rc, "%s", err);
            }
        }
    }
    return DANN_OK;
}

/* The beam search over B prepared query codes, with the invisible workspace-growth reruns.
 * vis_out != NULL selects build mode (dann_build.cuh). */
static int run_search(dann_index *ix, const uint64_t *d_q_codes, const int16_t *d_labels, const int32_t *d_label_off,
                      int B, uint32_t L, uint32_t c_target, dann_query_stats *d_stats, uint64_t *vis_out,
                      uint32_t *vis_out_len, uint32_t vis_out_cap, cudaStream_t st, const float *d_q_index = nullptr,
                      const QueryParam *d_qp = nullptr) {
    const IndexView &v = ix->v;
    uint32_t *d_ctl = ix->sc_ctl.as<uint32_t>(); /* [0]=work counter, [1]=overflow bits */
    int rc;
    std::vector<uint32_t> qlist;
    std::vector<dann_query_stats> hstats;
    uint32_t grow = 1;
    uint32_t nq = (uint32_t)B;
    for (int attempt = 0;; attempt++) {
        SearchPlan p;
        rc = make_plan(ix, nq, L, c_target, grow, d_label_off != nullptr, &p, false, vis_out == nullptr);
        if (rc) return rc;
        if (vis_out && !p.pairs) /* dann_search.cuh has no build mode: its launch would leave vis_out_len unwritten */
            return fail(DANN_ERR_STATE, "build mode needs the two-warp search kernel, which alone hands over its visited list: "
                                        "unset DANN_SEARCH_KERNEL=1");
        const size_t slots = (size_t)p.grid * p.W;
        if (!p.bitmap_words) CK(ix->ws_hash.reserve(slots * p.hash_cap * sizeof(uint32_t)));
        if (!p.lean) CK(ix->ws_cand.reserve(slots * p.cand_cap * sizeof(uint32_t))); /* lean entries carry their node */
        CK(ix->ws_heap.reserve(slots * p.cand_cap * (size_t)p.esize));
        if (p.bitmap_words) {
            CK(ix->ws_bitmap.reserve(slots * (size_t)p.bitmap_words * 4));
            if (ix->ws_bitmap.fresh) CK(cudaMemsetAsync(ix->ws_bitmap.p, 0, ix->ws_bitmap.cap, st));
            if (!p.lean) CK(ix->ws_ins.reserve(slots * (size_t)p.ins_cap * 4));
        }
        CK(cudaMemsetAsync(d_ctl, 0, 8, st));
        SearchArgs a = search_args_for_plan(v, ix->G, ix->Gshift, ix->lists_unique, p);
        a.q_codes = d_q_codes;
        a.q_labels = d_labels;
        a.q_label_off = d_label_off;
        a.qlist = attempt == 0 ? nullptr : ix->sc_qlist.as<uint32_t>();
        a.nq = nq;
        a.L = L;
        a.c_target = c_target;
        a.stream = ix->sc_stream.as<uint32_t>();
        a.stream_len = ix->sc_stream_len.as<uint32_t>();
        a.stats = d_stats;
        a.overflow = d_ctl + 1;
        a.counter = d_ctl;
        a.hash = ix->ws_hash.as<uint32_t>();
        a.bitmap = ix->ws_bitmap.as<uint32_t>();
        a.ins_list = ix->ws_ins.as<uint32_t>();
        a.cand_node = ix->ws_cand.as<uint32_t>();
        a.heap_tail = ix->ws_heap.p;
        a.build_mode = vis_out ? 1u : 0u;
        a.vis_out = vis_out;
        a.vis_out_len = vis_out_len;
        a.vis_out_cap = vis_out_cap;
        a.hv_flags = env_u32("DANN_HV_FLAGS", 4095);
        a.plain_vectors = ix->index_vectors;
        a.q_index = d_q_index;
        a.plain_dim = ix->plain ? v.dim_index : 0;
        a.qp = d_qp;
        if (attempt == 0) {
            dann_search_plan_info &pi = ix->last_plan;
            pi.kernel = p.lean ? 3u : p.pairs ? 2u : 1u;
            pi.slots_per_sm = p.W;
            pi.grid = p.grid;
            pi.heap_smem = p.hs;
            pi.visited_cap = p.vcap;
            pi.cand_cap = p.cand_cap;
            pi.entry_bytes = p.esize;
            pi.bitmap = p.bitmap_words ? 1u : 0u;
            pi.slot_hbm_bytes = (uint64_t)p.cand_cap * p.esize + (p.bitmap_words ? (uint64_t)p.bitmap_words * 4u : (uint64_t)p.hash_cap * 4u) +
                                (p.lean ? 0u : (uint64_t)p.cand_cap * 4u + (p.bitmap_words ? (uint64_t)p.ins_cap * 4u : 0u));
            pi.smem_per_slot = p.per_warp;
            pi.retries = 0;
        } else {
            ix->last_plan.retries = (uint32_t)attempt;
        }
        search_fn fn = p.lean ? pick_lean(p.entry, ix->NCH, p.maxw) : pick_kernel(p.pairs, p.entry, ix->NCH, ix->plain);
        size_t smem = (size_t)p.per_warp * p.W + DANN_SMEM_SLACK;
        CK(cudaFuncSetAttribute(fn, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
        fn<<<p.grid, p.W * (p.pairs ? 64 : 32), smem, st>>>(a);
        ix->launches++;
        CK(cudaGetLastError());
        uint32_t ctl[2] = {0, 0};
        {
            cudaError_t e_ = cudaMemcpyAsync(ctl, d_ctl, 8, cudaMemcpyDeviceToHost, st);
            if (e_ == cudaSuccess) e_ = cudaStreamSynchronize(st);
            if (e_ != cudaSuccess) { /* a faulting search kernel: say which one and how it was planned */
                ix->poisoned = true;
                return fail(DANN_ERR_CUDA, "search kernel %s failed: %s [attempt %d nq %u L %u c_target %u | n %u R %u Rp %u cw %u "
                            "keyed %d | grid %u W %u smem %zu per_warp %u hs %u vcap %u cand_cap %u hash_cap %u bitmap_words %u ins_cap %u entry %d]",
                            p.lean ? "lean" : p.pairs ? "two-warp" : "single-warp", cudaGetErrorString(e_), attempt, nq, L, c_target,
                            v.n, v.R, v.Rp, v.cw, d_label_off != nullptr, p.grid, p.W, smem, p.per_warp, p.hs, p.vcap, p.cand_cap,
                            p.hash_cap, p.bitmap_words, p.ins_cap, p.entry);
            }
        }
        if (ctl[1] == 0) break;
        if (getenv("DANN_DEBUG_STATUS")) fprintf(stderr, "[diskann_b200] search overflow bits 0x%x (attempt %d, plan need=%u vcap=%u)\n", ctl[1], attempt, p.need, p.vcap);
        if (ctl[1] & DANN_ST_INTERNAL) return fail(DANN_ERR_STATE, "internal error: next-node prediction mismatch in the two-warp search kernel");
        /* some queries outgrew their workspace: rerun exactly those with a larger one */
        if (attempt >= 8) return fail(DANN_ERR_CAPACITY, "search workspace still too small after %d growth steps", attempt);
        hstats.resize(B);
        CK(cudaMemcpy(hstats.data(), d_stats, (size_t)B * sizeof(dann_query_stats), cudaMemcpyDeviceToHost));
        qlist.clear();
        for (int b = 0; b < B; b++)
            if (hstats[b].status) qlist.push_back((uint32_t)b);
        nq = (uint32_t)qlist.size();
        CK(cudaMemcpyAsync(ix->sc_qlist.p, qlist.data(), nq * sizeof(uint32_t), cudaMemcpyHostToDevice, st)); /* ordered before the rerun on st */
        CK(cudaStreamSynchronize(st));
        grow *= 2;
        ix->timing.retries++;
    }
    return DANN_OK;
}

/* What a batch asks of its queries, checked and derived before anything runs.  A uniform batch (one k, L and rescore;
 * keyed when label_off is given) leaves qp empty.  A mixed batch (dann_search_batch_mixed) holds each query's own values
 * in qp, and k / L / rescore / c_target are the batch maxima: k is the row stride of the outputs, c_target that of the
 * stream.  rerank_smem is the largest single query's rerank window. */
struct BatchParams {
    int k = 0, L = 0, rescore = 0;
    uint32_t c_target = 0;
    size_t rerank_smem = 0;
    bool keyed = false; /* label_off goes to the kernels */
    std::vector<QueryParam> qp;
};

/* rows needed from the approximate stream: scan.rs:255-305 */
static uint32_t stream_rows(int k, int rescore) { return rescore == 0 ? (uint32_t)k : (uint32_t)rescore + (uint32_t)k - 1u; }

/* One query's k, search_list_size and rescore (`who` names it in the messages): the GUC ranges, the plain layout's rules
 * and the rerank kernel's shared memory.  *rescore becomes what the query reranks; *smem its rerank window. */
static int check_query(const dann_index *ix, const char *who, int k, int L, int *rescore, bool keyed, size_t *smem) {
    const IndexView &v = ix->v;
    if (k <= 0) return fail(DANN_ERR_INVALID_ARG, "%sk %d must be positive", who, k);
    if (L < 1 || L > 10000) return fail(DANN_ERR_INVALID_ARG, "%ssearch_list_size %d outside 1..10000 (guc.rs:11-26)", who, L);
    if (*rescore < 0 || *rescore > 1000) return fail(DANN_ERR_INVALID_ARG, "%srescore %d outside 0..1000 (guc.rs:28-43)", who, *rescore);
    if (ix->plain) {
        if (keyed) return fail(DANN_ERR_INVALID_ARG, "%splain storage does not support label filters (plain/storage.rs:260)", who);
        /* scan.rs:392-403: a plain index only resorts when it holds fewer dimensions than the heap column */
        if (v.dim == v.dim_index) *rescore = 0;
    }
    if (*rescore > 0 && v.n && !v.vectors)
        return fail(DANN_ERR_STATE, "%sindex has no heap vectors yet (dann_index_set_vectors): rescore must be 0", who);
    /* the rerank kernel keeps the query row, one f32 per streamed row and the window in shared memory; a request past
     * the limit is refused here, because a failed launch would poison the handle */
    *smem = rerank_smem_bytes(v.dim, stream_rows(k, *rescore), (uint32_t)*rescore);
    if (*smem > ix->rerank_smem_max)
        return fail(DANN_ERR_INVALID_ARG, "%sk=%d rows with rescore=%d need %zu B of shared memory per scan (limit %zu): "
                    "fetch fewer rows per scan", who, k, *rescore, *smem, ix->rerank_smem_max);
    return DANN_OK;
}

static int uniform_params(const dann_index *ix, int B, int k, int L, int rescore, bool keyed, BatchParams *bp) {
    if (B <= 0 || k <= 0) return fail(DANN_ERR_INVALID_ARG, "B and k must be positive");
    int rc = check_query(ix, "", k, L, &rescore, keyed, &bp->rerank_smem);
    if (rc) return rc;
    bp->k = k;
    bp->L = L;
    bp->rescore = rescore;
    bp->c_target = stream_rows(k, rescore);
    bp->keyed = keyed;
    bp->qp.clear();
    return DANN_OK;
}

/* The checks of dann_search_batch_mixed, on host copies of params [B] and label_off [B+1] (NULL: no query keyed).
 * kstride > 0 asks for that output row stride (a group slice writes into the whole batch's rows), else it is the largest
 * k.  Nothing is touched on the device. */
static int mixed_params(const dann_index *ix, int B, const dann_query_params *params, const int16_t *labels,
                        const int32_t *label_off, int kstride, BatchParams *bp) {
    if (B <= 0) return fail(DANN_ERR_INVALID_ARG, "B %d must be positive", B);
    if (!params) return fail(DANN_ERR_INVALID_ARG, "params is NULL");
    if (label_off && label_off[0] < 0) return fail(DANN_ERR_INVALID_ARG, "label_off[0] is negative");
    bp->qp.resize((size_t)B);
    bp->k = bp->L = bp->rescore = 0;
    bp->c_target = 0;
    bp->rerank_smem = 0;
    bp->keyed = false;
    for (int b = 0; b < B; b++) {
        const dann_query_params &p = params[b];
        char who[32];
        snprintf(who, sizeof who, "query %d: ", b);
        if (p.keyed != 0 && p.keyed != 1) return fail(DANN_ERR_INVALID_ARG, "%skeyed %d is not 0 or 1", who, p.keyed);
        if (p.keyed && !label_off) return fail(DANN_ERR_INVALID_ARG, "%skeyed, but label_off is NULL", who);
        if (label_off) {
            const int32_t o0 = label_off[b], o1 = label_off[b + 1];
            if (o1 < o0) return fail(DANN_ERR_INVALID_ARG, "%slabel_off is not monotone", who);
            if (!p.keyed && o1 > o0) return fail(DANN_ERR_INVALID_ARG, "%sunkeyed (keyed = 0), but its label_off range is not empty", who);
            if (o1 > o0 && !labels) return fail(DANN_ERR_INVALID_ARG, "%slabels is NULL but its key is not empty", who);
        }
        int rescore = p.rescore;
        size_t smem = 0;
        int rc = check_query(ix, who, p.k, p.search_list_size, &rescore, p.keyed != 0, &smem);
        if (rc) return rc;
        QueryParam &q = bp->qp[(size_t)b];
        q.L = (uint32_t)p.search_list_size;
        q.c_target = stream_rows(p.k, rescore);
        q.keyed = (uint32_t)p.keyed;
        q.k = (uint32_t)p.k;
        q.rescore = (uint32_t)rescore;
        bp->k = std::max(bp->k, p.k);
        bp->L = std::max(bp->L, p.search_list_size);
        bp->rescore = std::max(bp->rescore, rescore);
        bp->c_target = std::max(bp->c_target, q.c_target);
        bp->rerank_smem = std::max(bp->rerank_smem, smem);
        bp->keyed = bp->keyed || p.keyed;
    }
    if (kstride > 0) bp->k = std::max(bp->k, kstride);
    return DANN_OK;
}

/* B queries, the first k rows each (the first qp[b].k of a mixed batch).  All pointers are device pointers; d_labels /
 * d_label_off are used when bp.keyed. */
static int search_batch_device_locked(dann_index *ix, const float *d_queries, const int16_t *d_labels,
                                      const int32_t *d_label_off, int B, const BatchParams &bp,
                                      uint64_t *d_out_tid, float *d_out_dist, uint32_t *d_out_node,
                                      uint32_t *d_out_count, dann_query_stats *d_out_stats, cudaStream_t st) {
    const IndexView &v = ix->v;
    if (!d_queries || !d_out_tid) return fail(DANN_ERR_INVALID_ARG, "NULL query or output buffer");
    if (!bp.keyed) d_labels = nullptr, d_label_off = nullptr;
    const uint32_t c_target = bp.c_target;

    CK(ix->sc_qfull.reserve((size_t)B * v.dim * sizeof(float)));
    CK(ix->sc_qcodes.reserve((size_t)B * v.cw * sizeof(uint64_t)));
    CK(ix->sc_stream.reserve((size_t)B * c_target * sizeof(uint32_t)));
    CK(ix->sc_stream_len.reserve((size_t)B * sizeof(uint32_t)));
    CK(ix->sc_stats.reserve((size_t)B * sizeof(dann_query_stats)));
    CK(ix->sc_qlist.reserve((size_t)B * sizeof(uint32_t)));
    CK(ix->sc_ctl.reserve(64));
    const QueryParam *d_qp = nullptr;
    if (!bp.qp.empty()) { /* ordered on st behind the queries and keys the caller staged */
        CK(ix->sc_qparams.reserve(bp.qp.size() * sizeof(QueryParam)));
        CK(cudaMemcpyAsync(ix->sc_qparams.p, bp.qp.data(), bp.qp.size() * sizeof(QueryParam), cudaMemcpyHostToDevice, st));
        d_qp = ix->sc_qparams.as<QueryParam>();
    }
    dann_query_stats *d_stats = d_out_stats ? d_out_stats : ix->sc_stats.as<dann_query_stats>();

    ix->timing = dann_batch_timing{};
    CK(cudaEventRecord(ix->ev[0], st));
    if (ix->plain) CK(ix->sc_qindex.reserve((size_t)B * v.dim_index * sizeof(float)));
    int rc = launch_prepare(ix, d_queries, B, ix->sc_qfull.as<float>(), ix->sc_qcodes.as<uint64_t>(),
                            ix->sc_qindex.as<float>(), st);
    if (rc) return rc;
    CK(cudaEventRecord(ix->ev[1], st));

    rc = run_search(ix, ix->sc_qcodes.as<uint64_t>(), d_labels, d_label_off, B, (uint32_t)bp.L, c_target, d_stats, nullptr,
                    nullptr, 0, st, ix->sc_qindex.as<float>(), d_qp);
    if (rc) return rc;
    CK(cudaEventRecord(ix->ev[2], st));

    RerankArgs r;
    r.ix = v;
    r.q_full = ix->sc_qfull.as<float>();
    r.stream = ix->sc_stream.as<uint32_t>();
    r.stream_len = ix->sc_stream_len.as<uint32_t>();
    r.c_target = c_target;
    r.k = (uint32_t)bp.k;
    r.rescore = (uint32_t)bp.rescore;
    r.out_tid = d_out_tid;
    r.out_dist = d_out_dist;
    r.out_node = d_out_node;
    r.out_count = d_out_count;
    r.stats = d_stats;
    r.qp = d_qp;
    CK(allow_dynamic_smem(dann_rerank_kernel, bp.rerank_smem));
    dann_rerank_kernel<<<B, 128, bp.rerank_smem, st>>>(r);
    ix->launches++;
    CK(cudaGetLastError());
    if (ix->plain && bp.rescore > 0) {
        dann_plain_stats_kernel<<<(B + 127) / 128, 128, 0, st>>>(d_stats, B, d_qp);
        ix->launches++;
        CK(cudaGetLastError());
    }
    CK(cudaEventRecord(ix->ev[3], st));
    CK(cudaStreamSynchronize(st));
    float ms = 0;
    CK(cudaEventElapsedTime(&ms, ix->ev[0], ix->ev[1]));
    ix->timing.prepare_ms = ms;
    CK(cudaEventElapsedTime(&ms, ix->ev[1], ix->ev[2]));
    ix->timing.search_ms = ms;
    CK(cudaEventElapsedTime(&ms, ix->ev[2], ix->ev[3]));
    ix->timing.rerank_ms = ms;
    ix->timing.resort_ms = 0.0f; /* the rerank window runs inside the rerank kernel */
    CK(cudaEventElapsedTime(&ms, ix->ev[0], ix->ev[3]));
    ix->timing.total_ms = ms;
    return DANN_OK;
}

extern "C" int dann_search_batch_device(dann_index *ix, const float *d_queries, const int16_t *d_labels,
                                        const int32_t *d_label_off, int B, int k, int search_list_size,
                                        int rescore, uint64_t *d_out_tid, float *d_out_dist,
                                        uint32_t *d_out_count, dann_query_stats *d_out_stats, void *stream) try {
    int rc = check_live(ix);
    if (rc) return rc;
    BatchParams bp;
    rc = uniform_params(ix, B, k, search_list_size, rescore, d_label_off != nullptr, &bp);
    if (rc) return rc;
    std::lock_guard<std::mutex> lk(ix->mu);
    DANN_DEVICE_INPUT_STREAM(st, stream);
    return search_batch_device_locked(ix, d_queries, d_labels, d_label_off, B, bp, d_out_tid, d_out_dist, nullptr,
                                      d_out_count, d_out_stats, st);
} DANN_CATCH

extern "C" int dann_search_batch_mixed_device(dann_index *ix, const float *d_queries, const int16_t *d_labels,
                                              const int32_t *d_label_off, const dann_query_params *d_params, int B,
                                              uint64_t *d_out_tid, float *d_out_dist, uint32_t *d_out_count,
                                              dann_query_stats *d_out_stats, void *stream) try {
    int rc = check_live(ix);
    if (rc) return rc;
    if (B <= 0) return fail(DANN_ERR_INVALID_ARG, "B %d must be positive", B);
    if (!d_params) return fail(DANN_ERR_INVALID_ARG, "params is NULL");
    std::lock_guard<std::mutex> lk(ix->mu);
    DANN_DEVICE_INPUT_STREAM(st, stream);
    /* the checks read params and label_off on the host: one small read-back each, before anything runs */
    std::vector<dann_query_params> hp((size_t)B);
    std::vector<int32_t> hoff;
    CK(cudaMemcpyAsync(hp.data(), d_params, (size_t)B * sizeof(dann_query_params), cudaMemcpyDeviceToHost, st));
    if (d_label_off) {
        hoff.resize((size_t)B + 1);
        CK(cudaMemcpyAsync(hoff.data(), d_label_off, ((size_t)B + 1) * sizeof(int32_t), cudaMemcpyDeviceToHost, st));
    }
    CK(cudaStreamSynchronize(st));
    BatchParams bp;
    rc = mixed_params(ix, B, hp.data(), d_labels, d_label_off ? hoff.data() : nullptr, 0, &bp);
    if (rc) return rc;
    return search_batch_device_locked(ix, d_queries, d_labels, d_label_off, B, bp, d_out_tid, d_out_dist, nullptr,
                                      d_out_count, d_out_stats, st);
} DANN_CATCH

/* The device half of the host-buffer batch: stages B host queries (and label keys) on ix's device and runs the batch
 * there.  Returns with the rows in ix->st_tid / st_dist / sc_node / st_count / st_stats and ix->stream drained.  The
 * caller holds ix->mu. */
static int search_batch_staged_locked(dann_index *ix, const float *queries, const int16_t *labels,
                                      const int32_t *label_off, int B, const BatchParams &bp) {
    cudaStream_t st = ix->stream;
    const IndexView &v = ix->v;
    const size_t nk = (size_t)B * bp.k;
    CK(ix->st_queries.reserve((size_t)B * v.dim * sizeof(float)));
    CK(ix->st_tid.reserve(nk * sizeof(uint64_t)));
    CK(ix->st_dist.reserve(nk * sizeof(float)));
    CK(ix->sc_node.reserve(nk * sizeof(uint32_t)));
    CK(ix->st_count.reserve((size_t)B * sizeof(uint32_t)));
    CK(ix->st_stats.reserve((size_t)B * sizeof(dann_query_stats)));
    CK(cudaMemcpyAsync(ix->st_queries.p, queries, (size_t)B * v.dim * sizeof(float), cudaMemcpyHostToDevice, st));
    const int16_t *d_lab = nullptr;
    const int32_t *d_off = nullptr;
    std::vector<int16_t> nl;
    std::vector<int32_t> no;
    if (bp.keyed) {
        no.resize((size_t)B + 1);
        no[0] = 0;
        if (label_off[0] < 0) return fail(DANN_ERR_INVALID_ARG, "label_off[0] is negative");
        if (label_off[B] > label_off[0] && !labels) return fail(DANN_ERR_INVALID_ARG, "labels is NULL but label_off describes a non-empty key");
        for (int b = 0; b < B; b++) {
            int32_t o0 = label_off[b], o1 = label_off[b + 1];
            if (o1 < o0) return fail(DANN_ERR_INVALID_ARG, "label_off is not monotone");
            if (o1 > o0) append_label_set(nl, labels + o0, labels + o1);
            no[b + 1] = (int32_t)nl.size();
        }
        CK(ix->st_labels.reserve(std::max<size_t>(nl.size(), 1) * sizeof(int16_t)));
        CK(ix->st_label_off.reserve(no.size() * sizeof(int32_t)));
        if (!nl.empty()) CK(cudaMemcpyAsync(ix->st_labels.p, nl.data(), nl.size() * sizeof(int16_t), cudaMemcpyHostToDevice, st));
        CK(cudaMemcpyAsync(ix->st_label_off.p, no.data(), no.size() * sizeof(int32_t), cudaMemcpyHostToDevice, st));
        d_lab = ix->st_labels.as<int16_t>();
        d_off = ix->st_label_off.as<int32_t>();
    }
    return search_batch_device_locked(ix, ix->st_queries.as<float>(), d_lab, d_off, B, bp, ix->st_tid.as<uint64_t>(),
                                      ix->st_dist.as<float>(), ix->sc_node.as<uint32_t>(), ix->st_count.as<uint32_t>(),
                                      ix->st_stats.as<dann_query_stats>(), st);
}

/* the uniform batch of a caller that holds ix->mu (dann_shards) */
static int search_batch_staged_locked(dann_index *ix, const float *queries, const int16_t *labels,
                                      const int32_t *label_off, int B, int k, int L, int rescore) {
    BatchParams bp;
    const int rc = uniform_params(ix, B, k, L, rescore, label_off != nullptr, &bp);
    return rc ? rc : search_batch_staged_locked(ix, queries, labels, label_off, B, bp);
}

/* host-buffer batch with optional node ids; bp from uniform_params or mixed_params (rows of bp.k) */
static int search_batch_host(dann_index *ix, const float *queries, const int16_t *labels, const int32_t *label_off, int B,
                             const BatchParams &bp, uint64_t *out_tid, float *out_dist, uint32_t *out_node,
                             uint32_t *out_count, dann_query_stats *out_stats) {
    if (!queries || !out_tid) return fail(DANN_ERR_INVALID_ARG, "dann_search_batch: bad argument");
    std::lock_guard<std::mutex> lk(ix->mu);
    cudaStream_t st = ix->stream;
    const size_t nk = (size_t)B * bp.k;
    int rc = search_batch_staged_locked(ix, queries, labels, label_off, B, bp);
    if (rc) return rc;
    CK(cudaMemcpyAsync(out_tid, ix->st_tid.p, nk * sizeof(uint64_t), cudaMemcpyDeviceToHost, st));
    if (out_dist) CK(cudaMemcpyAsync(out_dist, ix->st_dist.p, nk * sizeof(float), cudaMemcpyDeviceToHost, st));
    if (out_node) CK(cudaMemcpyAsync(out_node, ix->sc_node.p, nk * sizeof(uint32_t), cudaMemcpyDeviceToHost, st));
    if (out_count) CK(cudaMemcpyAsync(out_count, ix->st_count.p, (size_t)B * sizeof(uint32_t), cudaMemcpyDeviceToHost, st));
    if (out_stats) CK(cudaMemcpyAsync(out_stats, ix->st_stats.p, (size_t)B * sizeof(dann_query_stats), cudaMemcpyDeviceToHost, st));
    CK(cudaStreamSynchronize(st));
    return DANN_OK;
}

static int search_batch_host(dann_index *ix, const float *queries, const int16_t *labels,
                             const int32_t *label_off, int B, int k, int L, int rescore, uint64_t *out_tid,
                             float *out_dist, uint32_t *out_node, uint32_t *out_count,
                             dann_query_stats *out_stats) {
    int rc = check_live(ix);
    if (rc) return rc;
    if (B <= 0 || k <= 0 || !queries || !out_tid) return fail(DANN_ERR_INVALID_ARG, "dann_search_batch: bad argument");
    BatchParams bp;
    rc = uniform_params(ix, B, k, L, rescore, label_off != nullptr, &bp);
    if (rc) return rc;
    return search_batch_host(ix, queries, labels, label_off, B, bp, out_tid, out_dist, out_node, out_count, out_stats);
}

extern "C" int dann_search_batch(dann_index *ix, const float *queries, const int16_t *labels,
                                 const int32_t *label_off, int B, int k, int search_list_size, int rescore,
                                 uint64_t *out_tid, float *out_dist, uint32_t *out_count,
                                 dann_query_stats *out_stats) try {
    return search_batch_host(ix, queries, labels, label_off, B, k, search_list_size, rescore, out_tid, out_dist,
                             nullptr, out_count, out_stats);
} DANN_CATCH

extern "C" int dann_search_batch_mixed(dann_index *ix, const float *queries, const int16_t *labels, const int32_t *label_off,
                                       const dann_query_params *params, int B, uint64_t *out_tid, float *out_dist,
                                       uint32_t *out_count, dann_query_stats *out_stats) try {
    int rc = check_live(ix);
    if (rc) return rc;
    BatchParams bp;
    rc = mixed_params(ix, B, params, labels, label_off, 0, &bp);
    if (rc) return rc;
    return search_batch_host(ix, queries, labels, label_off, B, bp, out_tid, out_dist, nullptr, out_count, out_stats);
} DANN_CATCH

/* ------------------------------------------------------------------------------------ */
/* index construction (SURVEY.md §8f row 1) — see dann_build.cuh                            */

extern "C" int dann_index_set_vectors(dann_index *ix, const float *vectors) try {
    int rc = check_live(ix);
    if (rc) return rc;
    if (!vectors) return fail(DANN_ERR_INVALID_ARG, "dann_index_set_vectors: NULL vectors");
    std::lock_guard<std::mutex> lk(ix->mu);
    IndexView &v = ix->v;
    if (!v.n) return DANN_OK;
    float *d = const_cast<float *>(v.vectors);
    if (!d) {
        void *p = nullptr;
        size_t bytes = (size_t)v.n * v.dim * sizeof(float);
        CK(cudaMalloc(&p, bytes));
        ix->owned.push_back(p);
        ix->hbm_bytes += bytes;
        d = reinterpret_cast<float *>(p);
        v.vectors = d;
    }
    CK(cudaMemcpyAsync(d, vectors, (size_t)v.n * v.dim * sizeof(float), cudaMemcpyHostToDevice, ix->stream)); /* ordered before the normalisation */
    CK(cudaStreamSynchronize(ix->stream));
    return normalize_rows(ix, d);
} DANN_CATCH

extern "C" int dann_index_set_vectors_device(dann_index *ix, float *d_vectors) try {
    int rc = check_live(ix);
    if (rc) return rc;
    if (!d_vectors) return fail(DANN_ERR_INVALID_ARG, "dann_index_set_vectors_device: NULL vectors");
    std::lock_guard<std::mutex> lk(ix->mu);
    IndexView &v = ix->v;
    if (!v.n) return DANN_OK;
    if (v.vectors) return fail(DANN_ERR_STATE, "dann_index_set_vectors_device: the index already owns a vector array");
    cudaPointerAttributes at{};
    if (cudaPointerGetAttributes(&at, d_vectors) != cudaSuccess || at.type != cudaMemoryTypeDevice || at.device != ix->device) {
        cudaGetLastError();
        return fail(DANN_ERR_INVALID_ARG, "dann_index_set_vectors_device: not a device pointer on device %d", ix->device);
    }
    v.vectors = d_vectors; /* borrowed: not in ix->owned */
    ix->hbm_bytes += (uint64_t)v.n * v.dim * sizeof(float);
    CK(order_after_default_stream(ix, ix->stream)); /* the caller's rows: see DANN_DEVICE_INPUT_STREAM */
    return normalize_rows(ix, d_vectors);
} DANN_CATCH

extern "C" int dann_index_download_nbrs(dann_index *ix, uint32_t *out) try {
    int rc = check_live(ix);
    if (rc) return rc;
    if (!out) return fail(DANN_ERR_INVALID_ARG, "dann_index_download_nbrs: NULL buffer");
    std::lock_guard<std::mutex> lk(ix->mu);
    const IndexView &v = ix->v;
    if (!v.n) return DANN_OK;
    CK(cudaMemcpy2D(out, (size_t)v.R * 4, v.nbrs, (size_t)v.Rp * 4, (size_t)v.R * 4, v.n, cudaMemcpyDeviceToHost));
    return DANN_OK;
} DANN_CATCH

extern "C" int dann_build_graph(dann_index *ix, int num_neighbors, int search_list_size, float max_alpha,
                                uint32_t max_batch, dann_build_stats *out) try {
    int rc = check_live(ix);
    if (rc) return rc;
    std::lock_guard<std::mutex> lk(ix->mu);
    IndexView &v = ix->v;
    if (ix->plain) return fail(DANN_ERR_STATE, "dann_build_graph builds over SBQ codes: not available for a plain-storage index");
    if (v.R != DANN_BUILD_SLACK || v.Rp != DANN_BUILD_SLACK)
        return fail(DANN_ERR_INVALID_ARG, "dann_build_graph needs an index loaded with R == %u neighbour slots", DANN_BUILD_SLACK);
    if (num_neighbors < 1 || num_neighbors > (int)DANN_BUILD_SLACK) return fail(DANN_ERR_INVALID_ARG, "num_neighbors must be 1..%u", DANN_BUILD_SLACK);
    if (search_list_size < 1 || search_list_size > 1000) return fail(DANN_ERR_INVALID_ARG, "build search_list_size must be 1..1000");
    if (v.has_labels && v.n_start_labels == 0)
        return fail(DANN_ERR_INVALID_ARG, "a labeled build needs the per-label start nodes (first node carrying each label)");
    if (v.n == 0) return DANN_OK;
    if (v.start_default != 0) return fail(DANN_ERR_INVALID_ARG, "dann_build_graph inserts in id order: start_default must be 0");
    if (max_batch == 0) max_batch = 1u << 20;
    cudaStream_t st = ix->stream;
    const uint32_t n = v.n;
    const uint32_t vis_cap = 2 * DANN_BUILD_CMAX;
    const uint32_t mb = std::min<uint32_t>(max_batch, n);
    /* a prune warp stages its 128 candidate codes in shared memory (row stride cw | 1): checked before anything is
     * allocated or the neighbour rows are reset, so a refused build leaves the index as it was */
    const size_t pw = ((size_t)DANN_BUILD_CMAX * 8 + (size_t)DANN_BUILD_CMAX * (v.cw | 1u) * 8 + DANN_BUILD_CMAX * 4 +
                       DANN_BUILD_SLACK * 4 + DANN_BUILD_SLACK * 2 + 15) & ~(size_t)15;
    const size_t budget = ix->smem_optin > 1024 ? ix->smem_optin - 1024 : ix->smem_optin;
    const int bw = (int)std::min<size_t>(8, budget / pw);
    if (bw < 1) return fail(DANN_ERR_CAPACITY, "SBQ code of %u words is too wide for the prune kernel's shared memory", v.words);

    DevBuf b_dist, b_deg, b_vis, b_vlen, b_k0, b_k1, b_v0, b_v1, b_heads, b_tmp, b_stream, b_slen, b_stats;
    struct Cleanup {
        std::vector<DevBuf *> v;
        ~Cleanup() {
            for (DevBuf *b : v) b->release();
        }
    } cleanup{{&b_dist, &b_deg, &b_vis, &b_vlen, &b_k0, &b_k1, &b_v0, &b_v1, &b_heads, &b_tmp, &b_stream, &b_slen, &b_stats}};
    const size_t ntrip = (size_t)mb * DANN_BUILD_SLACK;
    CK(b_dist.reserve((size_t)n * DANN_BUILD_SLACK * sizeof(uint16_t)));
    CK(b_deg.reserve((size_t)n));
    CK(b_vis.reserve((size_t)mb * vis_cap * sizeof(uint64_t)));
    CK(b_vlen.reserve((size_t)mb * 4));
    CK(b_k0.reserve(ntrip * 8));
    CK(b_k1.reserve(ntrip * 8));
    CK(b_v0.reserve(ntrip * 4));
    CK(b_v1.reserve(ntrip * 4));
    CK(b_heads.reserve(ntrip * 4 + 64));
    CK(ix->sc_stream.reserve((size_t)mb * 4)); /* run_search writes stream_len / stats even in build mode */
    CK(ix->sc_stream_len.reserve((size_t)mb * 4));
    CK(b_stats.reserve((size_t)mb * sizeof(dann_query_stats)));
    CK(ix->sc_qlist.reserve((size_t)mb * sizeof(uint32_t)));
    CK(ix->sc_ctl.reserve(64));
    size_t tmp_bytes = 0;
    CK(cub::DeviceRadixSort::SortPairs(nullptr, tmp_bytes, b_k0.as<uint64_t>(), b_k1.as<uint64_t>(), b_v0.as<uint32_t>(),
                                       b_v1.as<uint32_t>(), ntrip, 16, 64, st));
    CK(b_tmp.reserve(tmp_bytes));
    uint32_t *nbrs = const_cast<uint32_t *>(v.nbrs);
    CK(cudaMemsetAsync(nbrs, 0xFF, (size_t)n * DANN_BUILD_SLACK * 4, st));
    CK(cudaMemsetAsync(b_deg.p, 0, n, st));

    BuildArgs ba;
    ba.codes = v.codes;
    ba.cw = v.cw;
    ba.cws = v.cw | 1u;
    ba.n = n;
    ba.nbrs = nbrs;
    ba.nbr_dist = b_dist.as<uint16_t>();
    ba.deg = b_deg.as<uint8_t>();
    ba.R = (uint32_t)num_neighbors;
    ba.limit = std::min<uint32_t>(DANN_BUILD_SLACK, (uint32_t)std::ceil((double)num_neighbors * 1.3));
    ba.max_alpha = max_alpha;
    ba.label_off = v.has_labels ? v.label_off : nullptr;
    ba.labels = v.has_labels ? v.labels : nullptr;
    ba.per_warp_smem = (uint32_t)pw;
    const size_t bsmem = pw * bw + DANN_SMEM_SLACK;
    CK(cudaFuncSetAttribute(dann_build_prune_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)bsmem));
    CK(cudaFuncSetAttribute(dann_build_backlink_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)bsmem));
    CK(cudaFuncSetAttribute(dann_build_finalize_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)bsmem));
    const int bgrid = ix->sm_count * std::max<int>(1, (int)(budget / bsmem));

    dann_build_stats bs{};
    cudaEvent_t e[5];
    for (auto &x : e) CK(cudaEventCreate(&x));
    struct EvGuard {
        cudaEvent_t *e;
        ~EvGuard() {
            for (int i = 0; i < 5; i++) cudaEventDestroy(e[i]);
        }
    } evg{e};
    const uint32_t lists_unique_saved = ix->lists_unique;
    ix->lists_unique = 1; /* the builder never repeats an id within a list */
    const bool verbose = getenv("DANN_BUILD_VERBOSE") != nullptr;
    /* node 0 is the entry point (the reference's first inserted node); everything else arrives in
     * batches that grow with the graph (at most 1/16 of it) up to max_batch */
    for (uint32_t lo = 1; lo < n;) {
        uint32_t m = std::max<uint32_t>(1, lo / 16);
        m = std::min(std::min(m, mb), n - lo);
        /* graph/mod.rs:637-660: a labeled node is inserted twice — first from the label start nodes with the
         * label filter on, then from the default start node without it; the second pass merges with the
         * neighbours the first one left (add_neighbors) */
        uint32_t nheads = 0;
        for (int pass = v.has_labels ? 0 : 1; pass < 2; pass++) {
            const int16_t *qlab = pass == 0 ? v.labels : nullptr;
            const int32_t *qoff = pass == 0 ? reinterpret_cast<const int32_t *>(v.label_off + lo) : nullptr;
            CK(cudaEventRecord(e[0], st));
            rc = run_search(ix, v.codes + (size_t)lo * v.cw, qlab, qoff, (int)m, (uint32_t)search_list_size, 1u,
                            b_stats.as<dann_query_stats>(), b_vis.as<uint64_t>(), b_vlen.as<uint32_t>(), vis_cap, st);
            if (rc) {
                ix->lists_unique = lists_unique_saved;
                return rc;
            }
            CK(cudaEventRecord(e[1], st));
            dann_build_prune_kernel<<<bgrid, bw * 32, bsmem, st>>>(ba, lo, m, b_vis.as<uint64_t>(), b_vlen.as<uint32_t>(),
                                                                  vis_cap, b_k0.as<uint64_t>(), b_v0.as<uint32_t>());
            ix->launches++;
            CK(cudaGetLastError());
            CK(cudaEventRecord(e[2], st));
            const size_t cnt = (size_t)m * DANN_BUILD_SLACK;
            size_t tb = b_tmp.cap;
            CK(cub::DeviceRadixSort::SortPairs(b_tmp.p, tb, b_k0.as<uint64_t>(), b_k1.as<uint64_t>(), b_v0.as<uint32_t>(),
                                               b_v1.as<uint32_t>(), cnt, 16, 64, st));
            uint32_t *d_nheads = b_heads.as<uint32_t>() + ntrip;
            CK(cudaMemsetAsync(d_nheads, 0, 4, st));
            dann_build_heads_kernel<<<ix->sm_count * 4, 256, 0, st>>>(b_k1.as<uint64_t>(), cnt, b_heads.as<uint32_t>(), d_nheads);
            ix->launches += 2;
            CK(cudaMemcpyAsync(&nheads, d_nheads, 4, cudaMemcpyDeviceToHost, st));
            CK(cudaStreamSynchronize(st));
            CK(cudaEventRecord(e[3], st));
            if (nheads) {
                dann_build_backlink_kernel<<<bgrid, bw * 32, bsmem, st>>>(ba, b_k1.as<uint64_t>(), b_v1.as<uint32_t>(), cnt,
                                                                         b_heads.as<uint32_t>(), nheads);
                ix->launches++;
                CK(cudaGetLastError());
            }
            CK(cudaEventRecord(e[4], st));
            CK(cudaStreamSynchronize(st));
            float ms;
            CK(cudaEventElapsedTime(&ms, e[0], e[1]));
            bs.search_ms += ms;
            CK(cudaEventElapsedTime(&ms, e[1], e[2]));
            bs.prune_ms += ms;
            CK(cudaEventElapsedTime(&ms, e[2], e[3]));
            bs.sort_ms += ms;
            CK(cudaEventElapsedTime(&ms, e[3], e[4]));
            bs.backlink_ms += ms;
        }
        bs.batches++;
        if (verbose && (bs.batches % 16 == 0 || lo + m >= n))
            fprintf(stderr, "[dann_build] batch %u: nodes %u..%u (m=%u, %u destinations) search %.0f prune %.0f sort %.0f backlink %.0f ms\n",
                    bs.batches, lo, lo + m, m, nheads, bs.search_ms, bs.prune_ms, bs.sort_ms, bs.backlink_ms);
        lo += m;
    }
    dann_build_finalize_kernel<<<bgrid, bw * 32, bsmem, st>>>(ba);
    ix->launches++;
    CK(cudaGetLastError());
    CK(cudaStreamSynchronize(st));
    if (env_u32("DANN_BUILD_RESCUE", 0) == 1 && !v.has_labels) { /* opt-in: see dann_build.cuh "in-edge rescue" */
        DevBuf b_in, b_claim;
        struct Rel {
            DevBuf *a, *b;
            ~Rel() {
                a->release();
                b->release();
            }
        } rel{&b_in, &b_claim};
        CK(b_in.reserve((size_t)n * 4));
        CK(b_claim.reserve((size_t)n * 4 + 4));
        uint32_t *d_claim = b_claim.as<uint32_t>(), *d_resc = d_claim + n;
        for (int round = 0; round < 16; round++) {
            CK(cudaMemsetAsync(b_in.p, 0, (size_t)n * 4, st));
            CK(cudaMemsetAsync(d_claim, 0, (size_t)n * 4 + 4, st));
            dann_build_mark_indegree_kernel<<<ix->sm_count * 8, 256, 0, st>>>(nbrs, b_deg.as<uint8_t>(), n, b_in.as<uint32_t>());
            dann_build_rescue_kernel<<<ix->sm_count * 4, 256, 0, st>>>(nbrs, b_deg.as<uint8_t>(), n, (uint32_t)num_neighbors,
                                                                      b_in.as<uint32_t>(), d_claim, d_resc);
            dann_build_rescue_degrees_kernel<<<ix->sm_count * 4, 256, 0, st>>>(b_deg.as<uint8_t>(), d_claim, n, (uint32_t)num_neighbors);
            ix->launches += 3;
            CK(cudaGetLastError());
            uint32_t resc = 0;
            CK(cudaMemcpyAsync(&resc, d_resc, 4, cudaMemcpyDeviceToHost, st));
            CK(cudaStreamSynchronize(st));
            if (verbose) fprintf(stderr, "[dann_build] rescue round %d: %u nodes had no in-edge\n", round, resc);
            if (!resc) break;
        }
    }
    bs.total_ms = bs.search_ms + bs.prune_ms + bs.sort_ms + bs.backlink_ms;
    /* average degree */
    {
        std::vector<uint8_t> hdeg(std::min<uint32_t>(n, 1u << 20));
        CK(cudaMemcpy(hdeg.data(), b_deg.p, hdeg.size(), cudaMemcpyDeviceToHost));
        double sdeg = 0;
        for (uint8_t d : hdeg) sdeg += d;
        bs.avg_degree = sdeg / (double)hdeg.size();
    }
    if (out) *out = bs;
    return DANN_OK;
} DANN_CATCH

/* ------------------------------------------------------------------------------------ */
/* scan operator: ambeginscan / amrescan / amgettuple / amendscan (scan.rs:309-476)       */

extern "C" int dann_scan_begin(dann_index *ix, dann_scan **out) try {
    if (!ix || !out) return fail(DANN_ERR_INVALID_ARG, "dann_scan_begin: NULL argument");
    dann_scan *sc = new (std::nothrow) dann_scan();
    if (!sc) return fail(DANN_ERR_OOM, "host allocation failed");
    sc->ix = ix;
    *out = sc;
    return DANN_OK;
} DANN_CATCH

#define DANN_SCAN_BUFS(sc)                                                                                               \
    {&(sc)->d_qindex, &(sc)->d_step, &(sc)->d_query, &(sc)->d_qfull, &(sc)->d_qcodes, &(sc)->d_labels, &(sc)->d_label_off, \
     &(sc)->d_saved, &(sc)->d_heap_sm, &(sc)->d_vis, &(sc)->d_heap_tail, &(sc)->d_cnode, &(sc)->d_set, &(sc)->d_ins,       \
     &(sc)->d_stream, &(sc)->d_slen, &(sc)->d_stats, &(sc)->d_dist, &(sc)->d_win, &(sc)->d_winst, &(sc)->d_ctl,     \
     &(sc)->d_snap}

static void scan_release(dann_scan *sc) {
    DevBuf *bufs[] = DANN_SCAN_BUFS(sc);
    for (DevBuf *b : bufs) b->release();
}

/* (re)allocate the scan's private workspace for the current plan and reset the search state, enqueued on `st` */
static int scan_reset_search(dann_scan *sc, cudaStream_t st) {
    dann_index *ix = sc->ix;
    SearchPlan &p = sc->plan;
    int rc = make_plan(ix, 1, (uint32_t)sc->L, sc->plan_rows, sc->grow, sc->nlabels >= 0, &p, true);
    if (rc) return rc;
    CK(sc->d_saved.reserve(sizeof(SavedScan)));
    CK(sc->d_heap_sm.reserve((size_t)p.hs * p.esize + 16));
    CK(sc->d_vis.reserve((size_t)p.vcap * 8));
    CK(sc->d_heap_tail.reserve((size_t)p.cand_cap * p.esize));
    CK(sc->d_cnode.reserve((size_t)p.cand_cap * 4));
    CK(sc->d_ins.reserve((size_t)p.ins_cap * 4));
    if (p.bitmap_words) {
        CK(sc->d_set.reserve((size_t)p.bitmap_words * 4));
        CK(cudaMemsetAsync(sc->d_set.p, 0, (size_t)p.bitmap_words * 4, st));
    } else {
        CK(sc->d_set.reserve((size_t)p.hash_cap * 4));
    }
    CK(cudaMemsetAsync(sc->d_saved.p, 0, sizeof(SavedScan), st));
    return DANN_OK;
}

/* amrescan's checks of its arguments that do not depend on the index */
static int scan_rescan_check(const int16_t *labels, int nlabels, int search_list_size, int rescore) {
    if (search_list_size < 1 || search_list_size > 10000) return fail(DANN_ERR_INVALID_ARG, "search_list_size %d outside 1..10000", search_list_size);
    if (rescore < 0 || rescore > 1000) return fail(DANN_ERR_INVALID_ARG, "rescore %d outside 0..1000", rescore);
    if (nlabels > 0 && !labels) return fail(DANN_ERR_INVALID_ARG, "labels is NULL but nlabels > 0");
    return DANN_OK;
}

/* The enqueue half of amrescan: the scan's new query, key and parameters, and its vector preparation and search reset
 * enqueued on `st`, a stream of the index's device.  The caller has checked the arguments (scan_rescan_check), made the
 * device current and holds sc->ix->mu; the scan may step once `st` has been synchronised (scan_rescan_wait).  Several
 * scans may be enqueued on one stream and waited for with one synchronisation. */
static int scan_rescan_enqueue(dann_scan *sc, const float *query, const int16_t *labels, int nlabels,
                               int search_list_size, int rescore, cudaStream_t st) {
    dann_index *ix = sc->ix;
    const IndexView &v = ix->v;
    if (ix->plain) {
        if (query && nlabels >= 0) return fail(DANN_ERR_INVALID_ARG, "plain storage does not support label filters (plain/storage.rs:260)");
        if (v.dim == v.dim_index) rescore = 0; /* scan.rs:392-403: next() instead of next_with_resort */
    }
    if (rescore > 0 && v.n && !v.vectors) return fail(DANN_ERR_STATE, "index has no heap vectors yet: rescore must be 0");
    const uint32_t dim = v.dim;
    if (query) sc->query.assign(query, query + dim);
    else sc->query.assign(dim, 0.0f); /* NULL order-by argument: zero vector, no labels (labels/mod.rs:214-216) */
    sc->nlabels = query ? nlabels : -1;
    sc->labels.clear();
    if (sc->nlabels > 0) append_label_set(sc->labels, labels, labels + nlabels);
    sc->L = search_list_size;
    sc->rescore = rescore;
    sc->grow = 1;
    sc->plan_rows = (uint32_t)rescore + 64u;
    if (sc->deep) { /* back to the planned workspace: give the deep scan's buffers back (reserve() never shrinks) */
        DevBuf *deep_bufs[] = {&sc->d_heap_sm, &sc->d_vis, &sc->d_heap_tail, &sc->d_cnode, &sc->d_set, &sc->d_ins,
                               &sc->d_stream, &sc->d_dist, &sc->d_snap};
        for (DevBuf *b : deep_bufs) b->release();
        sc->deep = false;
    }
    sc->regrows = sc->growths = 0;
    sc->streamed = sc->win_len = 0;
    sc->exhausted = false;
    sc->stats = dann_query_stats{};
    /* amrescan's vector preparation runs once, here */
    CK(sc->d_query.reserve((size_t)dim * 4));
    CK(sc->d_qfull.reserve((size_t)dim * 4));
    CK(sc->d_qcodes.reserve((size_t)v.cw * 8));
    CK(sc->d_slen.reserve(16));
    CK(sc->d_stats.reserve(sizeof(dann_query_stats)));
    CK(sc->d_win.reserve((size_t)std::max(rescore, 1) * 8));
    CK(sc->d_winst.reserve(sizeof(ScanWindow)));
    CK(sc->d_step.reserve(sizeof(ScanStepOut) + sizeof(ScanRow)));
    CK(sc->d_ctl.reserve(64));
    CK(cudaMemcpyAsync(sc->d_query.p, sc->query.data(), (size_t)dim * 4, cudaMemcpyHostToDevice, st));
    if (sc->nlabels >= 0) {
        int32_t off[2] = {0, (int32_t)sc->labels.size()};
        CK(sc->d_labels.reserve(std::max<size_t>(sc->labels.size(), 1) * 2));
        CK(sc->d_label_off.reserve(8));
        if (!sc->labels.empty()) CK(cudaMemcpyAsync(sc->d_labels.p, sc->labels.data(), sc->labels.size() * 2, cudaMemcpyHostToDevice, st));
        CK(cudaMemcpyAsync(sc->d_label_off.p, off, 8, cudaMemcpyHostToDevice, st));
    }
    CK(cudaMemsetAsync(sc->d_winst.p, 0, sizeof(ScanWindow), st));
    if (ix->plain) CK(sc->d_qindex.reserve((size_t)v.dim_index * 4));
    int rc = launch_prepare(ix, sc->d_query.as<float>(), 1, sc->d_qfull.as<float>(), sc->d_qcodes.as<uint64_t>(),
                            sc->d_qindex.as<float>(), st);
    if (rc) return rc;
    return scan_reset_search(sc, st);
}

/* The wait half of amrescan: one synchronisation of `st`, on which the n scans of `ix`'s device were enqueued; then they
 * may step. */
static int scan_rescan_wait(dann_index *ix, cudaStream_t st, dann_scan *const *scans, size_t n) {
    CK(cudaStreamSynchronize(st));
    for (size_t i = 0; i < n; i++) scans[i]->active = true;
    return DANN_OK;
}

extern "C" int dann_scan_rescan(dann_scan *sc, const float *query, const int16_t *labels, int nlabels,
                                int search_list_size, int rescore) try {
    if (!sc) return fail(DANN_ERR_INVALID_ARG, "dann_scan_rescan: NULL scan");
    int rc = scan_rescan_check(labels, nlabels, search_list_size, rescore);
    if (rc) return rc;
    dann_index *ix = sc->ix;
    rc = check_live(ix);
    if (rc) return rc;
    std::lock_guard<std::mutex> lk(ix->mu);
    rc = scan_rescan_enqueue(sc, query, labels, nlabels, search_list_size, rescore, ix->stream);
    if (rc) return rc;
    return scan_rescan_wait(ix, ix->stream, &sc, 1);
} DANN_CATCH

/* The launch arguments of the scan's resumable search for rows [0, want) of this step: its plan, its private workspace
 * and its saved state (d_ctl[1] receives the overflow bits).  counters: the step yields several rows, and the search
 * records its counters at every row it appends (d_snap). */
static int scan_search_args(dann_scan *sc, uint32_t want, bool counters, SearchArgs *out) {
    dann_index *ix = sc->ix;
    const IndexView &v = ix->v;
    {
        const SearchPlan &p = sc->plan;
        CK(sc->d_stream.reserve((size_t)want * 4));
        uint32_t *d_ctl = sc->d_ctl.as<uint32_t>();
        SearchArgs a = search_args_for_plan(v, ix->G, ix->Gshift, ix->lists_unique, p);
        a.q_codes = sc->d_qcodes.as<uint64_t>();
        a.q_labels = sc->nlabels >= 0 ? sc->d_labels.as<int16_t>() : nullptr;
        a.q_label_off = sc->nlabels >= 0 ? sc->d_label_off.as<int32_t>() : nullptr;
        a.nq = 1;
        a.L = (uint32_t)sc->L;
        a.c_target = want;
        a.stream = sc->d_stream.as<uint32_t>();
        a.stream_len = sc->d_slen.as<uint32_t>();
        a.stats = sc->d_stats.as<dann_query_stats>();
        a.overflow = d_ctl + 1;
        a.counter = d_ctl;
        a.hash = sc->d_set.as<uint32_t>();
        a.bitmap = sc->d_set.as<uint32_t>();
        a.ins_list = sc->d_ins.as<uint32_t>();
        a.cand_node = sc->d_cnode.as<uint32_t>();
        a.heap_tail = sc->d_heap_tail.p;
        a.saved = sc->d_saved.as<SavedScan>();
        a.saved_heap_sm = sc->d_heap_sm.p;
        a.saved_vis = sc->d_vis.as<uint64_t>();
        a.plain_vectors = ix->index_vectors;
        a.q_index = sc->d_qindex.as<float>();
        a.plain_dim = ix->plain ? v.dim_index : 0;
        if (counters) {
            CK(sc->d_snap.reserve((size_t)want * sizeof(uint2)));
            a.row_counters = sc->d_snap.as<uint2>();
        }
        *out = a;
    }
    return DANN_OK;
}

/* Enqueue the resumable search for rows [0, want) of this launch (d_ctl[1] receives the overflow bits). */
static int scan_launch_search(dann_scan *sc, uint32_t want, bool counters) {
    dann_index *ix = sc->ix;
    cudaStream_t st = ix->stream;
    const SearchPlan &p = sc->plan;
    SearchArgs a;
    int rc = scan_search_args(sc, want, counters, &a);
    if (rc) return rc;
    CK(cudaMemsetAsync(sc->d_ctl.p, 0, 8, st));
    search_fn fn = pick_kernel(false, p.entry, ix->NCH, ix->plain, p.deep);
    CK(cudaFuncSetAttribute(fn, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)(p.per_warp + DANN_SMEM_SLACK)));
    fn<<<1, 32, p.per_warp + DANN_SMEM_SLACK, st>>>(a);
    ix->launches++;
    CK(cudaGetLastError());
    return DANN_OK;
}

/* rows a step of nrows amgettuple calls takes off the approximate stream: next_with_resort refills the window to
 * `rescore` (scan.rs:255-305) and each later call refills the one row its predecessor popped; next() takes one */
static uint32_t scan_step_need(const dann_scan *sc, uint32_t nrows) {
    const uint32_t rescore = (uint32_t)sc->rescore;
    return rescore == 0 ? nrows : (sc->win_len < rescore ? rescore - sc->win_len : 0u) + nrows - 1;
}

/* dynamic shared memory of a scan-distance CTA: the query row */
static size_t scan_distance_smem(const IndexView &v) { return (size_t)((v.dim + 3u) & ~3u) * sizeof(float) + DANN_SMEM_SLACK; }

/* the arguments of the exact distances of the rows [skip, want) a search step may append */
static int scan_distance_desc(dann_scan *sc, uint32_t want, uint32_t skip, ScanDistanceDesc *d) {
    dann_index *ix = sc->ix;
    CK(sc->d_dist.reserve((size_t)want * 4));
    *d = ScanDistanceDesc{sc->d_qfull.as<float>(), sc->d_stream.as<uint32_t>(), sc->d_slen.as<uint32_t>(),
                          sc->d_ctl.as<uint32_t>() + 1, sc->d_dist.as<float>(), skip, 0u /* view */};
    return DANN_OK;
}

/* the arguments of the window step; a step that does not search finds nothing new beyond `skip` */
static ScanFinishDesc scan_finish_desc(dann_scan *sc, bool searching, uint32_t skip) {
    ScanFinishDesc f;
    f.w = sc->d_winst.as<ScanWindow>();
    f.win = sc->d_win.as<uint64_t>();
    f.stream = sc->d_stream.as<uint32_t>();
    f.dist = sc->d_dist.as<float>();
    f.slen_p = searching ? sc->d_slen.as<uint32_t>() : nullptr;
    f.overflow_p = searching ? sc->d_ctl.as<uint32_t>() + 1 : nullptr;
    f.stats_p = sc->d_stats.as<dann_query_stats>();
    f.rescore = (uint32_t)sc->rescore;
    f.skip = skip;
    f.slen_fixed = skip;
    f.view = 0;
    return f;
}

/* Rebuild the scan's suspended search as the deep plan, with the candidate and visited capacity of the planned workspace
 * it leaves (its reset enqueued on `st`); the next search replays the stream up to sc->streamed, once, and grows the
 * workspace in place wherever that replay or a later step needs more (scan_grow_in_place). */
static int scan_enter_deep(dann_scan *sc, cudaStream_t st) {
    dann_index *ix = sc->ix;
    PlanInputs in{};
    in.n = ix->v.n;
    in.R = ix->v.R;
    in.plain_dim = ix->plain ? ix->v.dim_index : 0;
    /* the start nodes of a label key are staged before any visit: room for all of them and one visit */
    const uint64_t cand = std::max<uint64_t>(sc->plan.cand_cap, (uint64_t)sc->labels.size() + ix->v.R);
    SearchPlan &p = sc->plan;
    dann_make_deep_plan(in, (uint32_t)std::min<uint64_t>(cand, 0xFFFFFC00u), sc->plan.vcap, &p);
    sc->deep = true;
    sc->d_ins.release();
    CK(sc->d_saved.reserve(sizeof(SavedScan)));
    CK(sc->d_heap_sm.reserve((size_t)p.hs * p.esize + 16));
    CK(sc->d_vis.reserve((size_t)p.vcap * 8));
    CK(sc->d_heap_tail.reserve((size_t)p.cand_cap * p.esize));
    CK(sc->d_cnode.reserve((size_t)p.cand_cap * 4));
    CK(sc->d_set.reserve((size_t)p.bitmap_words * 4));
    CK(cudaMemsetAsync(sc->d_set.p, 0, (size_t)p.bitmap_words * 4, st));
    CK(cudaMemsetAsync(sc->d_saved.p, 0, sizeof(SavedScan), st));
    return DANN_OK;
}

/* The scan outgrew its workspace: rebuild it twice as large (its reset enqueued on `st`, the stream its next search
 * runs on); the next search replays the stream up to sc->streamed.  Where the planned workspace can grow no further -
 * an eighth regrow in one call, or a plan dann_make_plan refuses - the scan enters the deep mode instead
 * (DANN_DEBUG_DEEP_AFTER = k, a test hook: after k regrows of the scan). */
static int scan_regrow(dann_scan *sc, int attempt, cudaStream_t st) {
    if (sc->deep) /* a deep scan suspends before it could overflow (DANN_ST_GROW) */
        return fail(DANN_ERR_STATE, "internal error: a deep scan overflowed its workspace");
    if (attempt < 8 && sc->regrows < env_u32("DANN_DEBUG_DEEP_AFTER", UINT32_MAX)) {
        const SearchPlan last = sc->plan;
        sc->grow *= 2;
        const int rc = scan_reset_search(sc, st);
        if (rc != DANN_ERR_CAPACITY) {
            sc->regrows += rc == DANN_OK;
            return rc;
        }
        sc->plan = last;
    }
    return scan_enter_deep(sc, st);
}

/* A deep scan suspended before a visit its workspace might not fit (DANN_ST_GROW): at least double what lacks room,
 * keeping the live prefix of each array - the heap's HBM tail [hs, heap_len) (SplitStore indexes it by absolute
 * position), the seq->node table [0, ncand) and the visited list [0, vis_len) - so that the same step resumes where it
 * stopped.  The inserted-set bitmap and the heap top keep their size. */
static int scan_grow_in_place(dann_scan *sc, cudaStream_t st) {
    dann_index *ix = sc->ix;
    SearchPlan &p = sc->plan;
    SavedScan sv;
    CK(cudaMemcpyAsync(&sv, sc->d_saved.p, sizeof sv, cudaMemcpyDeviceToHost, st));
    CK(cudaStreamSynchronize(st));
    uint32_t cand = p.cand_cap, vcap = p.vcap;
    if ((uint64_t)sv.ncand + ix->v.R > cand)
        cand = (uint32_t)std::min<uint64_t>((std::max<uint64_t>(2ull * cand, (uint64_t)sv.ncand + ix->v.R) + 1023) & ~1023ull, 0xFFFFFC00u);
    if (sv.vis_len + 1ull > vcap) vcap = (uint32_t)std::min<uint64_t>(2ull * vcap, 0xFFFFFFFCu);
    if (cand == p.cand_cap && vcap == p.vcap)
        return fail(DANN_ERR_STATE, "internal error: a deep scan suspended with room for its next visit");
    const size_t hs_bytes = (size_t)p.hs * 8, tail_end = (size_t)sv.heap_len * 8;
    CK(sc->d_heap_tail.grow_keep((size_t)cand * 8, hs_bytes, std::max(tail_end, hs_bytes), st));
    CK(sc->d_cnode.grow_keep((size_t)cand * 4, 0, (size_t)sv.ncand * 4, st));
    CK(sc->d_vis.grow_keep((size_t)vcap * 8, 0, (size_t)sv.vis_len * 8, st));
    p.cand_cap = p.need = cand;
    p.vcap = vcap;
    sc->growths++;
    return DANN_OK;
}

/* The scan's counters after one amgettuple call: the search's (visits, candidates), the window's full-distance
 * comparisons and the rows streamed so far */
static void scan_set_counters(dann_scan *sc, uint32_t visits, uint32_t candidates, uint32_t d_full, uint32_t streamed) {
    const bool plain = sc->ix->plain;
    dann_query_stats &s = sc->stats;
    s.visits = visits;
    s.candidates = candidates;
    s.d_quantized = plain ? 0u : candidates;
    /* plain layout: every comparison of the beam search was a full-distance comparison (plain/storage.rs:238,288) */
    s.d_full = d_full + (plain ? candidates : 0u);
    s.stream_len = sc->streamed = streamed;
    s.status = 0;
}

/* The host side of a step of nrows calls that did not overflow, applied row by row: each record's stream position,
 * counters and row, then - when the step met the end of scan - the counters of the call that found it.  `want` = rows
 * [0, want) the search was asked for, the first `skip` of them replayed.  row i goes to the outputs' element i.
 * Returns the rows produced. */
static int scan_after_step(dann_scan *sc, const ScanStepOut &o, const ScanRow *rows, uint32_t nrows, bool searching,
                           uint32_t want, uint32_t skip, uint32_t *block, uint16_t *offset, uint32_t *node_id, float *dist,
                           dann_query_stats *row_stats) {
    const uint32_t streamed = sc->streamed;
    if (searching && o.slen < want) sc->exhausted = true;
    for (uint32_t r = 0; r < o.nrows; r++) {
        const ScanRow &x = rows[r];
        scan_set_counters(sc, x.visits, x.candidates, x.d_full, streamed + (x.end - skip));
        if (row_stats) row_stats[r] = sc->stats;
        if (block) block[r] = (uint32_t)(x.tid >> 16);
        if (offset) offset[r] = (uint16_t)(x.tid & 0xFFFFu);
        if (node_id) node_id[r] = x.node;
        if (dist) dist[r] = x.dist;
    }
    if (o.nrows < nrows)
        scan_set_counters(sc, o.stats.visits, o.stats.candidates, o.win.d_full, streamed + (o.slen > skip ? o.slen - skip : 0u));
    sc->win_len = o.win.len;
    return (int)o.nrows;
}

/* The next nrows rows of a scan in one step: exactly what nrows consecutive amgettuple calls return
 * (next_with_resort, scan.rs:244-305: `while resort_buffer.len() < resort_size { next() ... }` then pop; with
 * resort_size == 0 a plain next()).  The search, the exact distances of the rows it appended and the window step are
 * enqueued back to back (see dann_scan_finish_kernel), and one ScanStepOut with the step's records comes back: one host
 * synchronisation, more when the workspace must grow.  Returns the rows produced or < 0. */
static int scan_fetch(dann_scan *sc, uint32_t nrows, const char *what, uint32_t *block, uint16_t *offset, uint32_t *node_id,
                      float *dist, dann_query_stats *row_stats) {
    if (!sc) return fail(DANN_ERR_INVALID_ARG, "%s: NULL scan", what);
    if (!sc->active) return fail(DANN_ERR_STATE, "%s before dann_scan_rescan", what);
    dann_index *ix = sc->ix;
    int rc = check_live(ix);
    if (rc) return rc;
    std::lock_guard<std::mutex> lk(ix->mu);
    const IndexView &v = ix->v;
    cudaStream_t st = ix->stream;
    const uint32_t need = scan_step_need(sc, nrows);
    const bool searching = need && !sc->exhausted;
    const size_t out_bytes = sizeof(ScanStepOut) + (size_t)nrows * sizeof(ScanRow);
    CK(sc->d_step.reserve(out_bytes));
    sc->h_step.resize(out_bytes);
    if (searching && sc->streamed == 0 && !sc->deep && need > sc->plan_rows) {
        /* the first step after amrescan asks for more rows than the workspace is planned for: plan for them before
         * anything has streamed, instead of regrowing by replay; where no such plan exists, the planned workspace stays */
        const SearchPlan last = sc->plan;
        const uint32_t last_rows = sc->plan_rows;
        sc->plan_rows = need;
        rc = scan_reset_search(sc, st);
        if (rc == DANN_ERR_CAPACITY) {
            sc->plan = last;
            sc->plan_rows = last_rows;
        } else if (rc) {
            return rc;
        }
    }
    ScanStepOut o;
    uint32_t skip = 0; /* rows that are only re-generated because the workspace had to grow */
    for (int attempt = 0;;) {
        const uint32_t want = skip + need;
        if (searching) {
            rc = scan_launch_search(sc, want, nrows > 1);
            if (rc) return rc;
            if (sc->rescore > 0) {
                ScanDistanceDesc d;
                rc = scan_distance_desc(sc, want, skip, &d);
                if (rc) return rc;
                const uint32_t span = 256; /* rows per CTA */
                const size_t smem = scan_distance_smem(v);
                CK(allow_dynamic_smem(dann_scan_distance_kernel, smem));
                dann_scan_distance_kernel<<<(need + span - 1) / span, 128, smem, st>>>(v, d.q_full, d.stream, d.slen_p,
                                                                                      d.overflow_p, d.skip, span, d.out);
                ix->launches++;
                CK(cudaGetLastError());
            }
        }
        const ScanFinishDesc f = scan_finish_desc(sc, searching, skip);
        ScanStepOut *d_out = sc->d_step.as<ScanStepOut>();
        dann_scan_finish_kernel<<<1, 128, 0, st>>>(v, f.w, f.win, f.rescore, f.stream, f.dist,
                                                   nrows > 1 ? sc->d_snap.as<uint2>() : nullptr, f.skip, f.slen_p,
                                                   f.slen_fixed, f.overflow_p, f.stats_p, nrows, d_out,
                                                   reinterpret_cast<ScanRow *>(d_out + 1));
        ix->launches++;
        CK(cudaGetLastError());
        CK(cudaMemcpyAsync(sc->h_step.data(), d_out, out_bytes, cudaMemcpyDeviceToHost, st));
        CK(cudaStreamSynchronize(st));
        memcpy(&o, sc->h_step.data(), sizeof o);
        if (!o.overflow) break;
        if (o.overflow == DANN_ST_GROW) { /* the same step resumes after the rows it already appended */
            rc = scan_grow_in_place(sc, st);
            if (rc) return rc;
            continue;
        }
        rc = scan_regrow(sc, attempt++, st);
        if (rc) return rc;
        skip = sc->streamed;
    }
    return scan_after_step(sc, o, reinterpret_cast<const ScanRow *>(sc->h_step.data() + sizeof(ScanStepOut)), nrows,
                           searching, skip + need, skip, block, offset, node_id, dist, row_stats);
}

extern "C" int dann_scan_gettuple(dann_scan *sc, uint32_t *block, uint16_t *offset, uint32_t *node_id, float *dist) try {
    return scan_fetch(sc, 1u, "dann_scan_gettuple", block, offset, node_id, dist, nullptr);
} DANN_CATCH

extern "C" int dann_scan_fetch(dann_scan *sc, int max_rows, uint32_t *block, uint16_t *offset, uint32_t *node_id,
                               float *dist, dann_query_stats *row_stats) try {
    if (max_rows < 1 || max_rows > 65536)
        return fail(DANN_ERR_INVALID_ARG, "dann_scan_fetch: max_rows = %d outside 1..65536", max_rows);
    return scan_fetch(sc, (uint32_t)max_rows, "dann_scan_fetch", block, offset, node_id, dist, row_stats);
} DANN_CATCH

/* The device part of one dann_scan_gettuple_many round: one upload of [IndexView x views][SearchArgs x args]
 * [ScanDistanceDesc x ddesc][ScanFinishDesc x fdesc], one dann_scan_search_many_kernel launch per run of equal fns[]
 * (args is grouped by instantiation), one dann_scan_distance_many_kernel launch when ddesc is not empty, one
 * dann_scan_finish_many_kernel launch, one download of the fdesc.size() outcomes into outs and their rows into rows
 * (through back), and one synchronisation.
 * The descriptors' `view` fields index views[]: the indexes of the round's scans, all on the device of `ix`, whose
 * stream, sc_many buffer and launch counter the round uses. */
static int scan_many_round(dann_index *ix, const std::vector<IndexView> &views, const std::vector<scan_many_fn> &fns,
                           const std::vector<SearchArgs> &args, const std::vector<ScanDistanceDesc> &ddesc,
                           const std::vector<ScanFinishDesc> &fdesc, std::vector<unsigned char> &blob,
                           std::vector<ScanStepOut> &outs, std::vector<ScanRow> &rows, std::vector<unsigned char> &back) {
    cudaStream_t st = ix->stream;
    const size_t m = fdesc.size();
    auto align16 = [](size_t b) { return (b + 15) & ~(size_t)15; };
    const size_t o_args = align16(views.size() * sizeof(IndexView));
    const size_t o_dist = o_args + align16(args.size() * sizeof(SearchArgs));
    const size_t o_fin = o_dist + align16(ddesc.size() * sizeof(ScanDistanceDesc));
    const size_t o_out = o_fin + align16(m * sizeof(ScanFinishDesc));
    blob.assign(o_out, 0);
    memcpy(blob.data(), views.data(), views.size() * sizeof(IndexView));
    if (!args.empty()) memcpy(blob.data() + o_args, args.data(), args.size() * sizeof(SearchArgs));
    if (!ddesc.empty()) memcpy(blob.data() + o_dist, ddesc.data(), ddesc.size() * sizeof(ScanDistanceDesc));
    memcpy(blob.data() + o_fin, fdesc.data(), m * sizeof(ScanFinishDesc));
    const size_t o_rows = o_out + m * sizeof(ScanStepOut);
    CK(ix->sc_many.reserve(o_rows + m * sizeof(ScanRow)));
    unsigned char *dev = ix->sc_many.as<unsigned char>();
    const IndexView *d_views = reinterpret_cast<const IndexView *>(dev);
    CK(cudaMemcpyAsync(dev, blob.data(), o_out, cudaMemcpyHostToDevice, st));
    for (size_t g = 0; g < args.size();) {
        size_t e = g;
        uint32_t per_warp = 0;
        for (; e < args.size() && fns[e] == fns[g]; e++) per_warp = std::max(per_warp, args[e].per_warp_smem);
        const scan_many_fn fn = fns[g];
        const size_t smem = (size_t)per_warp + DANN_SMEM_SLACK;
        CK(cudaFuncSetAttribute(fn, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
        fn<<<(unsigned)(e - g), 32, smem, st>>>(reinterpret_cast<const SearchArgs *>(dev + o_args) + g, (uint32_t)(e - g));
        ix->launches++;
        CK(cudaGetLastError());
        g = e;
    }
    if (!ddesc.empty()) {
        size_t smem = 0;
        for (const IndexView &v : views) smem = std::max(smem, scan_distance_smem(v));
        CK(allow_dynamic_smem(dann_scan_distance_many_kernel, smem));
        dann_scan_distance_many_kernel<<<(unsigned)ddesc.size(), 128, smem, st>>>(
            d_views, reinterpret_cast<const ScanDistanceDesc *>(dev + o_dist));
        ix->launches++;
        CK(cudaGetLastError());
    }
    dann_scan_finish_many_kernel<<<(unsigned)((m + 127) / 128), 128, 0, st>>>(
        d_views, reinterpret_cast<const ScanFinishDesc *>(dev + o_fin), (uint32_t)m, reinterpret_cast<ScanStepOut *>(dev + o_out),
        reinterpret_cast<ScanRow *>(dev + o_rows));
    ix->launches++;
    CK(cudaGetLastError());
    outs.resize(m);
    rows.resize(m);
    back.resize(m * (sizeof(ScanStepOut) + sizeof(ScanRow)));
    CK(cudaMemcpyAsync(back.data(), dev + o_out, back.size(), cudaMemcpyDeviceToHost, st));
    CK(cudaStreamSynchronize(st));
    memcpy(outs.data(), back.data(), m * sizeof(ScanStepOut));
    memcpy(rows.data(), back.data() + m * sizeof(ScanStepOut), m * sizeof(ScanRow));
    return DANN_OK;
}

/* One amgettuple of each of n scans, in rounds (scan_many_round) on the stream of `lead`.  The scans may belong to
 * several indexes on the device of `lead`; the caller has checked the arguments, made the device current and holds
 * the mutex of every index involved.  The first round takes every scan; a scan whose search overflowed regrows alone
 * and replays in the next round, with the others done.
 * What fails for one scan (its workspace cannot grow, or its buffers cannot be allocated) goes to that scan's out_rc
 * and, when msgs != NULL, its message to (*msgs)[i]; the other scans go on.  A failure of a round as a whole fails the
 * call only while no scan has taken its step yet; after that it goes to the out_rc of every scan of the round, so that
 * no scan's row is lost. */
static int scan_gettuple_many_locked(dann_index *lead, dann_scan *const *scans, int n, int32_t *out_rc, uint32_t *block,
                                     uint16_t *offset, uint32_t *node_id, float *dist, std::vector<std::string> *msgs) {
    int rc = DANN_OK;
    struct Step {
        dann_scan *sc;
        int i;            /* position in the caller's arrays */
        uint32_t need, skip;
        bool searching;
        int attempt;
        scan_many_fn fn;  /* its search instantiation */
        uint32_t view;    /* its index in views[] */
    };
    /* everything the rounds use is allocated here, before any scan moves: a host allocation failure later would fail
     * the call after some scans have taken their step */
    std::vector<Step> steps((size_t)n);
    std::vector<Step *> round((size_t)n), searchers, live, next;
    std::vector<const dann_index *> indexes;
    std::vector<IndexView> views;
    std::vector<scan_many_fn> fns;
    std::vector<SearchArgs> args;
    std::vector<ScanDistanceDesc> ddesc;
    std::vector<ScanFinishDesc> fdesc;
    std::vector<unsigned char> blob;
    std::vector<ScanStepOut> outs;
    std::vector<ScanRow> rows;
    std::vector<unsigned char> back;
    searchers.reserve(n);
    live.reserve(n);
    next.reserve(n);
    fns.reserve(n);
    args.reserve(n);
    ddesc.reserve(n);
    fdesc.reserve(n);
    outs.reserve(n);
    rows.reserve(n);
    back.reserve((size_t)n * (sizeof(ScanStepOut) + sizeof(ScanRow)));
    if (msgs) msgs->assign((size_t)n, std::string());
    for (int i = 0; i < n; i++) {
        dann_scan *sc = scans[i];
        const size_t view = (size_t)(std::find(indexes.begin(), indexes.end(), sc->ix) - indexes.begin());
        if (view == indexes.size()) {
            indexes.push_back(sc->ix);
            views.push_back(sc->ix->v);
        }
        const uint32_t need = scan_step_need(sc, 1);
        steps[i] = Step{sc, i, need, 0u, need && !sc->exhausted, 0, nullptr, (uint32_t)view};
        round[i] = &steps[i];
    }
    blob.reserve(views.size() * sizeof(IndexView) +
                 (size_t)n * (sizeof(SearchArgs) + sizeof(ScanDistanceDesc) + sizeof(ScanFinishDesc)) + 64);
    bool moved = false; /* some scan has taken its step */
    auto scan_failed = [&](const Step *s, int code) {
        out_rc[s->i] = code;
        if (msgs) {
            try {
                (*msgs)[s->i] = g_err;
            } catch (...) { /* no memory for the message: the code still goes back */
            }
        }
    };
    while (!round.empty()) {
        /* the searching scans, grouped by instantiation: one launch per group */
        searchers.clear();
        for (Step *s : round)
            if (s->searching) {
                s->fn = pick_scan_many(s->sc->plan.entry, s->sc->ix->NCH, s->sc->ix->plain, s->sc->plan.deep);
                searchers.push_back(s);
            }
        std::stable_sort(searchers.begin(), searchers.end(),
                         [](const Step *a, const Step *b) { return (uintptr_t)a->fn < (uintptr_t)b->fn; });
        fns.clear();
        args.clear();
        ddesc.clear();
        for (Step *s : searchers) {
            const uint32_t want = s->skip + s->need;
            SearchArgs a;
            ScanDistanceDesc d{};
            rc = scan_search_args(s->sc, want, false, &a);
            if (!rc && s->sc->rescore > 0) rc = scan_distance_desc(s->sc, want, s->skip, &d);
            if (rc) { /* this scan's buffers: it leaves the round */
                scan_failed(s, rc);
                s->fn = nullptr;
                continue;
            }
            d.view = s->view;
            fns.push_back(s->fn);
            args.push_back(a);
            if (s->sc->rescore > 0) ddesc.push_back(d);
        }
        live.clear();
        fdesc.clear();
        for (Step *s : round)
            if (!s->searching || s->fn) {
                live.push_back(s);
                fdesc.push_back(scan_finish_desc(s->sc, s->searching, s->skip));
                fdesc.back().view = s->view;
            }
        if (live.empty()) break;
        rc = scan_many_round(lead, views, fns, args, ddesc, fdesc, blob, outs, rows, back);
        if (rc) {
            if (!moved) return rc;
            for (Step *s : live) scan_failed(s, rc);
            break;
        }
        next.clear();
        for (size_t j = 0; j < live.size(); j++) {
            Step *s = live[j];
            const int i = s->i;
            if (!outs[j].overflow) {
                out_rc[i] = scan_after_step(s->sc, outs[j], &rows[j], 1u, s->searching, s->skip + s->need, s->skip,
                                            block ? block + i : nullptr, offset ? offset + i : nullptr,
                                            node_id ? node_id + i : nullptr, dist ? dist + i : nullptr, nullptr);
                moved = true;
                continue;
            }
            const bool grow = outs[j].overflow == DANN_ST_GROW; /* a deep scan resumes its step where it stopped */
            rc = grow ? scan_grow_in_place(s->sc, lead->stream) : scan_regrow(s->sc, s->attempt++, lead->stream);
            if (rc) { /* memory, or a CUDA error that has poisoned the handle: this scan alone */
                scan_failed(s, rc);
                continue;
            }
            if (!grow) s->skip = s->sc->streamed;
            next.push_back(s);
        }
        round.swap(next);
    }
    return DANN_OK;
}

/* dann_scan_gettuple_many: n scans of one index */
static int scan_gettuple_many(dann_scan *const *scans, int n, int32_t *out_rc, uint32_t *block, uint16_t *offset,
                              uint32_t *node_id, float *dist, std::vector<std::string> *msgs) {
    if (!scans || !out_rc) return fail(DANN_ERR_INVALID_ARG, "dann_scan_gettuple_many: NULL argument");
    if (n < 1 || n > 65536) return fail(DANN_ERR_INVALID_ARG, "dann_scan_gettuple_many: n = %d outside 1..65536", n);
    for (int i = 0; i < n; i++)
        if (!scans[i]) return fail(DANN_ERR_INVALID_ARG, "dann_scan_gettuple_many: scan %d is NULL", i);
    dann_index *ix = scans[0]->ix;
    for (int i = 1; i < n; i++)
        if (scans[i]->ix != ix) return fail(DANN_ERR_INVALID_ARG, "dann_scan_gettuple_many: scans 0 and %d belong to different indexes", i);
    {
        std::vector<dann_scan *> sorted(scans, scans + n);
        std::sort(sorted.begin(), sorted.end(), std::less<dann_scan *>());
        if (std::adjacent_find(sorted.begin(), sorted.end()) != sorted.end())
            return fail(DANN_ERR_INVALID_ARG, "dann_scan_gettuple_many: a scan appears twice");
    }
    for (int i = 0; i < n; i++)
        if (!scans[i]->active) return fail(DANN_ERR_STATE, "dann_scan_gettuple_many: scan %d has not been rescanned", i);
    int rc = check_live(ix);
    if (rc) return rc;
    std::lock_guard<std::mutex> lk(ix->mu);
    return scan_gettuple_many_locked(ix, scans, n, out_rc, block, offset, node_id, dist, msgs);
}

extern "C" int dann_scan_gettuple_many(dann_scan *const *scans, int n, int32_t *out_rc, uint32_t *block, uint16_t *offset,
                                       uint32_t *node_id, float *dist) try {
    return scan_gettuple_many(scans, n, out_rc, block, offset, node_id, dist, nullptr);
} DANN_CATCH

extern "C" int dann_scan_stats(dann_scan *sc, dann_query_stats *out) try {
    if (!sc || !out) return fail(DANN_ERR_INVALID_ARG, "dann_scan_stats: NULL argument");
    *out = sc->stats;
    return DANN_OK;
} DANN_CATCH

extern "C" int dann_scan_workspace(dann_scan *sc, dann_scan_workspace_info *out) try {
    if (!sc || !out) return fail(DANN_ERR_INVALID_ARG, "dann_scan_workspace: NULL argument");
    *out = dann_scan_workspace_info{};
    out->mode = sc->deep ? 1u : 0u;
    out->regrows = sc->regrows;
    out->growths = sc->growths;
    const DevBuf *bufs[] = DANN_SCAN_BUFS(sc);
    for (const DevBuf *b : bufs) out->device_bytes += b->cap;
    return DANN_OK;
} DANN_CATCH

extern "C" void dann_scan_end(dann_scan *sc) {
    if (!sc) return;
    cudaSetDevice(sc->ix->device);
    scan_release(sc);
    cudaGetLastError();
    delete sc;
}

/* ------------------------------------------------------------------------------------ */
/* query coalescing for process-per-connection hosts (SURVEY.md §8f row 4)                */
#include "dann_coalescer.h"
#include "dann_group.h"

/* ------------------------------------------------------------------------------------ */
/* a table split into shards: every shard's batch, then one merge on the primary device   */
/* the merge launch lives in this file, not in dann_shards.h: tests/simt/cu2cpp.py rewrites this file's launches only */
static cudaError_t launch_shard_merge(const ShardMergeArgs &a, int sm_count, cudaStream_t st) {
    const unsigned grid = (unsigned)std::max(1, std::min<int>((int)((a.B + DANN_MERGE_WARPS - 1) / DANN_MERGE_WARPS), sm_count));
    dann_shard_merge_kernel<<<grid, DANN_MERGE_WARPS * 32, 0, st>>>(a);
    return cudaGetLastError();
}
#include "dann_shards.h"

/* ------------------------------------------------------------------------------------ */
/* reading an index relation file (SURVEY.md §8f row 2): host only                       */
#include "dann_pgreader.h"

struct dann_pg_relation {
    dannpg::Relation rel;
};

extern "C" int dann_pg_relation_open(const char *path, dann_pg_relation **out) try {
    if (!path || !out) return fail(DANN_ERR_INVALID_ARG, "dann_pg_relation_open: NULL argument");
    *out = nullptr;
    dann_pg_relation *r = new dann_pg_relation();
    const int rc = dannpg::open_relation(path, &r->rel);
    if (rc != DANN_OK) {
        const std::string msg = r->rel.err;
        delete r;
        return fail(rc, "dann_pg_relation_open: %s", msg.c_str());
    }
    *out = r;
    return DANN_OK;
} DANN_CATCH

extern "C" void dann_pg_relation_close(dann_pg_relation *rel) { delete rel; }

extern "C" int dann_pg_relation_stat(const dann_pg_relation *rel, dann_pg_relation_info *out) try {
    if (!rel || !out) return fail(DANN_ERR_INVALID_ARG, "dann_pg_relation_stat: NULL argument");
    dannpg::stat_relation(rel->rel, out);
    return DANN_OK;
} DANN_CATCH

extern "C" int dann_pg_read_chain(const dann_pg_relation *rel, uint32_t block, uint16_t offset, int page_type, void *buf,
                                  size_t cap, size_t *len) try {
    if (!rel || !len || (cap && !buf)) return fail(DANN_ERR_INVALID_ARG, "dann_pg_read_chain: NULL argument");
    std::vector<unsigned char> bytes;
    std::string err;
    const int rc = dannpg::read_chain(rel->rel, block, offset, page_type, bytes, err);
    if (rc != DANN_OK) return fail(rc, "dann_pg_read_chain (%u,%u): %s", block, (unsigned)offset, err.c_str());
    *len = bytes.size();
    if (cap) memcpy(buf, bytes.data(), std::min(cap, bytes.size()));
    return DANN_OK;
} DANN_CATCH

static int pg_extract(const dann_pg_relation *rel, const dann_pg_meta *meta, bool plain, dann_pg_snapshot **out, const char *who) {
    if (!rel || !meta || !out) return fail(DANN_ERR_INVALID_ARG, "%s: NULL argument", who);
    *out = nullptr;
    dannpg::SbqOut *o = new dannpg::SbqOut();
    memset(&o->pub, 0, sizeof o->pub);
    std::string err;
    int rc;
    try {
        rc = dannpg::extract_nodes(rel->rel, meta, plain, o, err);
    } catch (...) {
        delete o;
        throw;
    }
    if (rc != DANN_OK) {
        delete o;
        return fail(rc, "%s: %s", who, err.c_str());
    }
    o->pub.self = o;
    *out = &o->pub;
    return DANN_OK;
}

extern "C" int dann_pg_extract_sbq(const dann_pg_relation *rel, const dann_pg_meta *meta, dann_pg_snapshot **out) try {
    return pg_extract(rel, meta, false, out, "dann_pg_extract_sbq");
} DANN_CATCH

extern "C" int dann_pg_extract_plain(const dann_pg_relation *rel, const dann_pg_meta *meta, dann_pg_snapshot **out) try {
    return pg_extract(rel, meta, true, out, "dann_pg_extract_plain");
} DANN_CATCH

extern "C" void dann_pg_snapshot_free(dann_pg_snapshot *s) {
    if (s) delete static_cast<dannpg::SbqOut *>(s->self);
}

extern "C" int dann_pg_heap_fetch_vectors(const dann_pg_relation *heap, const dann_pg_relation *toast, const dann_pg_heap_layout *layout,
                                          const uint64_t *heap_tid, uint32_t n, float *out, uint32_t *n_missing) try {
    if (!heap || !layout || (n && (!heap_tid || !out)) || !layout->dim || (layout->natts_before && (!layout->attlen || !layout->attalign)))
        return fail(DANN_ERR_INVALID_ARG, "dann_pg_heap_fetch_vectors: bad argument");
    uint32_t missing = 0;
    std::string err;
    const int rc = dannpg::fetch_vectors(heap->rel, toast ? &toast->rel : nullptr, layout, heap_tid, n, out, &missing, err);
    if (rc != DANN_OK) return fail(rc, "dann_pg_heap_fetch_vectors: %s", err.c_str());
    if (n_missing) *n_missing = missing;
    return DANN_OK;
} DANN_CATCH
