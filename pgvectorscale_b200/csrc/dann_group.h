// dann_group.h — query-batch data parallelism inside ONE host process (SURVEY.md §8b/§8e): a group owns one full
// replica of the index per GPU; a batch is cut into contiguous slices (one per device), every device runs the whole
// hot path on its slice, and the "gather" is each device's D2H copy landing directly in the caller's arrays at the
// slice's offset - rows come back in query order without any device-to-device exchange (queries are independent
// units; the graph itself is replicas only, sharding it would put every hop on NVLink).  This is what a Rust host
// (one Postgres backend, or the sidecar that serves many) can call; torch.distributed / NCCL are only needed when
// ranks are separate PROCESSES (pgvectorscale_b200/group.py, bench.py under torchrun).
// Included at the end of diskann_b200.cu (it uses search_batch_host, fail() and DANN_CATCH); pure host code.
#pragma once
#include <condition_variable>
#include <thread>

/* One host thread per worker, driven by generations: each call publishes its arguments, bumps `gen` and waits until
 * every worker has run job(i) for that generation.  dann_group (one worker per replica) and dann_shards (one worker per
 * distinct device) both run on it. */
struct WorkerLoop {
    struct Worker {
        std::thread th;
        int rc = 0;
        std::string err;
        uint64_t seen = 0; /* generation this worker has finished */
    };
    std::vector<Worker> w;
    std::mutex mu;
    std::condition_variable cv_go, cv_done;
    uint64_t gen = 0;
    bool stop = false;
    std::function<int(size_t)> job; /* the work of worker i in the current generation; its error text is g_err */

    void start(size_t n, std::function<int(size_t)> fn) {
        job = std::move(fn);
        w.resize(n);
        for (size_t i = 0; i < n; i++) w[i].th = std::thread([this, i] { run(i); });
    }

    void run(size_t i) {
        Worker &me = w[i];
        uint64_t done = 0;
        std::unique_lock<std::mutex> lk(mu);
        for (;;) {
            cv_go.wait(lk, [&] { return stop || gen != done; });
            if (stop) return;
            const uint64_t g = gen;
            lk.unlock();
            int rc = DANN_OK;
            std::string err;
            try {
                rc = job(i);
                if (rc) err = g_err; /* thread-local message of this worker */
            } catch (const std::bad_alloc &) {
                rc = DANN_ERR_OOM;
            } catch (...) {
                rc = DANN_ERR_STATE;
            }
            lk.lock();
            me.rc = rc;
            try {
                me.err = err;
            } catch (...) {
            }
            done = g;
            me.seen = g;
            cv_done.notify_all();
        }
    }

    /* runs one generation; the caller has published the call's arguments (they are read after `mu` is taken) */
    void call() {
        std::unique_lock<std::mutex> lk(mu);
        const uint64_t g = ++gen;
        cv_go.notify_all();
        cv_done.wait(lk, [&] {
            for (const Worker &x : w)
                if (x.seen != g) return false;
            return true;
        });
    }

    void shutdown() {
        {
            std::lock_guard<std::mutex> lk(mu);
            stop = true;
        }
        cv_go.notify_all();
        for (Worker &x : w)
            if (x.th.joinable()) x.th.join();
    }
};

struct dann_group {
    std::vector<dann_index *> ix;
    std::vector<int> lo, hi; /* each replica's slice of the current call */
    WorkerLoop loop;
    std::mutex call_mu; /* one batch call at a time per group */
    /* arguments of the current call (borrowed from the caller for its duration) */
    const float *queries = nullptr;
    const int16_t *labels = nullptr;
    const int32_t *label_off = nullptr;
    int k = 0, L = 0, rescore = 0;
    const dann_query_params *params = nullptr; /* dann_group_search_batch_mixed; k is then the whole batch's row stride */
    uint32_t dim = 0;
    uint64_t *out_tid = nullptr;
    float *out_dist = nullptr;
    uint32_t *out_count = nullptr;
    dann_query_stats *out_stats = nullptr;

    int run(size_t i) {
        const int l = lo[i], h = hi[i];
        if (h <= l) return DANN_OK;
        const float *q = queries + (size_t)l * dim;
        const int32_t *off = label_off ? label_off + l : nullptr;
        uint64_t *tid = out_tid + (size_t)l * k;
        float *dist = out_dist ? out_dist + (size_t)l * k : nullptr;
        uint32_t *count = out_count ? out_count + l : nullptr;
        dann_query_stats *stats = out_stats ? out_stats + l : nullptr;
        if (!params) return search_batch_host(ix[i], q, labels, off, h - l, k, L, rescore, tid, dist, nullptr, count, stats);
        /* the slice's own parameters, with the rows laid out at the whole batch's stride */
        int rc = check_live(ix[i]);
        if (rc) return rc;
        BatchParams bp;
        rc = mixed_params(ix[i], h - l, params + l, labels, off, k, &bp);
        return rc ? rc : search_batch_host(ix[i], q, labels, off, h - l, bp, tid, dist, nullptr, count, stats);
    }
};

/* contiguous, balanced slice [lo, hi) of `total` queries for device `r` of `world` (the first ranks take the remainder;
 * the same rule as pgvectorscale_b200/group.py shard_bounds) */
static void group_bounds(int total, int world, int r, int *lo, int *hi) {
    const int base = total / world, rem = total % world;
    *lo = r * base + std::min(r, rem);
    *hi = *lo + base + (r < rem ? 1 : 0);
}

extern "C" void dann_group_free(dann_group *g) {
    if (!g) return;
    g->loop.shutdown();
    for (dann_index *x : g->ix) dann_index_free(x);
    delete g;
}

extern "C" int dann_group_create(const dann_snapshot_desc *snap, int ndev, const int *devices, dann_group **out) try {
    if (!snap || !out || ndev < 1 || ndev > 64) return fail(DANN_ERR_INVALID_ARG, "dann_group_create: bad argument");
    dann_group *g = new dann_group();
    g->ix.assign((size_t)ndev, nullptr);
    g->lo.assign((size_t)ndev, 0);
    g->hi.assign((size_t)ndev, 0);
    for (int i = 0; i < ndev; i++) {
        const int dev = devices ? devices[i] : i;
        int rc = dann_index_load(snap, dev, &g->ix[(size_t)i]);
        if (rc) {
            const std::string keep = g_err;
            dann_group_free(g); /* frees the replicas loaded so far */
            return fail(rc, "dann_group_create: replica %d (device %d): %s", i, dev, keep.c_str());
        }
    }
    g->dim = g->ix[0]->v.dim;
    g->loop.start(g->ix.size(), [g](size_t i) { return g->run(i); });
    *out = g;
    return DANN_OK;
} DANN_CATCH

extern "C" int dann_group_size(const dann_group *g) { return g ? (int)g->ix.size() : 0; }

extern "C" dann_index *dann_group_replica(dann_group *g, int i) {
    return (g && i >= 0 && (size_t)i < g->ix.size()) ? g->ix[(size_t)i] : nullptr;
}

/* one batch call over the replicas; the caller holds call_mu and has set k / L / rescore / params */
static int group_call(dann_group *g, int B, const float *queries, const int16_t *labels, const int32_t *label_off,
                      uint64_t *out_tid, float *out_dist, uint32_t *out_count, dann_query_stats *out_stats) {
    g->queries = queries;
    g->labels = labels;
    g->label_off = label_off;
    g->out_tid = out_tid;
    g->out_dist = out_dist;
    g->out_count = out_count;
    g->out_stats = out_stats;
    const int world = (int)g->ix.size();
    for (int r = 0; r < world; r++) group_bounds(B, world, r, &g->lo[(size_t)r], &g->hi[(size_t)r]);
    g->loop.call();
    for (int r = 0; r < world; r++)
        if (g->loop.w[(size_t)r].rc) return fail(g->loop.w[(size_t)r].rc, "replica %d: %s", r, g->loop.w[(size_t)r].err.c_str());
    return DANN_OK;
}

extern "C" int dann_group_search_batch(dann_group *g, const float *queries, const int16_t *labels, const int32_t *label_off,
                                       int B, int k, int search_list_size, int rescore, uint64_t *out_tid, float *out_dist,
                                       uint32_t *out_count, dann_query_stats *out_stats) try {
    if (!g || B <= 0 || k <= 0 || !queries || !out_tid) return fail(DANN_ERR_INVALID_ARG, "dann_group_search_batch: bad argument");
    std::lock_guard<std::mutex> one(g->call_mu);
    g->params = nullptr;
    g->k = k;
    g->L = search_list_size;
    g->rescore = rescore;
    return group_call(g, B, queries, labels, label_off, out_tid, out_dist, out_count, out_stats);
} DANN_CATCH

/* The slices are those of dann_group_search_batch, params sliced with the queries; the whole batch is checked on replica
 * 0 first (the replicas are copies of one index), so a refused batch runs nowhere. */
extern "C" int dann_group_search_batch_mixed(dann_group *g, const float *queries, const int16_t *labels, const int32_t *label_off,
                                             const dann_query_params *params, int B, uint64_t *out_tid, float *out_dist,
                                             uint32_t *out_count, dann_query_stats *out_stats) try {
    if (!g || !queries || !out_tid) return fail(DANN_ERR_INVALID_ARG, "dann_group_search_batch_mixed: bad argument");
    BatchParams bp;
    int rc = mixed_params(g->ix[0], B, params, labels, label_off, 0, &bp);
    if (rc) return rc;
    std::lock_guard<std::mutex> one(g->call_mu);
    g->params = params;
    g->k = bp.k;
    return group_call(g, B, queries, labels, label_off, out_tid, out_dist, out_count, out_stats);
} DANN_CATCH
