// dann_coalescer.h — query coalescing for process-per-connection hosts (SURVEY.md §8f row 4).
//
// Postgres runs one backend per connection and `amcanparallel = false` (mod.rs:63): every backend has exactly one
// index scan in flight, one query at a time, while the GPU reaches its throughput on batches (one query = one warp
// pair).  The coalescer is the piece a sidecar that owns the HBM-resident index would put between the two: any number
// of host threads (one per connected backend) submit single queries and block; a dispatcher thread gathers what
// arrives within a short window into ONE dann_search_batch_mixed call and hands every caller its own rows.  Queries are
// independent units, whatever their k, search_list_size, rescore or key, so each caller gets exactly what a private
// scan would have returned.
// The same dispatcher coalesces amgettuple calls: the gettuple requests of a window (any scans of the index, whatever
// their search_list_size, rescore or key) become ONE dann_scan_gettuple_many call, and each caller gets the row its
// own dann_scan_gettuple would have returned.  Search and gettuple requests never share a dispatch.
// Included at the end of diskann_b200.cu (it uses search_batch_host, scan_gettuple_many and fail()); pure host code.
#pragma once
#include <chrono>
#include <condition_variable>
#include <deque>
#include <thread>

struct CoalescedRequest {
    const float *query;
    const int16_t *labels;
    int nlabels; /* < 0: no scan key */
    int k, L, rescore;
    uint64_t *out_tid;
    float *out_dist;
    uint32_t *out_count;
    dann_query_stats *out_stats;
    /* gettuple request (scan != NULL): one amgettuple of `scan`, outputs as dann_scan_gettuple's */
    dann_scan *scan = nullptr;
    uint32_t *block = nullptr;
    uint16_t *offset = nullptr;
    uint32_t *node_id = nullptr;
    float *dist = nullptr;
    int row = 0; /* 1 row, 0 end of scan */
    int rc = 0;
    bool done = false;
    std::string err;
};

struct dann_coalescer {
    dann_index *ix = nullptr;
    int max_batch = 256;
    int max_wait_us = 200;
    std::mutex mu;
    std::condition_variable cv_work, cv_done, cv_idle;
    int callers = 0; /* threads inside dann_coalescer_search (guarded by mu) */
    std::deque<CoalescedRequest *> queue;
    bool stop = false;
    std::thread worker;
    uint64_t n_batches = 0, n_queries = 0, max_seen = 0;

    static bool compatible(const CoalescedRequest *a, const CoalescedRequest *b) {
        /* gettuple requests all go into one dann_scan_gettuple_many call, search requests into one mixed batch */
        return (a->scan != nullptr) == (b->scan != nullptr);
    }

    void run() {
        std::unique_lock<std::mutex> lk(mu);
        for (;;) {
            cv_work.wait(lk, [&] { return stop || !queue.empty(); });
            if (stop && queue.empty()) return;
            /* the window opens with the first request: wait for company, but never longer than max_wait_us */
            const auto deadline = std::chrono::steady_clock::now() + std::chrono::microseconds(max_wait_us);
            cv_work.wait_until(lk, deadline, [&] { return stop || (int)queue.size() >= max_batch; });
            std::vector<CoalescedRequest *> batch;
            CoalescedRequest *head = queue.front();
            try {
                batch.reserve(std::min<size_t>(queue.size(), (size_t)max_batch));
            } catch (...) { /* no memory for the batch list: fail the oldest request, keep serving */
                queue.pop_front();
                head->rc = DANN_ERR_OOM;
                head->err = "host allocation failed";
                head->done = true;
                cv_done.notify_all();
                continue;
            }
            for (auto it = queue.begin(); it != queue.end() && (int)batch.size() < max_batch;) {
                if (compatible(head, *it)) {
                    batch.push_back(*it); /* reserved above: does not allocate */
                    it = queue.erase(it);
                } else {
                    ++it; /* the other kind of request: next window */
                }
            }
            lk.unlock();
            /* the dispatcher is a std::thread: an exception escaping it would std::terminate the host process (the
             * sidecar and every backend behind it), so whatever execute() throws becomes the batch's status */
            int xrc = 0;
            try {
                execute(batch);
            } catch (const std::bad_alloc &) {
                xrc = DANN_ERR_OOM;
            } catch (...) {
                xrc = DANN_ERR_STATE;
            }
            lk.lock();
            n_batches++;
            n_queries += batch.size();
            max_seen = std::max<uint64_t>(max_seen, batch.size());
            for (CoalescedRequest *r : batch) {
                if (xrc) {
                    r->rc = xrc;
                    try {
                        r->err = xrc == DANN_ERR_OOM ? "host allocation failed" : "unexpected C++ exception in the coalescer";
                    } catch (...) {
                    }
                }
                r->done = true;
            }
            cv_done.notify_all();
        }
    }

    void execute(std::vector<CoalescedRequest *> &batch) {
        if (batch[0]->scan) return execute_gettuple(batch);
        const int B = (int)batch.size();
        const uint32_t dim = ix->v.dim;
        std::vector<float> q((size_t)B * dim);
        std::vector<int16_t> lab;
        std::vector<int32_t> off(1, 0);
        std::vector<dann_query_params> params((size_t)B);
        for (int b = 0; b < B; b++) {
            const CoalescedRequest *r = batch[b];
            memcpy(q.data() + (size_t)b * dim, r->query, (size_t)dim * sizeof(float));
            if (r->nlabels > 0) lab.insert(lab.end(), r->labels, r->labels + r->nlabels);
            off.push_back((int32_t)lab.size());
            params[(size_t)b] = dann_query_params{r->k, r->L, r->rescore, r->nlabels >= 0 ? 1 : 0};
        }
        if (lab.empty()) lab.push_back(0);
        /* each request was checked on its own at submission, so the batch is refused only if the index is */
        int rc = check_live(ix);
        BatchParams bp;
        if (!rc) rc = mixed_params(ix, B, params.data(), lab.data(), off.data(), 0, &bp);
        const int k = bp.k;
        std::vector<uint64_t> tid((size_t)B * k);
        std::vector<float> dist((size_t)B * k);
        std::vector<uint32_t> count(B);
        std::vector<dann_query_stats> stats(B);
        if (!rc)
            rc = search_batch_host(ix, q.data(), lab.data(), off.data(), B, bp, tid.data(), dist.data(), nullptr, count.data(),
                                   stats.data());
        const std::string err = rc ? g_err : std::string();
        for (int b = 0; b < B; b++) {
            CoalescedRequest *r = batch[b];
            r->rc = rc;
            r->err = err;
            if (rc) continue;
            memcpy(r->out_tid, tid.data() + (size_t)b * k, (size_t)r->k * sizeof(uint64_t));
            if (r->out_dist) memcpy(r->out_dist, dist.data() + (size_t)b * k, (size_t)r->k * sizeof(float));
            if (r->out_count) *r->out_count = count[b];
            if (r->out_stats) *r->out_stats = stats[b];
        }
    }

    void execute_gettuple(std::vector<CoalescedRequest *> &batch) {
        /* a scan is single-threaded: a second call on a scan that already has one in this dispatch breaks that, and is
         * refused alone (the first call, and everyone else's, go ahead) */
        std::vector<std::pair<dann_scan *, int>> order(batch.size());
        for (size_t i = 0; i < batch.size(); i++) order[i] = {batch[i]->scan, (int)i};
        std::sort(order.begin(), order.end(), [](const std::pair<dann_scan *, int> &a, const std::pair<dann_scan *, int> &b) {
            return std::less<dann_scan *>()(a.first, b.first) || (a.first == b.first && a.second < b.second);
        });
        std::vector<char> dup(batch.size(), 0);
        for (size_t j = 1; j < order.size(); j++)
            if (order[j].first == order[j - 1].first) dup[order[j].second] = 1;
        std::vector<CoalescedRequest *> run;
        run.reserve(batch.size());
        for (size_t i = 0; i < batch.size(); i++) {
            if (!dup[i]) {
                run.push_back(batch[i]);
                continue;
            }
            batch[i]->rc = DANN_ERR_INVALID_ARG;
            batch[i]->err = "dann_coalescer_gettuple: another call on the same scan is in flight (a scan is single-threaded)";
        }
        const int n = (int)run.size();
        std::vector<dann_scan *> scans(n);
        std::vector<int32_t> rcs(n, 0);
        std::vector<uint32_t> block(n, 0), node(n, 0);
        std::vector<uint16_t> offset(n, 0);
        std::vector<float> dist(n, 0.0f);
        std::vector<std::string> msgs;
        for (int i = 0; i < n; i++) scans[i] = run[i]->scan;
        const int rc = scan_gettuple_many(scans.data(), n, rcs.data(), block.data(), offset.data(), node.data(), dist.data(), &msgs);
        const std::string err = rc ? g_err : std::string(); /* the call's error */
        for (int i = 0; i < n; i++) {
            CoalescedRequest *r = run[i];
            r->rc = rc ? rc : std::min(rcs[i], 0);
            if (r->rc) {
                r->err = rc ? err : msgs[i]; /* a scan's own failure: its own message */
                continue;
            }
            r->row = rcs[i];
            if (!r->row) continue;
            if (r->block) *r->block = block[i];
            if (r->offset) *r->offset = offset[i];
            if (r->node_id) *r->node_id = node[i];
            if (r->dist) *r->dist = dist[i];
        }
    }

    /* queue `r` and block until the dispatcher has answered it */
    int submit(CoalescedRequest &r) {
        std::unique_lock<std::mutex> lk(mu);
        if (stop) return fail(DANN_ERR_STATE, "coalescer is shutting down");
        /* `callers` keeps dann_coalescer_destroy from deleting the object while this thread still holds (or is about
         * to re-acquire, inside cv_done.wait) its mutex */
        struct Leave {
            dann_coalescer *c;
            ~Leave() {
                if (--c->callers == 0) c->cv_idle.notify_all();
            }
        };
        callers++;
        Leave leave{this}; /* destroyed before lk: runs under the lock */
        queue.push_back(&r);
        cv_work.notify_one();
        cv_done.wait(lk, [&] { return r.done; });
        if (r.rc) return fail(r.rc, "%s", r.err.c_str());
        return DANN_OK;
    }
};

extern "C" int dann_coalescer_create(dann_index *ix, int max_batch, int max_wait_us, dann_coalescer **out) try {
    if (!ix || !out) return fail(DANN_ERR_INVALID_ARG, "dann_coalescer_create: NULL argument");
    if (max_batch < 1 || max_batch > 65536 || max_wait_us < 0) return fail(DANN_ERR_INVALID_ARG, "dann_coalescer_create: bad limits");
    dann_coalescer *c = new (std::nothrow) dann_coalescer();
    if (!c) return fail(DANN_ERR_OOM, "host allocation failed");
    c->ix = ix;
    c->max_batch = max_batch;
    c->max_wait_us = max_wait_us;
    c->worker = std::thread([c] { c->run(); });
    *out = c;
    return DANN_OK;
} DANN_CATCH

extern "C" int dann_coalescer_search(dann_coalescer *c, const float *query, const int16_t *labels, int nlabels, int k,
                                     int search_list_size, int rescore, uint64_t *out_tid, float *out_dist,
                                     uint32_t *out_count, dann_query_stats *out_stats) try {
    if (!c || !query || !out_tid || k <= 0) return fail(DANN_ERR_INVALID_ARG, "dann_coalescer_search: bad argument");
    if (nlabels > 0 && !labels) return fail(DANN_ERR_INVALID_ARG, "labels is NULL but nlabels > 0");
    /* a request the index would refuse is refused here, for this caller alone: the rest of its window goes ahead */
    int checked_rescore = rescore;
    size_t smem = 0;
    const int rc = check_query(c->ix, "", k, search_list_size, &checked_rescore, nlabels >= 0, &smem);
    if (rc) return rc;
    CoalescedRequest r;
    r.query = query;
    r.labels = labels;
    r.nlabels = nlabels;
    r.k = k;
    r.L = search_list_size;
    r.rescore = rescore;
    r.out_tid = out_tid;
    r.out_dist = out_dist;
    r.out_count = out_count;
    r.out_stats = out_stats;
    return c->submit(r);
} DANN_CATCH

extern "C" int dann_coalescer_gettuple(dann_coalescer *c, dann_scan *sc, uint32_t *block, uint16_t *offset, uint32_t *node_id,
                                       float *dist) try {
    if (!c || !sc) return fail(DANN_ERR_INVALID_ARG, "dann_coalescer_gettuple: NULL argument");
    /* what would fail the whole dispatch is refused here, for this caller alone */
    if (sc->ix != c->ix) return fail(DANN_ERR_INVALID_ARG, "dann_coalescer_gettuple: the scan belongs to another index");
    if (!sc->active) return fail(DANN_ERR_STATE, "dann_coalescer_gettuple before dann_scan_rescan");
    CoalescedRequest r{};
    r.scan = sc;
    r.block = block;
    r.offset = offset;
    r.node_id = node_id;
    r.dist = dist;
    const int rc = c->submit(r);
    return rc ? rc : r.row;
} DANN_CATCH

extern "C" int dann_coalescer_stats(dann_coalescer *c, uint64_t *batches, uint64_t *queries, uint64_t *largest_batch) try {
    if (!c) return fail(DANN_ERR_INVALID_ARG, "NULL coalescer");
    std::lock_guard<std::mutex> lk(c->mu);
    if (batches) *batches = c->n_batches;
    if (queries) *queries = c->n_queries;
    if (largest_batch) *largest_batch = c->max_seen;
    return DANN_OK;
} DANN_CATCH

extern "C" void dann_coalescer_destroy(dann_coalescer *c) {
    if (!c) return;
    {
        std::lock_guard<std::mutex> lk(c->mu);
        c->stop = true;
    }
    c->cv_work.notify_all();
    if (c->worker.joinable()) c->worker.join(); /* drains the queue: every queued request is answered */
    {
        std::unique_lock<std::mutex> lk(c->mu);
        c->cv_idle.wait(lk, [&] { return c->callers == 0; }); /* the answered callers have let go of the mutex */
    }
    delete c;
}
