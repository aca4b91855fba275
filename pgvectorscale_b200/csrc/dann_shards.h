// dann_shards.h — a table split into shards (include/diskann_b200.h, "a table split into shards").  Every shard is an
// ordinary dann_index over a disjoint set of rows; a batch runs the host-buffer search on every shard (one worker
// thread per distinct device, on WorkerLoop of dann_group.h), each worker copies its shards' rows into staging on the
// primary device (shard 0's), and dann_shard_merge_kernel (dann_shards.cuh) merges them there.  No graph hop crosses a
// device; only the merged k rows per query cross PCIe.
// A sharded scan (dann_shards_scan) is one dann_scan per shard whose rows are merged on the host, one row per call; its
// first step advances every device's shards in one dann_scan_gettuple_many round (scan_gettuple_many_locked).
// Included at the end of diskann_b200.cu, after dann_group.h and launch_shard_merge().
#pragma once

/* failures of the handle's own CUDA calls (staging, merge, result copies) poison the handle, not a shard */
#define SK(call)                                                                               \
    do {                                                                                       \
        cudaError_t e_ = (call);                                                               \
        if (e_ != cudaSuccess) {                                                               \
            g->poisoned = (e_ != cudaErrorMemoryAllocation);                                   \
            cudaGetLastError();                                                                \
            return fail(e_ == cudaErrorMemoryAllocation ? DANN_ERR_OOM : DANN_ERR_CUDA,        \
                        "%s:%d %s: %s", __FILE__, __LINE__, #call, cudaGetErrorString(e_));    \
        }                                                                                      \
    } while (0)

/* Copy of a shard's rows into the primary device's staging.  cudaMemcpyPeerAsync needs no peer access to be enabled (the
 * driver stages through the host when the devices cannot reach each other) and is an ordinary device copy when both
 * ends are on the same device.  The CPU SIMT emulator's fake runtime (tests/simt) has one host memory for every fake
 * device and no peer copy, so under DANN_SIMT_EMU the copy is a plain one. */
static cudaError_t copy_to_primary(void *dst, int dst_dev, const void *src, int src_dev, size_t bytes, cudaStream_t st) {
#ifdef DANN_SIMT_EMU
    (void)dst_dev;
    (void)src_dev;
    return cudaMemcpyAsync(dst, src, bytes, cudaMemcpyDeviceToDevice, st);
#else
    return cudaMemcpyPeerAsync(dst, dst_dev, src, src_dev, bytes, st);
#endif
}

struct dann_shards {
    std::vector<dann_index *> ix;         /* shard i */
    std::vector<std::vector<int>> of_dev; /* worker w's shards, ascending: one worker per distinct device */
    int primary = 0;                      /* device of shard 0: staging, merge and result copies */
    int sm_count = 0;
    cudaStream_t stream = nullptr;        /* on the primary device */
    bool poisoned = false;
    /* on the primary device: every shard's rows (shard-major [S][B][k], counts [S][B]) and the merged rows */
    DevBuf st_tid, st_dist, st_count, m_tid, m_dist, m_shard, m_count;
    WorkerLoop loop;
    std::mutex call_mu; /* one batch call at a time per handle */
    /* arguments of the current call (borrowed from the caller for its duration) */
    const float *queries = nullptr;
    const int16_t *labels = nullptr;
    const int32_t *label_off = nullptr;
    int B = 0, k = 0, L = 0, rescore = 0;
    dann_query_stats *out_stats = nullptr;

    /* shard s's batch on its own device, its rows copied to the primary device's staging */
    int run_shard(int s) {
        dann_index *ix = this->ix[(size_t)s];
        int rc = check_live(ix);
        if (rc) return rc;
        std::lock_guard<std::mutex> lk(ix->mu);
        rc = search_batch_staged_locked(ix, queries, labels, label_off, B, k, L, rescore);
        if (rc) return rc;
        cudaStream_t st = ix->stream;
        const size_t nk = (size_t)B * k;
        CK(copy_to_primary(st_tid.as<uint64_t>() + (size_t)s * nk, primary, ix->st_tid.p, ix->device, nk * sizeof(uint64_t), st));
        CK(copy_to_primary(st_dist.as<float>() + (size_t)s * nk, primary, ix->st_dist.p, ix->device, nk * sizeof(float), st));
        CK(copy_to_primary(st_count.as<uint32_t>() + (size_t)s * B, primary, ix->st_count.p, ix->device, (size_t)B * sizeof(uint32_t), st));
        if (out_stats)
            CK(cudaMemcpyAsync(out_stats + (size_t)s * B, ix->st_stats.p, (size_t)B * sizeof(dann_query_stats), cudaMemcpyDeviceToHost, st));
        CK(cudaStreamSynchronize(st));
        return DANN_OK;
    }

    int run(size_t w) {
        for (int s : of_dev[w]) {
            const int rc = run_shard(s);
            if (rc) {
                const std::string keep = g_err;
                return fail(rc, "shard %d: %s", s, keep.c_str());
            }
        }
        return DANN_OK;
    }
};

extern "C" void dann_shards_free(dann_shards *g) {
    if (!g) return;
    g->loop.shutdown();
    for (dann_index *x : g->ix) dann_index_free(x);
    cudaSetDevice(g->primary);
    DevBuf *bufs[] = {&g->st_tid, &g->st_dist, &g->st_count, &g->m_tid, &g->m_dist, &g->m_shard, &g->m_count};
    for (DevBuf *b : bufs) b->release();
    if (g->stream) cudaStreamDestroy(g->stream);
    cudaGetLastError();
    delete g;
}

extern "C" int dann_shards_create(const dann_snapshot_desc *const *shards, int nshards, const int *devices, dann_shards **out) try {
    if (!shards || !out || nshards < 1 || nshards > DANN_SHARDS_MAX)
        return fail(DANN_ERR_INVALID_ARG, "dann_shards_create: bad argument (1..%d shards)", DANN_SHARDS_MAX);
    *out = nullptr;
    for (int i = 0; i < nshards; i++) {
        const dann_snapshot_desc *a = shards[0], *b = shards[i];
        if (!b) return fail(DANN_ERR_INVALID_ARG, "dann_shards_create: shard %d is NULL", i);
        if (b->dim != a->dim || b->dim_index != a->dim_index || b->distance_type != a->distance_type ||
            !b->has_labels != !a->has_labels)
            return fail(DANN_ERR_INVALID_ARG, "dann_shards_create: shard %d differs from shard 0 in dim, dim_index, "
                        "distance_type or has_labels", i);
    }
    dann_shards *g = new dann_shards();
    g->ix.assign((size_t)nshards, nullptr);
    std::vector<int> devs;
    for (int i = 0; i < nshards; i++) {
        const int dev = devices ? devices[i] : i;
        int rc = dann_index_load(shards[i], dev, &g->ix[(size_t)i]);
        if (rc) {
            const std::string keep = g_err;
            dann_shards_free(g); /* frees the shards loaded so far */
            return fail(rc, "dann_shards_create: shard %d (device %d): %s", i, dev, keep.c_str());
        }
        const size_t w = (size_t)(std::find(devs.begin(), devs.end(), dev) - devs.begin());
        if (w == devs.size()) {
            devs.push_back(dev);
            g->of_dev.emplace_back();
        }
        g->of_dev[w].push_back(i);
    }
    g->primary = g->ix[0]->device;
    g->sm_count = g->ix[0]->sm_count;
    const cudaError_t e = [&] {
        cudaError_t r = cudaSetDevice(g->primary);
        return r == cudaSuccess ? cudaStreamCreateWithFlags(&g->stream, cudaStreamNonBlocking) : r;
    }();
    if (e != cudaSuccess) {
        cudaGetLastError();
        dann_shards_free(g);
        return fail(DANN_ERR_CUDA, "dann_shards_create: merge stream on device %d: %s", devs[0], cudaGetErrorString(e));
    }
    g->loop.start(g->of_dev.size(), [g](size_t w) { return g->run(w); });
    *out = g;
    return DANN_OK;
} DANN_CATCH

extern "C" int dann_shards_count(const dann_shards *g) { return g ? (int)g->ix.size() : 0; }

extern "C" dann_index *dann_shards_index(dann_shards *g, int i) {
    return (g && i >= 0 && (size_t)i < g->ix.size()) ? g->ix[(size_t)i] : nullptr;
}

extern "C" int dann_shards_search_batch(dann_shards *g, const float *queries, const int16_t *labels, const int32_t *label_off,
                                        int B, int k, int search_list_size, int rescore,
                                        uint64_t *out_tid, float *out_dist, int32_t *out_shard, uint32_t *out_count,
                                        dann_query_stats *out_stats) try {
    if (!g || B <= 0 || k <= 0 || !queries || !out_tid) return fail(DANN_ERR_INVALID_ARG, "dann_shards_search_batch: bad argument");
    if (rescore == 0) return fail(DANN_ERR_INVALID_ARG, "dann_shards_search_batch: rescore 0 leaves the rows without a distance to merge on");
    std::lock_guard<std::mutex> one(g->call_mu);
    if (g->poisoned) return fail(DANN_ERR_CUDA, "shards handle is poisoned by an earlier CUDA error");
    const size_t S = g->ix.size(), nk = (size_t)B * k;
    SK(cudaSetDevice(g->primary));
    SK(g->st_tid.reserve(S * nk * sizeof(uint64_t)));
    SK(g->st_dist.reserve(S * nk * sizeof(float)));
    SK(g->st_count.reserve(S * B * sizeof(uint32_t)));
    SK(g->m_tid.reserve(nk * sizeof(uint64_t)));
    SK(g->m_dist.reserve(nk * sizeof(float)));
    SK(g->m_shard.reserve(nk * sizeof(int32_t)));
    SK(g->m_count.reserve((size_t)B * sizeof(uint32_t)));
    g->queries = queries;
    g->labels = labels;
    g->label_off = label_off;
    g->B = B;
    g->k = k;
    g->L = search_list_size;
    g->rescore = rescore;
    g->out_stats = out_stats;
    g->loop.call();
    for (const WorkerLoop::Worker &x : g->loop.w)
        if (x.rc) return fail(x.rc, "%s", x.err.c_str());

    SK(cudaSetDevice(g->primary));
    ShardMergeArgs a;
    a.tid = g->st_tid.as<uint64_t>();
    a.dist = g->st_dist.as<float>();
    a.count = g->st_count.as<uint32_t>();
    a.S = (uint32_t)S;
    a.B = (uint32_t)B;
    a.k = (uint32_t)k;
    a.out_tid = g->m_tid.as<uint64_t>();
    a.out_dist = g->m_dist.as<float>();
    a.out_shard = g->m_shard.as<int32_t>();
    a.out_count = g->m_count.as<uint32_t>();
    SK(launch_shard_merge(a, g->sm_count, g->stream));
    SK(cudaMemcpyAsync(out_tid, g->m_tid.p, nk * sizeof(uint64_t), cudaMemcpyDeviceToHost, g->stream));
    if (out_dist) SK(cudaMemcpyAsync(out_dist, g->m_dist.p, nk * sizeof(float), cudaMemcpyDeviceToHost, g->stream));
    if (out_shard) SK(cudaMemcpyAsync(out_shard, g->m_shard.p, nk * sizeof(int32_t), cudaMemcpyDeviceToHost, g->stream));
    if (out_count) SK(cudaMemcpyAsync(out_count, g->m_count.p, (size_t)B * sizeof(uint32_t), cudaMemcpyDeviceToHost, g->stream));
    SK(cudaStreamSynchronize(g->stream));
    return DANN_OK;
} DANN_CATCH

#undef SK

/* ---- streaming scan of a sharded table (include/diskann_b200.h, "streaming scan of a sharded table") ---- */

/* f32::total_cmp as an unsigned key: total_ukey of dann_device.cuh, on the host */
static uint32_t host_total_ukey(float f) {
    uint32_t b;
    memcpy(&b, &f, sizeof b);
    return (b >> 31) ? ~b : (b | 0x80000000u);
}

struct dann_shards_scan {
    dann_shards *g = nullptr;
    std::vector<dann_scan *> sc; /* shard s's own scan */
    struct Head {
        uint32_t block = 0, node = 0;
        uint16_t offset = 0;
        float dist = 0.0f;
        bool live = false; /* a row of the shard is waiting to be merged */
    };
    std::vector<Head> head;
    int step_next = -1;  /* the shard whose head the last call returned: the next call steps it */
    bool first = true;   /* no shard has stepped since the rescan */
    bool active = false; /* rescanned, and no call has failed since */
};

extern "C" void dann_shards_scan_end(dann_shards_scan *ss) {
    if (!ss) return;
    for (dann_scan *sc : ss->sc) dann_scan_end(sc);
    delete ss;
}

extern "C" int dann_shards_scan_begin(dann_shards *g, dann_shards_scan **out) try {
    if (!g || !out) return fail(DANN_ERR_INVALID_ARG, "dann_shards_scan_begin: NULL argument");
    *out = nullptr;
    dann_shards_scan *ss = new dann_shards_scan();
    ss->g = g;
    ss->head.resize(g->ix.size());
    ss->sc.reserve(g->ix.size());
    for (dann_index *ix : g->ix) {
        dann_scan *sc = nullptr;
        const int rc = dann_scan_begin(ix, &sc);
        if (rc) {
            dann_shards_scan_end(ss);
            return rc;
        }
        ss->sc.push_back(sc);
    }
    *out = ss;
    return DANN_OK;
} DANN_CATCH

/* the failure of shard s's own call, with g_err as its message */
static int shard_failed(int s, int rc) {
    const std::string keep = g_err;
    return fail(rc, "shard %d: %s", s, keep.c_str());
}

extern "C" int dann_shards_scan_rescan(dann_shards_scan *ss, const float *query, const int16_t *labels, int nlabels,
                                       int search_list_size, int rescore) try {
    if (!ss) return fail(DANN_ERR_INVALID_ARG, "dann_shards_scan_rescan: NULL scan");
    int rc = scan_rescan_check(labels, nlabels, search_list_size, rescore);
    if (rc) return rc;
    if (rescore == 0) return fail(DANN_ERR_INVALID_ARG, "dann_shards_scan_rescan: rescore 0 leaves the rows without a distance to merge on");
    dann_shards *g = ss->g;
    ss->active = false;
    ss->first = true;
    ss->step_next = -1;
    for (dann_shards_scan::Head &h : ss->head) h = dann_shards_scan::Head{};
    std::vector<std::unique_lock<std::mutex>> locks;
    locks.reserve(g->ix.size());
    for (dann_index *ix : g->ix) locks.emplace_back(ix->mu); /* ascending shard order */
    /* each device's shards are enqueued on the stream of its first shard, then every device is waited for once */
    for (const std::vector<int> &dev : g->of_dev) {
        cudaStream_t st = g->ix[(size_t)dev[0]]->stream;
        for (int s : dev) {
            rc = check_live(g->ix[(size_t)s]);
            if (!rc) rc = scan_rescan_enqueue(ss->sc[(size_t)s], query, labels, nlabels, search_list_size, rescore, st);
            if (rc) return shard_failed(s, rc);
        }
    }
    std::vector<dann_scan *> scans;
    for (const std::vector<int> &dev : g->of_dev) {
        dann_index *lead = g->ix[(size_t)dev[0]];
        scans.clear();
        for (int s : dev) scans.push_back(ss->sc[(size_t)s]);
        rc = check_live(lead);
        if (!rc) rc = scan_rescan_wait(lead, lead->stream, scans.data(), scans.size());
        if (rc) return shard_failed(dev[0], rc);
    }
    ss->active = true;
    return DANN_OK;
} DANN_CATCH

/* The first step of the scans of device w's shards: one dann_scan_gettuple_many round (or a few, when a scan regrows)
 * that carries all of them, on the stream of the device's first shard, under the shards' mutexes in ascending order. */
static int shards_scan_first_step_on(dann_shards_scan *ss, size_t w) {
    dann_shards *g = ss->g;
    const std::vector<int> &dev = g->of_dev[w];
    const size_t n = dev.size();
    std::vector<std::unique_lock<std::mutex>> locks;
    std::vector<dann_scan *> scans;
    locks.reserve(n);
    for (int s : dev) {
        dann_index *ix = g->ix[(size_t)s];
        const int rc = check_live(ix);
        if (rc) return shard_failed(s, rc);
        locks.emplace_back(ix->mu);
        scans.push_back(ss->sc[(size_t)s]);
    }
    std::vector<int32_t> out_rc(n, 0);
    std::vector<uint32_t> block(n), node(n);
    std::vector<uint16_t> offset(n);
    std::vector<float> dist(n);
    std::vector<std::string> msgs;
    int rc = scan_gettuple_many_locked(g->ix[(size_t)dev[0]], scans.data(), (int)n, out_rc.data(), block.data(),
                                       offset.data(), node.data(), dist.data(), &msgs);
    if (rc) return shard_failed(dev[0], rc);
    for (size_t j = 0; j < n; j++) {
        if (out_rc[j] < 0) return fail(out_rc[j], "shard %d: %s", dev[j], msgs[j].c_str());
        ss->head[(size_t)dev[j]] = dann_shards_scan::Head{block[j], node[j], offset[j], dist[j], out_rc[j] == 1};
    }
    return DANN_OK;
}

/* The first step of every shard: one round per device, the devices at the same time (the first on this thread). */
static int shards_scan_first_step(dann_shards_scan *ss) {
    const size_t D = ss->g->of_dev.size();
    std::vector<int> rc(D, DANN_OK);
    std::vector<std::string> err(D);
    auto run = [&](size_t w) {
        try {
            rc[w] = shards_scan_first_step_on(ss, w);
            if (rc[w]) err[w] = g_err; /* thread-local message of this thread */
        } catch (const std::bad_alloc &) {
            rc[w] = DANN_ERR_OOM;
        } catch (...) {
            rc[w] = DANN_ERR_STATE;
        }
    };
    std::vector<std::thread> th;
    th.reserve(D);
    for (size_t w = 1; w < D; w++) th.emplace_back(run, w);
    run(0);
    for (std::thread &t : th) t.join();
    for (size_t w = 0; w < D; w++)
        if (rc[w]) return fail(rc[w], "%s", err[w].empty() ? "host failure in a first step" : err[w].c_str());
    return DANN_OK;
}

extern "C" int dann_shards_scan_gettuple(dann_shards_scan *ss, uint32_t *block, uint16_t *offset, uint32_t *node_id,
                                         float *dist, int32_t *shard) try {
    if (!ss) return fail(DANN_ERR_INVALID_ARG, "dann_shards_scan_gettuple: NULL scan");
    if (!ss->active) return fail(DANN_ERR_STATE, "dann_shards_scan_gettuple before dann_shards_scan_rescan, or after a failed call");
    ss->active = false; /* until this call has succeeded */
    if (ss->first) {
        const int rc = shards_scan_first_step(ss);
        if (rc) return rc;
        ss->first = false;
    } else if (ss->step_next >= 0) {
        const int s = ss->step_next;
        dann_shards_scan::Head &h = ss->head[(size_t)s];
        const int rc = dann_scan_gettuple(ss->sc[(size_t)s], &h.block, &h.offset, &h.node, &h.dist);
        if (rc < 0) return shard_failed(s, rc);
        h.live = rc == 1;
    }
    ss->active = true;
    ss->step_next = -1;
    int best = -1;
    uint32_t best_key = 0;
    for (size_t s = 0; s < ss->head.size(); s++) {
        const dann_shards_scan::Head &h = ss->head[s];
        if (!h.live) continue;
        const uint32_t key = host_total_ukey(h.dist);
        if (best < 0 || key < best_key) { /* ties: the lower shard */
            best = (int)s;
            best_key = key;
        }
    }
    if (best < 0) return 0;
    dann_shards_scan::Head &h = ss->head[(size_t)best];
    if (block) *block = h.block;
    if (offset) *offset = h.offset;
    if (node_id) *node_id = h.node;
    if (dist) *dist = h.dist;
    if (shard) *shard = best;
    h.live = false;
    ss->step_next = best;
    return 1;
} DANN_CATCH

extern "C" int dann_shards_scan_stats(dann_shards_scan *ss, dann_query_stats *out) try {
    if (!ss || !out) return fail(DANN_ERR_INVALID_ARG, "dann_shards_scan_stats: NULL argument");
    for (size_t s = 0; s < ss->sc.size(); s++) out[s] = ss->sc[s]->stats;
    return DANN_OK;
} DANN_CATCH
