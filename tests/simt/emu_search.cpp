// emu_search.cpp — runs the beam-search kernel SOURCES (pgvectorscale_b200/csrc/dann_search{,2,3}.cuh) under the CPU
// SIMT emulator with the product's own workspace plan (dann_plan.h), mirroring run_search() in diskann_b200.cu:
// same launch shape, same overflow/retry loop.  TEST INFRASTRUCTURE ONLY (see simt_emu.h); built by
// tests/simt/build_emu.py with g++, never by build.py, never loaded by the package.
#include <cuda_runtime.h> /* resolves to tests/simt/shim/cuda_runtime.h */

#include <string>
#include <vector>

#include "dann_search2.cuh"
#include "dann_search3.cuh"
#include "dann_plan.h"

alignas(128) unsigned char dann_smem[256 * 1024];

typedef void (*emu_kernel)(const SearchArgs);

template <typename T>
static emu_kernel pick1(uint32_t nch) {
    switch (nch) {
        case 1: return dann_search_kernel<T, 1>;
        case 2: return dann_search_kernel<T, 2>;
        case 3: return dann_search_kernel<T, 3>;
        default: return nullptr;
    }
}
template <typename T>
static emu_kernel pick2(uint32_t nch) {
    switch (nch) {
        case 1: return dann_search2_kernel<T, 1>;
        case 2: return dann_search2_kernel<T, 2>;
        case 3: return dann_search2_kernel<T, 3>;
        default: return nullptr;
    }
}
template <typename T, int MAXW>
static emu_kernel pick3(uint32_t nch) {
    switch (nch) {
        case 1: return dann_search3_kernel<T, 1, MAXW>;
        case 2: return dann_search3_kernel<T, 2, MAXW>;
        case 3: return dann_search3_kernel<T, 3, MAXW>;
        default: return nullptr;
    }
}
static emu_kernel pick_lean(int entry, uint32_t nch, int maxw) {
    if (maxw <= 16) return entry == 0 ? pick3<Ent32x21, 16>(nch) : pick3<Ent64, 16>(nch);
    return entry == 0 ? pick3<Ent32x21, 32>(nch) : pick3<Ent64, 32>(nch);
}
static emu_kernel pick(bool pairs, int entry, uint32_t nch, bool plain = false) {
    if (plain) return dann_search_kernel<Ent64, 1, 1>;
    if (pairs) return entry == 0 ? pick2<Ent32x21>(nch) : entry == 1 ? pick2<Ent32x16>(nch) : pick2<Ent64>(nch);
    return entry == 0 ? pick1<Ent32x21>(nch) : entry == 1 ? pick1<Ent32x16>(nch) : pick1<Ent64>(nch);
}

static std::string g_emu_err;
extern "C" const char *emu_last_error(void) { return g_emu_err.c_str(); }

struct emu_info {
    uint32_t retries, entry, W, hs, pairs, grid, cand_cap, vcap, bitmap_words, nch, G;
    uint32_t hv, lean, maxw, hash_cap;
    uint64_t switches;
    uint64_t coll_even, coll_odd; /* warp collectives completed by even / odd warps (controller / heap warp) */
};

/* One dann_search_batch-style search pass (no rerank): the approximate stream of every query.
 * q_codes [B][s->words]; qoff NULL = no scan key.  Returns 0, or a negative dann_status. */
extern "C" int emu_search(const dann_snapshot_desc *s, const uint64_t *q_codes, const int16_t *qlab, const int32_t *qoff,
                          uint32_t B, uint32_t L, uint32_t c_target, int force_single, uint32_t sm_count,
                          uint32_t smem_optin, uint32_t *stream, uint32_t *stream_len, dann_query_stats *stats,
                          emu_info *info, const float *index_vectors, const float *q_index) {
    const bool plain = index_vectors != nullptr; /* plain storage layout: q_codes / s->codes are not read */
    IndexView v{};
    v.n = s->n;
    v.dim = s->dim;
    v.dim_index = s->dim_index;
    v.bits = s->bits;
    v.words = s->words;
    v.cw = (s->words + 1u) & ~1u;
    v.R = s->R;
    v.Rp = (s->R + 7u) & ~7u;
    v.distance_type = s->distance_type;
    v.has_labels = s->has_labels ? 1 : 0;
    v.count = s->count;
    v.start_default = s->n ? s->start_default : DANN_INVALID_NODE;
    v.n_start_labels = s->start_labels && s->start_label_nodes ? s->n_start_labels : 0;
    uint32_t G = 1, Gshift = 0, NCH = 1;
    if (!plain && pick_code_mapping(v.cw, &G, &Gshift, &NCH) != 0) {
        g_emu_err = "code too wide";
        return DANN_ERR_INVALID_ARG;
    }
    /* HBM layout of dann_index_load: padded code rows and neighbour rows (16-byte aligned like cudaMalloc) */
    std::vector<ulonglong2> codes_store(((size_t)s->n * v.cw + 1) / 2 + 1);
    uint64_t *codes = reinterpret_cast<uint64_t *>(codes_store.data());
    for (size_t i = 0; i < s->n && !plain; i++)
        for (uint32_t w = 0; w < v.cw; w++) codes[i * v.cw + w] = w < s->words ? s->codes[i * s->words + w] : 0ull;
    std::vector<uint32_t> nbrs((size_t)s->n * v.Rp + 4, DANN_INVALID_NODE);
    uint32_t lists_unique = 1;
    for (size_t i = 0; i < s->n; i++) {
        for (uint32_t j = 0; j < s->R; j++) nbrs[i * v.Rp + j] = s->nbrs[i * s->R + j];
        for (uint32_t j = 0; j < s->R && s->nbrs[i * s->R + j] != DANN_INVALID_NODE; j++)
            for (uint32_t k = 0; k < j; k++)
                if (s->nbrs[i * s->R + k] == s->nbrs[i * s->R + j]) lists_unique = 0;
    }
    if (s->R > 64) lists_unique = 0;
    std::vector<ulonglong2> q_store(((size_t)B * v.cw + 1) / 2 + 1);
    uint64_t *qc = reinterpret_cast<uint64_t *>(q_store.data());
    for (size_t b = 0; b < B && !plain; b++)
        for (uint32_t w = 0; w < v.cw; w++) qc[b * v.cw + w] = w < s->words ? q_codes[b * s->words + w] : 0ull;
    v.codes = codes;
    v.nbrs = nbrs.data();
    v.tids = s->heap_tid;
    v.vectors = s->vectors;
    v.mean = s->mean;
    v.m2 = s->m2;
    v.start_labels = s->start_labels;
    v.start_label_nodes = s->start_label_nodes;
    v.label_off = s->label_off;
    v.labels = s->labels;
    if (!v.has_labels) v.label_off = nullptr, v.labels = nullptr;

    PlanInputs in;
    in.n = v.n;
    in.R = v.R;
    in.words = v.words;
    in.smem_optin = smem_optin;
    in.sm_count = (int)sm_count;
    in.plain_dim = plain ? s->dim_index : 0;
    in.allow_lean = true;
    in.ws_budget = 0;
    /* 16-byte aligned copies of the f32 rows, like cudaMalloc'ed memory */
    std::vector<float4> iv_store, qi_store;
    const float *ivp = nullptr, *qip = nullptr;
    if (plain) {
        iv_store.resize(((size_t)s->n * s->dim_index + 3) / 4 + 1);
        qi_store.resize(((size_t)B * s->dim_index + 3) / 4 + 1);
        memcpy(iv_store.data(), index_vectors, (size_t)s->n * s->dim_index * 4);
        memcpy(qi_store.data(), q_index, (size_t)B * s->dim_index * 4);
        ivp = reinterpret_cast<const float *>(iv_store.data());
        qip = reinterpret_cast<const float *>(qi_store.data());
    }

    std::vector<uint32_t> qlist;
    uint32_t nq = B, grow = 1, retries = 0;
    uint32_t ctl[2];
    SearchPlan p{};
    const uint64_t sw0 = simt::total_switches();
    uint64_t cp0[2];
    simt::collectives_by_warp_parity(cp0);
    for (int attempt = 0;; attempt++) {
        char err[256];
        int rc = dann_make_plan(in, nq, L, c_target, grow, qoff != nullptr, &p, force_single != 0, err, sizeof err);
        if (rc) {
            g_emu_err = err;
            return rc;
        }
        if ((size_t)p.per_warp * p.W > sizeof dann_smem) {
            g_emu_err = "plan needs more shared memory than the emulator provides";
            return DANN_ERR_CAPACITY;
        }
        const size_t slots = (size_t)p.grid * p.W;
        /* every workspace array sits between two guard zones that must come back untouched: an out-of-bounds
         * store of a kernel (heap tail, seq->node table, inserted-id list, hash set, stream) fails the run */
        const size_t GUARD = 256; /* bytes, keeps 16-byte alignment */
        struct Guarded {
            std::vector<ulonglong2> mem;
            size_t bytes = 0;
            void init(size_t nbytes, unsigned char fill) {
                bytes = nbytes;
                mem.assign((nbytes + 2 * 256 + 15) / 16 + 1, ulonglong2{0, 0});
                memset(mem.data(), 0xA5, mem.size() * 16);
                memset(reinterpret_cast<unsigned char *>(mem.data()) + 256, fill, nbytes);
            }
            unsigned char *p() { return reinterpret_cast<unsigned char *>(mem.data()) + 256; }
            bool intact() const {
                const unsigned char *b = reinterpret_cast<const unsigned char *>(mem.data());
                for (size_t i = 0; i < 256; i++)
                    if (b[i] != 0xA5 || b[256 + bytes + i] != 0xA5) return false;
                return true;
            }
        } g_hash, g_cand, g_bitmap, g_ins, g_heap;
        (void)GUARD;
        g_hash.init(p.bitmap_words ? 16 : slots * (size_t)p.hash_cap * 4, 0);
        g_cand.init(p.lean ? 16 : slots * (size_t)p.cand_cap * 4, 0);
        g_bitmap.init(slots * (size_t)p.bitmap_words * 4 + 16, 0);
        g_ins.init(p.bitmap_words && !p.lean ? slots * (size_t)p.ins_cap * 4 : 16, 0);
        g_heap.init(slots * (size_t)p.cand_cap * p.esize, 0);
        ctl[0] = ctl[1] = 0;
        SearchArgs a = search_args_for_plan(v, G, Gshift, lists_unique, p);
        a.q_codes = qc;
        a.q_labels = qlab;
        a.q_label_off = qoff;
        a.qlist = attempt == 0 ? nullptr : qlist.data();
        a.nq = nq;
        a.L = L;
        a.c_target = c_target;
        a.stream = stream;
        a.stream_len = stream_len;
        a.stats = stats;
        a.overflow = ctl + 1;
        a.counter = ctl;
        a.hash = reinterpret_cast<uint32_t *>(g_hash.p());
        a.bitmap = reinterpret_cast<uint32_t *>(g_bitmap.p());
        a.ins_list = reinterpret_cast<uint32_t *>(g_ins.p());
        a.cand_node = reinterpret_cast<uint32_t *>(g_cand.p());
        a.heap_tail = g_heap.p();
        a.hv_flags = env_u32("DANN_HV_FLAGS", 4095);
        a.plain_vectors = ivp;
        a.q_index = qip;
        a.plain_dim = in.plain_dim;
        emu_kernel fn = p.lean ? pick_lean(p.entry, NCH, p.maxw) : pick(p.pairs, p.entry, NCH, plain);
        if (!fn) {
            g_emu_err = "this code width is not instantiated in the emulator build";
            return DANN_ERR_INVALID_ARG;
        }
        simt::launch(p.grid, p.W * (p.pairs ? 64 : 32), [&] { fn(a); });
        for (size_t i = 0; i < slots * (size_t)p.bitmap_words; i++)
            if (a.bitmap[i]) {
                g_emu_err = "inserted-set bitmap not clean after the launch";
                return DANN_ERR_STATE;
            }
        if (!g_hash.intact() || !g_cand.intact() || !g_bitmap.intact() || !g_ins.intact() || !g_heap.intact()) {
            g_emu_err = "a kernel wrote outside one of its workspace arrays (guard zone damaged)";
            return DANN_ERR_STATE;
        }
        if (ctl[1] == 0) break;
        if (ctl[1] & DANN_ST_INTERNAL) {
            g_emu_err = "next-node prediction mismatch";
            return DANN_ERR_STATE;
        }
        if (attempt >= 8) {
            g_emu_err = "workspace still too small";
            return DANN_ERR_CAPACITY;
        }
        qlist.clear();
        for (uint32_t b = 0; b < B; b++)
            if (stats[b].status) qlist.push_back(b);
        nq = (uint32_t)qlist.size();
        grow *= 2;
        retries++;
    }
    if (info) {
        info->retries = retries;
        info->entry = (uint32_t)p.entry;
        info->W = p.W;
        info->hs = p.hs;
        info->pairs = p.pairs;
        info->grid = p.grid;
        info->cand_cap = p.cand_cap;
        info->vcap = p.vcap;
        info->bitmap_words = p.bitmap_words;
        info->nch = NCH;
        info->G = G;
        info->hv = 0;
        info->lean = p.lean ? 1u : 0u;
        info->maxw = (uint32_t)p.maxw;
        info->hash_cap = p.hash_cap;
        info->switches = simt::total_switches() - sw0;
        uint64_t cp1[2];
        simt::collectives_by_warp_parity(cp1);
        info->coll_even = cp1[0] - cp0[0];
        info->coll_odd = cp1[1] - cp0[1];
    }
    return 0;
}

/* the plan alone (host logic test): out[] = need, cand_cap, hash_cap, vcap, hs, W, grid, per_warp, esize, bitmap_words,
 * ins_cap, entry, pairs */
extern "C" int emu_plan(uint32_t n, uint32_t R, uint32_t words, uint32_t nq, uint32_t L, uint32_t c_target, uint32_t grow,
                        int keyed, int force_single, uint32_t sm_count, uint32_t smem_optin, int allow_lean, uint32_t *out) {
    PlanInputs in;
    in.n = n;
    in.R = R;
    in.words = words;
    in.smem_optin = smem_optin;
    in.sm_count = (int)sm_count;
    in.plain_dim = 0;
    in.allow_lean = allow_lean != 0; /* a one-shot batch search, as dann_search_batch plans it */
    in.ws_budget = 0;
    SearchPlan p{};
    char err[256];
    int rc = dann_make_plan(in, nq, L, c_target, grow, keyed != 0, &p, force_single != 0, err, sizeof err);
    if (rc) {
        g_emu_err = err;
        return rc;
    }
    const uint32_t v[15] = {p.need, p.cand_cap, p.hash_cap, p.vcap, p.hs, p.W, p.grid, p.per_warp, p.esize, p.bitmap_words,
                            p.ins_cap, (uint32_t)p.entry, (uint32_t)p.pairs, (uint32_t)p.lean, (uint32_t)p.maxw};
    for (int i = 0; i < 15; i++) out[i] = v[i];
    return 0;
}

/* ---- the heap warp's engine alone: a script of push pages and pops run through PairSearch::push_page and the pop of
 * run_heap, one warp, dumped after the last operation.  kinds[i]: 0 = push page of n[i] keys (taken from keys[] in
 * order), 1 = pop.  out_heap[len] receives the packed entries of slots 1..len, pops_seq[] the sequence number of
 * every popped root.  hs = entries kept in "shared memory", the rest in the tail. */
template <typename T>
static void heap_script_warp(const uint32_t *kinds, const uint32_t *n, uint32_t nops, const uint32_t *keys, uint32_t hs,
                             uint32_t cap, uint64_t *out_heap, uint32_t *out_len, uint32_t *pops_seq, SearchArgs &a,
                             typename T::E *tail) {
    using E = typename T::E;
    using H = RustHeap<E, T::KSHIFT>;
    const int lane = threadIdx.x & 31;
    unsigned char *base = dann_smem;
    PairSearch<T, 1> w(a, lane, 1u);
    E *hsm = reinterpret_cast<E *>(base);
    w.listp = reinterpret_cast<uint32_t *>(base + (size_t)hs * sizeof(E));
    w.dlp = w.listp + 2 * DANN_LIST_CAP;
    w.ctl = reinterpret_cast<PairCtl *>(w.dlp + 2 * DANN_LIST_CAP);
    w.cqp = reinterpret_cast<uint32_t *>(w.ctl + 1);
    w.cqe = reinterpret_cast<E *>(w.cqp + 32);
    w.heap.sm = hsm;
    w.heap.gl = tail;
    w.heap.hs = hs;
    w.heap_len = 0;
    uint32_t seq = 0, kpos = 0, npop = 0;
    for (uint32_t i = 0; i < nops; i++) {
        if (kinds[i] == 0) {
            for (uint32_t r = lane; r < n[i]; r += 32) w.dlp[r] = keys[kpos + r];
            if (lane == 0) {
                w.ctl->tn[0] = n[i];
                w.ctl->seq0[0] = seq;
            }
            __syncwarp();
            w.push_page(0);
            __syncwarp();
            seq += n[i];
            kpos += n[i];
        } else if (w.heap_len > 0) {
            if (lane == 0) pops_seq[npop] = T::seq(w.heap.get(1));
            npop++;
            __syncwarp();
            if (w.heap_len < w.heap.hs) {
                ArrayStore<E> sm{w.heap.sm};
                H::pop_warp1(sm, w.heap_len, lane);
            } else {
                H::pop_warp1(w.heap, w.heap_len, lane);
            }
            __syncwarp();
        }
    }
    for (uint32_t s = 1 + lane; s <= w.heap_len; s += 32) out_heap[s - 1] = (uint64_t)w.heap.get(s);
    if (lane == 0) *out_len = w.heap_len;
    (void)cap;
}

/* the same script through the lean kernel's heap code (LeanWarp::push_page - staged, cooperative - and ::pop) */
template <typename T>
static void heap_script_lean(const uint32_t *kinds, const uint32_t *n, uint32_t nops, const uint32_t *keys, uint32_t hs,
                             uint64_t *out_heap, uint32_t *out_len, uint32_t *pops_seq, SearchArgs &a, typename T::E *tail) {
    using E = typename T::E;
    const int lane = threadIdx.x & 31;
    unsigned char *base = dann_smem;
    LeanWarp<T, 1> w(a, lane);
    w.heap.sm = reinterpret_cast<E *>(base);
    w.ent = w.heap.sm + hs;
    w.stg = w.ent + DANN_LIST_CAP;
    w.list = reinterpret_cast<uint32_t *>(w.stg + DANN_STG_CAP);
    w.heap.gl = tail;
    w.heap.hs = hs;
    w.heap_len = 0;
    w.stg_async = false;
    uint32_t seq = 0, kpos = 0, npop = 0;
    for (uint32_t i = 0; i < nops; i++) {
        if (kinds[i] == 0) {
            for (uint32_t r = lane; r < n[i]; r += 32) w.ent[r] = T::make(keys[kpos + r], seq + r);
            __syncwarp();
            if (n[i] && (i & 1)) w.stage_ancestors_async(n[i]); /* every other page through the early-staging path */
            if (n[i]) w.push_page(n[i]);
            __syncwarp();
            seq += n[i];
            kpos += n[i];
        } else if (w.heap_len > 0) {
            if (lane == 0) pops_seq[npop] = T::seq(w.heap.get(1));
            npop++;
            w.pop();
            __syncwarp();
        }
    }
    for (uint32_t s = 1 + lane; s <= w.heap_len; s += 32) out_heap[s - 1] = (uint64_t)w.heap.get(s);
    if (lane == 0) *out_len = w.heap_len;
}

extern "C" int emu_heap_script(int entry, int hv, const uint32_t *kinds, const uint32_t *n, uint32_t nops, const uint32_t *keys,
                               uint32_t hs, uint32_t cap, uint64_t *out_heap, uint32_t *out_len, uint32_t *pops_seq) {
    if (hs % 4 || (size_t)hs * 8 + 4096 > sizeof dann_smem) {
        g_emu_err = "bad hs";
        return DANN_ERR_INVALID_ARG;
    }
    SearchArgs a{};
    a.hv_flags = env_u32("DANN_HV_FLAGS", 4095);
    std::vector<ulonglong2> tail((size_t)cap / 2 + 2);
    /* hv: 0 = the two-warp kernel's heap warp; 1 = the lean kernel's heap code with four-level pop rounds; 2 = the same
     * with lane 0 walking the pop's hole down */
    if (hv == 2) a.hv_flags &= ~DANN_HV_POP;
    auto run = [&](auto tag) {
        using T = decltype(tag);
        simt::launch(1, 32, [&] {
            if (hv == 0)
                heap_script_warp<T>(kinds, n, nops, keys, hs, cap, out_heap, out_len, pops_seq, a,
                                    reinterpret_cast<typename T::E *>(tail.data()));
            else
                heap_script_lean<T>(kinds, n, nops, keys, hs, out_heap, out_len, pops_seq, a,
                                    reinterpret_cast<typename T::E *>(tail.data()));
        });
    };
    if (entry == 0) run(Ent32x21{});
    else if (entry == 1 && hv == 0) run(Ent32x16{});
    else run(Ent64{});
    return 0;
}
