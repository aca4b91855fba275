/*
 * oracle.cpp — CPU oracle for the pgvectorscale StreamingDiskANN index-scan path.
 * TEST INFRASTRUCTURE ONLY (see oracle.h header).  "parity unpinned" for the two
 * third-party pieces named there (Rust std BinaryHeap sift order, simdeez hadd order).
 *
 * Reference paths are relative to pgvectorscale/src/access_method/.
 * Build: see oracle/Makefile  (-O2 -mavx2 -mfma -mpopcnt -ffp-contract=off).
 */
#include "oracle.h"

#include <immintrin.h>

#include <algorithm>
#include <atomic>
#include <cassert>
#include <cmath>
#include <cstring>
#include <map>
#include <thread>
#include <unordered_map>
#include <unordered_set>
#include <utility>
#include <vector>

/* ===================================================================== */
/* Rust std::collections::BinaryHeap clone (alloc/collections/binary_heap, 1.7x-1.8x).
 * Max-heap on `le(a,b)` == Rust `a <= b`.  parity unpinned: third-party (Rust std), see header.
 *   push  = Vec::push + sift_up(0, old_len)
 *   pop   = Vec::pop, swap with data[0], sift_down_to_bottom(0)
 *   sift_up: move hole up while !(elem <= parent)
 *   sift_down_to_bottom: always descend to the bottom picking
 *       child += (data[child] <= data[child+1])   (right child on ties), then sift_up.   */
template <class T, class LE>
struct RustBinaryHeap {
    std::vector<T> data;
    LE le;

    size_t len() const { return data.size(); }
    bool empty() const { return data.empty(); }
    const T &peek() const { return data[0]; }

    void push(const T &x) {
        size_t old_len = data.size();
        data.push_back(x);
        sift_up(0, old_len);
    }

    bool pop(T &out) {
        if (data.empty()) return false;
        T item = data.back();
        data.pop_back();
        if (!data.empty()) {
            std::swap(item, data[0]);
            sift_down_to_bottom(0);
        }
        out = item;
        return true;
    }

    size_t sift_up(size_t start, size_t pos) {
        T elem = data[pos];
        while (pos > start) {
            size_t parent = (pos - 1) / 2;
            if (le(elem, data[parent])) break;
            data[pos] = data[parent];
            pos = parent;
        }
        data[pos] = elem;
        return pos;
    }

    void sift_down_to_bottom(size_t pos) {
        size_t end = data.size();
        size_t start = pos;
        T elem = data[pos];
        size_t child = 2 * pos + 1;
        size_t lim = end >= 2 ? end - 2 : 0; /* end.saturating_sub(2) */
        while (child <= lim) {
            if (le(data[child], data[child + 1])) child += 1;
            data[pos] = data[child];
            pos = child;
            child = 2 * pos + 1;
        }
        if (child == end - 1) {
            data[pos] = data[child];
            pos = child;
        }
        data[pos] = elem;
        sift_up(start, pos);
    }
};

/* f32::total_cmp (core::f32): order by sign-magnitude integer transform. */
static inline int32_t total_key(float f) {
    int32_t b;
    std::memcpy(&b, &f, 4);
    b ^= (int32_t)(((uint32_t)(b >> 31)) >> 1);
    return b;
}
static inline int total_cmp(float a, float b) {
    int32_t ka = total_key(a), kb = total_key(b);
    return (ka > kb) - (ka < kb);
}

/* graph/neighbor_with_distance.rs:12-95 DistanceWithTieBreak */
struct Dwtb {
    float d;
    uint64_t tie; /* with_query => 0 (:31-43); new => ip_distance(from,to) (:45-49) */
};
static inline int dwtb_cmp(const Dwtb &a, const Dwtb &b) { /* :74-83 */
    if (a.d == 0.0f && b.d == 0.0f) return (a.tie > b.tie) - (a.tie < b.tie);
    return total_cmp(a.d, b.d);
}
static inline double dwtb_factor(const Dwtb &self, const Dwtb &divisor) { /* :55-65 */
    const float eps = 1.1920929e-07f; /* f32::EPSILON */
    if (divisor.d < 0.0f + eps) {
        if (self.d < 0.0f + eps) return (double)self.tie / (double)divisor.tie;
        return 1.7976931348623157e308; /* f64::MAX */
    }
    return (double)self.d / (double)divisor.d;
}

/* ===================================================================== */
/* leaf arithmetic                                                        */

extern "C" uint64_t orc_hamming(const uint64_t *a, const uint64_t *b, uint32_t words) {
    /* distance/mod.rs:255-323 : sum of (l ^ r).count_ones() as usize */
    uint64_t s = 0;
    for (uint32_t i = 0; i < words; i++) s += (uint64_t)__builtin_popcountll(a[i] ^ b[i]);
    return s;
}

/* simdeez 1.0.x Avx2::horizontal_add_ps — parity unpinned (third-party, un-vendored):
 * lo128+hi128, movehdup+add, movehl+add_ss  =>  ((a0+a4)+(a1+a5)) + ((a2+a6)+(a3+a7)) */
static inline float hadd8(const float *a) {
    float v0 = a[0] + a[4], v1 = a[1] + a[5], v2 = a[2] + a[6], v3 = a[3] + a[7];
    return (v0 + v1) + (v2 + v3);
}

static float l2_body(const float *x, const float *y, uint32_t n) {
    /* distance/mod.rs:325-377 with S = Avx2 (VF32_WIDTH = 8): sub, mul, add are separate ops */
    float acc[4][8];
    std::memset(acc, 0, sizeof(acc));
    uint32_t i = 0;
    for (; n - i >= 32; i += 32)
        for (int k = 0; k < 4; k++)
            for (int j = 0; j < 8; j++) {
                float d = x[i + 8 * k + j] - y[i + 8 * k + j];
                float p = d * d;
                acc[k][j] = acc[k][j] + p;
            }
    float dist = hadd8(acc[0]) + hadd8(acc[1]) + hadd8(acc[2]) + hadd8(acc[3]);
    for (; i < n; i++) {
        float diff = x[i] - y[i];
        float p = diff * diff;
        dist += p;
    }
    return dist;
}

static float ip_body(const float *x, const float *y, uint32_t n) {
    /* distance/mod.rs:380-434 : fmadd_ps in the body, plain mul+add in the tail */
    float acc[4][8];
    std::memset(acc, 0, sizeof(acc));
    uint32_t i = 0;
    for (; n - i >= 32; i += 32)
        for (int k = 0; k < 4; k++)
            for (int j = 0; j < 8; j++)
                acc[k][j] = std::fmaf(x[i + 8 * k + j], y[i + 8 * k + j], acc[k][j]);
    float dist = hadd8(acc[0]) + hadd8(acc[1]) + hadd8(acc[2]) + hadd8(acc[3]);
    for (; i < n; i++) {
        float p = x[i] * y[i];
        dist += p;
    }
    return dist;
}

static inline float finish_distance(int type, float v) {
    if (type == ORC_L2) return v;                 /* distance/mod.rs:88-104 (no sqrt) */
    if (type == ORC_IP) return -v;                /* :175-190 */
    float r = 1.0f - v;                           /* distance_x86.rs:34-36 (1.0 - ip).max(0.0) */
    return r > 0.0f ? r : 0.0f;                   /* f32::max: NaN-ignoring; r is never NaN here unless inputs are */
}

extern "C" float orc_distance(int type, const float *x, const float *y, uint32_t n) {
    return finish_distance(type, type == ORC_L2 ? l2_body(x, y, n) : ip_body(x, y, n));
}

static inline float hadd_avx2(__m256 a) {
    /* the classic simdeez/Agner sequence, same order as hadd8 */
    __m128 vlow = _mm256_castps256_ps128(a);
    __m128 vhigh = _mm256_extractf128_ps(a, 1);
    vlow = _mm_add_ps(vlow, vhigh);
    __m128 shuf = _mm_movehdup_ps(vlow);
    __m128 sums = _mm_add_ps(vlow, shuf);
    shuf = _mm_movehl_ps(shuf, sums);
    sums = _mm_add_ss(sums, shuf);
    return _mm_cvtss_f32(sums);
}

extern "C" float orc_distance_avx2(int type, const float *x, const float *y, uint32_t n) {
    __m256 a0 = _mm256_setzero_ps(), a1 = a0, a2 = a0, a3 = a0;
    uint32_t i = 0;
    float dist;
    if (type == ORC_L2) {
        for (; n - i >= 32; i += 32) {
            __m256 d0 = _mm256_sub_ps(_mm256_loadu_ps(x + i), _mm256_loadu_ps(y + i));
            __m256 d1 = _mm256_sub_ps(_mm256_loadu_ps(x + i + 8), _mm256_loadu_ps(y + i + 8));
            __m256 d2 = _mm256_sub_ps(_mm256_loadu_ps(x + i + 16), _mm256_loadu_ps(y + i + 16));
            __m256 d3 = _mm256_sub_ps(_mm256_loadu_ps(x + i + 24), _mm256_loadu_ps(y + i + 24));
            a0 = _mm256_add_ps(a0, _mm256_mul_ps(d0, d0));
            a1 = _mm256_add_ps(a1, _mm256_mul_ps(d1, d1));
            a2 = _mm256_add_ps(a2, _mm256_mul_ps(d2, d2));
            a3 = _mm256_add_ps(a3, _mm256_mul_ps(d3, d3));
        }
        dist = hadd_avx2(a0) + hadd_avx2(a1) + hadd_avx2(a2) + hadd_avx2(a3);
        for (; i < n; i++) {
            float diff = x[i] - y[i];
            float p = diff * diff;
            dist += p;
        }
    } else {
        for (; n - i >= 32; i += 32) {
            a0 = _mm256_fmadd_ps(_mm256_loadu_ps(x + i), _mm256_loadu_ps(y + i), a0);
            a1 = _mm256_fmadd_ps(_mm256_loadu_ps(x + i + 8), _mm256_loadu_ps(y + i + 8), a1);
            a2 = _mm256_fmadd_ps(_mm256_loadu_ps(x + i + 16), _mm256_loadu_ps(y + i + 16), a2);
            a3 = _mm256_fmadd_ps(_mm256_loadu_ps(x + i + 24), _mm256_loadu_ps(y + i + 24), a3);
        }
        dist = hadd_avx2(a0) + hadd_avx2(a1) + hadd_avx2(a2) + hadd_avx2(a3);
        for (; i < n; i++) {
            float p = x[i] * y[i];
            dist += p;
        }
    }
    return finish_distance(type, dist);
}

extern "C" float orc_distance_unoptimized(int type, const float *x, const float *y, uint32_t n) {
    /* distance/mod.rs:107-117 and :212-223 : sequential iterator sums */
    float s = 0.0f;
    if (type == ORC_L2) {
        for (uint32_t i = 0; i < n; i++) {
            float d = x[i] - y[i];
            float p = d * d;
            s += p;
        }
        return s;
    }
    for (uint32_t i = 0; i < n; i++) {
        float p = x[i] * y[i];
        s += p;
    }
    return finish_distance(type, s);
}

extern "C" void orc_preprocess_cosine(float *v, uint32_t n) {
    /* distance/mod.rs:225-253 */
    float norm = 0.0f;
    for (uint32_t i = 0; i < n; i++) {
        float p = v[i] * v[i];
        norm += p; /* sequential f32 sum (Iterator::sum) */
    }
    const float eps = 1.1920929e-07f;
    float adj = eps * (float)n;
    if (norm < eps) return;
    if (norm >= 1.0f - adj && norm <= 1.0f + adj) return;
    float s = std::sqrt(norm);
    for (uint32_t i = 0; i < n; i++) v[i] = v[i] / s;
}

extern "C" uint32_t orc_code_words(uint32_t dim, uint32_t bits) {
    uint64_t nb = (uint64_t)dim * bits; /* quantize.rs:38-46 */
    return (uint32_t)(nb % 64 == 0 ? nb / 64 : nb / 64 + 1);
}

extern "C" void orc_train(const float *vectors, uint32_t n, uint32_t dim, uint32_t bits,
                          float *mean, float *m2, uint64_t *count) {
    /* quantize.rs:104-148 : f32 Welford in heap-scan order */
    for (uint32_t d = 0; d < dim; d++) {
        mean[d] = 0.0f;
        if (m2) m2[d] = 0.0f;
    }
    uint64_t c = 0;
    for (uint32_t r = 0; r < n; r++) {
        const float *s = vectors + (size_t)r * dim;
        c += 1;
        float cf = (float)c;
        if (bits > 1) {
            for (uint32_t d = 0; d < dim; d++) {
                float delta = s[d] - mean[d];
                float q = (s[d] - mean[d]) / cf;
                mean[d] += q;
                float delta2 = s[d] - mean[d];
                float p = delta * delta2;
                m2[d] += p;
            }
        } else {
            for (uint32_t d = 0; d < dim; d++) {
                float q = (s[d] - mean[d]) / cf;
                mean[d] += q;
            }
        }
    }
    *count = c;
}

extern "C" void orc_quantize(const float *v, uint32_t dim, uint32_t bits, const float *mean,
                             const float *m2, uint64_t count, uint64_t *out) {
    /* quantize.rs:52-102 (use_mean == true) */
    uint32_t words = orc_code_words(dim, bits);
    for (uint32_t w = 0; w < words; w++) out[w] = 0;
    if (bits == 1) {
        for (uint32_t i = 0; i < dim; i++)
            if (v[i] > mean[i]) out[i / 64] |= 1ull << (i % 64);
        return;
    }
    float ranges = (float)(uint8_t)(bits + 1);
    for (uint32_t i = 0; i < dim; i++) {
        float variance = m2[i] / (float)count;
        float std_dev = std::sqrt(variance);
        float z = (v[i] - mean[i]) / std_dev;
        float index = (z + 2.0f) / (4.0f / ranges);
        size_t bit_position = (size_t)i * bits;
        if (index < 1.0f) {
            /* all zeros */
        } else {
            /* `index.floor() as usize`: saturating cast, NaN -> 0 */
            float fl = std::floor(index);
            uint64_t as_usize;
            if (fl != fl) as_usize = 0;
            else if (fl >= 18446744073709551616.0f) as_usize = UINT64_MAX;
            else if (fl <= 0.0f) as_usize = 0;
            else as_usize = (uint64_t)fl;
            uint64_t count_ones = std::min<uint64_t>(as_usize, bits);
            for (uint64_t j = 0; j < count_ones; j++)
                out[(bit_position + j) / 64] |= 1ull << ((bit_position + j) % 64);
        }
    }
}

extern "C" int orc_labels_overlap(const int16_t *a, uint32_t na, const int16_t *b, uint32_t nb) {
    /* labels/mod.rs:124-142 */
    uint32_t i = 0, j = 0;
    while (i < na && j < nb) {
        if (a[i] == b[j]) return 1;
        if (a[i] < b[j]) i++;
        else j++;
    }
    return 0;
}

extern "C" int orc_labels_contains_intersection(const int16_t *c, uint32_t nc, const int16_t *a,
                                                uint32_t na, const int16_t *b, uint32_t nb) {
    /* labels/mod.rs:84-111 : is (a ∩ b) ⊆ self */
    uint32_t i = 0, j = 0, k = 0;
    while (i < na && j < nb) {
        if (a[i] == b[j]) {
            while (k < nc && c[k] < a[i]) k++;
            if (k == nc || c[k] > a[i]) return 0;
            i++;
            j++;
        } else if (a[i] < b[j]) i++;
        else j++;
    }
    return 1;
}

extern "C" uint32_t orc_labels_normalize(int16_t *labels, uint32_t n) {
    std::sort(labels, labels + n); /* labels/mod.rs:30-37 */
    return (uint32_t)(std::unique(labels, labels + n) - labels);
}

struct KeyPayload {
    int64_t key, payload;
};
struct KeyLE {
    bool operator()(const KeyPayload &a, const KeyPayload &b) const { return a.key <= b.key; }
};
extern "C" uint32_t orc_binary_heap_script(const int64_t *ops, uint32_t nops, int64_t *out) {
    RustBinaryHeap<KeyPayload, KeyLE> h;
    uint32_t w = 0;
    for (uint32_t i = 0; i < nops; i++) {
        if (ops[i] >= 0) h.push(KeyPayload{ops[i], (int64_t)i});
        else {
            KeyPayload kp;
            if (h.pop(kp)) out[w++] = kp.payload;
        }
    }
    return w;
}

/* ===================================================================== */
/* ListSearchResult (graph/mod.rs:74-185)                                 */

struct Lsn { /* ListSearchNeighbor :22-72 */
    uint32_t node;
    Dwtb d;
};
struct LsnReverseLE { /* Reverse<Lsn>: a <= b  <=>  b.0 <= a.0 (core::cmp::Reverse) */
    bool operator()(const Lsn &a, const Lsn &b) const { return dwtb_cmp(b.d, a.d) <= 0; }
};

/* membership-only set (HashSet<ItemPointer>, graph/mod.rs:77,126-128): order independent */
struct NodeSet {
    std::vector<uint32_t> slots;
    uint32_t mask = 0, used = 0;
    void reset(uint32_t cap_pow2) {
        slots.assign(cap_pow2, ORC_INVALID_NODE);
        mask = cap_pow2 - 1;
        used = 0;
    }
    void grow() {
        std::vector<uint32_t> old;
        old.swap(slots);
        slots.assign(old.size() * 2, ORC_INVALID_NODE);
        mask = (uint32_t)slots.size() - 1;
        used = 0;
        for (uint32_t v : old)
            if (v != ORC_INVALID_NODE) insert(v);
    }
    bool insert(uint32_t v) {
        if ((used + 1) * 2 > slots.size()) grow();
        uint32_t h = (v * 2654435761u) & mask;
        while (true) {
            uint32_t cur = slots[h];
            if (cur == v) return false;
            if (cur == ORC_INVALID_NODE) {
                slots[h] = v;
                used++;
                return true;
            }
            h = (h + 1) & mask;
        }
    }
};

struct Lsr {
    RustBinaryHeap<Lsn, LsnReverseLE> candidates;
    std::vector<Lsn> visited;
    NodeSet inserted;
    orc_stats stats{};

    bool prepare_insert(uint32_t n) { return inserted.insert(n); } /* :126-128 */
    void insert_neighbor(const Lsn &n) {                            /* :144-147 */
        stats.candidates++;
        candidates.push(n);
    }
    /* :153-170 ; returns index into visited or -1 */
    long visit_closest(size_t pos_limit) {
        if (candidates.empty()) return -1;
        if (visited.size() > pos_limit) {
            const Lsn &node_at_pos = visited[pos_limit - 1];
            const Lsn &head = candidates.peek();
            if (dwtb_cmp(head.d, node_at_pos.d) >= 0) return -1;
        }
        Lsn head;
        candidates.pop(head);
        /* partition_point(|x| *x < head) */
        size_t lo = 0, hi = visited.size();
        while (lo < hi) {
            size_t mid = lo + (hi - lo) / 2;
            if (dwtb_cmp(visited[mid].d, head.d) < 0) lo = mid + 1;
            else hi = mid;
        }
        visited.insert(visited.begin() + (long)lo, head);
        return (long)lo;
    }
};

struct QueryCtx {
    const orc_snapshot *s;
    std::vector<float> q_full, q_index;
    std::vector<uint64_t> q_code;
    bool labels_some = false;
    std::vector<int16_t> labels;
    bool has_label_filter = false;
};

static inline const int16_t *node_labels(const orc_snapshot *s, uint32_t n, uint32_t *cnt) {
    if (!s->has_labels || !s->label_off) {
        *cnt = 0;
        return nullptr;
    }
    *cnt = s->label_off[n + 1] - s->label_off[n];
    return s->labels + s->label_off[n];
}

/* sbq/storage.rs:365-391 create_lsn_for_start_node + graph/mod.rs:117-122 */
/* plain/mod.rs:22-32 PlainDistanceMeasure::calculate_distance: distance_fn(query.to_index_slice(), node.vector) */
static inline float plain_distance(const QueryCtx &q, Lsr &l, uint32_t node) {
    const orc_snapshot *s = q.s;
    l.stats.d_full++; /* record_full_distance_comparison */
    return orc_distance_avx2(s->distance_type, q.q_index.data(), s->index_vectors + (size_t)node * s->dim_index,
                             s->dim_index);
}

static void lsr_add_start(const QueryCtx &q, Lsr &l, uint32_t node) {
    if (!l.prepare_insert(node)) return;
    const orc_snapshot *s = q.s;
    if (s->storage_type == ORC_STORAGE_PLAIN) { /* plain/storage.rs:223-252 */
        float d = plain_distance(q, l, node);
        l.insert_neighbor(Lsn{node, Dwtb{d, 0}});
        return;
    }
    l.stats.d_quantized++;
    float d = (float)orc_hamming(s->codes + (size_t)node * s->words, q.q_code.data(), s->words);
    l.insert_neighbor(Lsn{node, Dwtb{d, 0}});
}

/* sbq/storage.rs:125-190 visit_lsn_internal, GraphNeighborStore::Disk arm */
static void visit_lsn(const QueryCtx &q, Lsr &l, uint32_t visiting, bool no_filter) {
    const orc_snapshot *s = q.s;
    const uint32_t *nb = s->nbrs + (size_t)visiting * s->R;
    for (uint32_t j = 0; j < s->R; j++) {
        uint32_t n = nb[j];
        if (n == ORC_INVALID_NODE) break; /* sbq/node.rs:261-285 */
        if (!l.prepare_insert(n)) continue;
        if (s->storage_type == ORC_STORAGE_PLAIN) { /* plain/storage.rs:254-299 (asserts no_filter) */
            float d = plain_distance(q, l, n);
            l.insert_neighbor(Lsn{n, Dwtb{d, 0}});
            continue;
        }
        if (q.labels_some) {
            if (!no_filter) {
                uint32_t cnt;
                const int16_t *nl = node_labels(s, n, &cnt);
                if (!orc_labels_overlap(q.labels.data(), (uint32_t)q.labels.size(), nl, cnt))
                    continue;
            }
        }
        l.stats.d_quantized++;
        float d = (float)orc_hamming(s->codes + (size_t)n * s->words, q.q_code.data(), s->words);
        l.insert_neighbor(Lsn{n, Dwtb{d, 0}});
    }
}

/* graph/mod.rs:357-385 */
static void greedy_search_iterate(const QueryCtx &q, Lsr &l, size_t visit_n_closest,
                                  bool no_filter) {
    long idx;
    while ((idx = l.visit_closest(visit_n_closest)) >= 0) {
        l.stats.visits++;
        visit_lsn(q, l, l.visited[(size_t)idx].node, no_filter);
    }
}

struct ResortData { /* scan.rs:91-117 */
    uint64_t tid;
    uint32_t node;
    float distance;
};
struct ResortLE { /* Ord: other.distance.total_cmp(&self.distance) ; a <= b <=> cmp(a,b) != Greater */
    bool operator()(const ResortData &a, const ResortData &b) const {
        return total_cmp(b.distance, a.distance) <= 0;
    }
};

struct Scan { /* scan.rs TSVResponseIterator :162-306 */
    QueryCtx q;
    Lsr lsr;
    size_t L, resort_size;
    RustBinaryHeap<ResortData, ResortLE> resort;
    std::vector<float> tmp;
    std::vector<uint32_t> stream;

    void init(const orc_snapshot *s, const float *query, const int16_t *labels, int32_t nlabels,
              uint32_t search_list_size, uint32_t rescore) {
        q.s = s;
        L = search_list_size;
        resort_size = rescore;
        /* labels/mod.rs:209-238 from_scan_key_data */
        q.q_full.assign(s->dim, 0.0f);
        q.q_index.assign(s->dim_index, 0.0f);
        if (query == nullptr) { /* NULL query: zero vector, labels None (:214-216) */
            q.labels_some = false;
        } else {
            std::memcpy(q.q_full.data(), query, sizeof(float) * s->dim);
            std::memcpy(q.q_index.data(), query, sizeof(float) * s->dim_index);
            if (s->distance_type == ORC_COSINE) { /* pg_vector.rs:153-155, each copy separately */
                orc_preprocess_cosine(q.q_full.data(), s->dim);
                orc_preprocess_cosine(q.q_index.data(), s->dim_index);
            }
            q.labels_some = nlabels >= 0;
            if (q.labels_some) {
                q.labels.assign(labels, labels + nlabels);
                q.labels.resize(orc_labels_normalize(q.labels.data(), (uint32_t)nlabels));
            }
        }
        q.has_label_filter = q.labels_some && !q.labels.empty(); /* scan.rs:189 */
        tmp.resize(s->dim);

        /* graph/mod.rs:331-354 greedy_search_streaming_init */
        lsr.inserted.reset(4096);
        if (s->start_default == ORC_INVALID_NODE) return; /* no nodes in the graph */
        if (s->storage_type == ORC_STORAGE_PLAIN) {
            /* plain storage does not support label filters (plain/storage.rs:260): the key is ignored here */
            q.labels_some = false;
            q.labels.clear();
            q.has_label_filter = false;
        } else {
            /* sbq/mod.rs:145-148 */
            q.q_code.assign(s->words, 0);
            orc_quantize(q.q_index.data(), s->dim_index, s->bits, s->mean, s->m2, s->count, q.q_code.data());
        }
        /* start_nodes.rs:39-48 */
        if (q.labels_some) {
            for (int16_t lab : q.labels) {
                const int16_t *b = s->start_labels, *e = b + s->n_start_labels;
                const int16_t *it = std::lower_bound(b, e, lab);
                if (it != e && *it == lab) lsr_add_start(q, lsr, s->start_label_nodes[it - b]);
            }
        } else {
            lsr_add_start(q, lsr, s->start_default);
        }
    }

    /* scan.rs:210-242 next ; graph/mod.rs:174-184 consume ; sbq/storage.rs:404-414 return_lsn */
    bool next(uint64_t *tid, uint32_t *node) {
        while (true) {
            greedy_search_iterate(q, lsr, L, !q.has_label_filter);
            if (lsr.visited.empty()) return false;
            Lsn c = lsr.visited.front();
            lsr.visited.erase(lsr.visited.begin());
            uint64_t t = q.s->heap_tid[c.node];
            if ((t & 0xFFFFu) == 0) continue; /* InvalidOffsetNumber: deleted tuple */
            lsr.stats.stream_len++;
            stream.push_back(c.node);
            *tid = t;
            *node = c.node;
            return true;
        }
    }

    /* sbq/storage.rs:304-328 get_full_distance_for_resort */
    float full_distance(uint32_t node) {
        const orc_snapshot *s = q.s;
        std::memcpy(tmp.data(), s->vectors + (size_t)node * s->dim, sizeof(float) * s->dim);
        if (s->distance_type == ORC_COSINE) orc_preprocess_cosine(tmp.data(), s->dim);
        return orc_distance_avx2(s->distance_type, tmp.data(), q.q_full.data(), s->dim);
    }

    /* scan.rs:244-305 next_with_resort */
    bool next_with_resort(uint64_t *tid, uint32_t *node, float *dist) {
        /* scan.rs:392-403: plain storage only resorts when the index holds fewer dimensions than the heap */
        const bool plain_no_resort = q.s->storage_type == ORC_STORAGE_PLAIN && q.s->dim == q.s->dim_index;
        if (resort_size == 0 || plain_no_resort) { /* resort_buffer.capacity() == 0 */
            *dist = std::nanf("");
            return next(tid, node);
        }
        while (resort.len() < resort_size) {
            uint64_t t;
            uint32_t n;
            if (!next(&t, &n)) break;
            lsr.stats.d_full++;
            float d = full_distance(n);
            resort.push(ResortData{t, n, d});
        }
        ResortData rd;
        if (!resort.pop(rd)) return false;
        *tid = rd.tid;
        *node = rd.node;
        *dist = rd.distance;
        return true;
    }
};

extern "C" uint32_t orc_scan(const orc_snapshot *s, const float *query, const int16_t *labels,
                             int32_t nlabels, uint32_t search_list_size, uint32_t rescore,
                             uint32_t max_rows, uint64_t *out_tid, uint32_t *out_node,
                             float *out_dist, uint32_t *out_stream, uint32_t stream_cap,
                             orc_stats *out_stats) {
    Scan sc;
    sc.init(s, query, labels, nlabels, search_list_size, rescore);
    uint32_t rows = 0;
    while (rows < max_rows) {
        uint64_t t;
        uint32_t n;
        float d;
        if (!sc.next_with_resort(&t, &n, &d)) break;
        if (out_tid) out_tid[rows] = t;
        if (out_node) out_node[rows] = n;
        if (out_dist) out_dist[rows] = d;
        rows++;
    }
    if (out_stream)
        for (size_t i = 0; i < sc.stream.size() && i < stream_cap; i++) out_stream[i] = sc.stream[i];
    if (out_stats) *out_stats = sc.lsr.stats;
    return rows;
}

extern "C" void orc_scan_batch(const orc_snapshot *s, const float *queries,
                               const int16_t *labels, const int32_t *label_off, uint32_t B,
                               uint32_t search_list_size, uint32_t rescore, uint32_t k,
                               uint64_t *out_tid, float *out_dist, uint32_t *out_count,
                               orc_stats *out_stats, uint32_t threads) {
    if (threads == 0) threads = std::max(1u, std::thread::hardware_concurrency());
    threads = std::min(threads, std::max(1u, B));
    std::atomic<uint32_t> next{0};
    auto work = [&]() {
        while (true) {
            uint32_t b = next.fetch_add(1);
            if (b >= B) break;
            const int16_t *lab = nullptr;
            int32_t nl = -1;
            if (label_off) {
                lab = labels + label_off[b];
                nl = label_off[b + 1] - label_off[b];
            }
            for (uint32_t i = 0; i < k; i++) {
                out_tid[(size_t)b * k + i] = ~0ull;
                if (out_dist) out_dist[(size_t)b * k + i] = std::nanf("");
            }
            orc_stats st;
            uint32_t rows = orc_scan(s, queries + (size_t)b * s->dim, lab, nl, search_list_size,
                                     rescore, k, out_tid + (size_t)b * k, nullptr,
                                     out_dist ? out_dist + (size_t)b * k : nullptr, nullptr, 0,
                                     &st);
            if (out_count) out_count[b] = rows;
            if (out_stats) out_stats[b] = st;
        }
    };
    if (threads == 1) {
        work();
        return;
    }
    std::vector<std::thread> pool;
    for (uint32_t t = 0; t < threads; t++) pool.emplace_back(work);
    for (auto &t : pool) t.join();
}

/* ===================================================================== */
/* Serial Vamana build (index construction is OUT of the hot path; restated only so
 * that tests can obtain graphs the way the reference makes them).                */

struct Nwd { /* NeighborWithDistance, neighbor_with_distance.rs:97-155 */
    uint32_t node;
    Dwtb d;
};

struct Builder {
    uint32_t n, words, R, L;
    double max_alpha;
    bool has_labels;
    const uint64_t *codes;
    const uint32_t *label_off;
    const int16_t *labels;
    size_t max_during_build; /* meta_page.rs:253-255 ceil(R*1.3) */
    std::vector<std::vector<Nwd>> nbrs; /* BuilderNeighborCache (no eviction modelled) */
    bool have_start = false;
    uint32_t start_default = ORC_INVALID_NODE;
    std::map<int16_t, uint32_t> start_labeled; /* BTreeMap */
    orc_build_switches sw{};   /* all zero: the reference's rules (orc_build never sets one) */
    uint64_t bc[ORC_BC_N] = {}; /* branch counters, see oracle.h */

    const int16_t *labs(uint32_t i, uint32_t *cnt) const {
        if (!has_labels) {
            *cnt = 0;
            return nullptr;
        }
        *cnt = label_off[i + 1] - label_off[i];
        return labels + label_off[i];
    }
    static uint64_t ipd(uint32_t a, uint32_t b) { return a > b ? a - b : b - a; }
    float ham(uint32_t a, uint32_t b) const {
        return (float)orc_hamming(codes + (size_t)a * words, codes + (size_t)b * words, words);
    }

    void sort_candidates(std::vector<Nwd> &cand) const {
        if (sw.order_by_id)
            std::sort(cand.begin(), cand.end(), [](const Nwd &a, const Nwd &b) {
                return a.d.d != b.d.d ? a.d.d < b.d.d : a.node < b.node;
            });
        else
            std::stable_sort(cand.begin(), cand.end(),
                             [](const Nwd &a, const Nwd &b) { return dwtb_cmp(a.d, b.d) < 0; });
    }

    /* graph/mod.rs:392-488 */
    std::vector<Nwd> prune(uint32_t point, std::vector<Nwd> cand) {
        uint32_t np;
        const int16_t *pl = labs(point, &np);
        sort_candidates(cand);
        std::vector<Nwd> results;
        results.reserve(R);
        std::vector<double> max_factors(cand.size(), 0.0);
        double alpha = 1.0;
        while (alpha <= max_alpha && results.size() < R) {
            for (size_t i = 0; i < cand.size(); i++) {
                if (results.size() >= R) return results;
                if (max_factors[i] > alpha) continue;
                max_factors[i] = 1.7976931348623157e308;
                results.push_back(cand[i]);
                if (alpha > 1.0) bc[ORC_BC_ROUND2_KEPT]++;
                const Nwd &ex = cand[i];
                uint32_t ne;
                const int16_t *el = labs(ex.node, &ne);
                for (size_t j = i + 1; j < cand.size(); j++) {
                    if (max_factors[j] > max_alpha) continue;
                    if (has_labels) {
                        uint32_t nc;
                        const int16_t *cl = labs(cand[j].node, &nc);
                        if (!orc_labels_contains_intersection(el, ne, cl, nc, pl, np)) {
                            bc[ORC_BC_LABEL_SKIP]++;
                            continue;
                        }
                    }
                    float raw = ham(ex.node, cand[j].node);
                    if (raw == 0.0f) bc[cand[j].d.d == 0.0f ? ORC_BC_TIE_FACTOR : ORC_BC_ZERO_OCCLUDED]++;
                    Dwtb between{raw, ipd(cand[j].node, ex.node)};
                    double factor = dwtb_factor(cand[j].d, between);
                    max_factors[j] = std::max(max_factors[j], factor);
                }
            }
            alpha *= 1.2;
        }
        return results;
    }

    std::vector<Nwd> add_neighbors(uint32_t of, const std::vector<Nwd> &additional) {
        return add_neighbors(of, additional, max_during_build, false, nullptr);
    }

    /* graph/mod.rs:212-266.  `keep` = the length above which the list is pruned (the reference:
     * max_neighbors_during_build); `store_sorted` = the merged list is put in candidate order first */
    std::vector<Nwd> add_neighbors(uint32_t of, const std::vector<Nwd> &additional, size_t keep, bool store_sorted,
                                   bool *pruned) {
        std::vector<Nwd> cand = nbrs[of];
        std::unordered_set<uint32_t> hash;
        for (auto &c : cand) hash.insert(c.node);
        for (auto &a : additional)
            if (hash.insert(a.node).second) cand.push_back(a);
        if (!hash.insert(of).second) {
            for (size_t i = 0; i < cand.size(); i++)
                if (cand[i].node == of) {
                    cand.erase(cand.begin() + (long)i);
                    break;
                }
        }
        if (store_sorted) sort_candidates(cand);
        if (pruned) *pruned = cand.size() > keep;
        std::vector<Nwd> out = cand.size() > keep ? prune(of, cand) : cand;
        nbrs[of] = out;
        return out;
    }

    /* graph/mod.rs:285-327 greedy_search_for_build (one-shot, Builder arm of visit_lsn) */
    std::vector<Nwd> search_for_build(uint32_t ip, bool no_filter) {
        std::vector<Nwd> visited_nodes;
        if (!have_start) return visited_nodes;
        uint32_t nq;
        const int16_t *ql = labs(ip, &nq);
        bool q_some = has_labels;
        std::vector<uint32_t> starts;
        if (no_filter || !q_some) starts.push_back(start_default);
        else
            for (uint32_t i = 0; i < nq; i++) {
                auto it = start_labeled.find(ql[i]);
                if (it != start_labeled.end()) starts.push_back(it->second);
            }
        Lsr l;
        l.inserted.reset(4096);
        const uint64_t *qc = codes + (size_t)ip * words;
        for (uint32_t sn : starts) {
            if (!l.prepare_insert(sn)) continue;
            l.stats.d_quantized++;
            float d = (float)orc_hamming(codes + (size_t)sn * words, qc, words);
            l.insert_neighbor(Lsn{sn, Dwtb{d, sw.scan_ties ? 0 : ipd(sn, ip)}});
        }
        long idx;
        while ((idx = l.visit_closest(L)) >= 0) {
            Lsn e = l.visited[(size_t)idx];
            visited_nodes.push_back(Nwd{e.node, e.d});
            l.stats.visits++;
            for (const Nwd &nb : nbrs[e.node]) { /* sbq/storage.rs:191-228 */
                if (!l.prepare_insert(nb.node)) continue;
                if (q_some && !no_filter) {
                    uint32_t nn;
                    const int16_t *nl = labs(nb.node, &nn);
                    if (!orc_labels_overlap(ql, nq, nl, nn)) continue;
                }
                l.stats.d_quantized++;
                float d = (float)orc_hamming(codes + (size_t)nb.node * words, qc, words);
                l.insert_neighbor(Lsn{nb.node, Dwtb{d, sw.scan_ties ? 0 : ipd(nb.node, ip)}});
            }
        }
        if (sw.visited_cap || sw.cand_cap) { /* the distance-ordered visited list itself, possibly cut short */
            size_t nv = l.visited.size();
            if (sw.visited_cap && nv > sw.visited_cap) {
                nv = sw.visited_cap;
                bc[ORC_BC_VISITED_CUT]++;
            }
            visited_nodes.clear();
            for (size_t i = 0; i < nv; i++) visited_nodes.push_back(Nwd{l.visited[i].node, l.visited[i].d});
        }
        for (Nwd &v : visited_nodes) v.d.tie = ipd(v.node, ip); /* the prune's tie-break, whatever ordered the search */
        if (visited_nodes.empty()) bc[ORC_BC_EMPTY_SEARCH]++;
        /* HashSet<NeighborWithDistance> keyed by pointer: dedupe (cannot repeat here) */
        return visited_nodes;
    }

    /* graph/mod.rs:662-717 */
    void insert_internal(uint32_t ip, bool no_filter) {
        std::vector<Nwd> v = search_for_build(ip, no_filter);
        std::vector<Nwd> list = add_neighbors(ip, v);
        for (const Nwd &nb : list) /* update_back_pointer :720-737 */
            add_neighbors(nb.node, std::vector<Nwd>{Nwd{ip, nb.d}});
    }

    /* graph/mod.rs:490-533, 637-660 */
    void insert(uint32_t ip) {
        uint32_t nl;
        const int16_t *l = labs(ip, &nl);
        if (!have_start) {
            have_start = true;
            start_default = ip;
        }
        if (has_labels)
            for (uint32_t i = 0; i < nl; i++)
                if (!start_labeled.count(l[i])) start_labeled[l[i]] = ip;
        if (has_labels) insert_internal(ip, false);
        insert_internal(ip, true);
    }

    /* insert_internal for the nodes [lo, lo + m) at once: all searches first (none sees a batch mate's edges),
     * then the forward lists, then the back-links per destination in (distance, source) order */
    void insert_batch(uint32_t lo, uint32_t m, bool no_filter) {
        const size_t cap13 = max_during_build;
        const size_t back_keep = sw.slots ? std::min<size_t>(sw.slots, cap13) : cap13;
        const size_t fwd_keep = sw.fwd_keep_slots ? sw.slots : back_keep;
        std::vector<std::vector<Nwd>> vis(m);
        for (uint32_t b = 0; b < m; b++) vis[b] = search_for_build(lo + b, no_filter);
        struct Trip {
            uint32_t dst;
            float d;
            uint32_t src;
        };
        std::vector<Trip> trips;
        for (uint32_t b = 0; b < m; b++) {
            const uint32_t p = lo + b;
            std::vector<Nwd> &v = vis[b];
            const size_t deg = nbrs[p].size();
            if (deg) bc[ORC_BC_FWD_MERGED]++;
            if (sw.cand_cap && v.size() > sw.cand_cap - deg) {
                v.resize(sw.cand_cap - deg);
                bc[ORC_BC_CAND_CUT]++;
            }
            bool pruned;
            std::vector<Nwd> list = add_neighbors(p, v, fwd_keep, sw.order_by_id != 0, &pruned);
            bc[pruned ? ORC_BC_FWD_PRUNED : ORC_BC_FWD_KEPT]++;
            for (const Nwd &nb : list) trips.push_back(Trip{nb.node, nb.d.d, p}); /* update_back_pointer :720-737 */
        }
        std::sort(trips.begin(), trips.end(), [](const Trip &a, const Trip &b) {
            return a.dst != b.dst ? a.dst < b.dst : a.d != b.d ? a.d < b.d : a.src < b.src;
        });
        /* an unlabeled destination cannot already hold a source of this batch: appended as they come; the second
         * pass of a labeled batch can repeat an edge of the first, so its lists go through the merge */
        const bool merge = sw.order_by_id && has_labels;
        for (size_t s = 0; s < trips.size();) {
            size_t e = s;
            while (e < trips.size() && trips[e].dst == trips[s].dst) e++;
            const uint32_t q = trips[s].dst;
            size_t take = e - s;
            if (sw.back_src_cap && take > sw.back_src_cap) {
                take = sw.back_src_cap;
                bc[ORC_BC_BACK_SRC_CUT]++;
            }
            std::vector<Nwd> add;
            for (size_t i = s; i < s + take; i++) {
                add.push_back(Nwd{trips[i].src, Dwtb{trips[i].d, ipd(trips[i].src, q)}});
                for (const Nwd &x : nbrs[q])
                    if (x.node == trips[i].src) bc[ORC_BC_BACK_REPEAT]++;
            }
            bool pruned;
            add_neighbors(q, add, back_keep, merge, &pruned);
            bc[pruned ? ORC_BC_BACK_PRUNED : merge ? ORC_BC_BACK_MERGED : ORC_BC_BACK_APPENDED]++;
            s = e;
        }
    }
};

extern "C" void orc_build(uint32_t n, uint32_t words, const uint64_t *codes, uint32_t R,
                          uint32_t search_list_size, double max_alpha, int32_t has_labels,
                          const uint32_t *label_off, const int16_t *labels, uint32_t *out_nbrs,
                          uint32_t *out_start_default, int16_t *out_start_labels,
                          uint32_t *out_start_label_nodes, uint32_t *out_n_start_labels,
                          uint32_t start_label_cap) {
    Builder b;
    b.n = n;
    b.words = words;
    b.R = R;
    b.L = search_list_size;
    b.max_alpha = max_alpha;
    b.has_labels = has_labels != 0;
    b.codes = codes;
    b.label_off = label_off;
    b.labels = labels;
    b.max_during_build = (size_t)std::ceil((double)R * 1.3);
    b.nbrs.resize(n);
    for (uint32_t i = 0; i < n; i++) b.insert(i);
    /* build.rs:905-960 finalize_index_build: prune lists longer than R, write with sentinel */
    for (uint32_t i = 0; i < n; i++) {
        std::vector<Nwd> list = b.nbrs[i];
        if (list.size() > R) list = b.prune(i, list);
        for (uint32_t j = 0; j < R; j++)
            out_nbrs[(size_t)i * R + j] = j < list.size() ? list[j].node : ORC_INVALID_NODE;
    }
    *out_start_default = b.start_default;
    uint32_t k = 0;
    for (auto &kv : b.start_labeled) {
        if (k >= start_label_cap) break;
        out_start_labels[k] = kv.first;
        out_start_label_nodes[k] = kv.second;
        k++;
    }
    if (out_n_start_labels) *out_n_start_labels = k;
}

extern "C" void orc_build_batched(uint32_t n, uint32_t words, const uint64_t *codes, uint32_t R,
                                  uint32_t search_list_size, double max_alpha, int32_t has_labels,
                                  const uint32_t *label_off, const int16_t *labels, uint32_t max_batch,
                                  const orc_build_switches *sw, uint32_t *out_nbrs, uint32_t out_stride,
                                  uint64_t *out_counts) {
    Builder b;
    b.n = n;
    b.words = words;
    b.R = R;
    b.L = search_list_size;
    b.max_alpha = max_alpha;
    b.has_labels = has_labels != 0;
    b.codes = codes;
    b.label_off = label_off;
    b.labels = labels;
    b.max_during_build = (size_t)std::ceil((double)R * 1.3);
    b.nbrs.resize(n);
    if (sw) b.sw = *sw;
    if (max_batch == 0) max_batch = 0xFFFFFFFFu;
    /* node 0 alone (a batch of one is the reference's insert), then batches that grow with the graph */
    for (uint32_t lo = 0; lo < n;) {
        const uint32_t m = std::min(std::min(std::max<uint32_t>(1, lo / 16), max_batch), n - lo);
        for (uint32_t p = lo; p < lo + m; p++) { /* graph/mod.rs:490-533: start nodes, before the node's own search */
            if (!b.have_start) {
                b.have_start = true;
                b.start_default = p;
            }
            uint32_t nl;
            const int16_t *l = b.labs(p, &nl);
            for (uint32_t i = 0; i < nl; i++)
                if (!b.start_labeled.count(l[i])) b.start_labeled[l[i]] = p;
        }
        if (b.has_labels) b.insert_batch(lo, m, false);
        b.insert_batch(lo, m, true);
        lo += m;
    }
    for (uint32_t i = 0; i < n; i++) { /* build.rs:905-960 finalize_index_build */
        std::vector<Nwd> list = b.nbrs[i];
        if (list.size() > R) {
            list = b.prune(i, list);
            b.bc[ORC_BC_FINAL_PRUNED]++;
        }
        for (uint32_t j = 0; j < out_stride; j++)
            out_nbrs[(size_t)i * out_stride + j] = j < list.size() ? list[j].node : ORC_INVALID_NODE;
    }
    if (out_counts) std::memcpy(out_counts, b.bc, sizeof b.bc);
}
