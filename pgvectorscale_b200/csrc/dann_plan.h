// dann_plan.h — host-side planning of the search kernels' per-query workspace and launch shape.
//
// Pure host arithmetic (no CUDA calls), shared by the C ABI implementation (diskann_b200.cu) and by the CPU
// SIMT-emulation harness under tests/simt, so that the emulated kernels run with exactly the shapes and arguments the
// product launches.  It lays out the shared memory of all three search kernels, so it includes their headers
// (DANN_LIST_CAP and SearchArgs of dann_search_common.cuh, sizeof(PairCtl), DANN_STG_CAP).
#pragma once
#include <stdint.h>
#include <stdio.h>
#include <stdlib.h>

#include <algorithm>

#include "dann_search.cuh"
#include "dann_search2.cuh"
#include "dann_search3.cuh"

struct SearchPlan {
    uint32_t need, cand_cap, hash_cap, vcap, hs, W, grid, per_warp, esize, bitmap_words, ins_cap;
    int entry; /* 0 = Ent32x21, 1 = Ent32x16, 2 = Ent64 */
    bool pairs; /* two-warp kernel (memory warp + heap warp per query) */
    bool lean;  /* dann_search3.cuh: one warp and a few KB of shared memory per query, up to 32 queries per SM */
    int maxw;   /* lean: the instantiation's resident-warp bound (32 -> 64 registers per thread, 16 -> 128) */
};

/* what the plan depends on besides the request */
struct PlanInputs {
    uint32_t n, R, words; /* nodes, neighbour slots per node, u64 words per SBQ code */
    size_t smem_optin;    /* cudaDeviceProp::sharedMemPerBlockOptin */
    int sm_count;
    uint32_t plain_dim;   /* 0 = SBQ layout; else num_dimensions_to_index of a plain-storage index */
    bool allow_lean;      /* one-shot batch search (no suspended scan, no build mode): the lean kernel may serve it */
    uint64_t ws_budget;   /* bytes of HBM the per-slot workspaces may take together (0 = no limit) */
};

static uint32_t env_u32(const char *name, uint32_t dflt) {
    const char *s = getenv(name);
    if (!s || !*s) return dflt;
    return (uint32_t)strtoul(s, nullptr, 10);
}

static uint32_t pow2ceil(uint32_t x) {
    uint32_t p = 1;
    while (p < x) p <<= 1;
    return p;
}

static int pick_code_mapping(uint32_t cw, uint32_t *G, uint32_t *Gshift, uint32_t *NCH) {
    uint32_t C = cw / 2;
    uint32_t g = pow2ceil((C + 2) / 3);
    if (g > 32) g = 32;
    uint32_t n = (C + g - 1) / g;
    uint32_t sup;
    if (n <= 4) sup = n;
    else if (n <= 8) sup = 8;
    else return -1;
    *G = g;
    *Gshift = 0;
    while ((1u << *Gshift) < g) (*Gshift)++;
    *NCH = sup;
    return 0;
}

/* Workspace sizes and launch shape for `nq` queries.  `grow` doubles on every overflow retry; `keyed` = the
 * scan has a label key.  Returns DANN_OK or DANN_ERR_CAPACITY with a message in `err`. */
static int dann_make_plan(const PlanInputs &in, uint32_t nq, uint32_t L, uint32_t c_target, uint32_t grow, bool keyed,
                          SearchPlan *p, bool force_single, char *err, size_t errlen) {
    err[0] = 0;
    /* visits are about L + consumed; every visit stages at most R ids */
    uint64_t need = (((uint64_t)L + c_target) * 23 / 20 + 40u) * in.R * grow; /* 15% slack over L + consumed */
    /* test hook: start from a deliberately small workspace to exercise the growth path */
    const uint32_t shrink = std::max<uint32_t>(env_u32("DANN_DEBUG_SHRINK", 1), 1);
    need = std::max<uint64_t>(need / shrink, 256);
    if (need > (1ull << 30)) {
        snprintf(err, errlen, "per-query workspace would exceed 2^30 candidates");
        return DANN_ERR_CAPACITY;
    }
    p->need = (uint32_t)need;
    p->cand_cap = (uint32_t)((need + 1023) & ~1023ull);
    p->hash_cap = pow2ceil(2 * p->cand_cap);
    /* inserted-set: one bitmap over node ids per resident warp while that stays small
     * (<= 2 MB per warp, i.e. up to 16M nodes), else the CAS hash set */
    const bool use_bitmap = env_u32("DANN_SEARCH_BITMAP", in.n <= (16u << 20) ? 1 : 0) != 0;
    p->bitmap_words = use_bitmap ? ((in.n + 127u) / 128u) * 4u : 0u;
    /* every deduped id is recorded, also the ones a label filter then rejects: visits x R */
    p->ins_cap = keyed ? 2 * p->cand_cap : p->cand_cap;
    if (keyed) p->hash_cap = pow2ceil(4 * p->cand_cap);
    /* heap entry layout (dann_search.cuh): 4 bytes whenever the distance and the sequence number fit */
    const uint64_t maxdist = (uint64_t)in.words * 64;
    if (maxdist < 2048 && p->cand_cap <= (1u << 21)) p->entry = 0;
    else if (maxdist < 65536 && p->cand_cap <= 65536) p->entry = 1;
    else p->entry = 2;
    p->entry = (int)env_u32("DANN_SEARCH_ENTRY", (uint32_t)p->entry); /* test hook */
    if (in.plain_dim) p->entry = 2; /* f32 keys need the 32-bit key field of Ent64 */
    p->esize = p->entry == 2 ? 8 : 4;
    /* visited holds the not-yet-consumed visits: about L, more under a label filter */
    uint64_t vcap = std::max<uint64_t>(((uint64_t)L * (keyed ? 2 : 1) + 96u) * grow / shrink, 8);
    p->vcap = (uint32_t)((vcap + 3) & ~3ull);
    const size_t budget = in.smem_optin > 1024 ? in.smem_optin - 1024 : in.smem_optin;
    p->lean = false;
    p->maxw = 0;
    /* kernel choice, batch searches: the lean warp-per-query kernel (dann_search3.cuh) - up to 32 resident queries
     * per SM - whenever neighbour lists fit one 64-id page; DANN_SEARCH_KERNEL=1/2 select the round-1 kernels */
    /* at most 16 slots per SM by default: the 32-slot instantiation is held to 64 registers and spills on sm_90a
     * (~220 B stores / ~320 B loads per thread), the 16-slot one gets up to 128 and spills nothing - 4.5 % less search
     * time at the 20M x 768 headline point on an H100 (profiles/h100_tuning_ab.json); DANN_SEARCH_WARPS selects up to 32 */
    uint32_t wneed3 = (nq + in.sm_count - 1) / in.sm_count;
    wneed3 = std::min<uint32_t>(std::max<uint32_t>(wneed3, 1), 16u);
    /* batches that fit the 7 two-warp slots per SM of dann_search2.cuh in one wave stay there: with so few resident
     * queries the chain latency of a query is the step time, and two warps per query shorten it;
     * DANN_SEARCH_KERNEL=3 forces the lean kernel */
    const bool small_batch = wneed3 <= 7u && !getenv("DANN_SEARCH_KERNEL") && !getenv("DANN_SEARCH_WARPS");
    if (in.allow_lean && !force_single && in.R <= 64 && !in.plain_dim && ((in.words + 1u) & ~1u) <= 192u &&
        env_u32("DANN_SEARCH_KERNEL", 3) == 3 && !small_batch) {
        /* inserted-set: bitmap over node ids while a node id fits the 21-bit payload of a 4-byte entry and the
         * bitmap is not larger than the hash set; else an open-addressing set of 1.5 x the candidate bound
         * (3 x under a label key: rejected ids are recorded too), any multiple of 4 slots */
        const uint64_t hcap = ((uint64_t)p->cand_cap * (keyed ? 3u : 1u) * 3u / 2u + 3u) & ~3ull;
        const uint64_t bm_bytes = (uint64_t)((in.n + 127u) / 128u) * 16u;
        bool bm = in.n <= (1u << 21) && bm_bytes <= hcap * 4u;
        if (getenv("DANN_SEARCH_BITMAP")) bm = env_u32("DANN_SEARCH_BITMAP", 0) != 0 && in.n <= (16u << 20);
        const bool small = maxdist < 2048 && (bm ? in.n <= (1u << 21) : hcap <= (1u << 21)) && p->cand_cap <= (1u << 21);
        int entry3 = small ? 0 : 2;
        if (getenv("DANN_SEARCH_ENTRY") && env_u32("DANN_SEARCH_ENTRY", 0) == 2) entry3 = 2; /* test hook */
        const uint32_t esize3 = entry3 == 2 ? 8 : 4;
        uint32_t G3 = 1, Gs3 = 0, NCH3 = 1;
        pick_code_mapping((in.words + 1u) & ~1u, &G3, &Gs3, &NCH3);
        /* visited ring + page (entries, ids) + push staging area + the query's SBQ code (NCH x G 16-byte chunks) */
        const size_t fixed3 = (size_t)p->vcap * esize3 + (size_t)DANN_LIST_CAP * (esize3 + 4u) + (size_t)DANN_STG_CAP * esize3 +
                              (size_t)NCH3 * G3 * 16u + 16u;
        const uint32_t hs_floor = (uint32_t)std::min<uint64_t>((uint64_t)p->cand_cap, 256);
        if (fixed3 + (size_t)hs_floor * esize3 + 64 <= budget && hcap <= 0xFFFFFFFCull) {
            uint32_t W3 = env_u32("DANN_SEARCH_WARPS", wneed3);
            W3 = std::min<uint32_t>(std::max<uint32_t>(W3, 1), 32u);
            const uint64_t per_slot_hbm = (uint64_t)p->cand_cap * esize3 + (bm ? bm_bytes : hcap * 4u);
            for (;; W3--) {
                const uint64_t slots = (uint64_t)std::min<uint32_t>((uint32_t)in.sm_count, (nq + W3 - 1) / W3) * W3;
                const bool smem_ok = (budget / W3 & ~(size_t)15) >= fixed3 + (size_t)hs_floor * esize3;
                const bool hbm_ok = !in.ws_budget || slots * per_slot_hbm <= in.ws_budget;
                if ((smem_ok && hbm_ok) || W3 == 1) break;
            }
            const size_t per_warp3 = (budget / W3) & ~(size_t)15;
            uint32_t hs3 = (uint32_t)std::min<size_t>((size_t)p->cand_cap, (per_warp3 - fixed3) / esize3);
            hs3 = std::min<uint32_t>(env_u32("DANN_SEARCH_HS", hs3), (uint32_t)((per_warp3 - fixed3) / esize3));
            hs3 = std::max<uint32_t>(hs3 & ~3u, 4u);
            p->bitmap_words = bm ? ((in.n + 127u) / 128u) * 4u : 0u;
            p->hash_cap = bm ? 4u : (uint32_t)hcap;
            p->ins_cap = 0;
            p->entry = entry3;
            p->esize = esize3;
            p->hs = hs3;
            p->W = W3;
            p->per_warp = (uint32_t)((fixed3 + (size_t)hs3 * esize3 + 15) & ~(size_t)15);
            p->grid = std::min<uint32_t>((uint32_t)in.sm_count, (nq + W3 - 1) / W3);
            p->pairs = false;
            p->lean = true;
            p->maxw = W3 <= 16 ? 16 : 32;
            return DANN_OK;
        }
    }
    /* the two-warp kernel handles neighbour lists of up to 64 ids */
    p->pairs = !force_single && in.R <= 64 && env_u32("DANN_SEARCH_KERNEL", 2) != 1 && !in.plain_dim;
    const uint32_t wmax = p->pairs ? 7u : 12u; /* __launch_bounds__ of the two kernels */
    const size_t fixed = (size_t)p->vcap * 8 + (p->pairs ? 4 * DANN_LIST_CAP * 4 + sizeof(PairCtl) + 32 * 4 + 32 * 8 : 2 * DANN_LIST_CAP * 4) +
                         (size_t)((in.plain_dim + 3u) & ~3u) * 4; /* plain layout: the query's index slice */
    if (fixed + 1024 > budget) {
        snprintf(err, errlen, "visited list of %u entries does not fit shared memory", p->vcap);
        return DANN_ERR_CAPACITY;
    }
    uint32_t wneed = (nq + in.sm_count - 1) / in.sm_count;
    wneed = std::min<uint32_t>(std::max<uint32_t>(wneed, 1), wmax);
    /* Concurrency first: a batch should run in one wave (queries are latency-bound, one or two
     * warps each), so take as many query slots per SM as the batch needs and give each slot
     * whatever shared memory is left for the top of its heap; deeper heap levels spill to the
     * slot's HBM tail.  Only when that would leave fewer than 2048 in-smem entries (the top 11
     * levels) do we trade slots for shared memory. */
    const uint32_t hs_min = (uint32_t)std::min<uint64_t>(p->cand_cap, 2048);
    uint32_t wfit = (uint32_t)(budget / (fixed + (size_t)hs_min * p->esize));
    uint32_t W = std::min(wneed, std::max<uint32_t>(wfit, 1));
    W = env_u32("DANN_SEARCH_WARPS", W);
    W = std::min<uint32_t>(std::max<uint32_t>(W, 1), wmax);
    while (W > 1 && budget / W < fixed + 1024) W--;
    size_t per_warp = (budget / W) & ~(size_t)15;
    uint32_t hs = (uint32_t)std::min<size_t>(p->cand_cap, (per_warp - fixed) / p->esize);
    hs = std::min<uint32_t>(env_u32("DANN_SEARCH_HS", hs), (uint32_t)((per_warp - fixed) / p->esize)); /* test hook, never past the budget */
    hs = std::min(hs, p->cand_cap) & ~3u;
    p->hs = hs;
    p->W = W;
    p->per_warp = (uint32_t)((fixed + (size_t)hs * p->esize + 15) & ~(size_t)15);
    p->grid = std::min<uint32_t>((uint32_t)in.sm_count, (nq + W - 1) / W);
    return DANN_OK;
}

/* The launch arguments every search kernel takes from the index (its view, code mapping and list check) and from the
 * plan; the caller adds its request, its buffers and its mode. */
static SearchArgs search_args_for_plan(const IndexView &v, uint32_t G, uint32_t Gshift, uint32_t lists_unique, const SearchPlan &p) {
    SearchArgs a;
    a.ix = v;
    a.G = G;
    a.Gshift = Gshift;
    a.lists_unique = lists_unique;
    a.hash_cap = p.hash_cap;
    a.bitmap_words = p.bitmap_words;
    a.ins_cap = p.ins_cap;
    a.cand_cap = p.cand_cap;
    a.hs = p.hs;
    a.vcap = p.vcap;
    a.per_warp_smem = p.per_warp;
    return a;
}
