// dann_shards.cuh — the merge step of dann_shards_search_batch (host side: dann_shards.h).
//
// Inputs sit on the primary device, shard-major: tid[s][B][k], dist[s][B][k], count[s][B] (count <= k).  One warp per
// query, grid-stride over queries.  Lane l holds the heads of shards l, l+32, ... (DANN_SHARDS_PER_LANE slots, all
// indexed with compile-time constants so they stay in registers).  Each round the warp takes the 64-bit minimum of
// (total_ukey(dist) << 32 | s) over every live head with a shuffle butterfly (__reduce_min_sync is 32-bit only); the
// lane owning the winner writes the row and advances that shard's head.  Ties of distance go to the lower shard, and
// a shard's list is never re-sorted: its rows come out as a prefix of its own order.
#pragma once
#include "dann_device.cuh"

#define DANN_SHARDS_MAX 256
#define DANN_SHARDS_PER_LANE (DANN_SHARDS_MAX / 32)
#define DANN_MERGE_WARPS 8

struct ShardMergeArgs {
    const uint64_t *tid;
    const float *dist;
    const uint32_t *count;
    uint32_t S, B, k;
    uint64_t *out_tid;
    float *out_dist;
    int32_t *out_shard;
    uint32_t *out_count;
};

__global__ void __launch_bounds__(DANN_MERGE_WARPS * 32) dann_shard_merge_kernel(const ShardMergeArgs a) {
    const uint32_t lane = threadIdx.x & 31u;
    const size_t bk = (size_t)a.B * a.k;
    const uint32_t warps = gridDim.x * DANN_MERGE_WARPS;
    for (uint32_t b = blockIdx.x * DANN_MERGE_WARPS + (threadIdx.x >> 5); b < a.B; b += warps) {
        uint32_t head[DANN_SHARDS_PER_LANE], cnt[DANN_SHARDS_PER_LANE];
        uint64_t key[DANN_SHARDS_PER_LANE]; /* ~0: no head (shard absent or used up) */
#pragma unroll
        for (int j = 0; j < DANN_SHARDS_PER_LANE; j++) {
            const uint32_t s = lane + 32u * j;
            head[j] = 0;
            cnt[j] = s < a.S ? a.count[(size_t)s * a.B + b] : 0u;
            key[j] = cnt[j] ? ((uint64_t)total_ukey(a.dist[s * bk + (size_t)b * a.k]) << 32) | s : ~0ull;
        }
        uint32_t r = 0;
        for (; r < a.k; r++) {
            uint64_t m = key[0];
#pragma unroll
            for (int j = 1; j < DANN_SHARDS_PER_LANE; j++) m = key[j] < m ? key[j] : m;
#pragma unroll
            for (int o = 16; o > 0; o >>= 1) {
                const uint64_t x = __shfl_xor_sync(DANN_FULL, m, o);
                m = x < m ? x : m;
            }
            if (m == ~0ull) break; /* every list used up (uniform across the warp) */
            const uint32_t s = (uint32_t)m;
            if ((s & 31u) == lane) {
#pragma unroll
                for (int j = 0; j < DANN_SHARDS_PER_LANE; j++)
                    if ((uint32_t)j == (s >> 5)) {
                        const size_t at = (size_t)b * a.k;
                        a.out_tid[at + r] = a.tid[s * bk + at + head[j]];
                        if (a.out_dist) a.out_dist[at + r] = total_ukey_inverse((uint32_t)(m >> 32));
                        if (a.out_shard) a.out_shard[at + r] = (int32_t)s;
                        head[j]++;
                        key[j] = head[j] < cnt[j] ? ((uint64_t)total_ukey(a.dist[s * bk + at + head[j]]) << 32) | s : ~0ull;
                    }
            }
        }
        /* r rows merged: the rest of the row is "no row", as the rerank kernel leaves it */
        for (uint32_t i = r + lane; i < a.k; i += 32u) {
            const size_t at = (size_t)b * a.k + i;
            a.out_tid[at] = DANN_INVALID_TID;
            if (a.out_dist) a.out_dist[at] = __int_as_float(0x7fc00000);
            if (a.out_shard) a.out_shard[at] = -1;
        }
        if (lane == 0 && a.out_count) a.out_count[b] = r;
    }
}
