"""The model of dann_shards_search_batch (test infrastructure): every shard scanned by the oracle, then the shards' rows
merged by the rule include/diskann_b200.h states for the merge kernel.

The merge is a k-way merge of the shards' row lists by their heads, the way an executor merges ordered per-partition
scans: shard s's list is its first count_s[b] rows in its own order; k times, among the shards whose list is not used
up, take the head with the smallest key (f32::total_cmp key of its distance, s), output it and advance that shard.
Ties of distance go to the lower shard; a shard's list is never re-sorted."""
from __future__ import annotations

import heapq

import numpy as np

from oracle import oracle

INVALID_TID = np.uint64(0xFFFFFFFFFFFFFFFF)
NAN_BITS = 0x7FC00000          # distance past count, as the rerank kernel leaves it


def total_ukey(dist) -> np.ndarray:
    """f32::total_cmp as an unsigned 32-bit key (total_ukey in csrc/dann_device.cuh): negative floats have every bit
    flipped, the others only the sign bit."""
    b = np.ascontiguousarray(dist, dtype=np.float32).view(np.uint32)
    return np.where(b >> np.uint32(31), ~b, b | np.uint32(0x80000000)).astype(np.uint32)


def merge_shards(tids, dists, counts, k: int):
    """tids[S][B, >=k'] u64, dists[S][B, >=k'] f32, counts[S][B] -> tid[B,k], dist[B,k], shard[B,k] i32, count[B]."""
    S = len(tids)
    B = len(counts[0]) if S else 0
    tid = np.full((B, k), INVALID_TID, np.uint64)
    dist = np.full((B, k), NAN_BITS, np.uint32).view(np.float32)
    shard = np.full((B, k), -1, np.int32)
    count = np.zeros(B, np.uint32)
    keys = [total_ukey(d) for d in dists]
    for b in range(B):
        heads = [(int(keys[s][b, 0]), s, 0) for s in range(S) if counts[s][b] > 0]
        heapq.heapify(heads)
        r = 0
        while r < k and heads:
            _, s, j = heapq.heappop(heads)
            tid[b, r], dist[b, r], shard[b, r] = tids[s][b, j], dists[s][b, j], s
            r += 1
            if j + 1 < counts[s][b]:
                heapq.heappush(heads, (int(keys[s][b, j + 1]), s, j + 1))
        count[b] = r
    return tid, dist, shard, count


def scan_shards(snaps, queries, labels, label_off, L: int, rescore: int, k: int):
    """oracle.scan_batch on every shard, merged.  -> tid[B,k], dist[B,k], shard[B,k], count[B], stats[S, B]."""
    per = [oracle.scan_batch(s, queries, labels, label_off, L, rescore, k) for s in snaps]
    tid, dist, shard, count = merge_shards([p[0] for p in per], [p[1] for p in per], [p[2] for p in per], k)
    return tid, dist, shard, count, np.stack([p[3] for p in per])
