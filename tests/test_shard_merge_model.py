"""The shards' merge rule (tests/shard_model.py) on hand-made row lists: the model every sharded GPU test compares with.
CPU only."""
import numpy as np

from shard_model import INVALID_TID, NAN_BITS, merge_shards, total_ukey

NEG_NAN, POS_NAN = 0xFFC00000, 0x7FC00000


def _f(bits):
    return np.array(bits, np.uint32).view(np.float32)


def _lists(rows, k):
    """rows: one list per shard of (tid, dist) -> tids[S][1,k], dists[S][1,k], counts[S][1] (padding past count)."""
    tids, dists, counts = [], [], []
    for r in rows:
        t = np.full((1, k), INVALID_TID, np.uint64)
        d = np.full((1, k), np.nan, np.float32)
        for j, (tid, dist) in enumerate(r):
            t[0, j] = tid
            d[0, j] = dist
        tids.append(t)
        dists.append(d)
        counts.append(np.array([len(r)], np.uint32))
    return tids, dists, counts


def test_total_ukey_is_the_total_order():
    order = [NEG_NAN, 0xFF800000, 0xBF800000, 0x80000001, 0x80000000, 0x00000000, 0x00000001, 0x3F800000, 0x7F800000,
             POS_NAN]
    keys = total_ukey(_f(order))
    assert list(keys) == sorted(keys) and len(set(keys.tolist())) == len(order)


def test_ties_across_shards_go_to_the_lower_shard():
    tids, dists, counts = _lists([[(10, 1.0), (11, 2.0)], [(20, 1.0), (21, 1.5)], [(30, 1.0)]], 5)
    tid, dist, shard, count = merge_shards(tids, dists, counts, 5)
    assert tid[0].tolist() == [10, 20, 30, 21, 11]
    assert shard[0].tolist() == [0, 1, 2, 1, 0]
    assert dist[0].tolist() == [1.0, 1.0, 1.0, 1.5, 2.0]
    assert count.tolist() == [5]


def test_equal_keys_inside_one_shard_keep_their_order():
    tids, dists, counts = _lists([[(1, 0.5), (2, 0.5), (3, 0.5)], [(9, 0.5)]], 4)
    tid, _, shard, _ = merge_shards(tids, dists, counts, 4)
    assert tid[0].tolist() == [1, 2, 3, 9]            # shard 0's head keeps winning the tie until its list is used up
    assert shard[0].tolist() == [0, 0, 0, 1]


def test_used_up_and_empty_shards_and_k_past_the_total():
    tids, dists, counts = _lists([[], [(5, 3.0)], [(7, 1.0), (8, 4.0)], []], 6)
    tid, dist, shard, count = merge_shards(tids, dists, counts, 6)
    assert count.tolist() == [3]
    assert tid[0, :3].tolist() == [7, 5, 8] and shard[0, :3].tolist() == [2, 1, 2]
    assert (tid[0, 3:] == INVALID_TID).all() and (shard[0, 3:] == -1).all()
    assert (dist[0, 3:].view(np.uint32) == NAN_BITS).all()
    tids, dists, counts = _lists([[], []], 3)
    tid, _, shard, count = merge_shards(tids, dists, counts, 3)
    assert count.tolist() == [0] and (tid == INVALID_TID).all() and (shard == -1).all()


def test_signed_zeros_infinities_and_both_nans():
    nz, pz = _f([0x80000000])[0], _f([0])[0]
    nn, pn = _f([NEG_NAN])[0], _f([POS_NAN])[0]
    tids, dists, counts = _lists([[(1, pz), (2, np.inf), (3, pn)], [(4, nn), (5, -np.inf), (6, nz)]], 6)
    tid, dist, shard, _ = merge_shards(tids, dists, counts, 6)
    # -NaN < -inf < -0.0 < +0.0 < +inf < +NaN, each compared only at its shard's head
    assert tid[0].tolist() == [4, 5, 6, 1, 2, 3]
    assert dist[0].view(np.uint32).tolist() == [NEG_NAN, 0xFF800000, 0x80000000, 0, 0x7F800000, POS_NAN]


def test_the_merge_never_resorts_a_shard_and_keeps_its_prefix():
    """Lists that are not sorted by distance (the rerank window can give such): each shard's rows come out as a
    prefix of its own list, in its own order."""
    rng = np.random.default_rng(5)
    S, B, k = 6, 40, 9
    tids = [np.arange(B * k, dtype=np.uint64).reshape(B, k) + np.uint64(1000 * s) for s in range(S)]
    dists = [rng.integers(0, 4, (B, k)).astype(np.float32) for _ in range(S)]
    counts = [rng.integers(0, k + 1, B).astype(np.uint32) for _ in range(S)]
    tid, dist, shard, count = merge_shards(tids, dists, counts, k)
    for b in range(B):
        assert count[b] == min(k, sum(int(c[b]) for c in counts))
        for s in range(S):
            mine = tid[b][shard[b] == s]
            assert mine.tolist() == tids[s][b, :len(mine)].tolist()
        # the rule, restated: each output row is the smallest (key, shard) among the heads at that point
        heads = [0] * S
        keys = [total_ukey(d[b]) for d in dists]
        for r in range(int(count[b])):
            live = [(int(keys[s][heads[s]]), s) for s in range(S) if heads[s] < counts[s][b]]
            _, s = min(live)
            assert shard[b, r] == s and tid[b, r] == tids[s][b, heads[s]]
            assert dist[b, r].view(np.uint32) == dists[s][b, heads[s]].view(np.uint32)
            heads[s] += 1


def test_one_shard_is_the_identity():
    rng = np.random.default_rng(9)
    B, k = 30, 7
    t = rng.integers(0, 1 << 40, (B, k)).astype(np.uint64)
    d = rng.standard_normal((B, k)).astype(np.float32)
    c = rng.integers(0, k + 1, B).astype(np.uint32)
    for b in range(B):
        t[b, c[b]:] = INVALID_TID
        d[b, c[b]:] = _f([NAN_BITS])[0]
    tid, dist, shard, count = merge_shards([t], [d], [c], k)
    assert np.array_equal(tid, t) and np.array_equal(dist.view(np.uint32), d.view(np.uint32))
    assert np.array_equal(count, c)
    assert np.array_equal(shard, np.where(np.arange(k)[None, :] < c[:, None], 0, -1))
