"""dann_shards: a table split into shards, one independent index per shard, every query's rows merged on the device
(include/diskann_b200.h).  Every case is compared with tests/shard_model.scan_shards - the oracle's scan on every shard,
merged by the rule the merge kernel states - on tid, distance bits, shard, count and the per-shard counters."""
import os

import numpy as np
import pytest

from conftest import build_case, emulating
from oracle import fixtures, oracle
from shard_model import scan_shards

pytestmark = pytest.mark.gpu

COSINE, L2, IP = 0, 1, 2
K = 10
STAT_FIELDS = ("visits", "d_quantized", "candidates", "d_full")


@pytest.fixture(scope="module")
def lib(lib_built):
    from pgvectorscale_b200 import diskann
    if diskann.device_count() < 1:
        pytest.fail("no CUDA device visible: -m gpu tests need an H100")
    return diskann


def _global_tids(s, shard):
    """rows of different shards are different rows of the table: move shard i's heap blocks out of the others' way
    (the offset stays, so a deleted row stays deleted)"""
    s.heap_tid = s.heap_tid + (np.uint64(shard * 100000) << np.uint64(16))
    return s


def _shards(sizes, dist, bits, dim=48, seed=1, **kw):
    out = []
    for i, n in enumerate(sizes):
        s = build_case(n, dim, dist, bits=bits, seed=seed + 31 * i, R=16, L_build=32, deleted_every=9 if n > 50 else 0,
                       **kw)
        out.append(_global_tids(s, i))
    return out


def _labels_csr(labs):
    flat = np.array([x for ls in labs for x in ls], np.int16)
    off = np.cumsum([0] + [len(ls) for ls in labs]).astype(np.int32)
    return flat, off


def _search(lib, snaps, q, L, rescore, labels=None, devices=None, k=K):
    with lib.ShardedIndex(snaps, devices=[0] * len(snaps) if devices is None else devices) as g:
        assert g.count == len(snaps)
        return g.search_batch(q, labels=labels, k=k, search_list_size=L, rescore=rescore)


def _check(got, snaps, q, L, rescore, labels=None, k=K):
    flat, off = _labels_csr(labels) if labels is not None else (None, None)
    tid, dist, shard, count, stats = scan_shards(snaps, q, flat, off, L, rescore, k)
    assert np.array_equal(got["count"], count)
    assert np.array_equal(got["tid"], tid)
    assert np.array_equal(got["shard"], shard)
    assert np.array_equal(got["dist"].view(np.uint32), dist.view(np.uint32))
    assert got["stats"].shape == (len(snaps), q.shape[0])
    for f in STAT_FIELDS:
        assert np.array_equal(got["stats"][f].astype(np.uint64), stats[f]), f
    return tid, dist, shard, count


SIZES = {1: [700], 2: [600, 0], 3: [500, 7, 300], 5: [400, 0, 7, 250, 600]}
_CACHE = {}


@pytest.mark.parametrize("nshards", [1, 2, 3, 5])
@pytest.mark.parametrize("dist,bits", [(COSINE, 1), (COSINE, 2), (L2, 1), (L2, 2), (IP, 1), (IP, 2)],
                         ids=["cos1", "cos2", "l2-1", "l2-2", "ip1", "ip2"])
def test_shards_equal_the_model(lib, dist, bits, nshards):
    """shards of different sizes on device 0: deleted rows, an empty shard, a shard with fewer than k rows"""
    key = (dist, bits, nshards)
    if key not in _CACHE:
        _CACHE[key] = _shards(SIZES[nshards], dist, bits, seed=10 * dist + bits)
    snaps = _CACHE[key]
    if nshards > 1:
        assert any(s.n == 0 for s in snaps) or any(0 < s.n < K for s in snaps)
    q = fixtures.gen_vectors(13, 48, 100 + dist, "normal")
    got = _search(lib, snaps, q, 40, 20)
    tid, _, shard, count = _check(got, snaps, q, 40, 20)
    assert (count == K).all()
    if nshards > 2:
        assert len(np.unique(shard[shard >= 0])) > 1            # the merge took rows from more than one shard


def test_one_shard_is_dann_search_batch(lib):
    s = _global_tids(build_case(900, 64, L2, seed=5, R=16, L_build=32, deleted_every=7), 0)
    q = fixtures.gen_vectors(21, 64, 6, "normal")
    got = _search(lib, [s], q, 50, 30)
    with lib.DiskAnnIndex(s) as idx:
        one = idx.search_batch(q, k=K, search_list_size=50, rescore=30)
    assert np.array_equal(got["tid"], one["tid"])
    assert np.array_equal(got["dist"].view(np.uint32), one["dist"].view(np.uint32))
    assert np.array_equal(got["count"], one["count"])
    assert np.array_equal(got["stats"][0], one["stats"])
    assert np.array_equal(got["shard"], np.where(got["tid"] != lib.INVALID_TID, 0, -1))
    _check(got, [s], q, 50, 30)


def test_the_same_snapshot_twice_gives_every_row_twice_shard_0_first(lib):
    """every key ties across the two shards.  rescore 1000 > n keeps the whole stream in the rerank window, so each
    list is sorted and the merge alternates the shards row by row"""
    s = build_case(600, 32, COSINE, seed=8, R=16, L_build=32)
    q = fixtures.gen_vectors(9, 32, 9, "normal")
    got = _search(lib, [s, s], q, 40, 1000)
    with lib.DiskAnnIndex(s) as idx:
        one = idx.search_batch(q, k=K, search_list_size=40, rescore=1000)
    _check(got, [s, s], q, 40, 1000)
    assert (np.diff(one["dist"], axis=1) >= 0).all()
    assert np.array_equal(got["tid"], np.repeat(one["tid"][:, :K // 2], 2, axis=1))
    assert np.array_equal(got["shard"], np.tile([0, 1], (9, K // 2)))


def test_label_sets_that_differ_between_shards(lib):
    """shard 1 carries labels 21..36 instead of 1..16: keys only some shards hold, keys no shard holds"""
    snaps = _shards([500, 400, 300], L2, 2, dim=32, seed=40, labels=True)
    snaps[1].labels = snaps[1].labels + np.int16(20)
    snaps[1].start_labels = snaps[1].start_labels + np.int16(20)
    q = fixtures.gen_vectors(16, 32, 41, "normal")
    labs = [[3], [25], [3, 25], [40], [7, 8], [30, 31], [1], [36]] * 2
    got = _search(lib, snaps, q, 50, 25, labels=labs)
    _, _, shard, count = _check(got, snaps, q, 50, 25, labels=labs)
    assert count[3] == 0 and count[11] == 0                      # label 40: no shard has it
    assert set(shard[1][: count[1]]) == {1}                      # label 25: only shard 1
    assert 1 not in set(shard[0][: count[0]])                     # label 3: every shard but 1


def _special_rows(n, dim, seed, dist):
    """uniform rows with 10 % of their components at +-3e38: +inf L2 distances, and inner products of +-inf and NaN
    (inf + -inf).  For L2 also rows of +-inf and one of NaN (the scan path's L2 NaN is 0xFFC00000).  Inner products of
    such rows are left out: the emulated ABI's x86 arithmetic cannot give a NaN inner product's GPU bits."""
    rng = np.random.default_rng(seed)
    v = rng.uniform(-1, 1, (n, dim)).astype(np.float32)
    big = rng.random((n, dim)) < 0.1
    v[big] = np.where(rng.random(big.sum()) < 0.5, np.float32(3e38), np.float32(-3e38))
    if dist == L2:
        v[5] = np.inf
        v[6] = -np.inf
        v[7, ::2] = np.inf
        v[8] = np.nan
    return v


@pytest.mark.parametrize("dist", [L2, IP], ids=["l2", "ip"])
def test_nan_infinite_and_duplicate_rows(lib, dist):
    """keys the rerank window produces on such rows - NaN (both signs), +-inf, runs of equal distances - met by the
    merge, within a shard and across shards (shard 2 repeats rows of shard 0)"""
    v0 = _special_rows(300, 32, 50 + dist, dist)
    v1 = np.random.default_rng(51).uniform(-1, 1, (200, 32)).astype(np.float32)
    v2 = np.concatenate([v0[:40], v0[:40]])
    snaps = [_global_tids(fixtures.make_index(v, dist, bits=2, R=16, L_build=32), i) for i, v in enumerate((v0, v1, v2))]
    q = np.concatenate([v0[:6], v0[9:13], v1[:3], -v0[10:12]]).astype(np.float32)
    got = _search(lib, snaps, q, 60, 40)
    _, dist_, shard, count = _check(got, snaps, q, 60, 40)
    d = np.concatenate([dist_[b, :count[b]] for b in range(len(q))])
    assert not np.isfinite(d).all()
    assert len(d) - len(np.unique(d.view(np.uint32))) > 10       # ties


def _one_wave_of_warps():
    """warps the merge launch has at most: one 8-warp block per SM of device 0"""
    if emulating():
        return int(os.environ.get("SIMT_SM_COUNT") or 132) * 8
    import torch
    return torch.cuda.get_device_properties(0).multi_processor_count * 8


@pytest.mark.parametrize("nshards", [33, 256])
def test_many_tiny_shards_and_more_queries_than_one_wave_of_warps(lib, nshards):
    """more queries than the merge launch has warps (so warps take a second query), 33 shards (lane 0 holds two heads)
    and 256 shards of 1..12 rows (every lane holds eight)"""
    rng = np.random.default_rng(nshards)
    snaps = []
    for i in range(nshards):
        n = int(rng.integers(1, 13))
        v = fixtures.gen_vectors(n, 16, 1000 + i, "normal")
        snaps.append(_global_tids(fixtures.make_index(v, COSINE, bits=2, R=8, L_build=16), i))
    q = fixtures.gen_vectors(_one_wave_of_warps() + 44, 16, 77, "normal")
    got = _search(lib, snaps, q, 20, 12)
    _, _, shard, _ = _check(got, snaps, q, 20, 12)
    assert shard.max() >= 32


def test_shards_built_in_place_then_given_their_rows(lib):
    """dann_build_graph through dann_shards_index on each loaded shard, then set_vectors: the rows the model gives for
    the graphs the GPU built"""
    from pgvectorscale_b200.snapshot import INVALID_NODE
    snaps, rows = [], []
    for i, n in enumerate((300, 200, 120)):
        s = _global_tids(build_case(n, 32, L2, seed=60 + i, R=8, L_build=16), i)
        rows.append(s.vectors)
        s.R = 64
        s.nbrs = np.full((n, 64), INVALID_NODE, np.uint32)
        s.start_default = 0
        s.vectors = None
        snaps.append(s)
    q = fixtures.gen_vectors(11, 32, 61, "normal")
    with lib.ShardedIndex(snaps, devices=[0, 0, 0]) as g:
        for i, s in enumerate(snaps):
            ix = g.shard(i)
            assert ix.n == s.n and ix.R == 64
            ix.build_graph(24, 48, 1.2, 64)
            s.nbrs = ix.download_nbrs()
            ix.set_vectors(rows[i])
            s.vectors = rows[i]
        got = g.search_batch(q, k=K, search_list_size=40, rescore=20)
        timing = g.shard(2).last_batch_timing()
    assert timing["total_ms"] >= 0.0
    _check(got, snaps, q, 40, 20)


def test_refusals(lib):
    E = lib.DiskAnnError
    a = build_case(100, 32, L2, seed=70, R=8, L_build=16)
    other = {"dim": build_case(100, 48, L2, seed=71, R=8, L_build=16),
             "distance_type": build_case(100, 32, IP, seed=72, R=8, L_build=16),
             "has_labels": build_case(100, 32, L2, seed=73, R=8, L_build=16, labels=True)}
    for what, b in other.items():
        with pytest.raises(E) as ei:
            lib.ShardedIndex([a, b], devices=[0, 0])
        assert ei.value.code == -1, what
    for snaps in ([], [a] * 257):
        with pytest.raises(E) as ei:
            lib.ShardedIndex(snaps, devices=[0] * len(snaps))
        assert ei.value.code == -1
    q = fixtures.gen_vectors(4, 32, 74, "normal")
    with lib.ShardedIndex([a, a], devices=[0, 0]) as g:
        with pytest.raises(E) as ei:
            g.search_batch(q, k=K, search_list_size=40, rescore=0)
        assert ei.value.code == -1
        with pytest.raises(E) as ei:
            g.search_batch(q, k=K, search_list_size=0, rescore=10)
        assert ei.value.code == -1 and "shard 0:" in str(ei.value)
        ok = g.search_batch(q, k=K, search_list_size=40, rescore=10)       # a refused call leaves the handle usable
    _check(ok, [a, a], q, 40, 10)
    import copy
    bare = copy.copy(a)
    bare.vectors = None
    with lib.ShardedIndex([a, bare], devices=[0, 0]) as g:
        with pytest.raises(E) as ei:
            g.search_batch(q, k=K, search_list_size=40, rescore=10)
        assert ei.value.code == -6 and "shard 1:" in str(ei.value)


def test_a_missing_device_is_refused_without_a_leak(lib):
    a = build_case(2000, 64, L2, seed=80, R=16, L_build=32)
    free = None
    if not emulating():
        import torch
        torch.cuda.init()
        free = torch.cuda.mem_get_info(0)[0]
    for _ in range(3):
        with pytest.raises(lib.DiskAnnError) as ei:
            lib.ShardedIndex([a, a], devices=[0, 99])
        assert "shard 1 (device 99)" in str(ei.value)
    if free is not None:
        import torch
        assert free - torch.cuda.mem_get_info(0)[0] < (4 << 20)


def test_two_devices_equal_one(lib):
    if lib.device_count() < 2:
        pytest.skip("needs two CUDA devices (or SIMT_FAKE_DEVICES=2 under the emulated ABI)")
    snaps = _shards([400, 250, 7, 300], COSINE, 2, seed=90)
    q = fixtures.gen_vectors(17, 48, 91, "normal")
    one = _search(lib, snaps, q, 40, 20)
    for devs in ([0, 1, 0, 1], [1, 0, 1, 0]):                   # the second: the primary device is 1
        got = _search(lib, snaps, q, 40, 20, devices=devs)
        for f in ("tid", "shard", "count", "stats"):
            assert np.array_equal(got[f], one[f]), (devs, f)
        assert np.array_equal(got["dist"].view(np.uint32), one["dist"].view(np.uint32))
    _check(one, snaps, q, 40, 20)
