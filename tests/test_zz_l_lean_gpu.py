"""The lean warp-per-query search kernel (dann_search3.cuh) against the oracle, across every instantiation it ships.

The kernel serves every batch of more than 7 queries per SM, i.e. every batch bench.py times, but the other parity tests
use batches small enough for the two-warp kernel.  Here DANN_SEARCH_KERNEL=3 forces the lean kernel onto small batches,
and the plan of every call is read back, so a plan change that sends a case to another kernel fails instead of passing
quietly.  Bar, as in test_gpu_parity.py: bit-exact TIDs, bit-exact rerank distances (u32), counts, all five counters,
status 0.

Instantiations dann_search3_kernel<T, NCH, MAXW> (diskann_b200.cu pick_lean): T = Ent32x21 (4-byte entry, payload =
node id under the bitmap inserted-set, hash slot under the hash set) or Ent64; NCH = 1, 2, 3 16-byte chunks per lane
(dann_plan.h pick_code_mapping: words = ceil(dim * bits / 64), cw = (words + 1) & ~1); MAXW = 16 or 32 slots per SM.

   dim x bits | cw, G, NCH  | code gather | entry
   37 x 2     | 2, 1, 1     | exact       | 4 bytes
   100 x 2    | 4, 1, 2     | exact       | 4 bytes
   320 x 2    | 10, 2, 3    | bounds test | 4 bytes
   768 x 2    | 24, 4, 3    | exact       | 4 bytes (the benchmark's shape)
   992 x 2    | 32, 8, 2    | exact       | 4 bytes, the largest (max distance 1984 < 2048)
   1024 x 2   | 32, 8, 2    | exact       | 8 bytes, the smallest code that needs them
   1537 x 2   | 50, 16, 2   | bounds test | 8 bytes
   6144 x 2   | 192, 32, 3  | exact       | 8 bytes, the largest code the lean kernel takes
   6145 x 2   | 194         |             | two-warp kernel even under DANN_SEARCH_KERNEL=3

The tests whose names contain `gpu_built` build 2^21-node indexes with the GPU graph builder; the rest also run under
the CPU SIMT emulator (DANN_EMULATE=1, see tests/test_emulated_abi.py)."""
import copy
import functools
import os

import numpy as np
import pytest

from conftest import build_case, emulating
from test_gpu_parity import COSINE, IP, L2, _compare_batch, _queries

pytestmark = pytest.mark.gpu

HOOKS = ("DANN_SEARCH_KERNEL", "DANN_SEARCH_WARPS", "DANN_SEARCH_HS", "DANN_SEARCH_BITMAP", "DANN_SEARCH_ENTRY",
         "DANN_DEBUG_SHRINK")
INVALID = 0xFFFFFFFF


@pytest.fixture(scope="module")
def lib(lib_built):
    from pgvectorscale_b200 import diskann
    if diskann.device_count() < 1:
        pytest.fail("no CUDA device visible: -m gpu tests need an H100")
    return diskann


@pytest.fixture
def env(monkeypatch):
    """env(KERNEL=3, WARPS=16, ...) sets exactly these DANN_SEARCH_* / DANN_DEBUG_SHRINK hooks and clears the others."""
    def set_(**kv):
        for h in HOOKS:
            monkeypatch.delenv(h, raising=False)
        for key, val in kv.items():
            name = "DANN_DEBUG_SHRINK" if key == "SHRINK" else "DANN_SEARCH_" + key
            assert name in HOOKS, key
            monkeypatch.setenv(name, str(val))
    set_()
    return set_


def sm_count():
    if emulating():
        return int(os.environ.get("SIMT_SM_COUNT", "132"))
    import torch
    return torch.cuda.get_device_properties(0).multi_processor_count


def check(s, idx, q, k, L, rescore, labels=None, *, kernel=3, entry=None, bitmap=None, slots=None, retried=False):
    """Oracle parity of the whole batch, then proof of which kernel and which instantiation served it.
    last_search_plan() describes the first launch of the call; a growth retry only bumps `retries`.  The reruns of the
    overflowing queries are planned from the same hooks (every test here pins KERNEL, WARPS and BITMAP, and ENTRY where
    it matters), so their kernel and inserted-set are those asserted here; that is taken on trust, not read back."""
    g = _compare_batch(s, idx, q, k, L, rescore, labels)
    p = idx.last_search_plan()
    assert p["kernel"] == kernel, p
    if entry is not None:
        assert p["entry_bytes"] == entry, p
    if bitmap is not None:
        assert p["bitmap"] == bitmap, p
    if slots is not None:
        assert p["slots_per_sm"] == slots, p
    if retried:
        assert p["retries"] >= 1, p
    return g, p


@functools.lru_cache(maxsize=None)
def _case(n, dim, dist, kind, seed, R=24, L_build=48, **kw):
    return build_case(n, dim, dist, bits=2, seed=seed, kind=kind, R=R, L_build=L_build, **kw)


def case(*a, **kw):
    """A cached fixture index; a shallow copy, so that a test may replace an array without touching the cache."""
    return copy.copy(_case(*a, **kw))


def fill_lists(s, seed):
    """Every neighbour list full (R distinct ids, no terminator): what the builder leaves only for some nodes."""
    rng = np.random.default_rng(seed)
    nb = s.nbrs.copy()
    for i in range(s.n):
        have = [int(x) for x in nb[i] if x != INVALID]
        free = np.setdiff1d(np.arange(s.n), np.array(have + [i]))
        rng.shuffle(free)
        nb[i] = np.array(have + [int(x) for x in free[:s.R - len(have)]], np.uint32)
    s.nbrs = nb
    return s


# (dim, distance, data kind, entry bytes of the lean plan)
SHAPES = [(37, COSINE, "normal", 4), (100, L2, "uniform", 4), (320, IP, "uniform", 4), (768, COSINE, "normal", 4),
          (992, L2, "uniform", 4), (1024, IP, "uniform", 8), (1537, COSINE, "normal", 8), (6144, L2, "uniform", 8)]


@pytest.mark.parametrize("dim,dist,kind,entry", SHAPES, ids=[f"{d}x2" for d, *_ in SHAPES])
def test_instantiation_matrix(lib, env, dim, dist, kind, entry):
    """Every (entry, NCH) x both inserted-sets x both MAXW builds, heap tops of 4 / 16 / 256+ entries, a zero query.
    Codes that fit 4-byte entries run with DANN_SEARCH_ENTRY=2 as well: Ent64 never arises by itself at NCH = 1
    (at most 128 code bits) on an index this small."""
    s = case(400, dim, dist, kind, seed=dim)
    q = _queries(s, 40, dim + 1, kind)
    q[5] = 0.0                                                # NULL-like query: all-zero code
    hs = {37: 4, 100: 16, 320: 4, 768: 16, 992: None, 1024: 4, 1537: 16, 6144: 4}[dim]
    extra = {} if hs is None else {"HS": hs}
    layouts = [({}, entry)] + ([({"ENTRY": 2}, 8)] if entry == 4 else [])
    with lib.DiskAnnIndex(s) as idx:
        for hooks, e in layouts:
            for bitmap in (1, 0):
                for warps, (k, L, rescore) in ((16, (10, 40, 20)), (32, (7, 25, 0))):
                    env(KERNEL=3, WARPS=warps, BITMAP=bitmap, **extra, **hooks)
                    check(s, idx, q, k, L, rescore, entry=e, bitmap=bitmap, slots=warps)


def test_code_past_the_lean_bound_plans_the_two_warp_kernel(lib, env):
    """6145 x 2 bits = 194 code words: more than the lean kernel's 192, so even DANN_SEARCH_KERNEL=3 gets two warps."""
    s = case(300, 6145, COSINE, "normal", seed=6145)
    with lib.DiskAnnIndex(s) as idx:
        env(KERNEL=3)
        check(s, idx, _queries(s, 16, 3), 10, 40, 20, kernel=2)


@pytest.mark.parametrize("dim,dist,kind,entry", [SHAPES[3], SHAPES[6]], ids=["768x2", "1537x2"])
def test_each_slot_runs_several_queries(lib, env, dim, dist, kind, entry):
    """One slot per SM and more than 3 queries per slot: the bitmap is cleared and the hash set reset between a slot's
    queries; the heap lives almost wholly in the HBM tail (heap top of 4 or 16 entries)."""
    s = case(600, dim, dist, kind, seed=dim + 7)
    B = 3 * sm_count() + 5
    q = _queries(s, B, dim + 8, kind)
    q[B // 2] = 0.0
    with lib.DiskAnnIndex(s) as idx:
        for bitmap, hs in ((1, 4), (0, 16), (0, 4), (1, 16)):
            env(KERNEL=3, WARPS=1, BITMAP=bitmap, HS=hs)
            check(s, idx, q, 10, 50, 30, entry=entry, bitmap=bitmap, slots=1)
        env(KERNEL=3, WARPS=1, ENTRY=2, BITMAP=0)            # Ent64 on a code that fits 4 bytes: node id in the entry
        check(s, idx, q, 10, 50, 30, entry=8, bitmap=0, slots=1)


@pytest.mark.parametrize("dim,dist,kind,entry", [SHAPES[1], SHAPES[3], SHAPES[5]], ids=["100x2", "768x2", "1024x2"])
def test_growth_retries_through_the_query_list(lib, env, dim, dist, kind, entry):
    """DANN_DEBUG_SHRINK=8: first workspaces too small, the overflowing queries rerun through qlist with larger ones."""
    s = case(600, dim, dist, kind, seed=dim + 11)
    q = _queries(s, 3 * sm_count() + 1, dim + 12, kind)
    with lib.DiskAnnIndex(s) as idx:
        for bitmap, warps in ((1, 1), (0, 1), (0, 16), (1, 32)):
            env(KERNEL=3, WARPS=warps, BITMAP=bitmap, SHRINK=8, HS=16)
            check(s, idx, q, 10, 60, 40, entry=entry, bitmap=bitmap, slots=warps, retried=True)


@pytest.mark.parametrize("R", [1, 32, 33, 64])
def test_list_widths(lib, env, R):
    """Full lists of R ids: one id, exactly the first 32-lane chunk, one id in the second chunk, both chunks full (no
    terminator anywhere)."""
    s = fill_lists(case(300, 96, COSINE, "normal", seed=300 + R, R=R, L_build=max(2 * R, 8)), R)
    q = _queries(s, 24, R)
    with lib.DiskAnnIndex(s) as idx:
        for bitmap in (1, 0):
            env(KERNEL=3, WARPS=16, BITMAP=bitmap, HS=16)
            check(s, idx, q, 10, 40, 20, entry=4, bitmap=bitmap, slots=16)


def test_lists_wider_than_one_page_plan_away_from_lean(lib, env):
    """R = 70 > 64 ids: the single-warp kernel, whatever DANN_SEARCH_KERNEL asks for."""
    s = case(300, 64, L2, "uniform", seed=70, R=70, L_build=80)
    with lib.DiskAnnIndex(s) as idx:
        env(KERNEL=3)
        check(s, idx, _queries(s, 16, 70, "uniform"), 10, 40, 20, kernel=1)


def test_search_list_size_extremes(lib, env):
    """L = 1 (visited ring of one live entry) and L = 10000 (a visited ring of 40 KB per slot: the plan takes fewer
    slots than asked for, and the whole index is visited)."""
    s = case(500, 768, COSINE, "normal", seed=9)
    q = _queries(s, 24, 10)
    with lib.DiskAnnIndex(s) as idx:
        for bitmap in (1, 0):
            env(KERNEL=3, WARPS=16, BITMAP=bitmap)
            check(s, idx, q, 10, 1, 5, entry=4, bitmap=bitmap, slots=16)
            _, p = check(s, idx, q[:12], 10, 10000, 50, entry=4, bitmap=bitmap)
            assert 1 <= p["slots_per_sm"] < 16, p


def test_stream_exhaustion_and_rescore_bounds(lib, env):
    """k larger than the index (the stream runs dry), rescore 0 and 1000."""
    s = case(500, 100, L2, "uniform", seed=12)
    q = _queries(s, 20, 13, "uniform")
    with lib.DiskAnnIndex(s) as idx:
        for bitmap in (1, 0):
            env(KERNEL=3, WARPS=16, BITMAP=bitmap)
            g, _ = check(s, idx, q, 600, 50, 0, entry=4, bitmap=bitmap, slots=16)
            assert (g["count"] == s.n).all()
            g, _ = check(s, idx, q, 600, 50, 1000, entry=4, bitmap=bitmap, slots=16)
            assert (g["count"] == s.n).all()
            check(s, idx, q, 10, 100, 1000, entry=4, bitmap=bitmap, slots=16)


def test_deleted_tuples(lib, env):
    """Every third tuple deleted, then every tuple: deleted rows are skipped without a slot in the stream."""
    s = case(600, 320, COSINE, "normal", seed=14, deleted_every=3)
    q = _queries(s, 30, 15)
    with lib.DiskAnnIndex(s) as idx:
        for bitmap, hooks, entry in ((1, {}, 4), (0, {}, 4), (0, {"ENTRY": 2}, 8)):
            env(KERNEL=3, WARPS=16, BITMAP=bitmap, **hooks)
            g, _ = check(s, idx, q, 10, 50, 20, entry=entry, bitmap=bitmap, slots=16)
            assert ((g["tid"] & np.uint64(0xFFFF)) != 0).all()
    s.heap_tid = s.heap_tid & np.uint64(0xFFFFFFFFFFFF0000)
    with lib.DiskAnnIndex(s) as idx:
        for bitmap in (1, 0):
            env(KERNEL=3, WARPS=16, BITMAP=bitmap)
            g, _ = check(s, idx, q, 10, 50, 20, entry=4, bitmap=bitmap, slots=16)
            assert not g["count"].any()


def test_repeated_ids_inside_a_neighbour_list(lib, env):
    """The mutation of test_gpu_parity.test_duplicate_ids_inside_a_neighbour_list: lists that repeat an id take the
    strict list-order insert path; several queries per slot."""
    s = case(1500, 96, COSINE, "normal", seed=29, R=40, L_build=60)
    rng = np.random.default_rng(4)
    nb = s.nbrs.copy()
    mutated = 0
    for i in range(0, s.n, 3):
        deg = int((nb[i] != INVALID).sum())
        if deg >= 36:
            nb[i, deg - 1] = nb[i, int(rng.integers(0, 8))]
            nb[i, 33] = nb[i, 34]
            mutated += 1
    s.nbrs = nb
    repeats = sum(len(set(r[r != INVALID].tolist())) < int((r != INVALID).sum()) for r in nb)
    assert mutated >= 50 and repeats == mutated, (mutated, repeats)     # else the strict list-order path never runs
    q = _queries(s, 2 * sm_count() + 3, 7)
    with lib.DiskAnnIndex(s) as idx:
        for bitmap, warps in ((1, 1), (0, 1), (1, 16), (0, 32)):
            env(KERNEL=3, WARPS=warps, BITMAP=bitmap, HS=16)
            check(s, idx, q, 10, 60, 30, entry=4, bitmap=bitmap, slots=warps)


def test_label_keys(lib, env):
    """One label; unsorted keys with repeats; empty and unknown keys inside a keyed batch; a key of 40 distinct labels,
    34 of them unknown and sorting first, so the known ones are staged by the second 32-wide round."""
    s = case(2500, 128, COSINE, "normal", seed=21, R=32, L_build=64, labels=True)
    rng = np.random.default_rng(3)
    B = 36
    q = _queries(s, B, 5)
    one = [[int(rng.integers(1, 17))] for _ in range(B)]
    two = [[int(x) for x in rng.integers(1, 17, size=3)] + [int(rng.integers(1, 17))] * 2 for _ in range(B)]
    mixed = [[] if i % 4 == 0 else [999] if i % 4 == 1 else [-5, 1 + i % 16] if i % 4 == 2 else [1 + i % 16, 999]
             for i in range(B)]
    wide = []
    for i in range(B):
        key = list(range(-100, -66)) + [3, 7, 11, 14, 15, 16]
        rng.shuffle(key)
        wide.append([int(x) for x in key])
    with lib.DiskAnnIndex(s) as idx:
        for bitmap, hooks, e in ((1, {}, 4), (0, {}, 4), (1, {"ENTRY": 2}, 8), (0, {"ENTRY": 2}, 8)):
            env(KERNEL=3, WARPS=16, BITMAP=bitmap, HS=16, **hooks)
            check(s, idx, q, 10, 60, 30, labels=one, entry=e, bitmap=bitmap, slots=16)
            check(s, idx, q, 10, 40, 20, labels=two, entry=e, bitmap=bitmap, slots=16)
            g, _ = check(s, idx, q, 10, 60, 30, labels=mixed, entry=e, bitmap=bitmap, slots=16)
            assert not g["count"][0::4].any() and not g["count"][1::4].any()
            check(s, idx, q, 10, 60, 30, labels=wide, entry=e, bitmap=bitmap, slots=16)


def test_default_plan_at_the_lean_threshold(lib, env):
    """No hooks: the plan the benchmark gets.  7 queries per SM still take the two-warp kernel, one more query takes the
    lean one, up to 16 slots per SM.  Every query of every batch against the oracle, and the same bytes from all three
    kernels.  On an H100's 132 SMs the batches are 924, 925, 1024 (8 slots per SM) and 4096 (16 slots per SM, about two
    queries per slot); on fewer (emulated) SMs the last two shrink in proportion, to the same slot counts."""
    sm = sm_count()
    s = case(5000, 768, COSINE, "normal", seed=5000, R=50, L_build=100)
    q = _queries(s, 4096, 5001)
    with lib.DiskAnnIndex(s) as idx:
        for B in (7 * sm, 7 * sm + 1, round(1024 * sm / 132), round(4096 * sm / 132)):
            env()
            lean = B > 7 * sm
            want, _ = check(s, idx, q[:B], 10, 50, 30, kernel=3 if lean else 2, entry=4, bitmap=1,
                            slots=min(-(-B // sm), 16) if lean else 7)
            for kern in (1, 2, 3):
                env(KERNEL=kern)
                g = idx.search_batch(q[:B], k=10, search_list_size=50, rescore=30)
                assert idx.last_search_plan()["kernel"] == kern
                assert np.array_equal(g["tid"], want["tid"]) and np.array_equal(g["count"], want["count"])
                assert np.array_equal(g["dist"].view(np.uint32), want["dist"].view(np.uint32))
                assert np.array_equal(g["stats"], want["stats"])


# ---- past the 21-bit node-id boundary (GPU-built indexes) ------------------------------------------------------------

N21 = 1 << 21


@pytest.fixture(scope="module")
def big21(lib):
    """Two 64-d cosine indexes from the GPU graph builder: 2^21 nodes (the largest whose node ids fit the 21-bit field
    of a 4-byte entry) and 2^21 + 4096 nodes (ids that do not).  Queries: 960 random ones and, last, the vectors of the
    64 nodes below 2^21 (and, on the larger index, of the 64 nodes past it)."""
    if emulating():
        pytest.skip("2^21-node indexes are built with the GPU graph builder")
    import torch
    from tools import synth_index as si
    dev = torch.device("cuda", 0)
    out = {}
    for n in (N21, N21 + 4096):
        x = si.gen_dataset(n, 64, 0x5EED0021, "lowrank", device=dev)
        snap, _, _ = si.build_index_vamana(x, R=50, L_build=64)
        rnd = si.gen_dataset(1024, 64, 0x5EED0022, "lowrank", device=dev).cpu().numpy()
        src = np.arange(N21 - 64, N21) if n == N21 else np.arange(n - 64, n)
        q = np.concatenate([rnd[:960], snap.vectors[src]])
        out[n] = (snap, q, src)
        del x
        torch.cuda.empty_cache()
    return out


def _nodes(tid):
    """make_heap_tids: two tuples per block, offsets from 1."""
    return ((tid >> np.uint64(16)) * np.uint64(2) + (tid & np.uint64(0xFFFF)) - np.uint64(1)).astype(np.int64)


def _check_big(lib, env, snap, q, src, plans):
    from oracle import oracle
    k, L, rescore = 10, 100, 50
    sample = np.arange(len(q) - 64, len(q))                 # the node-derived queries
    with lib.DiskAnnIndex(snap) as idx:
        env(KERNEL=2)
        ref = idx.search_batch(q, k=k, search_list_size=L, rescore=rescore)
        assert idx.last_search_plan()["kernel"] == 2
        otid, odist, ocount, ostats = oracle.scan_batch(snap, q[sample], None, None, L, rescore, k, threads=0)
        for hooks, (entry, bitmap) in plans:
            env(**hooks)
            g = idx.search_batch(q, k=k, search_list_size=L, rescore=rescore)
            p = idx.last_search_plan()
            assert (p["kernel"], p["entry_bytes"], p["bitmap"], p["slots_per_sm"]) == \
                (3, entry, bitmap, min(-(-len(q) // sm_count()), 16)), (hooks, p)
            assert not g["stats"]["status"].any()
            assert np.array_equal(g["tid"], ref["tid"]) and np.array_equal(g["count"], ref["count"]), hooks
            assert np.array_equal(g["dist"].view(np.uint32), ref["dist"].view(np.uint32)), hooks
            assert np.array_equal(g["stats"], ref["stats"]), hooks
            assert np.array_equal(g["tid"][sample], otid), hooks
            assert np.array_equal(g["dist"][sample].view(np.uint32), odist.view(np.uint32)), hooks
            assert np.array_equal(g["count"][sample], ocount), hooks
            for f in ("visits", "d_quantized", "candidates", "d_full", "stream_len"):
                assert np.array_equal(g["stats"][f][sample].astype(np.uint64), ostats[f]), (hooks, f)
        # the high node ids come back: most node-derived queries find their own node
        found = [int(src[i]) in set(_nodes(ref["tid"][sample[i]]).tolist()) for i in range(64)]
        assert sum(found) >= 48, sum(found)
        return _nodes(ref["tid"][sample])


def test_gpu_built_2pow21_nodes_hash_and_bitmap_payloads(lib, env, big21):
    """n = 2^21: the default plan is the hash set with hash-slot payloads; DANN_SEARCH_BITMAP=1 gives the bitmap with
    node-id payloads of the full 21 bits."""
    snap, q, src = big21[N21]
    nodes = _check_big(lib, env, snap, q, src, [({}, (4, 0)), ({"BITMAP": 1}, (4, 1))])
    assert (nodes >= N21 - 64).any()


def test_gpu_built_past_2pow21_nodes_slot_payloads_and_ent64(lib, env, big21):
    """n = 2^21 + 4096: node ids no longer fit 21 bits.  The default plan keeps 4-byte entries carrying hash slots;
    DANN_SEARCH_BITMAP=1 needs the node id in the entry, i.e. Ent64."""
    snap, q, src = big21[N21 + 4096]
    nodes = _check_big(lib, env, snap, q, src, [({}, (4, 0)), ({"BITMAP": 1}, (8, 1))])
    assert (nodes >= N21).any()
