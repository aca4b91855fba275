"""The streaming scan's deep mode: a scan that outgrows every workspace dann_make_plan can give it streams on to the end
of the index, with the rows, distance bits and counters of the oracle's next_with_resort.

Bar: after every amgettuple the row (TID, node, rerank distance bits) and the five counters equal oracle.scan(.., i),
and a scan past its last row returns None.  The one exception is the hardware drain of a 300 000-node index, where
every row is compared with one oracle drain and the counters at every power-of-two row and at the end (oracle.scan
of i rows costs O(i), so a per-row comparison would cost O(n^2)).

Until a scan's planned workspace can grow no further, it regrows and replays as before; only then does it enter the
deep mode (workspace()["mode"] == 1).  On hardware, test_drain_past_the_replay_limit_without_hooks gets there by depth
alone.  Everywhere else DANN_DEBUG_SHRINK starts from a small workspace and DANN_DEBUG_DEEP_AFTER=k sends the scan
into the deep mode at its first overflow after k replay regrows: small indexes never reach the real limit.

Every test here except the hardware drain also runs under the CPU SIMT emulator (DANN_EMULATE=1,
tests/test_zz_s_deep_scan_emulated.py)."""
import functools
import threading

import numpy as np
import pytest

from conftest import build_case, emulating
from test_gpu_parity import COSINE, IP, L2, _queries

pytestmark = pytest.mark.gpu

FIELDS = ("visits", "d_quantized", "candidates", "d_full", "stream_len")
HOOKS = ("DANN_DEBUG_SHRINK", "DANN_DEBUG_DEEP_AFTER", "DANN_SEARCH_ENTRY", "DANN_SEARCH_BITMAP")


@pytest.fixture(scope="module")
def lib(lib_built):
    from pgvectorscale_b200 import diskann
    if diskann.device_count() < 1:
        pytest.fail("no CUDA device visible: -m gpu tests need an H100")
    return diskann


@pytest.fixture
def env(monkeypatch):
    """env(SHRINK=16, DEEP_AFTER=1, ENTRY=1, BITMAP=0) sets exactly these hooks and clears the others"""
    def set_(**kv):
        for h in HOOKS:
            monkeypatch.delenv(h, raising=False)
        for key, val in kv.items():
            name = "DANN_DEBUG_" + key if key in ("SHRINK", "DEEP_AFTER") else "DANN_SEARCH_" + key
            assert name in HOOKS, key
            monkeypatch.setenv(name, str(val))
    set_()
    return set_


@functools.lru_cache(maxsize=None)
def _case(n, dim, bits, dist, seed, R=16, labels=False, deleted_every=0, plain_dim=None):
    from oracle import fixtures
    s = build_case(n, dim, dist, bits=bits, seed=seed, R=R, L_build=2 * R, labels=labels, deleted_every=deleted_every,
                   dim_index=plain_dim)
    return fixtures.to_plain(s) if plain_dim else s


def index_a():
    """1500 nodes of 48 x 2 bits (Ent32x21, NCH 1), labels, every 7th tuple deleted: more candidates than the 1024 a
    shrunk workspace starts with, so a deep scan of it grows its candidate arrays in place"""
    return _case(1500, 48, 2, L2, seed=5, labels=True, deleted_every=7)


class Tracked:
    """One scan and the oracle's view of it: step() takes one amgettuple (or checks `row` from a many-scan call) and
    compares it and the counters with oracle.scan(.., i)."""

    def __init__(self, idx, s, q, labels=None, L=40, rescore=50):
        self.s, self.q, self.labels, self.L, self.rescore = s, q, labels, L, rescore
        self.sc = idx.begin_scan()
        self.rescan(q, labels, L, rescore)

    def rescan(self, q, labels=None, L=40, rescore=50):
        self.q, self.labels, self.L, self.rescore = q, labels, L, rescore
        self.sc.rescan(q, labels=labels, search_list_size=L, rescore=rescore)
        plain_no_resort = int(getattr(self.s, "storage_type", 0) or 0) != 0 and self.s.dim == self.s.dim_index
        self.with_dist = rescore > 0 and not plain_no_resort
        self.i = 0
        self.ended = False

    def step(self, row=False, stats=None):
        from oracle import oracle
        if row is False:
            row = self.sc.gettuple()
        self.i += 1
        ref = oracle.scan(self.s, self.q, self.labels, self.L, self.rescore, self.i)
        what = (self.i, self.labels, self.L, self.rescore)
        if len(ref["tid"]) < self.i:
            assert row is None, what
            self.ended = True
        else:
            assert row is not None, what
            assert ((row[0] << 16) | row[1]) == int(ref["tid"][-1]) and row[2] == int(ref["node"][-1]), what
            if self.with_dist:
                assert np.float32(row[3]).view(np.uint32) == ref["dist"][-1].view(np.uint32), what
        st = self.sc.stats() if stats is None else stats
        for f in FIELDS:
            assert st[f] == ref["stats"][f], (f,) + what
        return row

    def drain(self):
        while not self.ended:
            self.step()
        assert self.sc.gettuple() is None                     # end of scan stays the end
        return self.i - 1

    def end(self):
        self.sc.end()


# (id, fixture, hooks, key, L, rescore, the deep scan must have grown in place at least this often)
DRAINS = [
    ("x21-bitmap-r50", index_a, dict(SHRINK=16, DEEP_AFTER=1), None, 40, 50, 2),
    ("x21-bitmap-entry-at-first-overflow", index_a, dict(SHRINK=16, DEEP_AFTER=0), None, 60, 0, 1),
    ("x16-hash-r0", index_a, dict(SHRINK=16, DEEP_AFTER=1, ENTRY=1, BITMAP=0), None, 30, 0, 1),
    ("e64-key-r1000", index_a, dict(SHRINK=16, DEEP_AFTER=2, ENTRY=2), [3, 7], 40, 1000, 1),
    ("x21-key-hash", index_a, dict(SHRINK=16, DEEP_AFTER=1, BITMAP=0), [1, 2, 5, 11], 50, 50, 1),
    ("plain-truncated", lambda: _case(900, 48, None, L2, seed=9, deleted_every=11, plain_dim=32),
     dict(SHRINK=16, DEEP_AFTER=1), None, 40, 50, 1),
    ("nch8-8200x2", lambda: _case(320, 8200, 2, IP, seed=8202), dict(SHRINK=16, DEEP_AFTER=1), None, 30, 20, 1),
]


@pytest.mark.parametrize("case", DRAINS, ids=[c[0] for c in DRAINS])
def test_deep_scan_drains_like_the_oracle(lib, env, case):
    """Drained to the end of the index through the deep mode: every row and counter, the regrows before the deep mode,
    the in-place growths after it, and every live reachable row exactly once."""
    _, fixture, hooks, key, L, rescore, min_growths = case
    s = fixture()
    q = _queries(s, 1, s.dim + 11, "normal")[0]
    env(**hooks)
    with lib.DiskAnnIndex(s) as idx:
        t = Tracked(idx, s, q, key, L, rescore)
        try:
            rows = t.drain()
            ws = t.sc.workspace()
        finally:
            t.end()
    assert ws["mode"] == 1, ws
    assert ws["regrows"] == hooks["DEEP_AFTER"], ws
    assert ws["growths"] >= min_growths, ws
    if key is None:                                           # every live row is reachable in these graphs
        assert rows == int((s.heap_tid & 0xFFFF != 0).sum()), rows


def test_key_with_an_empty_start_list(lib, env):
    """A key none of whose labels has a start node: the stream is empty, no workspace ever overflows, so the scan ends
    at once in the planned mode; then a key with one such label and one that has a start node goes deep."""
    s = index_a()
    q = _queries(s, 1, 77, "normal")[0]
    env(SHRINK=16, DEEP_AFTER=0)
    with lib.DiskAnnIndex(s) as idx:
        t = Tracked(idx, s, q, [999], 40, 50)
        try:
            assert t.drain() == 0
            assert t.sc.workspace()["mode"] == 0
            t.rescan(q, [999, 3], 40, 50)
            assert t.drain() > 0
            assert t.sc.workspace()["mode"] == 1
        finally:
            t.end()


def _planned_bytes(idx, s, q, L, rescore):
    """device bytes of a fresh scan rescanned for a shallow query: the planned workspace"""
    sc = idx.begin_scan()
    try:
        sc.rescan(q, search_list_size=L, rescore=rescore)
        return sc.workspace()["device_bytes"]
    finally:
        sc.end()


def test_rescan_returns_a_deep_scan_to_the_planned_workspace(lib, env):
    """A scan driven deep is rescanned for a shallow query with every hook cleared: mode 0, no regrows or growths,
    exactly the device bytes of a fresh scan of that query (the same rescore: the rerank window, like every buffer a
    rescan reuses, keeps its largest size), and the rows still match."""
    s = index_a()
    q = _queries(s, 2, 31, "normal")
    with lib.DiskAnnIndex(s) as idx:
        env(SHRINK=16, DEEP_AFTER=1)
        t = Tracked(idx, s, q[0], None, 40, 50)
        try:
            while t.sc.workspace()["mode"] == 0:
                t.step()
            for _ in range(200):
                t.step()
            deep = t.sc.workspace()
            assert deep["mode"] == 1 and deep["growths"] >= 1, deep
            env()
            t.rescan(q[1], None, 20, 50)
            ws = t.sc.workspace()
            assert (ws["mode"], ws["regrows"], ws["growths"]) == (0, 0, 0), ws
            assert ws["device_bytes"] == _planned_bytes(idx, s, q[1], 20, 50), ws
            for _ in range(30):
                t.step()
            assert t.sc.workspace()["mode"] == 0
        finally:
            t.end()


def test_two_deep_scans_in_sequence_give_their_memory_back(lib, env):
    """Two scans of one index driven deep one after the other: each ends holding more than a planned workspace, and
    after end() the device's free memory is back within one planned workspace (at least the 2 MiB granularity of
    device allocations) of where it started."""
    s = index_a()
    q = _queries(s, 2, 41, "normal")
    with lib.DiskAnnIndex(s) as idx:
        planned = _planned_bytes(idx, s, q[0], 40, 50)
        free0 = None if emulating() else _free_bytes()
        for j in range(2):
            env(SHRINK=16, DEEP_AFTER=1)
            t = Tracked(idx, s, q[j], None, 40, 50)
            try:
                t.drain()
                ws = t.sc.workspace()
                assert ws["mode"] == 1 and ws["device_bytes"] > 0, ws
            finally:
                t.end()
            if free0 is not None:
                assert abs(_free_bytes() - free0) <= max(planned, 2 << 20), (j, free0, _free_bytes(), planned)


def _free_bytes():
    import torch
    torch.cuda.synchronize()
    return torch.cuda.mem_get_info(0)[0]


def test_many_scans_mixing_deep_and_shallow(lib, env):
    """dann_scan_gettuple_many over scans that go deep in the same round (identical plans), deep scans with other keys
    and rescores that go deep at other calls, and shallow ones that end early; every scan's row and counters after
    every call are those of its own oracle stream (so of its own dann_scan_gettuple sequence)."""
    s = index_a()
    q = _queries(s, 6, 53, "normal")
    env(SHRINK=16, DEEP_AFTER=1)
    specs = [(q[0], None, 40, 50), (q[0], None, 40, 50), (q[1], None, 60, 0), (q[2], [3, 7], 40, 1000),
             (q[3], [999], 40, 50), (q[4], None, 8, 0), (q[5], [5], 10, 20)]
    with lib.DiskAnnIndex(s) as idx:
        ts = [Tracked(idx, s, *sp) for sp in specs]
        try:
            entered = {}
            live = list(ts)
            calls = 0
            while live:
                calls += 1
                out = lib.gettuple_many([t.sc for t in live])
                for t, r in zip(live, out):
                    assert not isinstance(r, Exception), r
                    t.step(r)
                    if t.sc.workspace()["mode"] == 1:
                        entered.setdefault(id(t), calls)
                shallow_done = [t for t in live if t.ended or (t.L < 20 and t.i >= 300)]
                live = [t for t in live if t not in shallow_done]
            deep = [t for t in ts if id(t) in entered]
            assert ts[0] in deep and ts[1] in deep and ts[2] in deep and ts[3] in deep
            assert entered[id(ts[0])] == entered[id(ts[1])]   # the two identical scans went deep in the same round
            assert len(set(entered.values())) >= 2            # others at other calls, while the rest went on
            assert ts[4].i == 1 and id(ts[4]) not in entered  # the empty stream ended at its first call
        finally:
            for t in ts:
                t.end()


def test_coalescer_threads_with_one_deep_scan(lib, env):
    """Three threads drain their scans through one coalescer; one scan goes deep.  Each thread records its rows and
    counters; every call is then compared with the oracle."""
    s = index_a()
    q = _queries(s, 3, 61, "normal")
    env(SHRINK=16, DEEP_AFTER=1)
    specs = [(q[0], None, 40, 50, None), (q[1], None, 10, 0, 120), (q[2], [2], 20, 20, 120)]
    with lib.DiskAnnIndex(s) as idx, lib.Coalescer(idx, max_batch=8, max_wait_us=2000) as co:
        ts = [Tracked(idx, s, qq, key, L, rescore) for qq, key, L, rescore, _ in specs]
        logs = [[] for _ in ts]
        errors = []

        def run(j):
            try:
                limit = specs[j][4]
                while True:
                    r = co.gettuple(ts[j].sc)
                    logs[j].append((r, ts[j].sc.stats()))
                    if r is None or (limit and len(logs[j]) >= limit):
                        break
            except Exception as e:          # noqa: BLE001 - reported below
                errors.append(e)

        threads = [threading.Thread(target=run, args=(j,)) for j in range(len(ts))]
        try:
            for th in threads:
                th.start()
            for th in threads:
                th.join()
            assert not errors, errors
            for t, log in zip(ts, logs):
                for r, st in log:
                    t.step(r, st)
            assert ts[0].ended and ts[0].sc.workspace()["mode"] == 1
        finally:
            for t in ts:
                t.end()


def test_sharded_scan_drained_through_the_deep_mode(lib, env):
    """Two shards on one device, drained to the end: with DANN_DEBUG_DEEP_AFTER=0 a shard enters the deep mode at its
    first overflow, and the 1500-row shard must overflow a workspace of cand_cap candidates.  Every call equals the
    stream model of test_zz_r_shard_scan_gpu.py."""
    from oracle import fixtures
    from test_zz_m_wide_gpu import cand_cap
    from test_zz_q_shards_gpu import _shards
    from test_zz_r_shard_scan_gpu import Tracked as ShardTracked
    snaps = _shards([1500, 400], COSINE, 2, seed=91)
    L, rescore, shrink = 40, 20, 16
    assert cand_cap(L, rescore + 64, snaps[0].R, 1, shrink) < int((snaps[0].heap_tid & 0xFFFF != 0).sum())
    q = fixtures.gen_vectors(1, 48, 92, "normal")[0]
    env(SHRINK=shrink, DEEP_AFTER=0)
    with lib.ShardedIndex(snaps, devices=[0, 0]) as g:
        t = ShardTracked(g, snaps, q, L=L, rescore=rescore)
        try:
            rows = 0
            while t.step() is not None:
                rows += 1
        finally:
            t.end()
    assert rows == sum(int((s.heap_tid & 0xFFFF != 0).sum()) for s in snaps)


# ---- hardware: past the replay path's limit, no hooks ---------------------------------------------------------------

def _random_graph_index(n, dim, R, seed):
    """n uniform rows of `dim` dimensions (L2, 1 bit per dimension) and a random graph of R out-edges per node: the
    scan's rows do not depend on how good the graph is, and the oracle searches the same snapshot"""
    from oracle import oracle
    from pgvectorscale_b200.snapshot import Snapshot, code_words, make_heap_tids
    rng = np.random.default_rng(seed)
    v = rng.random((n, dim), dtype=np.float32)
    mean, m2, count = oracle.train(v, 1)
    codes = oracle.quantize_all(v, 1, mean, m2, count)
    nbrs = rng.integers(0, n, size=(n, R), dtype=np.uint32)
    return Snapshot(n=n, dim=dim, dim_index=dim, bits=1, words=code_words(dim, 1), R=R, distance_type=L2,
                    has_labels=False, count=count, mean=mean, m2=m2, codes=codes, nbrs=nbrs,
                    heap_tid=make_heap_tids(n), vectors=v, start_default=0)


def replay_limit(L, c_target, R, smem_optin):
    """the largest candidate capacity the replay path reaches: dann_make_plan's single-warp plan for the largest grow
    whose visited list still fits shared memory and whose candidates stay within 2^30"""
    from test_zz_m_wide_gpu import cand_cap
    budget = smem_optin - 1024
    grow, last = 1, None
    while True:
        vcap = ((L + 96) * grow + 3) & ~3
        need = ((L + c_target) * 23 // 20 + 40) * R * grow
        if vcap * 8 + 2 * 64 * 4 + 1024 > budget or need > 1 << 30:
            return last
        last = cand_cap(L, c_target, R, grow)
        grow *= 2


@pytest.mark.skipif(emulating(), reason="300 000 rows: hardware only")
def test_drain_past_the_replay_limit_without_hooks(lib, env):
    """300 000 nodes, R = 8, L = 100, rescore = 10: drained to the end with no hook set.  The scan's candidates pass
    the largest capacity the replay path reaches (where the parent commit's scan failed with DANN_ERR_CAPACITY), it is
    in the deep mode, and it returns every reachable row: every row and distance equal to one oracle drain, the
    counters equal at every power-of-two row and at the end."""
    import torch
    from oracle import oracle
    n, dim, R, L, rescore = 300_000, 32, 8, 100, 10
    s = _random_graph_index(n, dim, R, seed=2026)
    q = np.random.default_rng(7).random(dim, dtype=np.float32)
    ref = oracle.scan(s, q, None, L, rescore, n + 1)
    total = len(ref["tid"])
    limit = replay_limit(L, rescore + 64, R, torch.cuda.get_device_properties(0).shared_memory_per_block_optin)
    assert ref["stats"]["candidates"] > limit and total > limit, (ref["stats"], limit)
    env()
    with lib.DiskAnnIndex(s) as idx:
        sc = idx.begin_scan()
        try:
            sc.rescan(q, search_list_size=L, rescore=rescore)
            tid = np.zeros(total, np.uint64)
            node = np.zeros(total, np.uint32)
            dist = np.zeros(total, np.float32)
            checks = {}
            for i in range(total):
                r = sc.gettuple()
                assert r is not None, i
                tid[i], node[i], dist[i] = (r[0] << 16) | r[1], r[2], r[3]
                if (i + 1) & i == 0:
                    checks[i + 1] = sc.stats()
            assert sc.gettuple() is None
            checks[total + 1] = sc.stats()
            ws = sc.workspace()
        finally:
            sc.end()
    assert ws["mode"] == 1 and ws["regrows"] >= 7, ws
    assert np.array_equal(tid, ref["tid"]) and np.array_equal(node, ref["node"])
    assert np.array_equal(dist.view(np.uint32), ref["dist"].view(np.uint32))
    for i, st in checks.items():
        r = ref if i > total else oracle.scan(s, q, None, L, rescore, i)
        for f in FIELDS:
            assert st[f] == r["stats"][f], (f, i)
