"""dann_scan_fetch: the next n rows of a streaming scan in one GPU step, each with the counters its own amgettuple would
report.

Bar: two scans of the same query are driven side by side, one with IndexScan.fetch(n) and one with n gettuple calls.
They give equal rows (TID, node), equal distance bits, equal dann_scan_stats after every row, and equal counters
afterwards; a fetch after the end of scan returns no row.  Against the oracle, the rows of a fetch equal
oracle.scan(.., max_rows=i) and row_stats[i-1] equals its counters.  The only thing allowed to differ between the two
scans is dann_scan_workspace: the replay regrows before the deep mode are counted per call.

Every test here also runs under the CPU SIMT emulator (DANN_EMULATE=1, tests/test_zz_u_scan_fetch_emulated.py)."""
import numpy as np
import pytest

from test_gpu_parity import COSINE, IP, L2, _queries
from test_zz_p_values_gpu import duplicate_rows, overflow_rows, trained_index
from test_zz_s_deep_scan_gpu import _case, env, index_a, lib  # noqa: F401  (fixtures)

pytestmark = pytest.mark.gpu

FIELDS = ("visits", "d_quantized", "candidates", "d_full", "stream_len", "status")
INVALID_ARG, STATE = -1, -6     # DANN_ERR_INVALID_ARG, DANN_ERR_STATE


def _bits(x):
    return int(np.float32(x).view(np.uint32))


def fetch_vs_single(a, b, n):
    """a.fetch(n) against up to n gettuple calls of b: rows, distance bits and the counters after every row, then the
    counters after the step.  Returns the rows produced."""
    blk, off, node, dist, st = a.fetch(n)
    r = len(blk)
    assert len(off) == len(node) == len(dist) == len(st) == r <= n
    for i in range(r):
        row = b.gettuple()
        assert row is not None, (n, i)
        assert (row[0], row[1], row[2]) == (int(blk[i]), int(off[i]), int(node[i])), (n, i)
        assert _bits(row[3]) == _bits(dist[i]), (n, i)
        assert b.stats() == st[i], (n, i, b.stats(), st[i])
    if r < n:
        assert b.gettuple() is None, (n, r)
    else:
        assert a.stats() == st[-1]
    assert a.stats() == b.stats(), (n, a.stats(), b.stats())
    return r


def drain_side_by_side(idx, q, key, L, rescore, sizes):
    """fetch sizes in turn (cycling) against single calls until the end of scan, then fetches past it.  Returns the
    rows streamed and the fetch side's workspace."""
    a, b = idx.begin_scan(), idx.begin_scan()
    try:
        for sc in (a, b):
            sc.rescan(q, labels=key, search_list_size=L, rescore=rescore)
        total, i = 0, 0
        while True:
            n = sizes[i % len(sizes)]
            i += 1
            r = fetch_vs_single(a, b, n)
            total += r
            if r < n:
                break
        for n in (1, 7):                                  # past the end: no row, no change
            assert fetch_vs_single(a, b, n) == 0
        return total, a.workspace()
    finally:
        a.end()
        b.end()


def _sizes(rescore):
    return sorted({1, 2, 7, max(rescore - 1, 1), max(rescore, 1), rescore + 1, 1000}) + [65536]


@pytest.mark.parametrize("rescore", [0, 1, 50, 1000])
def test_fetch_equals_single_calls(lib, env, rescore):
    """Every fetch size of the issue, cycled until the index is drained; label-keyed and unkeyed; deleted tuples
    (every 7th)"""
    s = index_a()
    q = _queries(s, 2, 101 + rescore, "normal")
    with lib.DiskAnnIndex(s) as idx:
        rows, _ = drain_side_by_side(idx, q[0], None, 40, rescore, [1, 2, 7, max(rescore - 1, 1), rescore + 1])
        assert rows == int((s.heap_tid & 0xFFFF != 0).sum())
        drain_side_by_side(idx, q[1], [1, 2, 5], 30, rescore, _sizes(rescore))


# (id, fixture, hooks, key, L, rescore)
LAYOUTS = [
    ("x21-bitmap", index_a, {}, None, 40, 50),
    ("x16-hash", index_a, dict(ENTRY=1, BITMAP=0), None, 40, 50),
    ("e64-bitmap-key", index_a, dict(ENTRY=2), [3, 7], 40, 50),
    ("empty-start-list", index_a, {}, [999], 40, 50),
    ("plain-truncated", lambda: _case(900, 48, None, L2, seed=9, deleted_every=11, plain_dim=32), {}, None, 40, 50),
    ("plain-no-rerank", lambda: _case(600, 48, None, COSINE, seed=19, plain_dim=48), {}, None, 40, 50),
    ("nch8-8200x2", lambda: _case(320, 8200, 2, IP, seed=8202), {}, None, 30, 20),
]


@pytest.mark.parametrize("case", LAYOUTS, ids=[c[0] for c in LAYOUTS])
def test_fetch_layouts(lib, env, case):
    """Entry widths Ent32x21 / Ent32x16 / Ent64, bitmap and hash inserted-sets, a key with no start node, the plain
    layout with and without a truncated num_dimensions, NCH 8"""
    _, fixture, hooks, key, L, rescore = case
    s = fixture()
    q = _queries(s, 1, s.dim + 3, "normal")[0]
    env(**hooks)
    with lib.DiskAnnIndex(s) as idx:
        rows, _ = drain_side_by_side(idx, q, key, L, rescore, [3, 1, 64, 2, 500])
    if key == [999]:
        assert rows == 0


def test_replay_regrows_inside_one_fetch(lib, env):
    """A shrunk workspace overflows inside a long fetch: the step regrows, replays and still gives the single calls'
    rows and counters"""
    s = index_a()
    q = _queries(s, 1, 41, "normal")[0]
    env(SHRINK=16)
    with lib.DiskAnnIndex(s) as idx:
        a, b = idx.begin_scan(), idx.begin_scan()
        try:
            for sc in (a, b):
                sc.rescan(q, search_list_size=40, rescore=50)
            assert fetch_vs_single(a, b, 1) == 1             # past the first step: no planning ahead, the fetch regrows
            assert fetch_vs_single(a, b, 300) == 300
            ws = a.workspace()
            assert ws["regrows"] >= 1 and ws["mode"] == 0, ws
        finally:
            a.end()
            b.end()


@pytest.mark.parametrize("rescore", [0, 50])
def test_deep_mode_with_growths_inside_one_fetch(lib, env, rescore):
    """DANN_DEBUG_DEEP_AFTER sends the scan deep at its first overflow; later fetches grow the deep workspace in place
    mid-step"""
    s = index_a()
    q = _queries(s, 1, 43 + rescore, "normal")[0]
    env(SHRINK=16, DEEP_AFTER=0)
    with lib.DiskAnnIndex(s) as idx:
        rows, ws = drain_side_by_side(idx, q, None, 40, rescore, [200, 1, 333])
    assert ws["mode"] == 1 and ws["growths"] >= 1, ws
    assert rows == int((s.heap_tid & 0xFFFF != 0).sum())


def test_interleaving_and_rescan(lib, env):
    """fetch, gettuple and gettuple_many on one scan at arbitrary points, against a scan stepped by gettuple alone;
    then a rescan mid-stream with another rescore"""
    s = index_a()
    q = _queries(s, 2, 47, "normal")
    rng = np.random.default_rng(5)
    with lib.DiskAnnIndex(s) as idx:
        a, b, other = idx.begin_scan(), idx.begin_scan(), idx.begin_scan()
        try:
            for sc in (a, b, other):
                sc.rescan(q[0], search_list_size=40, rescore=20)
            for _ in range(40):
                op = rng.integers(0, 3)
                if op == 0:
                    fetch_vs_single(a, b, int(rng.integers(1, 40)))
                else:
                    row = a.gettuple() if op == 1 else lib.gettuple_many([a, other])[0]
                    ref = b.gettuple()
                    assert (row is None) == (ref is None)
                    if ref is not None:
                        assert row[:3] == ref[:3] and _bits(row[3]) == _bits(ref[3])
                    assert a.stats() == b.stats()
            for sc in (a, b):
                sc.rescan(q[1], labels=[2, 4], search_list_size=30, rescore=7)
            for n in (1, 6, 7, 8, 100, 65536):
                fetch_vs_single(a, b, n)
        finally:
            for sc in (a, b, other):
                sc.end()


def _value_case(kind, dist):
    if kind == "overflow":
        v, q = overflow_rows(600, 64, 3 + dist)
        return trained_index(v, dist, 2), q
    v, q = duplicate_rows(1200, 96, 37, 96 + dist, "normal" if dist == COSINE else "uniform")
    return trained_index(v, dist, 2, R=24, L_build=48), q


VALUES = [("overflow", L2), ("overflow", IP), ("duplicates", COSINE), ("duplicates", L2)]


@pytest.mark.parametrize("kind,dist", VALUES, ids=[f"{k}-{d}" for k, d in VALUES])
def test_window_staging_on_special_values(lib, env, kind, dist):
    """rescore = 1000: the window staged in shared memory for a multi-row step, on NaN / +-inf / tied distances"""
    s, q = _value_case(kind, dist)
    seen = []
    with lib.DiskAnnIndex(s) as idx:
        for qi in (1, 9, 13):
            a, b = idx.begin_scan(), idx.begin_scan()
            try:
                for sc in (a, b):
                    sc.rescan(q[qi], search_list_size=60, rescore=1000)
                seen.append(a.fetch(1)[3])
                b.gettuple()
                for n in (2, 999, 1000, 1001, 65536):
                    blk, off, node, dist_, st = a.fetch(n)
                    seen.append(dist_)
                    for i in range(len(blk)):
                        row = b.gettuple()
                        assert row[:3] == (int(blk[i]), int(off[i]), int(node[i]))
                        assert _bits(row[3]) == _bits(dist_[i]) and b.stats() == st[i]
                    if len(blk) < n:
                        assert b.gettuple() is None
                    assert a.stats() == b.stats()
            finally:
                a.end()
                b.end()
    d = np.concatenate(seen)
    if kind == "overflow" and dist == L2:
        assert np.isposinf(d).sum() > 50
    elif kind == "overflow":
        assert np.isnan(d).any() and np.isposinf(d).any() and np.isneginf(d).any()
    else:
        assert len(np.unique(d)) < len(d) // 4                  # runs of equal keys in the window


def test_fetch_against_the_oracle(lib):
    """At sampled row counts i, oracle.scan(.., max_rows=i) gives the fetch's first i rows and row_stats[i-1]"""
    from oracle import oracle
    s = index_a()
    q = _queries(s, 1, 53, "normal")[0]
    with lib.DiskAnnIndex(s) as idx:
        sc = idx.begin_scan()
        try:
            sc.rescan(q, labels=[1, 3, 6], search_list_size=40, rescore=30)
            blk, off, node, dist, st = sc.fetch(65536)
        finally:
            sc.end()
    r = len(blk)
    assert r > 100
    for i in sorted({1, 2, 29, 30, 31, 64, r // 2, r - 1, r}):
        ref = oracle.scan(s, q, [1, 3, 6], 40, 30, i)
        tid = (blk[:i].astype(np.uint64) << 16) | off[:i]
        assert np.array_equal(tid, ref["tid"]) and np.array_equal(node[:i], ref["node"]), i
        assert np.array_equal(dist[:i].view(np.uint32), ref["dist"].view(np.uint32)), i
        for f in FIELDS[:5]:
            assert st[i - 1][f] == ref["stats"][f], (i, f)
    ref = oracle.scan(s, q, [1, 3, 6], 40, 30, r + 1)
    assert len(ref["tid"]) == r


def test_argument_checks(lib):
    """max_rows of 0, -1 and 65537, a NULL scan and a fetch before rescan are refused before anything runs; every
    output may be NULL"""
    import ctypes as C
    s = index_a()
    q = _queries(s, 1, 59, "normal")[0]
    with lib.DiskAnnIndex(s) as idx:
        raw = lib.load_library()
        a, b = idx.begin_scan(), idx.begin_scan()
        try:
            assert raw.dann_scan_fetch(a._h, 1, None, None, None, None, None) == STATE
            for sc in (a, b):
                sc.rescan(q, search_list_size=40, rescore=10)
            launches = idx.kernel_launches
            for bad in (0, -1, 65537):
                assert raw.dann_scan_fetch(a._h, bad, None, None, None, None, None) == INVALID_ARG
                assert b"max_rows" in raw.dann_last_error()
            assert raw.dann_scan_fetch(None, 1, None, None, None, None, None) == INVALID_ARG
            assert idx.kernel_launches == launches
            assert raw.dann_scan_fetch(a._h, 25, None, None, None, None, None) == 25
            for _ in range(25):
                b.gettuple()
            assert a.stats() == b.stats()
            st = (C.c_uint32 * 6 * 3)()
            assert raw.dann_scan_fetch(a._h, 3, None, None, None, None, st) == 3
            for _ in range(3):
                b.gettuple()
            assert list(st[2]) == [b.stats()[f] for f in FIELDS]
        finally:
            a.end()
            b.end()


def test_first_fetch_plans_ahead(lib, env):
    """A first fetch after amrescan that asks for more rows than rescore + 64 is planned for them before anything
    streams; with a shrunk workspace the planned-ahead scan still regrows (by replay) no more often than single calls,
    and its rows and counters are theirs"""
    s = index_a()
    q = _queries(s, 1, 67, "normal")[0]
    env(SHRINK=4)
    with lib.DiskAnnIndex(s) as idx:
        a, b = idx.begin_scan(), idx.begin_scan()
        try:
            for sc in (a, b):
                sc.rescan(q, search_list_size=40, rescore=20)
            assert fetch_vs_single(a, b, 900) == 900
            assert fetch_vs_single(a, b, 65536) < 65536
            assert a.workspace()["regrows"] <= b.workspace()["regrows"]
        finally:
            a.end()
            b.end()


def test_one_step_whatever_the_row_count(lib):
    """A fetch that does not regrow costs the same kernel launches for every n"""
    s = index_a()
    q = _queries(s, 1, 61, "normal")[0]
    costs = {}
    with lib.DiskAnnIndex(s) as idx:
        for n in (1, 2, 16, 64):      # within the planned workspace of rescore + 64 streamed rows
            sc = idx.begin_scan()
            try:
                sc.rescan(q, search_list_size=100, rescore=50)
                before = idx.kernel_launches
                assert len(sc.fetch(n)[0]) == n
                costs[n] = idx.kernel_launches - before
                assert sc.workspace()["regrows"] == 0
            finally:
                sc.end()
    assert len(set(costs.values())) == 1, costs
