"""dann_shards_scan: the streaming scan of a sharded table (include/diskann_b200.h).  Bar: after EVERY gettuple, the row
(TID, node, distance bits, shard) and every shard's counters equal StreamModel - the oracle's scan of each shard
(oracle.scan(.., max_rows=j) is a shard's rows and counters after j steps), merged one row at a time by
tests/shard_model.total_ukey heads: the first call steps every shard, each later call the shard whose row the previous
call returned, ties to the lower shard.

Every test here also runs under the CPU SIMT emulator with two fake devices (tests/test_zz_r_shard_scan_emulated.py)."""
import threading

import numpy as np
import pytest

from conftest import build_case, emulating
from oracle import fixtures, oracle
from shard_model import total_ukey
from test_zz_q_shards_gpu import SIZES, _global_tids, _shards, _special_rows

pytestmark = pytest.mark.gpu

COSINE, L2, IP = 0, 1, 2
FIELDS = ("visits", "d_quantized", "candidates", "d_full", "stream_len")


@pytest.fixture(scope="module")
def lib(lib_built):
    from pgvectorscale_b200 import diskann
    if diskann.device_count() < 1:
        pytest.fail("no CUDA device visible: -m gpu tests need an H100")
    return diskann


class StreamModel:
    """The merged stream of one sharded scan, from the oracle's scan of every shard."""

    def __init__(self, snaps, q, labels, L, rescore):
        self.snaps, self.q, self.labels, self.L, self.rescore = snaps, q, labels, L, rescore
        S = len(snaps)
        self.steps = [0] * S
        self.heads = [None] * S
        self.stats = [None] * S
        self.first, self.next = True, None

    def _step(self, s):
        self.steps[s] += 1
        j = self.steps[s]
        ref = oracle.scan(self.snaps[s], self.q, self.labels, self.L, self.rescore, j)
        self.stats[s] = ref["stats"]
        self.heads[s] = None if len(ref["tid"]) < j else (int(ref["tid"][-1]), int(ref["node"][-1]), ref["dist"][-1])

    def gettuple(self):
        """-> (tid, node, dist f32, shard) or None"""
        if self.first:
            for s in range(len(self.snaps)):
                self._step(s)
            self.first = False
        elif self.next is not None:
            self._step(self.next)
        self.next = None
        live = [(int(total_ukey(np.array([h[2]], np.float32))[0]), s) for s, h in enumerate(self.heads) if h is not None]
        if not live:
            return None
        s = min(live)[1]
        tid, node, dist = self.heads[s]
        self.heads[s] = None
        self.next = s
        return tid, node, dist, s


class Tracked:
    """A ShardedScan and its model: step() compares the next row and every shard's counters."""

    def __init__(self, g, snaps, q, labels=None, L=40, rescore=20):
        self.sc = g.begin_scan()
        self.rescan(snaps, q, labels, L, rescore)

    def rescan(self, snaps, q, labels=None, L=40, rescore=20):
        self.sc.rescan(q, labels=labels, search_list_size=L, rescore=rescore)
        self.model = StreamModel(snaps, q, labels, L, rescore)
        self.calls = 0

    def step(self):
        self.calls += 1
        got, ref = self.sc.gettuple(), self.model.gettuple()
        what = (self.calls, self.model.labels, self.model.L, self.model.rescore)
        if ref is None:
            assert got is None, what
        else:
            assert got is not None, what
            assert ((got[0] << 16) | got[1], got[2], got[4]) == ref[:2] + (ref[3],), what
            assert np.float32(got[3]).view(np.uint32) == np.float32(ref[2]).view(np.uint32), what
        st = self.sc.stats()
        assert len(st) == len(self.model.snaps)
        for s, (a, b) in enumerate(zip(st, self.model.stats)):
            for f in FIELDS:
                assert a[f] == b[f], (s, f) + what
        return got

    def end(self):
        self.sc.end()


def _sharded(lib, snaps, devices=None):
    return lib.ShardedIndex(snaps, devices=[0] * len(snaps) if devices is None else devices)


_CACHE = {}


@pytest.mark.parametrize("nshards", [1, 2, 3, 5])
@pytest.mark.parametrize("dist,bits", [(COSINE, 1), (COSINE, 2), (L2, 1), (L2, 2), (IP, 1), (IP, 2)],
                         ids=["cos1", "cos2", "l2-1", "l2-2", "ip1", "ip2"])
def test_every_call_equals_the_stream_model(lib, dist, bits, nshards):
    """shards of 700 / 600+0 / 500+7+300 / 400+0+7+250+600 rows with deleted rows, drained 45 calls at rescore 20"""
    key = (dist, bits, nshards)
    if key not in _CACHE:
        _CACHE[key] = _shards(SIZES[nshards], dist, bits, seed=10 * dist + bits)
    snaps = _CACHE[key]
    q = fixtures.gen_vectors(2, 48, 200 + dist, "normal")
    with _sharded(lib, snaps) as g:
        for j in range(2):
            t = Tracked(g, snaps, q[j], L=40, rescore=20)
            shards = {t.step()[4] for _ in range(45)}
            if nshards > 2:
                assert len(shards) > 1
            t.end()


@pytest.mark.parametrize("dist,bits", [(L2, 2), (COSINE, 1)], ids=["l2-2", "cos1"])
def test_drained_to_end_of_scan(lib, dist, bits):
    """small shards with deleted rows, drained past their last row: each shard drops out where its own scan ends, and
    the merged scan ends when every shard has"""
    snaps = _shards([60, 0, 7, 30], dist, bits, seed=30 + dist, dim=32)
    for s in snaps:
        s.heap_tid[::4] &= np.uint64(0xFFFFFFFFFFFF0000)
    q = fixtures.gen_vectors(1, 32, 31, "normal")[0]
    with _sharded(lib, snaps) as g:
        t = Tracked(g, snaps, q, L=30, rescore=10)
        rows = 0
        while t.step() is not None:
            rows += 1
        assert rows > 10 and t.step() is None and t.step() is None
        t.end()


@pytest.mark.parametrize("k", [10, 50])
def test_first_k_rows_equal_the_batch(lib, k):
    snaps = _shards([500, 7, 300, 0], L2, 2, seed=41)
    q = fixtures.gen_vectors(5, 48, 42, "normal")
    with _sharded(lib, snaps) as g:
        b = g.search_batch(q, k=k, search_list_size=60, rescore=30)
        sc = g.begin_scan()
        for j in range(len(q)):
            sc.rescan(q[j], search_list_size=60, rescore=30)
            rows = [sc.gettuple() for _ in range(k)]
            n = int(b["count"][j])
            assert all(r is None for r in rows[n:])
            assert [(r[0] << 16) | r[1] for r in rows[:n]] == b["tid"][j, :n].tolist()
            assert [r[4] for r in rows[:n]] == b["shard"][j, :n].tolist()
            assert np.array([r[3] for r in rows[:n]], np.float32).view(np.uint32).tolist() == \
                b["dist"][j, :n].view(np.uint32).tolist()
        sc.end()


def test_one_shard_is_a_private_index_scan(lib):
    s = _global_tids(build_case(900, 64, L2, seed=5, R=16, L_build=32, deleted_every=7), 0)
    q = fixtures.gen_vectors(1, 64, 6, "normal")[0]
    with _sharded(lib, [s]) as g, lib.DiskAnnIndex(s) as idx:
        sc, one = g.begin_scan(), idx.begin_scan()
        sc.rescan(q, search_list_size=50, rescore=30)
        one.rescan(q, search_list_size=50, rescore=30)
        for _ in range(60):
            a, b = sc.gettuple(), one.gettuple()
            assert a[:3] == b[:3] and a[4] == 0
            assert np.float32(a[3]).view(np.uint32) == np.float32(b[3]).view(np.uint32)
            assert sc.stats() == [one.stats()]
        sc.end()
        one.end()


def test_the_same_snapshot_twice_alternates_shard_0_first(lib):
    """rescore 1000 > n keeps each shard's whole stream in its rerank window, so each shard's rows come sorted and every
    key ties across the two shards"""
    s = build_case(600, 32, COSINE, seed=8, R=16, L_build=32)
    q = fixtures.gen_vectors(1, 32, 9, "normal")[0]
    with _sharded(lib, [s, s]) as g:
        t = Tracked(g, [s, s], q, L=40, rescore=1000)
        rows = [t.step() for _ in range(40)]
        t.end()
    assert [r[4] for r in rows] == [0, 1] * 20
    assert [r[:4] for r in rows[0::2]] == [r[:4] for r in rows[1::2]]


def test_label_keys_and_query_forms(lib):
    """shard 1 carries labels 21..36 instead of 1..16: keys only some shards hold, a key no shard holds, an empty key, a
    NULL query, all on one sharded scan rescanned between them"""
    snaps = _shards([500, 400, 300], L2, 2, dim=32, seed=40, labels=True)
    snaps[1].labels = snaps[1].labels + np.int16(20)
    snaps[1].start_labels = snaps[1].start_labels + np.int16(20)
    q = fixtures.gen_vectors(8, 32, 41, "normal")
    with _sharded(lib, snaps) as g:
        t = None
        for j, labs in enumerate([[3], [25], [3, 25], [40], [], None, [7, 8, 30]]):
            if t is None:
                t = Tracked(g, snaps, q[j], labels=labs, L=50, rescore=25)
            else:
                t.rescan(snaps, q[j], labels=labs, L=50, rescore=25)
            rows = [t.step() for _ in range(30)]
            got = [r for r in rows if r is not None]
            if labs == [40] or labs == []:
                assert not got
            if labs == [25]:
                assert got and {r[4] for r in got} == {1}
            if labs == [3]:
                assert got and 1 not in {r[4] for r in got}
        t.rescan(snaps, None, labels=None, L=50, rescore=25)    # NULL order-by argument
        for _ in range(30):
            t.step()
        t.end()


@pytest.mark.parametrize("dist", [L2, IP], ids=["l2", "ip"])
def test_nan_infinite_and_duplicate_rows(lib, dist):
    """NaN (both signs), +-inf and runs of equal distances met by the merge, within a shard and across shards (shard 2
    repeats rows of shard 0); NaN keys sort where f32::total_cmp puts them"""
    v0 = _special_rows(300, 32, 50 + dist, dist)
    v1 = np.random.default_rng(51).uniform(-1, 1, (200, 32)).astype(np.float32)
    v2 = np.concatenate([v0[:40], v0[:40]])
    snaps = [_global_tids(fixtures.make_index(v, dist, bits=2, R=16, L_build=32), i) for i, v in enumerate((v0, v1, v2))]
    q = np.concatenate([v0[:3], v0[9:11], -v0[10:11]]).astype(np.float32)
    d = []
    with _sharded(lib, snaps) as g:
        for j in range(len(q)):
            t = Tracked(g, snaps, q[j], L=60, rescore=40)
            d += [r[3] for r in (t.step() for _ in range(50)) if r is not None]
            t.end()
    d = np.array(d, np.float32)
    assert not np.isfinite(d).all()
    assert len(d) - len(np.unique(d.view(np.uint32))) > 10       # ties


def test_workspace_growth_keeps_the_stream(lib, monkeypatch):
    """DANN_DEBUG_SHRINK=8: every first workspace is too small, so the first (many-scan) step and later single steps
    regrow and replay"""
    monkeypatch.setenv("DANN_DEBUG_SHRINK", "8")
    snaps = _shards([500, 7, 300], COSINE, 2, seed=77)
    q = fixtures.gen_vectors(2, 48, 78, "normal")
    with _sharded(lib, snaps) as g:
        for j in range(2):
            t = Tracked(g, snaps, q[j], L=(60, 150)[j], rescore=50)
            for _ in range(120):
                t.step()
            t.end()


def test_rescan_mid_stream(lib):
    snaps = _shards([400, 300], IP, 2, seed=61)
    q = fixtures.gen_vectors(3, 48, 62, "normal")
    with _sharded(lib, snaps) as g:
        t = Tracked(g, snaps, q[0], L=40, rescore=20)
        for _ in range(25):
            t.step()
        t.rescan(snaps, q[1], L=80, rescore=30)
        for _ in range(40):
            t.step()
        t.rescan(snaps, q[2], labels=None, L=20, rescore=5)
        for _ in range(10):
            t.step()
        t.end()


def test_launch_counts(lib):
    """The first gettuple of S shards on one device is one many-scan round: at most (distinct search instantiations + 2)
    launches over every shard's count, on the count of the device's first shard.  Later calls move only the stepped
    shard's count."""
    for bits, most in ((2, 3), ((1, 2, 1, 2), 4)):             # one instantiation; two code widths of 768-d rows
        bs = bits if isinstance(bits, tuple) else (bits,) * 4
        snaps = [_global_tids(build_case(n, 768, COSINE, bits=b, seed=90 + i, R=16, L_build=32), i)
                 for i, (n, b) in enumerate(zip((300, 200, 250, 120), bs))]
        q = fixtures.gen_vectors(1, 768, 95, "normal")[0]
        with _sharded(lib, snaps) as g:
            shards = [g.shard(i) for i in range(4)]
            t = Tracked(g, snaps, q, L=40, rescore=20)
            before = [x.kernel_launches for x in shards]
            t.step()
            moved = [x.kernel_launches - b for x, b in zip(shards, before)]
            assert sum(moved) <= most and moved[1:] == [0, 0, 0], moved
            for _ in range(15):
                before = [x.kernel_launches for x in shards]
                stepped = t.model.next
                t.step()
                moved = [x.kernel_launches - b for x, b in zip(shards, before)]
                assert moved[stepped] > 0 and sum(moved) == moved[stepped], (stepped, moved)
            t.end()


def test_refusals(lib):
    import copy
    import ctypes as C
    E = lib.DiskAnnError
    a = build_case(100, 32, L2, seed=70, R=8, L_build=16)
    q = fixtures.gen_vectors(1, 32, 74, "normal")[0]
    raw = lib.load_library()
    with _sharded(lib, [a, a]) as g:
        sc = g.begin_scan()
        with pytest.raises(E) as ei:                              # gettuple before rescan
            sc.gettuple()
        assert ei.value.code == -6
        for L, rescore in ((40, 0), (0, 10), (40, 1001)):
            with pytest.raises(E) as ei:
                sc.rescan(q, search_list_size=L, rescore=rescore)
            assert ei.value.code == -1, (L, rescore)
        assert raw.dann_shards_scan_rescan(sc._h, C.c_void_p(q.ctypes.data), None, 2, 40, 10) == -1   # labels NULL
        h = C.c_void_p()
        assert raw.dann_shards_scan_begin(None, C.byref(h)) == -1
        assert raw.dann_shards_scan_begin(g._h, None) == -1
        assert raw.dann_shards_scan_rescan(None, C.c_void_p(q.ctypes.data), None, -1, 40, 10) == -1
        assert raw.dann_shards_scan_gettuple(None, None, None, None, None, None) == -1
        assert raw.dann_shards_scan_stats(None, None) == -1
        assert raw.dann_shards_scan_stats(sc._h, None) == -1
        raw.dann_shards_scan_end(None)
        sc.rescan(q, search_list_size=40, rescore=10)             # refusals leave the scan usable
        assert raw.dann_shards_scan_gettuple(sc._h, None, None, None, None, None) == 1   # NULL outputs are allowed
        sc.end()
    bare = copy.copy(a)
    bare.vectors = None
    with _sharded(lib, [a, bare]) as g:
        sc = g.begin_scan()
        with pytest.raises(E) as ei:
            sc.rescan(q, search_list_size=40, rescore=10)
        assert ei.value.code == -6 and "shard 1:" in str(ei.value)
        with pytest.raises(E) as ei:                              # a failed rescan leaves no usable scan
            sc.gettuple()
        assert ei.value.code == -6
        sc.end()


def test_two_scans_and_a_batch_from_three_threads(lib):
    snaps = _shards([500, 7, 300], L2, 1, seed=83)
    q = fixtures.gen_vectors(6, 48, 84, "normal")
    errors = []
    with _sharded(lib, snaps) as g:
        want = g.search_batch(q, k=10, search_list_size=40, rescore=20)
        scans = [Tracked(g, snaps, q[j], L=(40, 90)[j], rescore=(20, 40)[j]) for j in range(2)]
        bar = threading.Barrier(3)

        def drain(t):
            try:
                bar.wait()
                for _ in range(40):
                    t.step()
            except Exception as e:                                # reported below
                errors.append(e)

        def batches():
            try:
                bar.wait()
                for _ in range(6):
                    got = g.search_batch(q, k=10, search_list_size=40, rescore=20)
                    for f in ("tid", "shard", "count"):
                        assert np.array_equal(got[f], want[f]), f
            except Exception as e:
                errors.append(e)

        th = [threading.Thread(target=drain, args=(t,)) for t in scans] + [threading.Thread(target=batches)]
        for t in th:
            t.start()
        for t in th:
            t.join()
        for t in scans:
            t.end()
    assert not errors, errors


def test_two_devices_equal_one(lib):
    if lib.device_count() < 2:
        pytest.skip("needs two CUDA devices (or SIMT_FAKE_DEVICES=2 under the emulated ABI)")
    snaps = _shards([400, 250, 7, 300], COSINE, 2, seed=90)
    q = fixtures.gen_vectors(2, 48, 91, "normal")
    for j in range(2):
        runs = []
        for devs in ([0, 0, 0, 0], [0, 1, 0, 1], [1, 0, 1, 0]):   # the last: the first shard is on device 1
            with _sharded(lib, snaps, devices=devs) as g:
                t = Tracked(g, snaps, q[j], L=40, rescore=20)
                runs.append([t.step() for _ in range(40)])
                t.end()
        assert runs[1] == runs[0] and runs[2] == runs[0]
