"""dann_scan_gettuple_many - one amgettuple of each of many scans in one call - and its coalescer front end, against the
oracle.  Bar: after EVERY call, every scan's row (TID, node, rerank distance bits) and its five counters equal the
oracle's scan of that many rows (oracle.scan(.., i)), and a scan past its last row returns None.

Covered: 40+ scans per call that mix search_list_size 1..200, rescore 0 / 1 / 50, no key / an empty key / an unknown
label / one or two labels, a NULL and a zero query, on cosine / L2 / IP indexes of 1 and 2 bits with deleted tuples;
scans ending at different calls; two entry layouts in one call (the launch count per round: one search launch per
instantiation, one distance launch, one finish launch); workspace regrowth under DANN_DEBUG_SHRINK=8; the hash-set
inserted-set; plain storage; NCH 1, 2, 3, 4 and 8; more scans than one wave; single and many calls interleaved on the
same scans; every call-level error, each leaving every scan where it was; the coalescer with 12 threads, and a second
call on a scan inside one coalescer dispatch, refused alone.

Every test here also runs under the CPU SIMT emulator (DANN_EMULATE=1, tests/test_zz_n_scan_many_emulated.py)."""
import threading

import numpy as np
import pytest

from conftest import build_case, emulating
from test_gpu_parity import COSINE, IP, L2, _queries

pytestmark = pytest.mark.gpu

FIELDS = ("visits", "d_quantized", "candidates", "d_full", "stream_len")


@pytest.fixture(scope="module")
def lib(lib_built):
    from pgvectorscale_b200 import diskann
    if diskann.device_count() < 1:
        pytest.fail("no CUDA device visible: -m gpu tests need an H100")
    return diskann


class Tracked:
    """One scan and the oracle's view of it: check(row) compares the row of the scan's i-th amgettuple and its counters
    with oracle.scan(.., i)."""

    def __init__(self, idx, s, q, labels=None, L=40, rescore=20):
        self.s, self.q, self.labels, self.L, self.rescore = s, q, labels, L, rescore
        self.sc = idx.begin_scan()
        self.sc.rescan(q, labels=labels, search_list_size=L, rescore=rescore)
        plain_no_resort = int(getattr(s, "storage_type", 0) or 0) != 0 and s.dim == s.dim_index
        self.with_dist = rescore > 0 and not plain_no_resort
        self.i = 0
        self.ended = False

    def check(self, row):
        from oracle import oracle
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
        st = self.sc.stats()
        for f in FIELDS:
            assert st[f] == ref["stats"][f], (f,) + what

    def end(self):
        self.sc.end()


def many(lib, tracked):
    """one gettuple_many over `tracked`, every result checked"""
    out = lib.gettuple_many([t.sc for t in tracked])
    assert len(out) == len(tracked)
    for t, r in zip(tracked, out):
        assert not isinstance(r, Exception), r
        t.check(r)
    return out


def mixed_scans(idx, s, seed):
    """42 scans: L 1..200 x rescore 0 / 1 / 50 x five keys, a NULL query and a zero query"""
    q = _queries(s, 40, seed)
    keys = [None, [], [999], [3], [2, 7]]
    Ls = [1, 7, 30, 100, 200]
    out = []
    for j in range(40):
        out.append(Tracked(idx, s, q[j], keys[j % 5], Ls[(j // 5) % 5], (0, 1, 50)[j % 3]))
    out.append(Tracked(idx, s, None, None, 50, 50))
    out.append(Tracked(idx, s, np.zeros(s.dim, np.float32), [3], 20, 1))
    return out


@pytest.mark.parametrize("dist,bits", [(COSINE, 2), (L2, 1), (IP, 2)])
def test_many_mixed_scans_every_call(lib, dist, bits):
    s = build_case(500, 64, dist, bits=bits, seed=40 + dist + bits, kind="uniform" if dist == IP else "normal",
                   labels=True, R=20, L_build=40, deleted_every=7)
    with lib.DiskAnnIndex(s) as idx:
        tr = mixed_scans(idx, s, 100 + dist)
        for _ in range(12):
            many(lib, tr)
        for t in tr:
            t.end()


def test_scans_end_at_different_calls(lib):
    """A 60-node index with every 4th tuple deleted: scans with different keys run dry after different numbers of rows;
    the finished ones keep returning None while the others go on."""
    s = build_case(60, 32, L2, bits=2, seed=9, kind="uniform", labels=True, R=12, L_build=24, deleted_every=4)
    q = _queries(s, 8, 19, "uniform")
    with lib.DiskAnnIndex(s) as idx:
        tr = [Tracked(idx, s, q[j], [None, [1], [2, 5], [7], [999]][j % 5], (5, 30, 80)[j % 3], (0, 10, 50)[j % 3])
              for j in range(8)]
        ends = set()
        for call in range(70):
            many(lib, tr)
            ends |= {t.i for t in tr if t.ended and t.i == call + 1}
            if all(t.ended for t in tr):
                break
        assert all(t.ended for t in tr)
        assert len(ends) >= 3, ends                    # the scans ran dry at different calls
        for t in tr:
            t.end()


def test_two_entry_layouts_in_one_call_and_the_launch_count(lib):
    """1024 x 2 codes: L = 10 plans Ent32x16, L = 3000 Ent64 (cand_cap > 65536, as in test_zz_m_wide_gpu.py).  A call
    that mixes them is one search launch per layout + one distance launch + one finish launch; a call of one layout
    is exactly 3 launches."""
    s = build_case(320, 1024, IP, bits=2, seed=1031, kind="uniform", R=24, L_build=48)
    q = _queries(s, 8, 1033, "uniform")
    with lib.DiskAnnIndex(s) as idx:
        small = [Tracked(idx, s, q[j], None, 10, (20, 0)[j % 2]) for j in range(4)]
        large = [Tracked(idx, s, q[4 + j], None, 3000, (20, 0)[j % 2]) for j in range(4)]
        for _ in range(3):
            before = idx.kernel_launches
            many(lib, small + large)
            assert idx.kernel_launches - before == 2 + 1 + 1
        for group in (small, large):
            before = idx.kernel_launches
            many(lib, group)
            assert idx.kernel_launches - before == 3
        for t in small + large:
            t.end()


def test_regrowth_at_different_calls_leaves_the_rows_unchanged(lib, monkeypatch):
    """DANN_DEBUG_SHRINK=8: every first workspace is too small; each scan overflows, regrows alone and replays in a
    later round of the same call, at its own calls."""
    monkeypatch.setenv("DANN_DEBUG_SHRINK", "8")
    s = build_case(500, 64, COSINE, bits=2, seed=77, labels=True, R=20, L_build=40, deleted_every=9)
    q = _queries(s, 10, 78)
    with lib.DiskAnnIndex(s) as idx:
        tr = [Tracked(idx, s, q[j], [None, [4]][j % 2], (10, 40, 120, 200, 60)[j % 5], (30, 50)[j % 2])
              for j in range(10)]
        rounds = []
        for _ in range(40):
            before = idx.kernel_launches
            many(lib, tr)
            rounds.append(idx.kernel_launches - before)
        assert max(rounds) > 3, rounds                 # some call needed a second round
        for t in tr:
            t.end()


SHAPES = [  # (dim, bits, distance, data kind): NCH 1, 2, 3, 4, 8 (test_zz_m_wide_gpu.py's code-mapping table)
    (37, 2, COSINE, "normal"), (100, 2, L2, "uniform"), (768, 2, COSINE, "normal"), (6145, 2, L2, "uniform"),
    (8200, 2, IP, "uniform"),
]


@pytest.mark.parametrize("shape", SHAPES, ids=[f"{d}x{b}" for d, b, *_ in SHAPES])
def test_every_code_width(lib, shape):
    dim, bits, dist, kind = shape
    s = build_case(200, dim, dist, bits=bits, seed=dim, kind=kind, R=16, L_build=32)
    q = _queries(s, 6, dim + 5, kind)
    with lib.DiskAnnIndex(s) as idx:
        tr = [Tracked(idx, s, q[j], None, (8, 40, 150)[j % 3], (0, 20)[j % 2]) for j in range(6)]
        for _ in range(8):
            many(lib, tr)
        for t in tr:
            t.end()


def test_hash_set_inserted_set(lib, monkeypatch):
    monkeypatch.setenv("DANN_SEARCH_BITMAP", "0")
    s = build_case(400, 48, L2, bits=2, seed=5, kind="uniform", labels=True, R=16, L_build=32, deleted_every=5)
    with lib.DiskAnnIndex(s) as idx:
        tr = mixed_scans(idx, s, 55)[::3]
        for _ in range(8):
            many(lib, tr)
        for t in tr:
            t.end()


@pytest.mark.parametrize("dist,dim,dim_index", [(COSINE, 96, None), (L2, 70, 38)])
def test_plain_storage(lib, dist, dim, dim_index):
    from oracle import fixtures
    s = fixtures.to_plain(build_case(400, dim, dist, seed=8, R=16, L_build=32, deleted_every=11, dim_index=dim_index))
    q = _queries(s, 6, 15)
    with lib.DiskAnnIndex(s) as idx:
        tr = [Tracked(idx, s, q[j], None, (10, 60, 150)[j % 3], (0, 20)[j % 2]) for j in range(6)]
        tr.append(Tracked(idx, s, None, None, 30, 10))
        for _ in range(10):
            many(lib, tr)
        for t in tr:
            t.end()


def test_more_scans_than_one_wave(lib):
    """800 scans at L = 200 on a 24-slot graph: each scan's plan takes about 42 KB of shared memory, so an H100 holds
    about 5 per SM and 660 in one wave.  (Fewer scans under the CPU emulator, which has no waves.)"""
    s = build_case(400, 32, L2, bits=2, seed=3, kind="uniform", R=24, L_build=48)
    n = 120 if emulating() else 800
    q = _queries(s, n, 4, "uniform")
    with lib.DiskAnnIndex(s) as idx:
        tr = [Tracked(idx, s, q[j], None, 200, (50, 0)[j % 2]) for j in range(n)]
        for _ in range(2):
            many(lib, tr)
        for t in tr:
            t.end()


def test_single_and_many_calls_interleave(lib):
    s = build_case(500, 64, COSINE, bits=2, seed=61, labels=True, R=20, L_build=40)
    q = _queries(s, 8, 62)
    with lib.DiskAnnIndex(s) as idx:
        tr = [Tracked(idx, s, q[j], [None, [5]][j % 2], (20, 80)[j % 2], (0, 50, 1)[j % 3]) for j in range(8)]
        for step in range(12):
            if step % 3 == 2:
                for t in tr[step % 2::2]:               # half of the scans take a single amgettuple
                    t.check(t.sc.gettuple())
            else:
                many(lib, tr)
        for t in tr:
            t.end()


def test_call_level_errors_move_no_scan(lib):
    import ctypes as C
    s = build_case(300, 32, L2, bits=2, seed=17, kind="uniform", R=16, L_build=32)
    q = _queries(s, 4, 18, "uniform")
    with lib.DiskAnnIndex(s) as idx, lib.DiskAnnIndex(s) as other:
        tr = [Tracked(idx, s, q[j], None, 30, (0, 20)[j % 2]) for j in range(4)]
        many(lib, tr)
        launches = idx.kernel_launches
        stats = [t.sc.stats() for t in tr]
        fresh = idx.begin_scan()                        # never rescanned
        foreign = Tracked(other, s, q[0], None, 30, 20)
        ended = idx.begin_scan()
        ended.end()                                     # its handle is NULL now
        scans = [t.sc for t in tr]
        cases = [([], -1), (scans * 16385 + [scans[0]], -1), (scans + [ended], -1), (scans + [foreign.sc], -1),
                 (scans + [scans[1]], -1), (scans + [fresh], -6)]
        for lst, code in cases:
            with pytest.raises(lib.DiskAnnError) as e:
                lib.gettuple_many(lst)
            assert e.value.code == code, (len(lst), e.value)
        lib_ = lib.load_library()
        handles = (C.c_void_p * 4)(*[t.sc._h for t in tr])
        assert lib_.dann_scan_gettuple_many(handles, 4, None, None, None, None, None) == -1   # NULL out_rc
        rc = np.zeros(4, np.int32)
        assert lib_.dann_scan_gettuple_many(None, 4, C.c_void_p(rc.ctypes.data), None, None, None, None) == -1
        assert idx.kernel_launches == launches
        assert [t.sc.stats() for t in tr] == stats
        for _ in range(3):                              # and the scans go on from where they were
            many(lib, tr)
        for t in tr + [foreign]:
            t.end()
        fresh.end()


def test_coalescer_gettuple_from_many_threads(lib):
    """12 threads behind a barrier, each draining its own scan through Coalescer.gettuple: the rows are the oracle's,
    and the dispatcher served more than one thread per dann_scan_gettuple_many."""
    s = build_case(400, 64, COSINE, bits=2, seed=23, labels=True, R=16, L_build=32, deleted_every=6)
    q = _queries(s, 12, 24)
    with lib.DiskAnnIndex(s) as idx, lib.DiskAnnIndex(s) as other:
        tr = [Tracked(idx, s, q[j], [None, [2]][j % 2], (10, 50, 120)[j % 3], (0, 1, 30)[j % 3]) for j in range(12)]
        rows = [[] for _ in tr]
        errors = []
        co = lib.Coalescer(idx, max_batch=64, max_wait_us=20000)
        bar = threading.Barrier(len(tr))

        def drain(j):
            try:
                bar.wait()
                for _ in range(15):
                    rows[j].append(co.gettuple(tr[j].sc))
            except Exception as e:                      # reported below
                errors.append(e)

        th = [threading.Thread(target=drain, args=(j,)) for j in range(len(tr))]
        for t in th:
            t.start()
        for t in th:
            t.join()
        assert not errors, errors
        st = co.stats()
        foreign = Tracked(other, s, q[0], None, 30, 20)
        with pytest.raises(lib.DiskAnnError) as e:      # a scan of another index
            co.gettuple(foreign.sc)
        assert e.value.code == -1
        co.close()
        from oracle import oracle
        for t, got in zip(tr, rows):
            ref = oracle.scan(s, t.q, t.labels, t.L, t.rescore, 15)
            n = len(ref["tid"])
            assert all(r is None for r in got[n:])
            assert [(r[0] << 16) | r[1] for r in got[:n]] == ref["tid"].tolist()
            assert [r[2] for r in got[:n]] == ref["node"].tolist()
            if t.rescore:
                assert np.array([r[3] for r in got[:n]], np.float32).view(np.uint32).tolist() == \
                    ref["dist"].view(np.uint32).tolist()
            stt = t.sc.stats()
            for f in FIELDS:
                assert stt[f] == ref["stats"][f], f
        assert st["queries"] == 12 * 15 and st["largest_batch"] > 1, st
        for t in tr + [foreign]:
            t.end()


def test_coalescer_refuses_a_second_call_on_a_scan_alone(lib):
    """Two threads call gettuple on the same scan inside one dispatch (max_batch = 3 holds the window until all three
    requests are queued): one of them is refused with DANN_ERR_INVALID_ARG, the other one and the third thread, on a
    scan of its own, get their rows, and the shared scan took exactly one step."""
    s = build_case(300, 32, L2, bits=2, seed=29, kind="uniform", R=16, L_build=32)
    q = _queries(s, 2, 30, "uniform")
    with lib.DiskAnnIndex(s) as idx:
        shared, own = Tracked(idx, s, q[0], None, 30, 20), Tracked(idx, s, q[1], None, 30, 0)
        co = lib.Coalescer(idx, max_batch=3, max_wait_us=5_000_000)
        bar = threading.Barrier(3)
        got = [None] * 3

        def call(j, t):
            bar.wait()
            try:
                got[j] = co.gettuple(t.sc)
            except lib.DiskAnnError as e:
                got[j] = e

        th = [threading.Thread(target=call, args=(j, t)) for j, t in enumerate((shared, shared, own))]
        for t in th:
            t.start()
        for t in th:
            t.join()
        st = co.stats()
        co.close()
        refused = [g for g in got[:2] if isinstance(g, Exception)]
        assert len(refused) == 1 and refused[0].code == -1 and "in flight" in str(refused[0]), got
        assert st["largest_batch"] == 3, st
        shared.check([g for g in got[:2] if not isinstance(g, Exception)][0])
        own.check(got[2])
        many(lib, [shared, own])                         # both go on from where they were
        shared.end()
        own.end()
