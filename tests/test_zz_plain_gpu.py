"""GPU parity of the plain (uncompressed) storage layout - SURVEY.md §8f row 3: plain/storage.rs:223-307,
scan.rs:392-403 - and of the one-synchronisation amgettuple, through the C ABI: batch calls, the streaming scan
operator with counters after every row, golden vectors, edge-case fuzz.  Part of the regular `-m gpu` run."""
import os

import numpy as np
import pytest

from conftest import build_case
from test_gpu_parity import _compare_batch, _queries

pytestmark = pytest.mark.gpu

COSINE, L2, IP = 0, 1, 2


@pytest.fixture(scope="module")
def lib(lib_built):
    from pgvectorscale_b200 import diskann
    if diskann.device_count() < 1:
        pytest.fail("no CUDA device visible: -m gpu tests need an H100")
    return diskann


# ---- plain storage layout (dann_index_load_plain) ---------------------------------------------------------------
def _compare_plain(s, idx, q, k, L, rescore):
    from oracle import oracle
    g = idx.search_batch(q, k=k, search_list_size=L, rescore=rescore)
    for b in range(q.shape[0]):
        r = oracle.scan(s, q[b], None, L, rescore, k)
        n = len(r["tid"])
        assert int(g["count"][b]) == n
        assert g["tid"][b, :n].tolist() == r["tid"].tolist()
        if rescore and s.dim != s.dim_index:       # scan.rs:392-403: only then is there a rerank and a distance
            assert g["dist"][b, :n].view(np.uint32).tolist() == r["dist"].view(np.uint32).tolist()
        for f in ("visits", "d_quantized", "candidates", "d_full", "stream_len"):
            assert int(g["stats"][f][b]) == r["stats"][f], f


@pytest.mark.parametrize("dist,dim,dim_index", [(COSINE, 768, None), (L2, 256, None), (COSINE, 256, 100), (L2, 70, 38)])
def test_plain_storage_batch_and_scan_match_oracle(lib, monkeypatch, dist, dim, dim_index):
    from oracle import fixtures, oracle
    s = fixtures.to_plain(build_case(2000, dim, dist, seed=8, kind="normal", R=32, L_build=64, deleted_every=13,
                                     dim_index=dim_index))
    q = _queries(s, 24, 5)
    with lib.DiskAnnIndex(s) as idx:
        _compare_plain(s, idx, q, k=10, L=50, rescore=20)
        _compare_plain(s, idx, q[:8], k=15, L=20, rescore=0)
        scan = idx.begin_scan()                       # the streaming operator, counters after every row
        scan.rescan(q[0], search_list_size=40, rescore=10)
        want = oracle.scan(s, q[0], None, 40, 10, 30)
        got = []
        for _ in range(30):
            row = scan.gettuple()
            if row is None:
                break
            got.append((row[0] << 16) | row[1])
        assert got == want["tid"].tolist()
        st = scan.stats()
        for f in ("visits", "d_quantized", "candidates", "d_full"):
            assert st[f] == want["stats"][f], f
        scan.end()
        with pytest.raises(lib.DiskAnnError, match="label"):
            idx.search_batch(q[:2], labels=[[1], [2]], k=5)


@pytest.mark.parametrize("name", ["plain_cos128", "plain_l2_96x40", "plain_cos70x38"])
def test_plain_storage_golden_vectors(lib, monkeypatch, name):
    import os as _os
    from golden.make_plain_golden import make_case
    z = np.load(_os.path.join(_os.path.dirname(__file__), "golden", "plain_golden.npz"))
    s, q, L, rescore, k = make_case(name)
    with lib.DiskAnnIndex(s) as idx:
        g = idx.search_batch(q, k=k, search_list_size=L, rescore=rescore)
    assert np.array_equal(g["count"], z[f"{name}/count"])
    assert np.array_equal(g["tid"], z[f"{name}/tid"])
    if rescore > 0 and s.dim != s.dim_index:
        for b in range(len(q)):
            n = int(g["count"][b])
            assert g["dist"][b, :n].view(np.uint32).tolist() == z[f"{name}/dist_bits"][b, :n].tolist()
    assert np.array_equal(g["stats"]["visits"], z[f"{name}/visits"])
    assert np.array_equal(g["stats"]["d_full"], z[f"{name}/d_full"])


@pytest.mark.parametrize("seed", range(30))
def test_plain_storage_random_small_indexes(lib, monkeypatch, seed):
    """Edge-case fuzz of the plain layout: tiny graphs, 1..100 dimensions, truncated slices, deleted tuples."""
    from oracle import fixtures, oracle
    rng = np.random.default_rng(7000 + seed)
    n = int(rng.choice([1, 2, 5, 33, 200]))
    dim = int(rng.choice([1, 2, 3, 8, 31, 33, 64, 100]))
    dist = int(rng.choice([COSINE, L2]))
    dim_index = None if dim < 3 or rng.random() < 0.5 else int(rng.integers(1, dim))
    R = int(rng.choice([1, 3, 16, 40, 70]))
    s = fixtures.to_plain(build_case(n, dim, dist, seed=seed, kind="normal", R=R, L_build=max(2 * R, 8),
                                     dim_index=dim_index, deleted_every=int(rng.choice([0, 0, 3, 1]))))
    B = int(rng.integers(1, 5))
    q = fixtures.gen_vectors(B, dim, 300 + seed, "normal")
    if rng.random() < 0.3:
        q[0] = 0.0
    with lib.DiskAnnIndex(s) as idx:
        for _ in range(2):
            _compare_plain(s, idx, q, k=int(rng.choice([1, 3, 20])), L=int(rng.choice([1, 2, 5, 50])),
                           rescore=int(rng.choice([0, 1, 7, 100])))
        L, rescore = int(rng.choice([1, 4, 30])), int(rng.choice([0, 2, 50]))
        want = oracle.scan(s, q[0], None, L, rescore, 10_000)
        sc = idx.begin_scan()
        sc.rescan(q[0], search_list_size=L, rescore=rescore)
        got = []
        while True:
            row = sc.gettuple()
            if row is None:
                break
            got.append((row[0] << 16) | row[1])
            assert len(got) <= n
        assert got == want["tid"].tolist()
        st = sc.stats()
        for f in ("visits", "d_quantized", "candidates", "d_full"):
            assert st[f] == want["stats"][f], f
        sc.end()


def test_one_synchronisation_gettuple_rows_and_counters_match_oracle(lib):
    """amgettuple (dann_scan_distance_kernel / dann_scan_finish_kernel, one synchronisation per row): the row and all
    four counters equal oracle.scan's after every call, across rescans with and without a window and a label key."""
    from oracle import oracle
    s = build_case(3000, 128, COSINE, seed=21, kind="normal", labels=True, deleted_every=9)
    q = _queries(s, 4, 3)
    with lib.DiskAnnIndex(s) as idx:
        sc = idx.begin_scan()
        for qi, (L, rescore, key) in enumerate(((40, 10, None), (25, 0, None), (60, 50, [3, 9]), (30, 5, None))):
            sc.rescan(q[qi], labels=key, search_list_size=L, rescore=rescore)
            for i in range(1, 40):
                row = sc.gettuple()
                want = oracle.scan(s, q[qi], key, L, rescore, i)
                if row is None:
                    assert len(want["tid"]) < i
                    break
                assert ((row[0] << 16) | row[1]) == int(want["tid"][i - 1])
                st = sc.stats()
                for f in ("visits", "d_quantized", "candidates", "d_full"):
                    assert st[f] == want["stats"][f], (qi, i, f)
        sc.end()
