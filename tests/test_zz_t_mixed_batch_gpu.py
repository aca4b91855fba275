"""dann_search_batch_mixed - one batch whose queries differ in k, search_list_size, rescore and key - its device and group
entry points and the coalescer that now merges every waiting search request into one such batch.  Bar: every query's
rows (TID, distance bits when it reranks), count and counters equal the oracle's scan with that query's own parameters,
and every dann_query_stats field equals a private one-query dann_search_batch; past its own k a row is DANN_INVALID_TID
and NaN up to the batch's largest k.

Covered: cosine / L2 / IP indexes of 1 and 2 bits with labels and deleted tuples; k 1..40, L 1..300, rescore 0..200 and
no key / an empty key / labels with and without a start node in one batch; growth reruns inside a mixed batch
(DANN_DEBUG_SHRINK); the lean, two-warp and single-warp kernels; the plain layout with dim_index < dim and == dim; a
mixed call with equal parameters against dann_search_batch, bit for bit; the device entry point; every refusal, each
leaving the handle usable; 12 coalescer callers of 12 parameter classes in one dispatch; a two-replica group.

Every test here also runs under the CPU SIMT emulator (DANN_EMULATE=1, tests/test_zz_t_mixed_batch_emulated.py)."""
import ctypes as C
import os
import threading

import numpy as np
import pytest

from conftest import build_case, buffer_device, dptr, emulating
from test_gpu_parity import COSINE, IP, L2, _queries

pytestmark = pytest.mark.gpu

FIELDS = ("visits", "d_quantized", "candidates", "d_full")
ALL_FIELDS = FIELDS + ("stream_len", "status")
INVALID_TID = 0xFFFFFFFFFFFFFFFF
NAN_BITS = 0x7FC00000
# labels of the fixture are 1..16: 999 has no start node (nor any row)
KEYS = [None, [], [3], [2, 7], [999], [5, 999], [1, 4, 9]]


@pytest.fixture(scope="module")
def lib(lib_built):
    from pgvectorscale_b200 import diskann
    if diskann.device_count() < 1:
        pytest.fail("no CUDA device visible: -m gpu tests need an H100")
    return diskann


def sm_count():
    if emulating():
        return int(os.environ.get("SIMT_SM_COUNT", "132"))
    import torch
    return torch.cuda.get_device_properties(0).multi_processor_count


def labeled_case(dist, bits, seed=0):
    return build_case(500, 64, dist, bits=bits, seed=60 + 3 * dist + bits + seed, kind="uniform" if dist == IP else "normal",
                      labels=True, R=20, L_build=40, deleted_every=7)


def draw(B, seed, keyed=True):
    """per-query k 1..40, L 1..300, rescore 0..200 and (keyed) a key of KEYS"""
    rng = np.random.default_rng(seed)
    k = rng.integers(1, 41, B)
    L = rng.integers(1, 301, B)
    rescore = rng.integers(0, 201, B)
    labels = [KEYS[int(i)] for i in rng.integers(0, len(KEYS), B)] if keyed else None
    return k, L, rescore, labels


def check_rows(g, b, kmax, n, tids, dist_bits=None):
    """query b's n rows, then INVALID / NaN up to kmax"""
    assert g["tid"].shape[1] == kmax
    assert int(g["count"][b]) == n, b
    assert g["tid"][b, :n].tolist() == list(tids), b
    assert all(int(t) == INVALID_TID for t in g["tid"][b, n:]), b
    assert all(int(d) == NAN_BITS for d in g["dist"][b, n:].view(np.uint32)), b
    if dist_bits is not None:
        assert g["dist"][b, :n].view(np.uint32).tolist() == list(dist_bits), b


def check_oracle(s, q, g, k, L, rescore, labels, with_dist=True):
    from oracle import oracle
    kmax = int(np.max(k))
    for b in range(q.shape[0]):
        lab = None if labels is None else labels[b]
        r = oracle.scan(s, q[b], lab, int(L[b]), int(rescore[b]), int(k[b]))
        dist = r["dist"].view(np.uint32).tolist() if with_dist and rescore[b] > 0 else None
        check_rows(g, b, kmax, len(r["tid"]), r["tid"].tolist(), dist)
        for f in FIELDS:
            assert int(g["stats"][f][b]) == r["stats"][f], (b, f, int(k[b]), int(L[b]), int(rescore[b]), lab)


def check_private(idx, q, g, k, L, rescore, labels):
    """g equals B private one-query dann_search_batch calls, on every output and every dann_query_stats field"""
    kmax = int(np.max(k))
    for b in range(q.shape[0]):
        lab = None if labels is None or labels[b] is None else [labels[b]]
        p = idx.search_batch(q[b:b + 1], labels=lab, k=int(k[b]), search_list_size=int(L[b]), rescore=int(rescore[b]))
        n = int(p["count"][0])
        check_rows(g, b, kmax, n, p["tid"][0, :n].tolist(), p["dist"][0, :n].view(np.uint32).tolist())
        for f in ALL_FIELDS:
            assert int(g["stats"][f][b]) == int(p["stats"][f][0]), (b, f)


@pytest.mark.parametrize("dist,bits", [(COSINE, 1), (COSINE, 2), (L2, 1), (L2, 2), (IP, 1), (IP, 2)])
def test_mixed_batch_matches_oracle(lib, dist, bits):
    s = labeled_case(dist, bits)
    q = _queries(s, 48, 200 + dist, "uniform" if dist == IP else "normal")
    k, L, rescore, labels = draw(48, 300 + 10 * dist + bits)
    with lib.DiskAnnIndex(s) as idx:
        g = idx.search_batch(q, labels=labels, k=k, search_list_size=L, rescore=rescore)
    check_oracle(s, q, g, k, L, rescore, labels)


@pytest.mark.parametrize("shrink", [None, "8"], ids=["planned", "growth_reruns"])
def test_mixed_batch_equals_private_batches(lib, monkeypatch, shrink):
    if shrink:
        monkeypatch.setenv("DANN_DEBUG_SHRINK", shrink)
    s = labeled_case(COSINE, 2, seed=1)
    q = _queries(s, 40, 17)
    k, L, rescore, labels = draw(40, 18)
    with lib.DiskAnnIndex(s) as idx:
        g = idx.search_batch(q, labels=labels, k=k, search_list_size=L, rescore=rescore)
        plan = idx.last_search_plan()
        if shrink:
            assert plan["retries"] > 0, plan     # some queries overflowed and reran inside the mixed batch
        check_private(idx, q, g, k, L, rescore, labels)
    check_oracle(s, q, g, k, L, rescore, labels)


@pytest.mark.parametrize("kernel", ["lean", "two_warp", "single_warp"])
def test_every_search_kernel(lib, monkeypatch, kernel):
    s = labeled_case(L2, 2, seed=2)
    B = 8 * sm_count() if kernel == "lean" else 16       # more than 7 queries per SM: the lean plan
    if kernel == "single_warp":
        monkeypatch.setenv("DANN_SEARCH_KERNEL", "1")
    q = _queries(s, B, 23)
    k, L, rescore, labels = draw(B, 24)
    with lib.DiskAnnIndex(s) as idx:
        g = idx.search_batch(q, labels=labels, k=k, search_list_size=L, rescore=rescore)
        assert idx.last_search_plan()["kernel"] == {"lean": 3, "two_warp": 2, "single_warp": 1}[kernel]
    check_oracle(s, q, g, k, L, rescore, labels)


@pytest.mark.parametrize("dim,dim_index", [(96, 40), (96, None)], ids=["dim_index_lt_dim", "dim_index_eq_dim"])
def test_plain_layout(lib, dim, dim_index):
    """k, L and rescore per query; a plain index reranks only when dim_index < dim (scan.rs:392-403)"""
    from oracle import fixtures
    s = fixtures.to_plain(build_case(600, dim, COSINE, seed=31, R=24, L_build=48, deleted_every=11, dim_index=dim_index))
    q = _queries(s, 32, 32)
    k, L, rescore, _ = draw(32, 33, keyed=False)
    with lib.DiskAnnIndex(s) as idx:
        g = idx.search_batch(q, k=k, search_list_size=L, rescore=rescore)
        assert idx.last_search_plan()["kernel"] == 1
        check_private(idx, q, g, k, L, rescore, None)
    check_oracle(s, q, g, k, L, rescore, None, with_dist=s.dim != s.dim_index)


@pytest.mark.parametrize("keyed", [False, True])
def test_equal_parameters_give_the_uniform_batch_bit_for_bit(lib, keyed):
    s = labeled_case(COSINE, 1, seed=3)
    B = 24
    q = _queries(s, B, 41)
    labels = [KEYS[1 + b % (len(KEYS) - 1)] for b in range(B)] if keyed else None
    with lib.DiskAnnIndex(s) as idx:
        u = idx.search_batch(q, labels=labels, k=12, search_list_size=70, rescore=30)
        m = idx.search_batch(q, labels=labels, k=[12] * B, search_list_size=[70] * B, rescore=[30] * B)
    assert np.array_equal(u["tid"], m["tid"])
    assert np.array_equal(u["dist"].view(np.uint32), m["dist"].view(np.uint32))
    assert np.array_equal(u["count"], m["count"])
    assert np.array_equal(u["stats"], m["stats"])


def test_device_entry_point_equals_host_entry_point(lib):
    import torch
    from pgvectorscale_b200.diskann import QUERY_PARAMS_DTYPE, STATS_DTYPE
    s = labeled_case(L2, 2, seed=4)
    B = 20
    q = _queries(s, B, 51)
    k, L, rescore, labels = draw(B, 52)
    labels = [sorted(set(x)) if x is not None else None for x in labels]     # the device entry point takes sorted keys
    kmax = int(k.max())
    p = np.zeros(B, QUERY_PARAMS_DTYPE)
    p["k"], p["search_list_size"], p["rescore"] = k, L, rescore
    p["keyed"] = [0 if x is None else 1 for x in labels]
    off = np.zeros(B + 1, np.int32)
    off[1:] = np.cumsum([0 if x is None else len(x) for x in labels])
    flat = np.asarray([v for x in labels if x is not None for v in x] or [0], np.int16)
    dev = buffer_device()
    d_q = torch.from_numpy(q).to(dev)
    d_p = torch.from_numpy(p.view(np.int32).reshape(B, 4).copy()).to(dev)
    d_lab = torch.from_numpy(flat).to(dev)
    d_off = torch.from_numpy(off).to(dev)
    d_tid = torch.zeros((B, kmax), dtype=torch.int64, device=dev)
    d_dist = torch.zeros((B, kmax), dtype=torch.float32, device=dev)
    d_count = torch.zeros(B, dtype=torch.int32, device=dev)
    d_stats = torch.zeros((B, 6), dtype=torch.int32, device=dev)
    with lib.DiskAnnIndex(s) as idx:
        h = idx.search_batch(q, labels=labels, k=k, search_list_size=L, rescore=rescore)
        idx.search_batch_mixed_device(dptr(d_q), dptr(d_p), dptr(d_tid), dptr(d_dist), dptr(d_count), dptr(d_stats),
                                      d_labels=dptr(d_lab), d_label_off=dptr(d_off))
    assert np.array_equal(d_tid.cpu().numpy().view(np.uint64), h["tid"])
    assert np.array_equal(d_dist.cpu().numpy().view(np.uint32), h["dist"].view(np.uint32))
    assert np.array_equal(d_count.cpu().numpy().view(np.uint32), h["count"])
    assert np.array_equal(d_stats.cpu().numpy().view(np.uint32).reshape(-1).view(STATS_DTYPE), h["stats"])


def _raw_mixed(lib, idx, q, params, labels=None, label_off=None, B=None, null_params=False):
    """dann_search_batch_mixed on raw arrays -> (rc, message)"""
    B = q.shape[0] if B is None else B
    kmax = max(1, int(params["k"].max())) if len(params) else 1
    tid = np.zeros((max(B, 1), kmax), np.uint64)
    p = lambda a: None if a is None else C.c_void_p(a.ctypes.data)     # noqa: E731
    rc = lib.load_library().dann_search_batch_mixed(idx._h, p(q), p(labels), p(label_off), None if null_params else p(params),
                                                    B, p(tid), None, None, None)
    return rc, lib.load_library().dann_last_error().decode()


def test_refusals_leave_the_handle_usable(lib):
    from oracle import fixtures
    from pgvectorscale_b200.diskann import QUERY_PARAMS_DTYPE
    s = labeled_case(COSINE, 2, seed=5)
    B = 6
    q = _queries(s, B, 61)

    def params(all_keyed=False, **bad):
        p = np.zeros(B, QUERY_PARAMS_DTYPE)
        p["k"], p["search_list_size"], p["rescore"], p["keyed"] = 5, 40, 10, int(all_keyed)
        for f, v in bad.items():
            p[f][3] = v
        return p

    empty_off = np.zeros(B + 1, np.int32)
    bad_off = np.array([0, 1, 2, 3, 1, 4, 5], np.int32)          # falls at query 3
    one_lab = np.array([3], np.int16)
    unkeyed_lab_off = np.array([0, 0, 0, 0, 1, 1, 1], np.int32)   # query 3 has a key range but keyed = 0
    cases = [
        (dict(), dict(B=0), "B"),
        (dict(), dict(null_params=True), "params"),
        (dict(k=0), {}, "query 3"),
        (dict(k=-2), {}, "query 3"),
        (dict(search_list_size=0), {}, "query 3"),
        (dict(search_list_size=10001), {}, "query 3"),
        (dict(rescore=-1), {}, "query 3"),
        (dict(rescore=1001), {}, "query 3"),
        (dict(keyed=2), dict(label_off=empty_off), "query 3"),
        (dict(keyed=1), {}, "query 3"),                                               # keyed without label_off
        (dict(all_keyed=True), dict(labels=np.arange(1, 6, dtype=np.int16), label_off=bad_off), "query 3"),
        (dict(), dict(labels=one_lab, label_off=unkeyed_lab_off), "query 3"),
        (dict(k=200000, rescore=1000), {}, "query 3"),                                # past the rerank window
    ]
    with lib.DiskAnnIndex(s) as idx:
        for bad, kw, who in cases:
            rc, msg = _raw_mixed(lib, idx, q, params(**bad), **kw)
            assert rc == -1, (bad, kw, rc, msg)
            assert who in msg, (bad, kw, msg)
        k, L, rescore, labels = draw(B, 62)
        g = idx.search_batch(q, labels=labels, k=k, search_list_size=L, rescore=rescore)
    check_oracle(s, q, g, k, L, rescore, labels)
    # the plain layout refuses a keyed query, alone among unkeyed ones
    sp = fixtures.to_plain(build_case(300, 48, L2, seed=63, R=16, L_build=32, dim_index=20))
    qp = _queries(sp, B, 64)
    with lib.DiskAnnIndex(sp) as idx:
        rc, msg = _raw_mixed(lib, idx, qp, params(keyed=1), labels=one_lab, label_off=unkeyed_lab_off)
        assert rc == -1 and "query 3" in msg, msg
        k, L, rescore, _ = draw(B, 65, keyed=False)
        g = idx.search_batch(qp, k=k, search_list_size=L, rescore=rescore)
    check_oracle(sp, qp, g, k, L, rescore, None)


def test_coalescer_merges_every_parameter_class_into_one_dispatch(lib):
    from oracle import oracle
    s = labeled_case(L2, 2, seed=6)
    q = _queries(s, 12, 71)
    classes = [(k, L, r, key) for k, L, r, key in zip((1, 5, 10, 20, 40, 3, 7, 12, 25, 33, 9, 15),
                                                       (10, 40, 100, 300, 60, 1, 150, 80, 200, 35, 120, 50),
                                                       (0, 10, 50, 200, 1, 0, 30, 100, 0, 20, 5, 75),
                                                       (None, [3], None, [], [2, 7], [999], None, [1, 4, 9], [5],
                                                        None, [3], [6, 999]))]
    assert len(set((k, L, r, str(key)) for k, L, r, key in classes)) == 12
    results, errors = {}, []
    with lib.DiskAnnIndex(s) as idx, lib.Coalescer(idx, max_batch=64, max_wait_us=2_000_000) as co:
        start = threading.Barrier(12)

        def backend(t):
            try:
                k, L, rescore, key = classes[t]
                start.wait()
                results[t] = co.search(q[t], labels=key, k=k, search_list_size=L, rescore=rescore)
            except Exception as e:      # noqa: BLE001
                errors.append(e)

        th = [threading.Thread(target=backend, args=(t,)) for t in range(12)]
        for x in th:
            x.start()
        for x in th:
            x.join()
        st = co.stats()
    assert not errors, errors
    assert st == dict(batches=1, queries=12, largest_batch=12), st
    for t, (k, L, rescore, key) in enumerate(classes):
        r = oracle.scan(s, q[t], key, L, rescore, k)
        g = results[t]
        n = len(r["tid"])
        assert g["count"] == n and g["tid"][:n].tolist() == r["tid"].tolist(), t
        assert all(int(x) == INVALID_TID for x in g["tid"][n:]), t
        if rescore:
            assert g["dist"][:n].view(np.uint32).tolist() == r["dist"].view(np.uint32).tolist(), t
        for f in FIELDS:
            assert g["stats"][f] == r["stats"][f], (t, f)


def test_group_of_two_replicas_equals_one_index(lib):
    if lib.device_count() < 2:
        pytest.skip("needs two devices (runs under the emulator with SIMT_FAKE_DEVICES=2)")
    s = labeled_case(COSINE, 2, seed=7)
    B = 33
    q = _queries(s, B, 81)
    k, L, rescore, labels = draw(B, 82)
    with lib.DiskAnnIndex(s) as idx:
        one = idx.search_batch(q, labels=labels, k=k, search_list_size=L, rescore=rescore)
    with lib.IndexGroup(s, ndev=2) as grp:
        two = grp.search_batch(q, labels=labels, k=k, search_list_size=L, rescore=rescore)
    for f in ("tid", "count", "stats"):
        assert np.array_equal(one[f], two[f]), f
    assert np.array_equal(one["dist"].view(np.uint32), two["dist"].view(np.uint32))
    check_oracle(s, q, two, k, L, rescore, labels)
