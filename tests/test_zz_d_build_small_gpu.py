"""dann_build_graph on a small index whose inputs come from the oracle (numpy only): structural validity, recall of
scans over the built graph, parity oracle vs CUDA on the built snapshot - unlabeled and labeled.  Small enough to run
under CPU emulation too (tests/test_emulated_abi.py), where it is the only check of the builder's kernels.
Written after this round's GPU minutes were spent; the file name sorts it after the tests that have been on hardware."""
import numpy as np
import pytest

from conftest import build_case

pytestmark = pytest.mark.gpu

L2 = 1


def _build(lib, n, dim, labels, R=24, L_build=48):
    from oracle import fixtures
    from pgvectorscale_b200.snapshot import INVALID_NODE
    s = build_case(n, dim, L2, seed=77, kind="normal", R=8, L_build=16, labels=labels)   # codes/means/labels from the oracle
    slots = 64
    s.R = slots
    s.nbrs = np.full((n, slots), INVALID_NODE, np.uint32)
    s.start_default = 0
    if labels:                      # per-label start node = first node carrying the label (graph/start_nodes.rs)
        first = {}
        for i in range(n):
            for l in s.labels[s.label_off[i]:s.label_off[i + 1]]:
                first.setdefault(int(l), i)
        ks = sorted(first)
        s.start_labels = np.array(ks, np.int16)
        s.start_label_nodes = np.array([first[k] for k in ks], np.uint32)
    idx = lib.DiskAnnIndex(s)
    st = idx.build_graph(R, L_build, 1.2, 256)
    s.nbrs = idx.download_nbrs()
    return s, idx, st


def _check_structure(s, R):
    n = s.n
    nb = s.nbrs
    valid = nb != 0xFFFFFFFF
    deg = valid.sum(1)
    assert deg.max() <= R and deg[1:].min() >= 1
    assert (valid[:, :-1] >= valid[:, 1:]).all()                      # INVALID-terminated prefixes
    assert (nb[valid] < n).all()
    assert not (nb == np.arange(n, dtype=np.uint32)[:, None]).any()   # no self loops
    for i in range(n):                                                # no duplicates
        row = nb[i][valid[i]]
        assert len(set(row.tolist())) == len(row)


@pytest.fixture(scope="module")
def lib(lib_built):
    from pgvectorscale_b200 import diskann
    if diskann.device_count() < 1:
        pytest.fail("no CUDA device visible: -m gpu tests need an H100")
    return diskann


def test_small_built_graph_valid_recall_parity(lib):
    from oracle import fixtures, oracle
    n, dim, R = 1500, 48, 24
    s, idx, st = _build(lib, n, dim, labels=False, R=R)
    try:
        _check_structure(s, R)
        assert st["batches"] >= 5 and st["avg_degree"] > 0.5 * R
        q = fixtures.gen_vectors(32, dim, 5, "normal")
        g = idx.search_batch(q, k=10, search_list_size=60, rescore=60)
        otid, odist, _, ostats = oracle.scan_batch(s, q, None, None, 60, 60, 10)
        assert np.array_equal(g["tid"], otid)
        assert np.array_equal(g["dist"].view(np.uint32), odist.view(np.uint32))
        assert np.array_equal(g["stats"]["visits"].astype(np.uint64), ostats["visits"])
        node_of = {int(t): i for i, t in enumerate(s.heap_tid)}
        hits = 0
        for b in range(len(q)):
            d = ((s.vectors - q[b]) ** 2).sum(1)
            truth = set(np.argsort(d, kind="stable")[:10].tolist())
            hits += len(truth & set(node_of[int(t)] for t in g["tid"][b, :int(g["count"][b])]))
        # iid Gaussian vectors are a hard case for SBQ; the yardstick is the reference's SERIAL build on the same data
        ser = build_case(n, dim, L2, seed=77, kind="normal", R=R, L_build=48)
        ser_hits = 0
        for b in range(len(q)):
            d = ((s.vectors - q[b]) ** 2).sum(1)
            truth = set(np.argsort(d, kind="stable")[:10].tolist())
            ser_hits += len(truth & set(oracle.scan(ser, q[b], None, 60, 60, 10)["node"].tolist()))
        assert hits >= ser_hits - 0.1 * 10 * len(q), (hits, ser_hits)
    finally:
        idx.close()


def test_small_built_labeled_graph_valid_and_parity(lib):
    from oracle import fixtures, oracle
    n, dim, R = 1200, 32, 24
    s, idx, st = _build(lib, n, dim, labels=True, R=R)
    try:
        _check_structure(s, R)
        q = fixtures.gen_vectors(16, dim, 6, "normal")
        labels = [[1 + (i % 16)] for i in range(16)]
        off = np.arange(17, dtype=np.int32)
        lab = np.array([l[0] for l in labels], np.int16)
        g = idx.search_batch(q, labels=labels, k=10, search_list_size=60, rescore=40)
        otid, odist, ocount, _ = oracle.scan_batch(s, q, lab, off, 60, 40, 10)
        assert np.array_equal(g["count"], ocount) and np.array_equal(g["tid"], otid)
        for b in range(16):                                   # every returned row carries the label
            for t in g["tid"][b, :int(g["count"][b])]:
                node = int(np.nonzero(s.heap_tid == t)[0][0])
                assert labels[b][0] in s.labels[s.label_off[node]:s.label_off[node + 1]]
    finally:
        idx.close()


# floors leave room for the rescue's run-to-run variation on hardware (its kernels race by design; without it the
# build is deterministic, tests/test_zz_o_build_model_gpu.py); under emulation the five cases return 997, 446, 1000, 1000
# and 750 of 1000 rows
@pytest.mark.parametrize("dim,R,rescue,floor", [(8, 10, 0, 0.98), (2, 10, 0, 0.3), (8, 10, 1, 0.995), (2, 20, 1, 0.99),
                                                 (2, 10, 1, 0.6)])
def test_small_accuracy_connectivity_of_the_gpu_builder(lib, monkeypatch, dim, R, rescue, floor):
    """build.rs:1717-1853 (1000 random low-dimensional vectors, num_neighbors = 10, search_list_size = 10, unbounded scan
    at query_search_list_size = 2 must return every row) applied to dann_build_graph.  The reference's SERIAL build - and
    the oracle's restatement of it, tests/test_oracle_kats.py - keeps every node reachable.  The batch builder matches
    that at 8 dimensions; at 2 dimensions (2-bit SBQ leaves 9 distinct codes for 1000 points, every batch is a crowd of
    zero-distance duplicates that do not see each other) it does NOT: a known limit of batched insertion, recorded
    here with the floor it currently reaches (DESIGN.md section 6b).  DANN_BUILD_RESCUE=1 (opt-in, not the reference's
    algorithm) hands every node without an in-edge a slot in a neighbour's list after the build: everything but the
    most degenerate case (5 distinct codes, R = 10) then comes back complete."""
    monkeypatch.setenv("DANN_BUILD_RESCUE", str(rescue))
    from pgvectorscale_b200.snapshot import INVALID_NODE
    n = 1000
    s = build_case(n, dim, 0, seed=5, kind="uniform", R=4, L_build=8)
    s.R = 64
    s.nbrs = np.full((n, 64), INVALID_NODE, np.uint32)
    s.start_default = 0
    with lib.DiskAnnIndex(s) as idx:
        idx.build_graph(R, 10 if R == 10 else 40, 1.2, 256)
        nb = idx.download_nbrs()
        valid = nb != INVALID_NODE
        assert valid.sum(1).max() <= R and (nb[valid] < n).all()
        assert (valid[:, :-1] >= valid[:, 1:]).all()          # still INVALID-terminated prefixes after the rescue
        sc = idx.begin_scan()
        sc.rescan(np.ones(dim, np.float32), search_list_size=2, rescore=50)
        got = set()
        while True:
            row = sc.gettuple()
            if row is None:
                break
            got.add((row[0], row[1]))
        sc.end()
    assert len(got) >= floor * n, len(got)


@pytest.mark.parametrize("seed", range(12))
def test_random_small_builds_are_valid_graphs_with_scan_parity(lib, monkeypatch, seed):
    """Builder fuzz: 1..1200 nodes, num_neighbors 1..64, build search lists 1..100, batch limits 1..unbounded, with and
    without labels and the in-edge rescue - every result is a structurally valid graph (INVALID-terminated lists of at
    most R distinct in-range ids, no self loops) and scans over it equal the oracle's on the same snapshot."""
    from oracle import fixtures, oracle
    from pgvectorscale_b200.snapshot import INVALID_NODE
    rng = np.random.default_rng(90000 + seed)
    n = int(rng.choice([1, 2, 5, 70, 400, 1200]))
    dim = int(rng.choice([2, 8, 48, 200]))
    dist = int(rng.integers(0, 3))
    labels = bool(rng.random() < 0.4)
    R, Lb, mb = int(rng.choice([1, 4, 12, 32, 50, 64])), int(rng.choice([1, 5, 30, 100])), int(rng.choice([1, 7, 64, 1 << 20]))
    monkeypatch.setenv("DANN_BUILD_RESCUE", str(int(rng.integers(0, 2))))
    s = build_case(n, dim, dist, bits=int(rng.choice([1, 2])), seed=seed, kind=str(rng.choice(["normal", "uniform"])), R=4,
                   L_build=8, labels=labels)
    s.R = 64
    s.nbrs = np.full((n, 64), INVALID_NODE, np.uint32)
    s.start_default = 0
    if labels:
        first = {}
        for i in range(n):
            for l in s.labels[s.label_off[i]:s.label_off[i + 1]]:
                first.setdefault(int(l), i)
        ks = sorted(first)
        s.start_labels = np.array(ks, np.int16)
        s.start_label_nodes = np.array([first[k] for k in ks], np.uint32)
    with lib.DiskAnnIndex(s) as idx:
        idx.build_graph(R, Lb, 1.2, mb)
        s.nbrs = idx.download_nbrs()
        _check_structure_general(s, R)
        q = fixtures.gen_vectors(2, dim, 3 + seed, "normal")
        key = [[1], [2, 3]] if labels else None
        g = idx.search_batch(q, labels=key, k=5, search_list_size=20, rescore=10)
    for b in range(2):
        r = oracle.scan(s, q[b], None if key is None else key[b], 20, 10, 5)
        nrow = len(r["tid"])
        assert int(g["count"][b]) == nrow and g["tid"][b, :nrow].tolist() == r["tid"].tolist(), (seed, b)


def _check_structure_general(s, R):
    n, nb = s.n, s.nbrs
    valid = nb != 0xFFFFFFFF
    assert valid.sum(1).max() <= R
    assert (valid[:, :-1] >= valid[:, 1:]).all()
    assert (nb[valid] < n).all()
    assert not (nb == np.arange(n, dtype=np.uint32)[:, None]).any()
    for i in range(n):
        row = nb[i][valid[i]]
        assert len(set(row.tolist())) == len(row)
