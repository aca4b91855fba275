"""dann_build_graph edge for edge against a CPU model of the batched build.

The model (oracle.build_graph_batched) runs the oracle's restatement of the reference's prune / add_neighbors /
search_for_build under the builder's batch schedule, with each of the builder's departures from the reference as one
named switch (oracle.GPU_BUILDER_SWITCHES); with every switch off and max_batch = 1 it IS the serial reference build
(tests/test_oracle_kats.py).  Without the in-edge rescue the device build is a pure function of its inputs, so
download_nbrs() must equal the model's array exactly, order inside every list included.

Every case names the branch it is there for and asserts, from the model's branch counters, that the branch ran.
Runs under CPU emulation too (tests/test_zz_o_build_model_emulated.py), except the cases marked hardware_only."""
import copy

import numpy as np
import pytest

from conftest import build_case

pytestmark = pytest.mark.gpu

INVALID = 0xFFFFFFFF
UNBOUNDED = 1 << 20


@pytest.fixture(scope="module")
def lib(lib_built):
    from pgvectorscale_b200 import diskann
    if diskann.device_count() < 1:
        pytest.fail("no CUDA device visible: -m gpu tests need an H100")
    return diskann


def _start_labels(s):
    """per-label start node = first node carrying the label (graph/start_nodes.rs)"""
    first = {}
    for i in range(s.n):
        for l in s.labels[s.label_off[i]:s.label_off[i + 1]]:
            first.setdefault(int(l), i)
    ks = sorted(first)
    s.start_labels = np.array(ks, np.int16)
    s.start_label_nodes = np.array([first[k] for k in ks], np.uint32)


def _empty_graph(s):
    s.R = 64
    s.nbrs = np.full((s.n, 64), INVALID, np.uint32)
    s.start_default = 0
    if s.has_labels:
        _start_labels(s)
    return s


def _case(n, dim, bits=None, kind="normal", labels=False, seed=11):
    """codes / means / labels from the oracle; the graph is left empty for the builder"""
    return _empty_graph(build_case(n, dim, 1, bits=bits, seed=seed, kind=kind, R=2, L_build=4, labels=labels))


def _custom_labels_case(n, dim, label_sets, seed=11):
    from oracle import fixtures
    off = np.zeros(n + 1, np.uint32)
    flat = []
    for i, ls in enumerate(label_sets):
        flat.extend(sorted(ls))
        off[i + 1] = len(flat)
    v = fixtures.gen_vectors(n, dim, seed, "normal")
    s = fixtures.make_index(v, 1, R=2, L_build=4, label_off=off, labels=np.asarray(flat, np.int16))
    return _empty_graph(s)


def _prefix(s, k):
    p = copy.copy(s)
    p.n = k
    p.codes, p.heap_tid, p.vectors = s.codes[:k], s.heap_tid[:k], s.vectors[:k]
    if s.has_labels:
        p.label_off = s.label_off[:k + 1]
        p.labels = s.labels[:int(s.label_off[k])]
    return _empty_graph(p)


def _model(s, R, L, mb):
    from oracle import oracle
    return oracle.build_graph_batched(s.codes, R, L, 1.2, s.label_off if s.has_labels else None,
                                      s.labels if s.has_labels else None, 0 if mb >= UNBOUNDED else mb,
                                      oracle.GPU_BUILDER_SWITCHES, stride=64)


def _device(lib, s, R, L, mb):
    with lib.DiskAnnIndex(s) as idx:
        idx.build_graph(R, L, 1.2, mb)
        return idx.download_nbrs()


def _row(a, i):
    return a[i][a[i] != INVALID].tolist()


def _assert_equal(lib, s, R, L, mb, got, want):
    if np.array_equal(got, want):
        return
    i = int(np.nonzero((got != want).any(1))[0][0])
    lo, hi = 1, s.n              # builds are in id order: the smallest differing prefix localises the batch
    while lo < hi:
        mid = (lo + hi) // 2
        p = _prefix(s, mid)
        if np.array_equal(_device(lib, p, R, L, mb), _model(p, R, L, mb)[0]):
            lo = mid + 1
        else:
            hi = mid
    pytest.fail(f"first differing node {i} of {s.n}: device {_row(got, i)} model {_row(want, i)}; "
                f"{int((got != want).any(1).sum())} lists differ; smallest differing prefix n' = {lo}")


def _check(lib, s, R, L, mb, expect=()):
    want, counts = _model(s, R, L, mb)
    for name in expect:      # the case reaches the branch it is there for
        assert counts[name] > 0, (name, counts)
    got = _device(lib, s, R, L, mb)
    _assert_equal(lib, s, R, L, mb, got, want)
    return got, counts


# ---- schedule: max_batch and n ------------------------------------------------------------------------------------
@pytest.mark.parametrize("mb,expect", [
    (1, ("back_pruned", "final_pruned")),            # serial: one head per launch, back-link overflow at ceil(1.3 R)
    (7, ("back_pruned", "fwd_pruned")),              # batches cut by max_batch, not by lo / 16
    (256, ("back_pruned", "round2_kept")),           # the setting the other builder tests use
    (UNBOUNDED, ("back_pruned", "final_pruned")),    # batches of lo / 16 throughout
])
def test_batch_limits(lib, mb, expect):
    _check(lib, _case(1500 if mb > 1 else 500, 48), 12, 100, mb, expect)


@pytest.mark.parametrize("n", [1, 2, 17, 33])        # nothing to insert / one insert / batch size still 1 / first batch of 2
def test_smallest_graphs(lib, n):
    _check(lib, _case(n, 16), 4, 10, UNBOUNDED, ("fwd_kept",))


# ---- num_neighbors on both sides of ceil(1.3 R) = 64 ---------------------------------------------------------------
@pytest.mark.parametrize("R,expect", [
    (1, ("back_pruned",)),                   # limit 2: every second back-link prunes to one neighbour
    (4, ("back_pruned", "final_pruned")),
    (10, ("back_pruned", "final_pruned")),   # limit 13 < 64: forward lists longer than the back-link limit survive to finalize
    (24, ("back_pruned", "final_pruned")),
    (49, ("back_pruned", "fwd_pruned")),     # limit = ceil(63.7) = 64: the last R whose limit is its own
    (50, ("back_pruned", "fwd_pruned")),     # limit = min(64, 65): the benchmark's setting
    (64, ("back_pruned", "fwd_pruned")),     # limit = slots = R: finalize has nothing to do
])
def test_num_neighbors(lib, R, expect):
    _, counts = _check(lib, _case(700, 40), R, 100, 256, expect)
    if R == 64:
        assert counts["final_pruned"] == 0


# ---- build search list: the visited list's hand-over ----------------------------------------------------------------
@pytest.mark.parametrize("L,expect", [
    (1, ("fwd_kept",)),                       # the search stops after two visits
    (10, ("fwd_kept", "back_pruned")),
    (100, ("fwd_pruned", "back_pruned")),     # more than 64 candidates: the forward prune
    (150, ("cand_cut", "fwd_pruned")),        # more than 128 visited nodes: the closest, in the visited list's order, are kept
    (300, ("visited_cut", "cand_cut")),       # more than 2 x 128 visited nodes: cut by the search kernel at the hand-over
])
def test_build_search_list(lib, L, expect):
    _check(lib, _case(1500, 32), 16, L, 256, expect)


# ---- code widths: rows are stored padded to an even word count cw, the prune kernel's shared-memory rows have stride
# cw | 1; 1920 + 1024 (cw | 1) bytes per prune warp out of 226 KB -------------------------------------------------
@pytest.mark.parametrize("words,n,expect", [
    (1, 600, ("fwd_pruned", "back_pruned")),    # one word + one of padding: lanes 2..31 of the staging loop idle
    (2, 600, ("fwd_pruned", "back_pruned")),    # even: no padding, stride 3
    (3, 600, ("fwd_pruned", "back_pruned")),    # odd: padded to 4, stride 5
    (24, 400, ("fwd_pruned", "back_pruned")),   # widest code with eight prune warps per block (stride 25)
    (25, 400, ("fwd_pruned", "back_pruned")),   # first width that costs a warp (padded to 26, stride 27: seven warps)
    (222, 300, ("fwd_pruned", "back_pruned")),  # widest code that fits at all (stride 223): one warp per block
])
def test_code_widths(lib, words, n, expect):
    _check(lib, _case(n, 64 * words, bits=1), 8, 100, 64, expect)


def test_code_too_wide_for_the_prune_kernel_is_refused_and_the_graph_is_left_alone(lib):
    """223 words (padded to 224): 128 staged rows of stride 225 outgrow the opt-in shared memory of an SM.  DANN_ERR_CAPACITY, and the
    index keeps the graph it had: scans still return the oracle's rows."""
    from oracle import fixtures, oracle
    s = build_case(80, 64 * 223, 1, bits=1, seed=4, kind="normal", R=64, L_build=20)
    assert s.start_default == 0
    q = fixtures.gen_vectors(2, s.dim, 9, "normal")
    with lib.DiskAnnIndex(s) as idx:
        with pytest.raises(lib.DiskAnnError) as e:
            idx.build_graph(8, 20, 1.2, 64)
        assert e.value.code == -5 and "too wide" in str(e.value)        # DANN_ERR_CAPACITY
        assert np.array_equal(idx.download_nbrs(), s.nbrs)
        g = idx.search_batch(q, k=5, search_list_size=20, rescore=10)
    otid, _, _, _ = oracle.scan_batch(s, q, None, None, 20, 10, 5)
    assert np.array_equal(g["tid"], otid)


# ---- code types and ties ------------------------------------------------------------------------------------------
@pytest.mark.parametrize("bits", [1, 2])
def test_one_and_two_bit_codes(lib, bits):
    _check(lib, _case(800, 48, bits=bits), 12, 100, 256, ("fwd_pruned", "back_pruned", "round2_kept"))


@pytest.mark.parametrize("R,L,mb", [(10, 10, 256), (10, 40, UNBOUNDED), (20, 100, 7)])
def test_tie_heavy_codes(lib, R, L, mb):
    """2-d uniform data at 2 bits: a handful of distinct codes.  Zero distances to the point and to the kept neighbour
    (the |id - p| / |id - kept| factor, the infinite factor), destinations with more than 64 new sources in one batch."""
    expect = ["tie_factor", "zero_occluded", "back_pruned", "final_pruned"] + (["back_src_cut"] if mb > 64 else [])
    _check(lib, _case(2000, 2, kind="uniform", seed=5), R, L, mb, expect)   # batches of more than 64 nodes from n = 1040 on


# ---- labels ---------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("mb", [1, 256])
def test_labeled_two_pass_insert(lib, mb):
    """1-2 of 16 labels per node: the filtered pass, the unfiltered pass merging with what it left (repeated sources
    dropped in the back-link path), contains_intersection in the prune."""
    _check(lib, _case(900, 32, labels=True), 12, 60, mb,
           ("fwd_merged", "back_merged", "back_repeat", "back_pruned", "label_skip", "final_pruned"))


def test_labeled_edge_sets(lib):
    """Nodes without any label (their filtered search has no start node and visits nothing), a label that one node
    alone carries (its filtered search starts - and ends - at itself), nodes carrying many labels."""
    rng = np.random.default_rng(3)
    n = 500
    sets = []
    for i in range(n):
        r = rng.random()
        if i % 7 == 0:
            sets.append([])
        elif r < 0.5:
            sets.append([int(rng.integers(1, 5))])
        else:
            sets.append(rng.integers(1, 9, size=int(rng.integers(2, 6))).tolist())
    sets[0] = []
    sets[123] = [1, 99]        # 99: carried by this node only
    sets = [sorted(set(x)) for x in sets]
    _check(lib, _custom_labels_case(n, 24, sets), 8, 40, 64,
           ("empty_search", "fwd_merged", "back_repeat", "label_skip", "back_pruned"))


# ---- determinism, kernel selection, the rescue ----------------------------------------------------------------------
def test_same_input_built_twice_on_one_handle(lib):
    s = _case(1200, 24)
    want, _ = _model(s, 16, 60, 256)
    with lib.DiskAnnIndex(s) as idx:
        idx.build_graph(16, 60, 1.2, 256)
        a = idx.download_nbrs()
        idx.build_graph(16, 60, 1.2, 256)
        b = idx.download_nbrs()
    assert np.array_equal(a, b)
    assert np.array_equal(a, want)


@pytest.mark.parametrize("kernel", ["1", "2"])
def test_build_under_a_forced_search_kernel(lib, monkeypatch, kernel):
    """Only the two-warp kernel hands over its visited list.  DANN_SEARCH_KERNEL=2 builds the model's graph;
    DANN_SEARCH_KERNEL=1 (the single-warp kernel) is refused, never a graph pruned from a buffer nobody wrote."""
    monkeypatch.setenv("DANN_SEARCH_KERNEL", kernel)
    s = _case(300, 24)
    if kernel == "2":
        _check(lib, s, 8, 30, 64, ("back_pruned",))
        return
    with lib.DiskAnnIndex(s) as idx:
        with pytest.raises(lib.DiskAnnError) as e:
            idx.build_graph(8, 30, 1.2, 64)
        assert e.value.code == -6 and "two-warp" in str(e.value)       # DANN_ERR_STATE


@pytest.mark.parametrize("dim,R", [(8, 10), (2, 10), (2, 20)])
def test_rescued_lists_stay_consistent_with_their_degrees(lib, monkeypatch, dim, R):
    """DANN_BUILD_RESCUE=1 races by design and is outside the exact comparison.  What must still hold: every row is a
    prefix of valid distinct ids, and the degrees the builder keeps (their mean is the returned avg_degree) count exactly
    the valid entries."""
    monkeypatch.setenv("DANN_BUILD_RESCUE", "1")
    s = _case(1000, dim, kind="uniform", seed=5)
    with lib.DiskAnnIndex(s) as idx:
        st = idx.build_graph(R, 10, 1.2, 256)
        nb = idx.download_nbrs()
    valid = nb != INVALID
    assert (valid[:, :-1] >= valid[:, 1:]).all() and valid.sum(1).max() <= R and (nb[valid] < s.n).all()
    assert not (nb == np.arange(s.n, dtype=np.uint32)[:, None]).any()
    for i in range(s.n):
        row = nb[i][valid[i]]
        assert len(set(row.tolist())) == len(row), i
    assert round(st["avg_degree"] * s.n) == int(valid.sum())


def test_large_build_hardware_only(lib):
    """40 000 nodes, batches of up to 2 353: many blocks per launch, heads spread over every SM.  The serial C++ model takes
    about 10 s for this size; the emulated device build would take far longer, so the emulated run
    deselects this case by its name."""
    _check(lib, _case(40000, 64), 32, 64, UNBOUNDED, ("fwd_pruned", "back_pruned", "final_pruned"))
