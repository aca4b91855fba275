"""CPU tests that pin the oracle (oracle/oracle.cpp) before it is trusted as the checker.

Sources of truth, in order:
  * the reference's own portable known-answer tests, restated as data:
      labels/mod.rs:249-425 (overlap / intersection truth tables),
      distance_x86.rs:40-63 (SIMD order vs scalar within 1e-6),
      build.rs:1419-1556 (rescore semantics, L2 / IP 3-vector sanity checks),
      build.rs:2016-2044 (NULL query returns every row),
      build.rs:1311-1396 and labels/filtering_tests.rs:880-1024 (recall properties);
  * a second, independent Python restatement (tests/pyref.py) of the scan written from the
    reference sources;
  * committed golden outputs (tests/golden/, regenerate with tests/golden/make_golden.py).
The two third-party pieces the reference does not vendor (Rust std BinaryHeap sift order,
simdeez horizontal_add_ps order) cannot be executed here: for them parity is "unpinned" and
these tests only prove that both restatements implement the same published algorithm.
"""
import os

import numpy as np
import pytest

import pyref
from conftest import build_case
from oracle import fixtures, oracle

COSINE, L2, IP = 0, 1, 2


# ---- labels/mod.rs:253-425 -------------------------------------------------------------
OVERLAP_KATS = [
    ([], [1, 2, 3], False), ([1, 2], [2, 3], True), ([1, 2], [3, 4], False),
    ([1, 2, 3, 4, 5], [1, 2, 3, 4], True), ([1, 2, 3, 4, 5], [6, 7, 8, 9, 10], False),
    ([1, 2, 3, 4, 5], [2, 3, 4, 5, 6], True), ([1, 3, 5, 10, 11], [2, 4, 6, 8, 11], True),
]
INTERSECTION_KATS = [  # (a, b, c, c.contains_intersection(a, b))
    ([1, 3, 5, 10, 11], [2, 4, 6, 8, 11], list(range(1, 12)), True),
    ([], [1, 2, 3], [1, 2, 3], True),
    ([1, 2, 3], [4, 5, 6], [1, 2, 3, 4, 5, 6], True),
    ([1, 2, 3], [2, 3, 4], [1, 3, 4], False),
    ([1, 2, 3, 4], [2, 3, 4, 5], [1, 2, 4, 5], False),
    ([1, 2, 3], [2, 3, 4], [], False),
    ([1, 2, 3], [2, 3, 4], [2, 4], False),
    ([1], [1], [1], True),
    ([], [], [], True),
    (list(range(1, 101)), list(range(50, 151)), list(range(1, 201)), True),
    ([1, 1, 2, 2, 3, 3], [2, 2, 3, 3, 4, 4], [1, 2, 3, 4], True),
    ([-3, -2, -1, 0], [-2, -1, 0, 1], [-3, -2, -1, 0, 1], True),
]


@pytest.mark.parametrize("a,b,want", OVERLAP_KATS)
def test_label_overlap_truth_table(a, b, want):
    assert oracle.labels_overlap(a, b) is want
    assert oracle.labels_overlap(b, a) is want
    assert pyref.overlaps(a, b) is want


@pytest.mark.parametrize("a,b,c,want", INTERSECTION_KATS)
def test_label_contains_intersection_truth_table(a, b, c, want):
    a, b, c = (oracle.labels_normalize(x) for x in (a, b, c))      # LabelSet::from: sort + dedup
    assert oracle.labels_contains_intersection(c, a, b) is want
    assert oracle.labels_contains_intersection(c, b, a) is want


def test_label_normalize_sorts_and_dedups():
    assert list(oracle.labels_normalize([5, -1, 5, 3, 3, 0])) == [-1, 0, 3, 5]


# ---- Rust BinaryHeap clone ---------------------------------------------------------------
def test_binary_heap_hand_traced_tie_order():
    # push 5 equal keys then pop all: sift_up never moves an equal element, pop swaps the last
    # element to the root and walks it to the bottom preferring the RIGHT child on ties.
    #   data=[0,1,2,3,4]
    #   pop -> 0: last=4 takes the root, hole walks to child 2 (right on tie)   -> [2,1,4,3]
    #   pop -> 2: last=3 takes the root, children (1,4) tie -> right child (4)  -> [4,1,3]
    #   pop -> 4: last=3 takes the root, only child 1 moves up (child==end-1)   -> [1,3]
    #   pop -> 1: last=3 takes the root                                          -> [3]
    #   pop -> 3
    ops = [7, 7, 7, 7, 7, -1, -1, -1, -1, -1]
    assert list(oracle.binary_heap_script(ops)) == [0, 2, 4, 1, 3]
    # distinct keys: plain max-heap order
    ops = [3, 9, 1, 7, -1, -1, -1, -1]
    assert list(oracle.binary_heap_script(ops)) == [1, 3, 0, 2]


def test_binary_heap_matches_independent_python_clone():
    rng = np.random.default_rng(5)
    for trial in range(40):
        n = int(rng.integers(1, 400))
        ops = []
        live = 0
        for i in range(n):
            if live and rng.random() < 0.4:
                ops.append(-1)
                live -= 1
            else:
                ops.append(int(rng.integers(0, 6)))     # few distinct keys => many ties
                live += 1
        ops += [-1] * live
        h = pyref.RustBinaryHeap(lambda a, b: a[0] <= b[0])
        want = []
        for i, o in enumerate(ops):
            if o >= 0:
                h.push((o, i))
            else:
                want.append(h.pop()[1])
        assert list(oracle.binary_heap_script(ops)) == want


# ---- distances ---------------------------------------------------------------------------
def test_simd_order_vs_scalar_reference_tolerance():
    """distance_x86.rs:40-63: 2000-d normalised ramps, |simd - scalar| < 1e-6."""
    r = np.arange(2000, dtype=np.float32) + 1.0
    l = np.arange(2000, dtype=np.float32) + 2.0
    r = r / np.float32(np.sqrt(np.float32(np.sum(r * r, dtype=np.float32))))
    l = l / np.float32(np.sqrt(np.float32(np.sum(l * l, dtype=np.float32))))
    for kind in (COSINE, L2):
        for impl in ("emu", "avx2"):
            assert abs(oracle.distance(kind, r, l, impl) - oracle.distance(kind, r, l, "unoptimized")) < 1e-6


@pytest.mark.parametrize("n", [1, 7, 31, 32, 33, 64, 100, 768, 1536, 2000])
def test_scalar_emulation_equals_real_avx2_bits(n):
    rng = np.random.default_rng(n)
    for _ in range(20):
        x = rng.standard_normal(n).astype(np.float32)
        y = rng.standard_normal(n).astype(np.float32)
        for kind in (COSINE, L2, IP):
            a = np.float32(oracle.distance(kind, x, y, "emu"))
            b = np.float32(oracle.distance(kind, x, y, "avx2"))
            assert a.view(np.uint32) == b.view(np.uint32)
    x = rng.standard_normal(n).astype(np.float32)
    y = rng.standard_normal(n).astype(np.float32)
    for kind in (COSINE, L2, IP):
        assert np.float32(pyref.distance(kind, x, y)).view(np.uint32) == \
            np.float32(oracle.distance(kind, x, y, "emu")).view(np.uint32)


def test_preprocess_cosine_edge_cases():
    z = np.zeros(16, np.float32)
    assert np.array_equal(oracle.preprocess_cosine(z), z)               # zero vector untouched
    u = np.zeros(16, np.float32)
    u[3] = 1.0
    assert np.array_equal(oracle.preprocess_cosine(u), u)               # already unit: untouched
    v = np.arange(1, 17, dtype=np.float32)
    w = oracle.preprocess_cosine(v)
    assert np.array_equal(w, pyref.preprocess_cosine(v))
    assert np.array_equal(oracle.preprocess_cosine(w), w)               # idempotent (debug_assert in the reference)


# ---- quantizer -----------------------------------------------------------------------------
def test_quantizer_layout_and_buckets():
    assert oracle.code_words(768, 2) == 24 and oracle.code_words(768, 1) == 12
    assert oracle.code_words(100, 1) == 2 and oracle.code_words(3, 2) == 1
    mean = np.zeros(4, np.float32)
    m2 = np.full(4, 4.0, np.float32)                   # count 4 => variance 1, std 1
    # z = -3 -> idx<1 -> 00 ; z = -0.5 -> idx 1.125 -> 1 one ; z = 1 -> idx 2.25 -> 2 ones ; z=5 -> min(5,2)
    v = np.array([-3.0, -0.5, 1.0, 5.0], np.float32)
    code = oracle.quantize(v, 2, mean, m2, 4)
    assert int(code[0]) == (0b00) | (0b01 << 2) | (0b11 << 4) | (0b11 << 6)
    # 1 bit: strictly greater than the mean
    code = oracle.quantize(np.array([0.0, 1e-9, -1.0, 2.0], np.float32), 1, mean, m2, 4)
    assert int(code[0]) == 0b1010
    # index built on an empty table: count = 0 => std = NaN => every bucket is 0 (build.rs:1419-1433)
    code = oracle.quantize(v, 2, mean, np.zeros(4, np.float32), 0)
    assert int(code[0]) == 0


def test_quantizer_matches_python_restatement():
    rng = np.random.default_rng(2)
    data = rng.standard_normal((50, 70)).astype(np.float32)
    for bits in (1, 2, 3):
        mean, m2, count = oracle.train(data, bits)
        for i in range(5):
            a = oracle.quantize(data[i], bits, mean, m2, count)
            b = pyref.quantize(data[i], bits, mean, m2, count, len(a))
            assert [int(x) for x in a] == b


# ---- values the uniform / Gaussian fixtures never produce (tests/test_zz_p_values_gpu.py) -----------------------------
def _bits(x):
    return int(np.float32(x).view(np.uint32))


def _value_cases():
    """(name, kind, x, y, expected bits or a predicate) at a tail-only, a body + tail and a body-only length."""
    f = np.float32
    out = []
    for n in (7, 40, 96):
        z = np.zeros(n, f)
        x, y = z.copy(), z.copy()
        # x86: inf + -inf = 0xFFC00000, and the inner product's `-dist` flips it to 0x7FC00000
        x[0] = y[0] = x[1] = f(3e38)
        y[1] = f(-3e38)
        if n >= 32:
            x[1] = y[1] = 0.0
            x[8] = y[0] = x[0] = f(3e38)
            y[8] = f(-3e38)
        out += [("nan", IP, x, y, 0x7FC00000), ("nan-cos", COSINE, x, y, 0)]
        x, y = z.copy(), z.copy()
        x[0], y[0], x[n - 1], y[n - 1] = f(3e38), f(3e38), f(-3e38), f(-3e38)
        out += [("inf", IP, x, y, 0xFF800000), ("inf-l2", L2, x, -y, 0x7F800000), ("equal-l2", L2, x, x, 0)]
        x = np.full(n, f(1e-20))
        h = np.full(n, f(5e-21))
        out += [("subnormal-ip", IP, x, x, lambda b: 0x80000000 < b < 0x80800000),
                ("subnormal-l2", L2, h, -h, lambda b: 0 < b < 0x00800000),
                ("denormal-in", IP, np.full(n, f(1e-40)), np.full(n, f(0.5)), lambda b: 0x80000000 < b < 0x80800000)]
        x, y = z.copy(), z.copy()
        x[0], y[n - 1] = 1.0, -1.0
        out += [("orthogonal-ip", IP, x, y, 0x80000000), ("orthogonal-cos", COSINE, x, y, _bits(1.0)),
                ("neg-zeros-ip", IP, np.full(n, f(-0.0)), z, 0x80000000), ("self-cos", COSINE, x, x, 0)]
    return out


@pytest.mark.parametrize("case", range(len(_value_cases())))
def test_distance_bits_on_nan_inf_subnormal_and_signed_zero_inputs(case):
    """The scalar restatement, the real AVX2 build and the Python restatement give the same bits, and the bits the
    x86 reference gives: NaN inner products 0x7FC00000, +-inf, subnormal sums kept, -0.0 for an exactly zero product."""
    name, kind, x, y, want = _value_cases()[case]
    with np.errstate(all="ignore"):
        got = {impl: _bits(oracle.distance(kind, x, y, impl)) for impl in ("emu", "avx2")}
        got["pyref"] = _bits(pyref.distance(kind, x, y))
    assert len(set(got.values())) == 1, (name, {k: hex(v) for k, v in got.items()})
    b = got["avx2"]
    assert want(b) if callable(want) else b == want, (name, len(x), hex(b))


def test_preprocess_cosine_of_overflowing_and_subnormal_rows():
    """A norm that overflows divides every component by +inf: the row becomes signed zeros.  A norm below f32::EPSILON
    (subnormal or underflowed to zero) leaves the row untouched."""
    f = np.float32
    rows = {"3e38": np.array([3e38, 1.0, -2.0, 0.5, -0.0], f), "1e20": np.full(40, f(1e20)),
            "-1e20": np.full(40, f(-1e20)), "1e-40": np.array([1e-40, -1e-40, 0.0, -0.0, 3e-39], f),
            "1e-20": np.full(40, f(1e-20))}
    for name, v in rows.items():
        with np.errstate(all="ignore"):
            a, b = oracle.preprocess_cosine(v), pyref.preprocess_cosine(v)
        assert np.array_equal(a.view(np.uint32), b.view(np.uint32)), name
        if name.endswith("e20") or name == "3e38":
            assert not a.any() and np.array_equal(np.signbit(a), np.signbit(v)), name
        else:
            assert np.array_equal(a.view(np.uint32), v.view(np.uint32)), name


def test_quantizer_edges_match_python_restatement():
    """Constant columns (m2 = 0: z = +-inf, or NaN at the mean), +-0 means, count 0 / 1 / 2^24 + 3 / 2^53 + 1, query
    components on every bucket edge and its nextafter neighbours: the fixtures of tests/test_zz_p_values_gpu.py."""
    from test_zz_p_values_gpu import COUNTS, quantizer_case
    for count in COUNTS:
        for bits in (1, 2, 3, 4):
            s, q, _, _ = quantizer_case(count, bits)
            for r in q:
                with np.errstate(all="ignore"):
                    want = pyref.quantize(r, bits, s.mean, s.m2, count, s.words)
                assert [int(x) for x in oracle.quantize(r, bits, s.mean, s.m2, count)] == want, (count, bits)
    # hand-worked: count 0 (std = +inf, z = 0, index = ranges / 2), a constant column, `count as f32` to nearest
    one = np.ones(1, np.float32)
    assert int(oracle.quantize(np.array([5.0], np.float32), 3, 0 * one, one, 0)[0]) == 0b011       # index 2.0
    assert int(oracle.quantize(np.array([5.0], np.float32), 2, 0 * one, one, 0)[0]) == 0b01        # index 1.5
    assert [int(oracle.quantize(np.array([v], np.float32), 4, one, 0 * one, 7)[0]) for v in (2.0, 1.0, 0.0)] == \
        [0b1111, 0, 0]
    # count 2^24 + 3 converts to 2^24 + 4 = m2: variance 1, z = 1, index (1 + 2) / (4 / 3) = 2.2499998 -> 2 ones
    m2 = np.array([16777220.0], np.float32)
    assert int(oracle.quantize(np.array([1.0], np.float32), 2, 0 * one, m2, (1 << 24) + 3)[0]) == 0b11


@pytest.mark.parametrize("bits", [3, 4, 5, 7, 8, 16, 31, 32])
def test_quantizer_wide_bits_match_python_restatement(bits):
    """3 to 32 bits per dimension, trained on data, at 13 dimensions (a dimension's bits straddle a word unless
    64 % bits == 0), rows far past the last edge included."""
    rng = np.random.default_rng(bits)
    data = rng.standard_normal((60, 13)).astype(np.float32)
    mean, m2, count = oracle.train(data, bits)
    rows = np.concatenate([data[:10], 4 * data[10:12], np.zeros((1, 13), np.float32)])
    full = 0
    for r in rows:
        a = oracle.quantize(r, bits, mean, m2, count)
        assert [int(x) for x in a] == pyref.quantize(r, bits, mean, m2, count, len(a))
        full += sum(bin(int(w)).count("1") for w in a)
    assert full > 13 * bits


@pytest.mark.parametrize("family", ["duplicates", "overflow"])
def test_cpp_oracle_equals_python_restatement_on_ties_and_overflow(family):
    """Whole scans on 160 rows drawn from 9 distinct vectors (cosine, L2: zero distances and runs of equal exact
    distances in the rerank window) and on rows with +-3e38 components (inner product: +-inf and NaN distances)."""
    from test_zz_p_values_gpu import duplicate_rows, overflow_rows, trained_index
    if family == "duplicates":
        v, q = duplicate_rows(160, 24, 9, 5, "normal")
        cases = [(trained_index(v, COSINE, 2, R=12, L_build=24), q[[0, 1, 13, 24]]),
                 (trained_index(v, L2, 1, R=12, L_build=24), q[[2, 14, 24]])]
    else:
        v, q = overflow_rows(160, 40, 7)
        cases = [(trained_index(v, IP, 2, R=12, L_build=24), q[[0, 8, 10, 16]]),
                 (trained_index(v, L2, 2, R=12, L_build=24), q[[1, 9, 11]])]
    special = 0
    for s, qs in cases:
        for qi in qs:
            for (L, rescore, rows) in ((20, 10, 15), (40, 60, 30)):
                with np.errstate(all="ignore"):
                    a = oracle.scan(s, qi, None, L, rescore, rows)
                    b_rows, b_stats = pyref.scan(s, qi, None, L, rescore, rows)
                assert a["tid"].tolist() == [r[0] for r in b_rows]
                assert a["node"].tolist() == [r[1] for r in b_rows]
                assert a["dist"].view(np.uint32).tolist() == \
                    np.array([r[2] for r in b_rows], np.float32).view(np.uint32).tolist()
                assert a["stats"] == b_stats
                d = a["dist"]
                special += int((d == 0).sum() + (d[1:] == d[:-1]).sum()) if family == "duplicates" else \
                    int(np.isnan(d).sum() + np.isinf(d).sum())
    assert special > 20, special


# ---- reference SQL KATs restated (index created BEFORE the inserts => zero means) -----------
def _three_vector_index(dist):
    v = np.array([[1, 1, 1], [2, 2, 2], [3, 3, 3]], np.float32)
    return fixtures.make_index(v, dist, R=10, L_build=10, train_on_data=False), v


def _top1(s, v, q, rescore=50):
    r = oracle.scan(s, np.asarray(q, np.float32), None, 100, rescore, 1)
    return v[r["node"][0]].tolist()


def test_l2_sanity_check_kat():        # build.rs:1475-1516
    s, v = _three_vector_index(L2)
    for q in ([1, 1, 1], [2, 2, 2], [3, 3, 3]):
        assert _top1(s, v, q) == q


def test_ip_sanity_check_kat():        # build.rs:1518-1556
    s, v = _three_vector_index(IP)
    for q in ([1, 1, 1], [2, 2, 2], [3, 3, 3]):
        assert _top1(s, v, q) == [3, 3, 3]


def test_no_rescore_kat():             # build.rs:1419-1473
    v = np.array([[1, 1, 1], [2, 2, 2]], np.float32)
    s = fixtures.make_index(v, L2, train_on_data=False)
    assert not s.codes.any()           # SBQ cannot tell the two rows apart
    wrong_a = _top1(s, v, [1, 1, 1], rescore=0) != [1, 1, 1]
    wrong_b = _top1(s, v, [2, 2, 2], rescore=0) != [2, 2, 2]
    assert wrong_a or wrong_b
    assert _top1(s, v, [1, 1, 1], rescore=2) == [1, 1, 1]
    assert _top1(s, v, [2, 2, 2], rescore=2) == [2, 2, 2]


def test_null_query_returns_all_rows():    # build.rs:2016-2044
    s = build_case(300, 48, COSINE, seed=3, kind="uniform", R=20, L_build=40)
    r = oracle.scan(s, None, None, 100, 50, 1000)
    assert len(r["tid"]) == 300 and len(set(r["tid"].tolist())) == 300


def test_recall_scaffold_property():       # build.rs:1311-1396: > 9 of 10 at L=25 on 300 vectors
    s = build_case(300, 1536, L2, seed=4, kind="uniform")
    q = np.ones(1536, np.float32)
    r = oracle.scan(s, q, None, 25, 50, 10)
    truth = np.argsort(((s.vectors - q) ** 2).sum(1), kind="stable")[:10]
    assert len(set(r["node"].tolist()) & set(truth.tolist())) > 9 - 1   # reference asserts > 9 with pg's RNG; >= 9 here


def test_labeled_recall_property():        # labels/filtering_tests.rs:880-1024: recall >= 0.9
    s = build_case(1000, 128, L2, seed=6, kind="uniform", labels=True)
    rng = np.random.default_rng(0)
    hits = tot = 0
    for t in range(20):
        q = rng.random(128, dtype=np.float32)
        lab = [int(rng.integers(1, 17))]
        r = oracle.scan(s, q, lab, 100, 50, 10)
        ok = np.array([oracle.labels_overlap(lab, s.labels[s.label_off[i]:s.label_off[i + 1]]) for i in range(s.n)])
        d = ((s.vectors - q) ** 2).sum(1)
        d[~ok] = np.inf
        truth = np.argsort(d, kind="stable")[:10]
        hits += len(set(r["node"].tolist()) & set(truth.tolist()))
        tot += 10
        assert all(ok[n] for n in r["node"])       # every returned row satisfies `labels && ARRAY[l]`
    assert hits / tot >= 0.9


def _null_and_empty_labels_index():
    """labels/filtering_tests.rs:23-110 as data: `CREATE INDEX ... USING diskann (embedding, labels)` on the empty table
    (zero-mean quantizer), then four rows: {1,2}, NULL, {}, {1,NULL,3} (NULL array = no labels, NULL element dropped,
    labels/mod.rs:209-238)."""
    v = np.array([[1, 2, 3], [4, 5, 6], [7, 8, 9], [10, 11, 12]], np.float32)
    sets = [[1, 2], [], [], [1, 3]]
    off = np.zeros(5, np.uint32)
    off[1:] = np.cumsum([len(x) for x in sets])
    lab = np.array([x for st in sets for x in st], np.int16)
    return fixtures.make_index(v, COSINE, R=10, L_build=10, label_off=off, labels=lab, train_on_data=False)


@pytest.mark.parametrize("key,want", [([1], 2), ([], 0), ([3], 1), (None, 4)])
def test_null_and_empty_labels_kat(key, want):     # labels/filtering_tests.rs:23-110
    s = _null_and_empty_labels_index()
    r = oracle.scan(s, np.zeros(3, np.float32), key, 100, 50, 100)
    assert len(r["tid"]) == want
    b_rows, _ = pyref.scan(s, np.zeros(3, np.float32), key, 100, 50, 100)
    assert [x[0] for x in b_rows] == r["tid"].tolist()


def test_mixed_filtering_with_null_labels_kat():    # labels/filtering_tests.rs:170-213 (the index part: `labels && '{1}'`)
    v = np.array([[1, 2, 3], [4, 5, 6], [7, 8, 9], [10, 11, 12], [13, 14, 15], [16, 17, 18]], np.float32)
    sets = [[1, 2], [], [], [1, 3], [2, 3], []]          # NULL, {} and {NULL} all carry no label
    off = np.zeros(7, np.uint32)
    off[1:] = np.cumsum([len(x) for x in sets])
    lab = np.array([x for st in sets for x in st], np.int16)
    s = fixtures.make_index(v, COSINE, R=10, L_build=10, label_off=off, labels=lab, train_on_data=False)
    r = oracle.scan(s, np.zeros(3, np.float32), [1], 100, 50, 100)
    assert sorted(r["node"].tolist()) == [0, 3]      # the executor's `category = 'blog'` then keeps row 3 only: count 1


@pytest.mark.parametrize("train_on_data", [True, False])
def test_small_accuracy_connectivity_property(train_on_data):
    """build.rs:1717-1853 (test_index_small_accuracy / ..._insert_after_index_created): 1000 random 2-d vectors,
    num_neighbors = 10, search_list_size = 10; with diskann.query_search_list_size = 2 an unbounded scan still returns
    every row - no node may get disconnected.  (Postgres' random() stream is not reproducible: our RNG, same property.)"""
    s = build_case(1000, 2, COSINE, seed=5, kind="uniform", R=10, L_build=10, train_on_data=train_on_data)
    r = oracle.scan(s, np.ones(2, np.float32), None, 2, 50, 5000)
    assert len(r["tid"]) == 1000 and len(set(r["tid"].tolist())) == 1000


# ---- the model of the batched builder is the serial restatement when nothing departs from it ----
@pytest.mark.parametrize("n,dim,kind,labels,R,L", [
    (1, 8, "normal", False, 4, 4), (2, 8, "normal", True, 4, 4), (400, 16, "normal", False, 10, 20),
    (600, 2, "uniform", False, 10, 10),      # tie-heavy: the stable sort by DistanceWithTieBreak, the tie factor
    (400, 24, "normal", True, 8, 20),        # both passes of a labeled insert, contains_intersection
    (300, 40, "normal", False, 50, 100)])    # max_neighbors_during_build = 65: lists longer than 64
def test_batched_build_model_with_no_switch_and_batches_of_one_is_the_serial_build(n, dim, kind, labels, R, L):
    """oracle.build_graph_batched runs orc_build's own prune / add_neighbors / search_for_build under the GPU builder's
    schedule (tests/test_zz_o_build_model_gpu.py compares dann_build_graph with it).  With every departure switched off
    and max_batch = 1 that schedule is the reference's serial insert: the neighbour arrays are identical."""
    s = build_case(n, dim, L2, seed=3, kind=kind, R=R, L_build=L, labels=labels)
    nb, counts = oracle.build_graph_batched(s.codes, R, L, 1.2, s.label_off if labels else None,
                                            s.labels if labels else None, max_batch=1)
    assert np.array_equal(nb, s.nbrs)
    assert n < 100 or (counts["back_pruned"] and counts["final_pruned"])
    if kind == "uniform":
        assert counts["tie_factor"] and counts["zero_occluded"]
    if labels and n > 100:
        assert counts["fwd_merged"] and counts["back_repeat"] and counts["label_skip"]


def test_batched_build_model_switches_each_change_the_graph():
    """Every named departure is live: switching it on alone moves at least one edge of a build that exercises it."""
    s = build_case(1500, 2, L2, seed=5, kind="uniform", R=10, L_build=10)
    s2 = build_case(1200, 32, L2, seed=11, kind="normal", R=16, L_build=150)
    for code, R, L in ((s.codes, 10, 10), (s2.codes, 16, 300)):
        base, _ = oracle.build_graph_batched(code, R, L, 1.2, max_batch=0)
        moved = {k: not np.array_equal(base, oracle.build_graph_batched(code, R, L, 1.2, max_batch=0, switches={k: v})[0])
                 for k, v in (("scan_ties", 1), ("order_by_id", 1), ("visited_cap", 256), ("cand_cap", 128),
                              ("back_src_cap", 64), ("slots", 12))}
        if L == 10:
            assert moved["scan_ties"] and moved["order_by_id"] and moved["slots"], moved
        else:
            assert moved["visited_cap"] and moved["cand_cap"], moved
    a = oracle.build_graph_batched(s2.codes, 16, 150, 1.2, max_batch=0, switches=dict(slots=64))[0]
    b = oracle.build_graph_batched(s2.codes, 16, 150, 1.2, max_batch=0, switches=dict(slots=64, fwd_keep_slots=1))[0]
    assert not np.array_equal(a, b)


# ---- the two restatements agree on whole scans ---------------------------------------------
@pytest.mark.parametrize("dist,bits,labels,dim_index", [(COSINE, 2, False, None), (L2, 1, False, None),
                                                        (IP, 2, True, None), (COSINE, 2, True, 40)])
def test_cpp_oracle_equals_python_restatement(dist, bits, labels, dim_index):
    s = build_case(400, 72, dist, bits=bits, seed=9 + dist, kind="normal", R=12, L_build=24,
                   labels=labels, dim_index=dim_index, deleted_every=7)
    q = fixtures.gen_vectors(6, 72, 33, "normal")
    for i in range(6):
        lab = None if not labels or i % 3 == 0 else [1 + i, 3]
        for (L, rescore, rows) in ((20, 10, 15), (5, 0, 30), (40, 60, 12)):
            a = oracle.scan(s, q[i], lab, L, rescore, rows)
            b_rows, b_stats = pyref.scan(s, q[i], lab, L, rescore, rows)
            assert a["tid"].tolist() == [r[0] for r in b_rows]
            assert a["node"].tolist() == [r[1] for r in b_rows]
            if rescore:
                assert a["dist"].view(np.uint32).tolist() == \
                    np.array([r[2] for r in b_rows], np.float32).view(np.uint32).tolist()
            assert a["stats"] == b_stats


# ---- plain storage layout (SURVEY §8f row 3: oracle groundwork, no CUDA path yet) ---------------
@pytest.mark.parametrize("dist,dim_index", [(COSINE, None), (L2, None), (COSINE, 40), (L2, 40)])
def test_plain_storage_scan_cpp_equals_python(dist, dim_index):
    s = fixtures.to_plain(build_case(300, 64, dist, seed=21 + dist, kind="normal", R=12, L_build=24,
                                     dim_index=dim_index, deleted_every=9))
    q = fixtures.gen_vectors(4, 64, 77, "normal")
    for i in range(4):
        for (L, rescore, rows) in ((20, 10, 15), (5, 0, 25), (30, 40, 12)):
            a = oracle.scan(s, q[i], None, L, rescore, rows)
            b_rows, b_stats = pyref.scan(s, q[i], None, L, rescore, rows)
            assert a["node"].tolist() == [r[1] for r in b_rows]
            assert a["stats"] == b_stats
            assert a["stats"]["d_quantized"] == 0
            resorts = rescore > 0 and s.dim != s.dim_index          # scan.rs:392-403
            if resorts:
                assert a["dist"].view(np.uint32).tolist() == \
                    np.array([r[2] for r in b_rows], np.float32).view(np.uint32).tolist()
                assert a["stats"]["d_full"] > a["stats"]["candidates"]
            else:
                assert a["stats"]["d_full"] == a["stats"]["candidates"]  # every comparison is a full distance


def test_plain_storage_l2_sanity_kat():       # build.rs:1475-1516 run with storage_layout = plain (plain/tests.rs)
    s, v = _three_vector_index(L2)
    p = fixtures.to_plain(s)
    for q in ([1, 1, 1], [2, 2, 2], [3, 3, 3]):
        assert _top1(p, v, q, rescore=0) == q   # exact distances: no rescore needed, unlike the SBQ layout


def test_plain_storage_exact_order_on_full_graph_walk():
    s = fixtures.to_plain(build_case(200, 32, L2, seed=5, kind="normal", R=16, L_build=40))
    q = fixtures.gen_vectors(1, 32, 6, "normal")[0]
    r = oracle.scan(s, q, None, 400, 0, 200)     # L >= n: the stream is the exact order of every reachable node
    d = np.array([oracle.distance(L2, q, s.index_vectors[n]) for n in r["node"]], np.float32)
    assert len(r["node"]) == 200 and np.all(np.diff(d) >= 0)


# ---- committed golden vectors -----------------------------------------------------------------
def test_golden_vectors():
    path = os.path.join(os.path.dirname(__file__), "golden", "scan_golden.npz")
    z = np.load(path)
    from golden.make_golden import CASES, run_case
    for name in CASES:
        got = run_case(name)
        for key, val in got.items():
            assert np.array_equal(z[f"{name}/{key}"], val), (name, key)


def test_march_native_build_of_the_oracle_returns_the_same_rows():
    """bench.py's optional CPU arm (BASELINE.md §3) times oracle.cpp built with -march=native; it is never used for
    parity, but it must still be the same algorithm: rows, distance bits and counters equal the reference-flag build."""
    from conftest import build_case
    from oracle import fixtures, oracle
    from pgvectorscale_b200.snapshot import COSINE
    s = build_case(1200, 96, COSINE, seed=14, R=24, L_build=48, labels=True, deleted_every=7)
    q = fixtures.gen_vectors(12, 96, 4, "normal")
    a = oracle.scan_batch(s, q, None, None, 40, 30, 10, threads=2)
    b = oracle.scan_batch(s, q, None, None, 40, 30, 10, threads=2, native=True)
    assert np.array_equal(a[0], b[0]) and np.array_equal(a[1].view(np.uint32), b[1].view(np.uint32))
    assert np.array_equal(a[2], b[2]) and np.array_equal(a[3], b[3])
