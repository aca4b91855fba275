"""The scan path against the oracle on the VALUES that uniform and Gaussian fixtures never produce.

The other parity files pin the kernels across shapes with `oracle.fixtures.gen_vectors` data: uniform [0, 1) or unit
Gaussian rows quantized at 1 or 2 bits per dimension.  Here the rows and queries are made by hand so that they reach
the value-dependent branches of the path:

  family      | rows                                          | what it reaches
  quantizer   | quantizer set directly: constant columns      | sbq_count_ones branch by branch (1 bit: strict `>`;
              | (m2 = 0), means of +0.0 and -0.0, count 0, 1, | `index < 1.0`; the floor and the `bits` cap; z = +-inf
              | 2^24 + 3 and 2^53 + 1; queries at the mean,   | and NaN) and `count as f32` (__ull2float_rn: 2^24 + 3
              | on every bucket boundary of 2, 3 and 4 bits   | rounds to 2^24 + 4, toward zero it would be 2^24 + 2)
              | and on their nextafter neighbours             |
  multi-bit   | 3, 4, 5, 8, 16 and 32 bits per dimension;     | the prepare kernel's multi-bit packing (a dimension's
              | 40 x 3 and 13 x 5 (bits straddle a word),     | bits across two 64-bit words), wider codes at one dim
              | 7 x 32, up to 768 x 8                         |
  overflow    | 10 % of components at +-3e38; whole rows of   | +inf L2 distances and their ties, NaN and +-inf inner
              | 1e20 (finite, the norm overflows)             | products, cosine rows and queries normalised to zeros
  tiny        | +-1e-40, -0.0, +0.0; rows of tiny components; | subnormal arithmetic (whole distances subnormal), the
              | all-zero rows; one-hot rows                   | cosine `norm < eps` branch, -0.0 inner products
  duplicates  | 2000 rows drawn from 37 distinct vectors, at  | zero distances, the cosine (1 - ip).max(0) clamp, runs
              | 96-d and 768 x 2 (the benchmark's NCH = 3)    | of equal keys in both heaps and the rerank window

Every family runs through search_batch on the two-warp kernel (the default at small batches), the lean kernel
(DANN_SEARCH_KERNEL=3) with both inserted-sets and both entry widths where the code allows, and the single-warp kernel
(DANN_SEARCH_KERNEL=1); the plan of every call is read back.  The quantizer, multi-bit and overflow families also
compare the stand-alone prepare_queries (q_full bits, codes) and full_distance (distance bits).  The overflow, tiny
and duplicate families also run search_batch_device, the streaming scan drained to the end with the counters after
every row, gettuple_many over a mix of scans, and (cosine and L2) the plain layout.

Bar, as in test_gpu_parity.py: bit-exact TIDs, bit-exact rerank distances (u32), counts, all five counters, status 0.
Every case also asserts, from the fixture or the oracle's output, that its degeneracy happened: an m2 = 0 column, a
query component on a bucket boundary and at the mean, NaN and +-inf rows, a subnormal distance, a -0.0 distance, tied
rerank rows.  Without that a case could pass without testing anything.

The parity target is the reference's x86 build: a NaN inner product there is `-(0xFFC00000)` = 0x7FC00000, which the
GPU's float unit would canonicalise to 0x7FFFFFFF without the mapping in full_distance_group8.

Every test here also runs under the CPU SIMT emulator (DANN_EMULATE=1, tests/test_zz_p_values_emulated.py); that run
has x86 arithmetic, so it can see neither the NaN bits nor a flush of subnormals to zero."""
import functools

import numpy as np
import pytest

from conftest import buffer_device, dptr, emulating
from test_gpu_parity import COSINE, IP, L2

pytestmark = pytest.mark.gpu

F = np.float32
HOOKS = ("DANN_SEARCH_KERNEL", "DANN_SEARCH_WARPS", "DANN_SEARCH_HS", "DANN_SEARCH_BITMAP", "DANN_SEARCH_ENTRY",
         "DANN_DEBUG_SHRINK")
FIELDS = ("visits", "d_quantized", "candidates", "d_full", "stream_len")
FLT_MIN = F(1.17549435e-38)
NEG_ZERO_BITS = 0x80000000


@pytest.fixture(scope="module")
def lib(lib_built):
    from pgvectorscale_b200 import diskann
    if diskann.device_count() < 1:
        pytest.fail("no CUDA device visible: -m gpu tests need an H100")
    return diskann


@pytest.fixture
def env(monkeypatch):
    """env(KERNEL=3, BITMAP=0, ...) sets exactly these DANN_SEARCH_* hooks and clears the others."""
    def set_(**kv):
        for h in HOOKS:
            monkeypatch.delenv(h, raising=False)
        for key, val in kv.items():
            monkeypatch.setenv("DANN_SEARCH_" + key, str(val))
    set_()
    return set_


# ---- index construction ----------------------------------------------------------------------------------------------

def index_with_quantizer(v, dist, bits, mean, m2, count, R=16, L_build=32):
    """What CREATE INDEX leaves behind for rows `v`, with the SBQ quantizer (mean, m2, count) given instead of trained:
    rows cosine-normalised for the build, quantized by the oracle, serial Vamana over the codes."""
    from oracle import oracle
    from pgvectorscale_b200.snapshot import Snapshot, code_words, make_heap_tids
    v = np.ascontiguousarray(v, F)
    n, dim = v.shape
    iv = np.array([oracle.preprocess_cosine(r) for r in v], F) if dist == COSINE else v.copy()
    mean, m2 = np.ascontiguousarray(mean, F), np.ascontiguousarray(m2, F)
    codes = oracle.quantize_all(iv, bits, mean, m2, count)
    nbrs, sd, _, _ = oracle.build_graph(codes, R, L_build, 1.2)
    return Snapshot(n=n, dim=dim, dim_index=dim, bits=bits, words=code_words(dim, bits), R=R, distance_type=dist,
                    has_labels=False, count=count, mean=mean, m2=m2, codes=codes, nbrs=nbrs, heap_tid=make_heap_tids(n),
                    vectors=v, start_default=sd)


def trained_index(v, dist, bits, R=16, L_build=32):
    from oracle import fixtures
    return fixtures.make_index(np.ascontiguousarray(v, F), dist, bits=bits, R=R, L_build=L_build)


# ---- the quantizer in f32, one operation at a time (sbq/quantize.rs:52-102) -----------------------------------------

def bucket_index(v, mean, m2, count_f, bits):
    """`(z + 2.0) / (4.0 / ranges)` with z = (v - mean) / sqrt(m2 / count_f), every step rounded to f32."""
    with np.errstate(all="ignore"):
        std = np.sqrt(F(m2) / F(count_f), dtype=F)
        z = (np.asarray(v, F) - F(mean)) / std
        return (z + F(2.0)) / (F(4.0) / F(bits + 1))


def boundary_values(mean, m2, count_f, bits, k, reach=256):
    """Per dimension, the f32 value nearest the k-th bucket edge whose bucket index is exactly k (1 <= k <= bits), or
    NaN where none lies within `reach` ulps: the `index < 1.0` test at k = 1, the floor above."""
    mean, m2 = np.asarray(mean, F), np.asarray(m2, F)
    with np.errstate(all="ignore"):
        std = np.sqrt(m2.astype(np.float64) / float(F(count_f)))
        v0 = (mean.astype(np.float64) + (k * 4.0 / (bits + 1) - 2.0) * std).astype(F)
    cols, up, down = [v0], v0, v0
    for _ in range(reach):
        up, down = np.nextafter(up, F(np.inf)), np.nextafter(down, F(-np.inf))
        cols += [up, down]
    c = np.stack(cols, 1)
    hit = bucket_index(c, mean[:, None], m2[:, None], count_f, bits) == F(k)
    out = c[np.arange(len(mean)), hit.argmax(1)]
    out[~hit.any(1)] = np.nan
    return out


def code_ones(code, dim, bits):
    """The number of ones of each dimension of one SBQ code."""
    bitv = [(int(code[p // 64]) >> (p % 64)) & 1 for p in range(dim * bits)]
    return np.array([sum(bitv[i * bits:(i + 1) * bits]) for i in range(dim)])


# ---- comparison with the oracle ---------------------------------------------------------------------------------------

def oracle_batch(s, q, k, L, rescore):
    from oracle import oracle
    return oracle.scan_batch(s, q, None, None, L, rescore, k, threads=0)


def compare(g, ref, rescore, with_dist=True):
    otid, odist, ocount, ostats = ref
    assert np.array_equal(g["count"], ocount)
    assert np.array_equal(g["tid"], otid), "row ids differ from the oracle"
    if rescore > 0 and with_dist:
        bad = np.argwhere(g["dist"].view(np.uint32) != odist.view(np.uint32))
        assert not len(bad), [(int(b), int(i), hex(int(g["dist"][b, i].view(np.uint32))),
                               hex(int(odist[b, i].view(np.uint32)))) for b, i in bad[:6]]
    for f in FIELDS:
        assert np.array_equal(g["stats"][f].astype(np.uint64), ostats[f]), f
    assert not g["stats"]["status"].any()


def plans(words):
    """(hooks, kernel, entry bytes, inserted-set) of every kernel a batch can be sent to: the default (two-warp at
    this batch size), the lean kernel with the bitmap and the hash set at its natural entry and, where that is 4
    bytes, at 8 bytes too, and the single-warp kernel."""
    natural = 4 if words * 64 < 2048 else 8
    out = [({}, 2, None, None), ({"KERNEL": 1}, 1, None, None)]
    for bitmap in (1, 0):
        out.append(({"KERNEL": 3, "BITMAP": bitmap}, 3, natural, bitmap))
        if natural == 4:
            out.append(({"KERNEL": 3, "BITMAP": bitmap, "ENTRY": 2}, 3, 8, bitmap))
    return out


RUNS = ((10, 40, 20), (30, 60, 60), (10, 30, 0))


def every_kernel(env, idx, s, q, runs=RUNS):
    """Each (k, L, rescore) of `runs` on every plan, against one oracle batch; -> the oracle's output per run."""
    refs = {}
    for k, L, rescore in runs:
        refs[(k, L, rescore)] = ref = oracle_batch(s, q, k, L, rescore)
        for hooks, kernel, entry, bitmap in plans(s.words):
            env(**hooks)
            g = idx.search_batch(q, k=k, search_list_size=L, rescore=rescore)
            compare(g, ref, rescore)
            p = idx.last_search_plan()
            assert p["kernel"] == kernel, (hooks, p)
            if entry is not None:
                assert p["entry_bytes"] == entry, (hooks, p)
            if bitmap is not None:
                assert p["bitmap"] == bitmap, (hooks, p)
    env()
    return refs


def prepare_and_full_distance(idx, s, q, seed):
    """prepare_queries: q_full bits against preprocess_cosine, codes against oracle.quantize; full_distance bits
    against oracle.distance(.., "avx2") for 48 rows per query.  -> the oracle's distances [B, 48]"""
    import torch
    from oracle import oracle
    dev = buffer_device()
    B, dim, m = q.shape[0], s.dim, min(48, s.n)
    d_q = torch.from_numpy(np.ascontiguousarray(q)).to(dev)
    d_full = torch.empty((B, dim), dtype=torch.float32, device=dev)
    d_codes = torch.empty((B, idx.code_stride), dtype=torch.int64, device=dev)
    idx.prepare_queries(dptr(d_q), dptr(d_full), dptr(d_codes))
    if not emulating():
        torch.cuda.synchronize()
    full = d_full.cpu().numpy()
    codes = d_codes.cpu().numpy().view(np.uint64)
    for b in range(B):
        qf = oracle.preprocess_cosine(q[b]) if s.distance_type == COSINE else q[b]
        assert np.array_equal(full[b].view(np.uint32), qf.view(np.uint32)), b
        want = oracle.quantize(qf, s.bits, s.mean, s.m2, s.count)
        assert np.array_equal(codes[b, :s.words], want), (b, codes[b, :s.words], want)
        assert not codes[b, s.words:].any()
    rng = np.random.default_rng(seed)
    nodes = np.stack([rng.permutation(s.n)[:m] for _ in range(B)]).astype(np.uint32)
    d_nodes = torch.from_numpy(nodes.view(np.int32)).to(dev)
    d_out = torch.empty((B, m), dtype=torch.float32, device=dev)
    idx.full_distance(dptr(d_full), dptr(d_nodes), dptr(d_out))
    if not emulating():
        torch.cuda.synchronize()
    out = d_out.cpu().numpy()
    ref = np.zeros((B, m), F)
    for b in range(B):
        for i in range(m):
            x = s.vectors[nodes[b, i]]
            if s.distance_type == COSINE:
                x = oracle.preprocess_cosine(x)
            ref[b, i] = oracle.distance(s.distance_type, x, full[b], "avx2")
    bad = np.argwhere(out.view(np.uint32) != ref.view(np.uint32))
    assert not len(bad), [(int(b), int(i), hex(int(out[b, i].view(np.uint32))), hex(int(ref[b, i].view(np.uint32))))
                          for b, i in bad[:6]]
    return ref


def device_entry_point(idx, s, q, k, L, rescore):
    """search_batch_device (buffers in HBM, the caller's stream) against the oracle."""
    import torch
    B = q.shape[0]
    dev = buffer_device()
    d_q = torch.from_numpy(np.ascontiguousarray(q)).to(dev)
    d_tid = torch.empty((B, k), dtype=torch.int64, device=dev)
    d_dist = torch.empty((B, k), dtype=torch.float32, device=dev)
    d_cnt = torch.empty(B, dtype=torch.int32, device=dev)
    d_st = torch.empty((B, 6), dtype=torch.int32, device=dev)
    if emulating():
        idx.search_batch_device(dptr(d_q), k, L, rescore, dptr(d_tid), dptr(d_dist), dptr(d_cnt), dptr(d_st))
    else:
        side = torch.cuda.Stream(device=dev)
        with torch.cuda.stream(side):
            idx.search_batch_device(d_q, k, L, rescore, d_tid, d_dist, d_cnt, d_st, stream=side.cuda_stream)
        side.synchronize()
    st = d_st.cpu().numpy().view(np.uint32)
    stats = np.zeros(B, [(f, "<u4") for f in FIELDS + ("status",)])
    for j, f in enumerate(FIELDS + ("status",)):
        stats[f] = st[:, j]
    g = dict(tid=d_tid.cpu().numpy().view(np.uint64), dist=d_dist.cpu().numpy(),
             count=d_cnt.cpu().numpy().view(np.uint32), stats=stats)
    compare(g, oracle_batch(s, q, k, L, rescore), rescore)


def scan_check(s, sc, q, L, rescore, i, row, with_dist=True):
    """The i-th row of a streaming scan and its counters against the oracle's scan of i rows; -> False at the end."""
    from oracle import oracle
    ref = oracle.scan(s, q, None, L, rescore, i)
    if len(ref["tid"]) < i:
        assert row is None, i
        return False
    assert row is not None, i
    assert ((row[0] << 16) | row[1]) == int(ref["tid"][-1]) and row[2] == int(ref["node"][-1]), i
    if rescore and with_dist:
        assert np.float32(row[3]).view(np.uint32) == ref["dist"][-1].view(np.uint32), \
            (i, hex(int(np.float32(row[3]).view(np.uint32))), hex(int(ref["dist"][-1].view(np.uint32))))
    st = sc.stats()
    for f in FIELDS:
        assert st[f] == ref["stats"][f], (f, i)
    return True


def drain(idx, s, q, L, rescore, with_dist=True):
    """amrescan, then amgettuple until the scan ends, every row and the counters after it checked; -> rows"""
    sc = idx.begin_scan()
    try:
        sc.rescan(q, search_list_size=L, rescore=rescore)
        i = 0
        while True:
            i += 1
            if not scan_check(s, sc, q, L, rescore, i, sc.gettuple(), with_dist):
                return i - 1
    finally:
        sc.end()


def many_scans(lib, idx, s, qs, calls):
    """gettuple_many over scans of `qs` with a mix of (L, rescore); every row and counter after every call."""
    mix = [(1, 0), (40, 20), (15, 1), (60, 60)]
    scans = []
    try:
        for j, q in enumerate(qs):
            L, rescore = mix[j % len(mix)]
            sc = idx.begin_scan()
            scans.append((sc, q, L, rescore))
            sc.rescan(q, search_list_size=L, rescore=rescore)
        for i in range(1, calls + 1):
            out = lib.gettuple_many([t[0] for t in scans])
            for (sc, q, L, rescore), row in zip(scans, out):
                assert not isinstance(row, Exception), row
                scan_check(s, sc, q, L, rescore, i, row)
    finally:
        for t in scans:
            t[0].end()


def other_entry_points(lib, env, s, q, small, q_small):
    """search_batch_device on `s`; on the smaller index `small`: the streaming scan drained to the end for two
    queries, gettuple_many over six scans, and (cosine, L2) the plain layout's batch and drained scan."""
    from oracle import fixtures
    env()
    with lib.DiskAnnIndex(s) as idx:
        device_entry_point(idx, s, q, 10, 40, 20)
    with lib.DiskAnnIndex(small) as idx:
        for j, (L, rescore) in enumerate(((30, 20), (10, 0))):
            assert drain(idx, small, q_small[j], L, rescore) > 0
        many_scans(lib, idx, small, q_small[:6], 25)
    if small.distance_type != IP:
        p = fixtures.to_plain(small)
        with lib.DiskAnnIndex(p) as idx:
            for k, L, rescore in ((10, 40, 20), (25, 30, 0)):
                g = idx.search_batch(q_small, k=k, search_list_size=L, rescore=rescore)
                compare(g, oracle_batch(p, q_small, k, L, rescore), rescore, with_dist=False)
            assert drain(idx, p, q_small[0], 30, 10, with_dist=False) > 0


def returned(ref):
    """The rerank distances of the rows a batch with rescore > 0 returned (a flat f32 array)."""
    _, dist, count, _ = ref
    return np.concatenate([dist[b, :count[b]] for b in range(len(count))]).astype(F)


def tied_rows(ref):
    """Number of returned rows whose distance bits equal those of the row before them in the same result."""
    _, dist, count, _ = ref
    bits = dist.view(np.uint32)
    return sum(int((bits[b, 1:count[b]] == bits[b, :count[b] - 1]).sum()) for b in range(len(count)))


# ---- family 1: the quantizer's edges -----------------------------------------------------------------------------------

COUNTS = [0, 1, (1 << 24) + 3, (1 << 53) + 1]
# No f32 value lies exactly on the first edge of 4 bits: there z is about -1.2, so z + 2 is exact and a multiple of
# 2^-23, while 4 / 5 in f32 (13421773 * 2^-24) is not, and the neighbours of that quotient round to 1 -+ 2^-23 / 2^-24.
UNREACHABLE_EDGE = (4, 1)
QDIM, QROWS = 48, 256


@functools.lru_cache(maxsize=None)
def quantizer_case(count, bits):
    """A 48-d index whose quantizer is set directly: every 8th column constant (m2 = 0, every row at the mean), means
    of +0.0 (columns 0, 7, ...) and -0.0 (columns 3, 10, ...), standard deviations 0.5 to 2 over `count`.  Queries put
    each component at the mean, -0.0 / +0.0, 3 std away, or (count > 0, bits > 1) on a bucket edge k = 1..bits as the
    f32 arithmetic computes it for this count, or on that edge's nextafter neighbours."""
    rng = np.random.default_rng(count % 1000 + 17 * bits)
    count_f = float(F(count))                                    # `count as f32`, round to nearest
    mean = (rng.standard_normal(QDIM) * 0.5).astype(F)
    mean[0::7] = F(0.0)
    mean[3::7] = F(-0.0)
    sigma = rng.uniform(0.5, 2.0, QDIM).astype(F)
    m2 = (sigma.astype(np.float64) ** 2 * max(count_f, 1.0)).astype(F)
    const = np.arange(QDIM) % 8 == 5
    m2[const] = 0.0
    rows = (mean + sigma * rng.standard_normal((QROWS, QDIM)).astype(F)).astype(F)
    rows[:, const] = mean[const]
    dist = L2 if bits % 2 else IP
    s = index_with_quantizer(rows, dist, bits, mean, m2, count)
    edges = [boundary_values(mean, m2, count, bits, k) for k in range(1, bits + 1)] if bits > 1 and count else []
    opts = [mean, np.full(QDIM, F(-0.0)), np.full(QDIM, F(0.0)), mean + 3 * sigma, mean - 3 * sigma]
    for e in edges:
        opts += [e, np.nextafter(e, F(np.inf)), np.nextafter(e, F(-np.inf))]
    B = 2 * len(opts) + 2
    q = np.empty((B, QDIM), F)
    for j in range(B):
        for i in range(QDIM):
            v = opts[(j + i) % len(opts)][i]
            q[j, i] = mean[i] if np.isnan(v) else v
    return s, q, edges, const


@pytest.mark.parametrize("count", COUNTS, ids=["count0", "count1", "count2p24p3", "count2p53p1"])
def test_quantizer_edges(lib, env, count):
    """1 to 4 bits per dimension at one `count`: prepare_queries' codes (sbq_count_ones) and every kernel's scans."""
    import pyref
    for bits in (1, 2, 3, 4):
        s, q, edges, const = quantizer_case(count, bits)
        # the degeneracies: constant columns with query components above, below and at the mean; +-0 means met by
        # +-0 components; every bucket edge hit exactly
        assert const.any() and not s.m2[const].any()
        for cols in (const, s.mean.view(np.uint32) == 0, s.mean.view(np.uint32) == NEG_ZERO_BITS):
            assert cols.any()
            at = q[:, cols] == s.mean[cols]
            assert at.any() and (q[:, cols] > s.mean[cols]).any() and (q[:, cols] < s.mean[cols]).any()
        assert (q[:, s.mean.view(np.uint32) == 0].view(np.uint32) == NEG_ZERO_BITS).any()
        if bits > 1 and count:
            for k, e in enumerate(edges, 1):
                live = ~const
                if (bits, k) == UNREACHABLE_EDGE:
                    assert not np.isfinite(e).any()
                    continue
                assert np.isfinite(e[live]).sum() >= live.sum() // 2, (bits, k)
                on = np.isin(q.view(np.uint32), e[np.isfinite(e)].view(np.uint32))
                assert (bucket_index(q[on], np.broadcast_to(s.mean, q.shape)[on], np.broadcast_to(s.m2, q.shape)[on],
                                     count, bits) == F(k)).any(), (bits, k)
        if count == (1 << 24) + 3 and bits > 1:
            # `count as f32` rounds to nearest: toward zero (2^24 + 2) the query codes would differ
            assert float(F(count)) == count + 1
            rz = [pyref.quantize(r, bits, s.mean, s.m2, count - 1, s.words) for r in q]
            rn = [pyref.quantize(r, bits, s.mean, s.m2, count, s.words) for r in q]
            assert rz != rn
        with lib.DiskAnnIndex(s) as idx:
            prepare_and_full_distance(idx, s, q, seed=bits)
            every_kernel(env, idx, s, q)


# ---- family 2: 3 to 32 bits per dimension --------------------------------------------------------------------------

MULTI = [(40, 3, COSINE, 600), (64, 4, L2, 600), (13, 5, IP, 600), (96, 8, L2, 600), (24, 16, COSINE, 600),
         (7, 32, IP, 600), (768, 8, COSINE, 1000)]


@pytest.mark.parametrize("dim,bits,dist,n", MULTI, ids=[f"{d}x{b}" for d, b, _, _ in MULTI])
def test_multi_bit_codes(lib, env, dim, bits, dist, n):
    """Trained quantizers of 3 to 32 bits per dimension: prepare_queries packs each dimension's leading ones across
    64-bit words, and every kernel scans the wider codes."""
    from oracle import fixtures, oracle
    rows = fixtures.gen_vectors(n, dim, 7 * dim + bits, "normal" if dist == COSINE else "uniform")
    s = trained_index(rows, dist, bits, R=20, L_build=40)
    with np.errstate(all="ignore"):
        std = np.sqrt(s.m2 / F(s.count))
    far = [s.mean + F(3) * std, s.mean - F(3) * std]              # past the last edge and below the first
    q = np.concatenate([fixtures.gen_vectors(20, dim, dim + bits, "normal"),
                        fixtures.gen_vectors(12, dim, dim + bits + 1, "uniform"), far, rows[:4]]).astype(F)
    q[-1] = 0.0
    straddle = [i for i in range(dim) if (i * bits) // 64 != (i * bits + bits - 1) // 64]
    assert bool(straddle) == (64 % bits != 0), straddle           # 3, 5 bits: some dimension's bits cross a word
    iq = [oracle.preprocess_cosine(r) if dist == COSINE else r for r in q]
    ones = np.stack([code_ones(oracle.quantize(r, bits, s.mean, s.m2, s.count), dim, bits) for r in iq])
    assert ones.max() == bits and len(np.unique(ones)) >= min(bits + 1, 4), np.unique(ones)
    if straddle:
        assert (ones[:, straddle] > 0).any() and (ones[:, straddle] < bits).any()
    with lib.DiskAnnIndex(s) as idx:
        assert idx.code_stride == (s.words + 1) & ~1
        prepare_and_full_distance(idx, s, q, seed=dim)
        every_kernel(env, idx, s, q)


# ---- family 3: overflow --------------------------------------------------------------------------------------------

def overflow_rows(n, dim, seed):
    """Uniform [-1, 1) rows with 10 % of their components at +-3e38, and every 16th row all 1e20 (finite components
    whose norm and whose products overflow).  Queries: table rows, a row of -1e20, rows with +-3e38, plain rows."""
    rng = np.random.default_rng(seed)
    v = rng.uniform(-1, 1, (n, dim)).astype(F)
    big = rng.random((n, dim)) < 0.1
    v[big] = np.where(rng.random(big.sum()) < 0.5, F(3e38), F(-3e38))
    v[::16] = F(1e20)
    q = np.concatenate([v[1:9], -v[::16][:2], rng.uniform(-1, 1, (6, dim)).astype(F)])
    qb = rng.random(q[-6:].shape) < 0.1
    q[-6:][qb] = np.where(rng.random(qb.sum()) < 0.5, F(3e38), F(-3e38))
    q = np.concatenate([q, rng.uniform(-1, 1, (4, dim)).astype(F)])
    return v, q


@pytest.mark.parametrize("dist", [COSINE, L2, IP], ids=["cosine", "l2", "ip"])
def test_overflow(lib, env, dist):
    """+inf L2 distances and their ties; inner products of +-inf and NaN (inf + -inf), whose bits must be the x86
    build's 0x7FC00000; cosine rows and queries that normalise to zeros."""
    from oracle import oracle
    v, q = overflow_rows(600, 64, 3 + dist)
    s = trained_index(v, dist, 2)
    with lib.DiskAnnIndex(s) as idx:
        full = prepare_and_full_distance(idx, s, q, seed=dist)
        refs = every_kernel(env, idx, s, q)
    d = np.concatenate([returned(r) for (_, _, rescore), r in refs.items() if rescore] + [full.ravel()])
    if dist == COSINE:
        zero = [r for r in v if not oracle.preprocess_cosine(r).any()]
        assert len(zero) >= len(v) // 2                            # every row with a +-3e38 or 1e20 component
        assert not oracle.preprocess_cosine(q[8]).any()             # -1e20 query
        assert (d == F(1.0)).sum() > 50 and not np.isnan(d).any()
    elif dist == L2:
        assert np.isposinf(d).sum() > 50 and tied_rows(refs[(30, 60, 60)]) > 20
    else:
        assert np.isnan(d).any() and np.isposinf(d).any() and np.isneginf(d).any()
        assert (d[np.isnan(d)].view(np.uint32) == 0x7FC00000).all()
    small_v, small_q = overflow_rows(300, 40, 30 + dist)
    other_entry_points(lib, env, s, q, trained_index(small_v, dist, 2), small_q)


# ---- family 4: tiny components and signed zeros ----------------------------------------------------------------------

def tiny_rows(n, dim, seed):
    """A quarter each: rows of tiny components (+-1e-20 scale, so that products and squared differences are
    subnormal), rows of +-1e-40 / -0.0 / +0.0, one-hot rows of +-1 (integer-valued, so inner products are exactly
    zero or +-1), and all-zero rows.  Queries of the same four kinds."""
    rng = np.random.default_rng(seed)
    kinds = np.arange(n) % 4
    v = np.zeros((n, dim), F)
    t = kinds == 0
    v[t] = (rng.uniform(-1, 1, (t.sum(), dim)) * 1e-20).astype(F)
    t = kinds == 1
    v[t] = rng.choice(np.array([1e-40, -1e-40, -0.0, 0.0, 3e-39], F), (t.sum(), dim))
    t = np.flatnonzero(kinds == 2)
    v[t, rng.integers(0, dim, len(t))] = rng.choice(np.array([1.0, -1.0], F), len(t))
    q = np.concatenate([(rng.uniform(-1, 1, (6, dim)) * 1e-20).astype(F),
                        rng.choice(np.array([1e-40, -1e-40, -0.0, 0.0], F), (4, dim)),
                        v[2:40:4][:6], np.full((2, dim), F(-0.0))]).astype(F)
    return v, q


@pytest.mark.parametrize("dist", [COSINE, L2, IP], ids=["cosine", "l2", "ip"])
def test_tiny_components_and_signed_zeros(lib, env, dist):
    """Subnormal products and sums kept (not flushed), the cosine `norm < eps` branch on tiny and zero rows, -0.0
    inner products of one-hot rows."""
    from oracle import oracle
    v, q = tiny_rows(600, 64, 5 + dist)
    s = trained_index(v, dist, 2 if dist != IP else 1)
    with lib.DiskAnnIndex(s) as idx:
        refs = every_kernel(env, idx, s, q)
    d = np.concatenate([returned(r) for (_, _, rescore), r in refs.items() if rescore])
    if dist == COSINE:
        assert np.array_equal(oracle.preprocess_cosine(v[0]), v[0]) and v[0].any()    # norm < eps: untouched
        assert (d == F(0.0)).any() and (d == F(1.0)).any()
    else:
        sub = (d != 0) & (np.abs(d) < FLT_MIN)
        assert sub.sum() > 20, sub.sum()
        if dist == IP:
            assert (d.view(np.uint32) == NEG_ZERO_BITS).sum() > 20
    small_v, small_q = tiny_rows(240, 40, 50 + dist)
    other_entry_points(lib, env, s, q, trained_index(small_v, dist, 2), small_q)


# ---- family 5: duplicates and exact ties -----------------------------------------------------------------------------

def duplicate_rows(n, dim, distinct, seed, kind):
    """n rows drawn from `distinct` vectors; queries: table rows, table rows perturbed by 1e-3, the zero vector.  Half
    the distinct unit vectors have an inner product with themselves above 1 in the AVX2 order, so that a row's cosine
    distance to itself goes through the (1 - ip).max(0) clamp."""
    from oracle import fixtures, oracle
    base = fixtures.gen_vectors(distinct * 8, dim, seed, kind)
    if kind == "normal":
        over = np.array([oracle.distance(IP, x, x, "avx2") < -1.0 for x in base])
        base = np.concatenate([base[over][:distinct // 2], base[~over][:distinct - distinct // 2]])
    base = base[:distinct]
    rng = np.random.default_rng(seed)
    v = base[rng.integers(0, distinct, n)]
    q = np.concatenate([v[:12], v[12:24] + (rng.standard_normal((12, dim)) * 1e-3).astype(F),
                        np.zeros((1, dim), F)]).astype(F)
    return np.ascontiguousarray(v, F), q


DUPS = [(96, COSINE, "normal"), (96, L2, "uniform"), (96, IP, "uniform"), (768, COSINE, "normal")]


@pytest.mark.parametrize("dim,dist,kind", DUPS, ids=["96-cosine", "96-l2", "96-ip", "768-cosine"])
def test_duplicates(lib, env, dim, dist, kind):
    """2000 rows of 37 distinct vectors: zero distances (through the cosine clamp), and runs of equal Hamming
    distances and of equal exact distances in the beam's heaps and the rerank window."""
    from oracle import oracle
    v, q = duplicate_rows(2000, dim, 37, dim + dist, kind)
    s = trained_index(v, dist, 2, R=24, L_build=48)
    with lib.DiskAnnIndex(s) as idx:
        refs = every_kernel(env, idx, s, q, runs=((10, 40, 20), (40, 80, 100), (10, 30, 0)))
    assert len(np.unique(v, axis=0)) == 37
    assert tied_rows(refs[(40, 80, 100)]) > 12 * 30
    d = returned(refs[(40, 80, 100)])
    if dist == IP:
        assert len(np.unique(d)) < 60
    else:
        assert (d == F(0.0)).sum() >= 100
    if dist == COSINE:
        # the clamp: a row's inner product with itself (both normalised) above 1, so 1 - ip < 0 -> 0.0
        _, dist_, count, _ = refs[(40, 80, 100)]
        over = [i for i in range(12) if oracle.distance(IP, oracle.preprocess_cosine(q[i]),
                                                        oracle.preprocess_cosine(q[i]), "avx2") < -1.0
                and (dist_[i, :count[i]] == 0).sum() >= 10]
        assert over, "no query of this fixture returns its duplicates through the cosine clamp"
    small_v, small_q = duplicate_rows(300, dim, 12, dim + dist + 1, kind)
    other_entry_points(lib, env, s, q[:16], trained_index(small_v, dist, 2), small_q)
