"""The two-warp and single-warp search kernels, the streaming scan, the exact-distance kernels and the stand-alone SBQ
distance kernel against the oracle, at every code width and shared-memory size they ship, up to the reference's 16000
dimensions (build.rs:192, MAX_DIMENSION).

Bar, as in test_gpu_parity.py: bit-exact TIDs, bit-exact rerank distances (u32), counts, all five counters, status 0.
Every batch pins its kernel (DANN_SEARCH_KERNEL=2 two-warp, =1 single-warp) and inserted-set (DANN_SEARCH_BITMAP), and
reads the plan back, so a plan change that moves a case to another kernel or entry layout fails instead of passing.

Code mapping (dann_plan.h pick_code_mapping): words = ceil(dim * bits / 64), cw = (words + 1) & ~1, C = cw / 2 16-byte
chunks, G = min(32, pow2ceil((C + 2) / 3)) lanes per row, NCH = ceil(C / G), rounded up to 8 when it is 5 to 8.  Entry
layout (dann_make_plan): Ent32x21 while the maximum distance words * 64 < 2048, Ent32x16 while it is < 65536 and
cand_cap <= 65536, else Ent64.  The plan reports entry_bytes only (4 for both 4-byte layouts), so the layout a batch
ran is that rule applied to its plan's cand_cap, and entry_bytes confirms it.

   dim x bits | words / cw | G, NCH | chunk rows          | natural entry
   37 x 2     | 2 / 2      | 1, 1   | exact              | Ent32x21
   100 x 2    | 4 / 4      | 1, 2   | exact              | Ent32x21
   768 x 2    | 24 / 24    | 4, 3   | exact              | Ent32x21 (the benchmark's shape)
   992 x 2    | 31 / 32    | 8, 2   | exact              | Ent32x21, the largest (max distance 1984)
   1024 x 2   | 32 / 32    | 8, 2   | exact              | Ent32x16, the smallest
   6145 x 2   | 193 / 194  | 32, 4  | 97 of 128 chunks   | Ent32x16
   8192 x 2   | 256 / 256  | 32, 4  | exact              | Ent32x16
   16000 x 1  | 250 / 250  | 32, 4  | 125 of 128         | Ent32x16 (the reference's default at its maximum)
   8200 x 2   | 257 / 258  | 32, 8  | 129 of 256: 5-7 idle | Ent32x16
   16000 x 2  | 500 / 500  | 32, 8  | 250 of 256         | Ent32x16 (the widest code the reference makes)

Instantiations of dann_search2_kernel<T, NCH> (pick_search2) and dann_search_kernel<T, NCH> (pick_search), 15 each, and
which batches run them (both kernels alike):
   Ent32x21 x NCH 1, 2, 3   natural entry of 37, 100, 768 and 992 x 2
   Ent32x16 x NCH 1, 2, 3   DANN_SEARCH_ENTRY=1 on those (the keys fit 16 bits); NCH 2 also natural at 1024 x 2
   Ent32x16 x NCH 4, 8      natural entry of the codes of 193 words and more
   Ent64    x NCH 1 .. 8    DANN_SEARCH_ENTRY=2 everywhere; natural at L = 3000 (cand_cap > 65536) on 1024 x 2 and wider
   Ent32x21 x NCH 4, 8      UNREACHABLE: NCH 4 needs at least 193 words, a maximum distance of 12352 or more, which
                            does not fit the 11-bit key.  Not tested.
INSTANTIATIONS below is this table; test_instantiation_table_matches_the_batches checks that the batches assert it.

The streaming scan always runs the single-warp kernel.  It does not publish its plan: its entry layout is asserted
through a proxy, a one-query DANN_SEARCH_KERNEL=1 batch with the scan's L, rescore and key and c_target = rescore + 64
(k = rescore + 65, or 64 when rescore is 0), which is the make_plan(nq = 1, c_target = rescore + 64) of the scan.

The exact-distance kernels (prepare, full-distance, rerank, scan-distance) stage the query row in dynamic shared
memory: dim4 * 4 + 128 bytes.  Dimensions 12256 (a window of 48 KB exactly, which with the kernel's static shared
memory is past the default limit: the first opt-in launch), 12260 (TMA staging), 12289 (dim % 4 != 0: plain-copy
staging and the scalar tail) and 16000 run them around that bound.

Every test here also runs under the CPU SIMT emulator (DANN_EMULATE=1, tests/test_emulated_abi.py)."""
import copy
import functools
import os

import numpy as np
import pytest

from conftest import buffer_device, build_case, dptr, emulating
from test_gpu_parity import COSINE, IP, L2, _compare_batch, _queries

pytestmark = pytest.mark.gpu

HOOKS = ("DANN_SEARCH_KERNEL", "DANN_SEARCH_WARPS", "DANN_SEARCH_HS", "DANN_SEARCH_BITMAP", "DANN_SEARCH_ENTRY",
         "DANN_DEBUG_SHRINK", "DANN_SBQ_UNR", "DANN_SBQ_BLOCKS_PER_SM")
INVALID = 0xFFFFFFFF
NAN_BITS = 0x7FC00000
X21, X16, E64 = 0, 1, 2
LAYOUT = {X21: "Ent32x21", X16: "Ent32x16", E64: "Ent64"}

# (kernel, layout, NCH) that the batches of test_search_kernels_at_every_code_width assert: the docstring's table
INSTANTIATIONS = {(kern, lay, nch) for kern in (1, 2) for lay, nch in
                  [(X21, 1), (X21, 2), (X21, 3), (X16, 1), (X16, 2), (X16, 3), (X16, 4), (X16, 8),
                   (E64, 1), (E64, 2), (E64, 3), (E64, 4), (E64, 8)]}
UNREACHABLE = {(kern, X21, nch) for kern in (1, 2) for nch in (4, 8)}


@pytest.fixture(scope="module")
def lib(lib_built):
    from pgvectorscale_b200 import diskann
    if diskann.device_count() < 1:
        pytest.fail("no CUDA device visible: -m gpu tests need an H100")
    return diskann


@pytest.fixture
def env(monkeypatch):
    """env(KERNEL=1, HS=4, SBQ_UNR=2, ...) sets exactly these hooks (DANN_SEARCH_*, DANN_DEBUG_SHRINK, DANN_SBQ_*) and
    clears the others."""
    def set_(**kv):
        for h in HOOKS:
            monkeypatch.delenv(h, raising=False)
        for key, val in kv.items():
            name = "DANN_DEBUG_SHRINK" if key == "SHRINK" else "DANN_" + key if key.startswith("SBQ") \
                else "DANN_SEARCH_" + key
            assert name in HOOKS, key
            monkeypatch.setenv(name, str(val))
    set_()
    return set_


def pow2ceil(x):
    p = 1
    while p < x:
        p <<= 1
    return p


def code_mapping(dim, bits):
    """words, cw, G, NCH, chunks used: dann_plan.h pick_code_mapping restated."""
    words = -(-dim * bits // 64)
    cw = (words + 1) & ~1
    C = cw // 2
    G = min(32, pow2ceil((C + 2) // 3))
    nch = -(-C // G)
    assert nch <= 8, (dim, bits)
    return words, cw, G, 8 if nch > 4 else nch, C


def planned_layout(words, cand_cap, hook=None):
    """dann_make_plan's entry layout of a two-warp / single-warp plan."""
    if hook is not None:
        return hook
    maxdist = words * 64
    if maxdist < 2048 and cand_cap <= 1 << 21:
        return X21
    if maxdist < 65536 and cand_cap <= 65536:
        return X16
    return E64


def cand_cap(L, c_target, R, grow=1, shrink=1):
    """dann_make_plan's per-query candidate capacity."""
    need = ((L + c_target) * 23 // 20 + 40) * R * grow
    need = max(need // shrink, 256)
    return (need + 1023) & ~1023


@functools.lru_cache(maxsize=None)
def _case(n, dim, bits, dist, kind, seed, R=24, L_build=48, **kw):
    return build_case(n, dim, dist, bits=bits, seed=seed, kind=kind, R=R, L_build=L_build, **kw)


def case(*a, **kw):
    """A cached fixture index; a shallow copy, so that a test may replace an array without touching the cache."""
    return copy.copy(_case(*a, **kw))


# (dim, bits, distance, data kind, (words, cw, G, NCH, chunks used), natural layout, label key or None)
SHAPES = [
    (37, 2, COSINE, "normal", (2, 2, 1, 1, 1), X21, None),
    (100, 2, L2, "uniform", (4, 4, 1, 2, 2), X21, None),
    (768, 2, COSINE, "normal", (24, 24, 4, 3, 12), X21, [3, 7]),
    (992, 2, L2, "uniform", (31, 32, 8, 2, 16), X21, None),
    (1024, 2, IP, "uniform", (32, 32, 8, 2, 16), X16, None),
    (6145, 2, COSINE, "normal", (193, 194, 32, 4, 97), X16, [2, 11]),
    (8192, 2, L2, "uniform", (256, 256, 32, 4, 128), X16, None),
    (16000, 1, COSINE, "normal", (250, 250, 32, 4, 125), X16, None),
    (8200, 2, IP, "uniform", (257, 258, 32, 8, 129), X16, None),
    (16000, 2, L2, "uniform", (500, 500, 32, 8, 250), X16, [5, 9, 14]),
]
SHAPE_IDS = [f"{d}x{b}" for d, b, *_ in SHAPES]
N_NODES = 320


def shape_case(shape):
    dim, bits, dist, kind, mapping, natural, key = shape
    return case(N_NODES, dim, bits, dist, kind, seed=dim + bits, labels=key is not None)


def assert_mapping(idx, s, shape):
    """The fixture has the code this shape stands for: a drifting fixture fails here instead of testing another."""
    dim, bits, _, _, mapping, natural, _ = shape
    words, cw, G, nch, used = code_mapping(dim, bits)
    assert (s.words, idx.code_stride) == (words, cw)
    assert (words, cw, G, nch, used) == mapping, (shape, (words, cw, G, nch, used))
    assert planned_layout(words, 1024) == natural
    return words, nch


def check(s, idx, q, k, L, rescore, labels=None, *, kernel, words, layout, hook=None, bitmap=None, hs=None):
    """Oracle parity of the whole batch, then proof of the kernel, entry layout, inserted-set and heap top it ran."""
    g = _compare_batch(s, idx, q, k, L, rescore, labels)
    p = idx.last_search_plan()
    assert p["kernel"] == kernel, p
    lay = planned_layout(words, p["cand_cap"], hook)
    assert lay == layout, (LAYOUT[lay], p)
    assert p["entry_bytes"] == (8 if lay == E64 else 4), p
    if bitmap is not None:
        assert p["bitmap"] == bitmap, p
    if hs is not None:
        assert p["heap_smem"] == hs, p
    return g, p


def batch_plans(natural):
    """(kernel, hook, layout, [(bitmap, heap top, (k, L, rescore))]) of one shape's batch matrix."""
    layouts = [(None, natural), (E64, E64)] + ([(X16, X16)] if natural == X21 else [])
    out = []
    for kernel in (2, 1):
        for hook, layout in layouts:
            runs = [(1, 4 if kernel == 2 else 16, (10, 40, 20)), (0, 16 if kernel == 2 else 4, (7, 25, 0))]
            out.append((kernel, hook, layout, runs))
    return out


def test_instantiation_table_matches_the_batches():
    """The batches of test_search_kernels_at_every_code_width run exactly the docstring's instantiations, and every
    one of the 2 x 15 that is not listed there as unreachable."""
    ran = set()
    for shape in SHAPES:
        dim, bits, _, _, mapping, natural, _ = shape
        for kernel, hook, layout, _ in batch_plans(natural):
            ran.add((kernel, layout, code_mapping(dim, bits)[3]))
    every = {(kern, lay, nch) for kern in (1, 2) for lay in (X21, X16, E64) for nch in (1, 2, 3, 4, 8)}
    assert ran == INSTANTIATIONS == every - UNREACHABLE
    for kern, lay, nch in UNREACHABLE:      # the smallest code of NCH 4 (193 words) has distances past 11 bits
        assert min(w for w in range(1, 513) if code_mapping(32 * w, 2)[3] == nch) * 64 >= 2048


# ---- 1. search kernels and the streaming scan at every code width ---------------------------------------------------

@pytest.mark.parametrize("shape", SHAPES, ids=SHAPE_IDS)
def test_search_kernels_at_every_code_width(lib, env, shape):
    """Both kernels x the natural entry, Ent64 and (for 4-byte Ent32x21 codes) Ent32x16 x both inserted-sets, heap
    tops of 4 and 16 entries, a zero query; k > n on some shapes; Ent64 without the hook on the wide codes."""
    dim, bits, dist, kind, mapping, natural, key = shape
    s = shape_case(shape)
    q = _queries(s, 24, dim + 1, kind)
    q[5] = 0.0                                                # NULL-like query: all-zero code
    with lib.DiskAnnIndex(s) as idx:
        words, nch = assert_mapping(idx, s, shape)
        for kernel, hook, layout, runs in batch_plans(natural):
            for bitmap, hs, (k, L, rescore) in runs:
                env(KERNEL=kernel, BITMAP=bitmap, HS=hs, **({} if hook is None else {"ENTRY": hook}))
                check(s, idx, q, k, L, rescore, kernel=kernel, words=words, layout=layout, hook=hook, bitmap=bitmap,
                      hs=hs)
        if dim in (100, 8200):                                # k > n: the stream runs dry
            for kernel in (2, 1):
                env(KERNEL=kernel)
                g, _ = check(s, idx, q[:8], s.n + 40, 60, 50, kernel=kernel, words=words, layout=natural)
                assert (g["count"] == s.n).all()
        if natural == X16:                                    # cand_cap > 65536: Ent64 by the plan's own rule
            assert cand_cap(3000, 10 + 20 - 1, s.R) > 65536
            for kernel in (2, 1):
                env(KERNEL=kernel)
                check(s, idx, q[:6], 10, 3000, 20, kernel=kernel, words=words, layout=E64)


def scan_rows(s, sc, q, labels, L, rescore, rows):
    """rescan, then `rows` gettuples, each checked (row, node, distance bits, the four counters and the stream length)
    against the oracle's scan of that many rows."""
    from oracle import oracle
    sc.rescan(q, labels=labels, search_list_size=L, rescore=rescore)
    got = 0
    for i in range(1, rows + 1):
        row = sc.gettuple()
        ref = oracle.scan(s, q, labels, L, rescore, i)
        if len(ref["tid"]) < i:
            assert row is None
            break
        got += 1
        assert row is not None, i
        assert ((row[0] << 16) | row[1]) == int(ref["tid"][-1]) and row[2] == int(ref["node"][-1]), i
        if rescore:
            assert np.float32(row[3]).view(np.uint32) == ref["dist"][-1].view(np.uint32), i
        st = sc.stats()
        for f in ("visits", "d_quantized", "candidates", "d_full", "stream_len"):
            assert st[f] == ref["stats"][f], (f, i, labels, L, rescore)
    return got


@pytest.mark.parametrize("shape", SHAPES, ids=SHAPE_IDS)
def test_streaming_scan_at_every_code_width(lib, env, shape):
    """amrescan + 41 amgettuples, rescore 50 and 0, a label key where the fixture has labels; the entry layout of the
    scan's single-warp search through the proxy batch (module docstring)."""
    dim, bits, dist, kind, mapping, natural, key = shape
    s = shape_case(shape)
    q = _queries(s, 2, dim + 3, kind)
    with lib.DiskAnnIndex(s) as idx:
        words, _ = assert_mapping(idx, s, shape)
        sc = idx.begin_scan()
        try:
            for qi, labels, L, rescore in ((0, None, 40, 50), (1, key, 30, 0)):
                env()
                got = scan_rows(s, sc, q[qi], labels, L, rescore, 41)
                assert got == 41 or labels is not None, got
                env(KERNEL=1)                                 # proxy: the scan's plan, published by a batch
                check(s, idx, q[qi:qi + 1], rescore + 65 if rescore else 64, L, rescore,
                      None if labels is None else [labels], kernel=1, words=words, layout=natural)
        finally:
            sc.end()


def test_scan_drained_through_the_switch_to_ent64(lib, env):
    """A 1024 x 2 code (Ent32x16) scanned to the end of a 2000-node index with 64-id lists.  Under
    DANN_DEBUG_SHRINK=8 the first workspace is too small, and each regrow-and-replay doubles it; the visited list
    overflows until it holds the scan's unconsumed visits, and with rescore 1000 the candidate capacity that goes with
    it is past 65536, so the last regrow rebuilds the suspended search as Ent64, which replays the stream.  The number
    of regrowths is read from the kernel launch counter: a gettuple that searches launches the search, the distance
    kernel and the window step once per attempt, one that does not launches the window step alone.  The layouts are
    dann_make_plan's rule."""
    from oracle import oracle
    L, rescore, shrink = 100, 1000, 8
    s = case(2000, 1024, 2, IP, "uniform", seed=1024 + 7, R=64, L_build=72)
    q = _queries(s, 1, 1031, "uniform")[0]
    with lib.DiskAnnIndex(s) as idx:
        assert planned_layout(s.words, cand_cap(L, rescore + 64, s.R, 1, shrink)) == X16
        env(SHRINK=shrink)
        sc = idx.begin_scan()
        try:
            sc.rescan(q, search_list_size=L, rescore=rescore)
            ref = oracle.scan(s, q, None, L, rescore, s.n + 1)
            rows, regrows = [], 0
            while True:
                before = idx.kernel_launches
                r = sc.gettuple()
                launches = idx.kernel_launches - before
                assert launches == 1 or launches % 3 == 0, launches
                regrows += max(launches // 3 - 1, 0)
                if r is None:
                    break
                rows.append(r)
            st = sc.stats()
        finally:
            sc.end()
    assert len(rows) == len(ref["tid"]) == s.n
    assert np.array_equal(np.array([(b << 16) | o for b, o, _, _ in rows], np.uint64), ref["tid"])
    assert np.array_equal(np.array([n for _, _, n, _ in rows], np.uint32), ref["node"])
    assert np.array_equal(np.array([d for *_, d in rows], np.float32).view(np.uint32), ref["dist"].view(np.uint32))
    for f in ("visits", "d_quantized", "candidates", "d_full", "stream_len"):
        assert st[f] == ref["stats"][f], f
    assert regrows >= 1
    assert planned_layout(s.words, cand_cap(L, rescore + 64, s.R, 1 << (regrows - 1), shrink)) == X16, regrows
    assert planned_layout(s.words, cand_cap(L, rescore + 64, s.R, 1 << regrows, shrink)) == E64, regrows


# ---- 2. exact-distance kernels around and past 48 KB of shared memory ----------------------------------------------

# (dim, dim_index, distance, data kind): the query window dim4 * 4 + 128 is 48 KB exactly (an opt-in launch only
# because of the kernel's static shared memory), TMA staging past 48 KB, a row that is not a multiple of 4 (plain
# copy, scalar tail), the reference's maximum
WIDE_ROWS = [(12256, 12256, L2, "uniform"), (12260, 12260, COSINE, "normal"), (12289, 12289, IP, "uniform"),
             (12289, 12289, COSINE, "normal"), (16000, 12289, COSINE, "normal"), (16000, 16000, L2, "uniform")]


@pytest.mark.parametrize("dim,dim_index,dist,kind", WIDE_ROWS, ids=[f"{d}-{i}-{t}" for d, i, t, _ in WIDE_ROWS])
def test_exact_distance_kernels_around_48kb_of_shared_memory(lib, env, dim, dim_index, dist, kind):
    """prepare_queries and full_distance bit-equal to the oracle (a zero query, DANN_INVALID_NODE -> NaN), a batch
    with rescore > 0 (dann_rerank_kernel) and a streaming scan with rescore > 0 (dann_scan_distance_kernel)."""
    import torch
    from oracle import oracle
    s = case(160, dim, None, dist, kind, seed=dim + dim_index + dist, R=16, L_build=32, dim_index=dim_index)
    B, m = 5, 13
    q = _queries(s, B, dim + 5, kind) * 3.0
    q[0] = 0.0
    with lib.DiskAnnIndex(s) as idx:
        dev = buffer_device()
        d_q = torch.from_numpy(q).to(dev)
        d_full = torch.empty((B, dim), dtype=torch.float32, device=dev)
        d_codes = torch.empty((B, idx.code_stride), dtype=torch.int64, device=dev)
        idx.prepare_queries(dptr(d_q), dptr(d_full), dptr(d_codes))
        full = d_full.cpu().numpy()
        codes = d_codes.cpu().numpy().view(np.uint64)
        for b in range(B):
            qf = oracle.preprocess_cosine(q[b]) if dist == COSINE else q[b]
            qi = q[b, :dim_index].copy()
            if dist == COSINE:
                qi = oracle.preprocess_cosine(qi)
            assert np.array_equal(full[b].view(np.uint32), qf.view(np.uint32)), b
            assert np.array_equal(codes[b, :s.words], oracle.quantize(qi, s.bits, s.mean, s.m2, s.count)), b
            assert not codes[b, s.words:].any()
        rng = np.random.default_rng(dim)
        nodes = rng.integers(0, s.n, size=(B, m), dtype=np.uint32)
        nodes[1, 4] = nodes[3, 0] = nodes[3, m - 1] = INVALID
        d_nodes = torch.from_numpy(nodes.view(np.int32)).to(dev)
        d_out = torch.empty((B, m), dtype=torch.float32, device=dev)
        idx.full_distance(dptr(d_full), dptr(d_nodes), dptr(d_out))
        out = d_out.cpu().numpy().view(np.uint32)
        for b in range(B):
            for i in range(m):
                if nodes[b, i] == INVALID:
                    assert out[b, i] == NAN_BITS, (b, i)
                    continue
                x = s.vectors[nodes[b, i]]
                if dist == COSINE:
                    x = oracle.preprocess_cosine(x)
                ref = np.float32(oracle.distance(dist, x, full[b], "avx2"))
                assert out[b, i] == ref.view(np.uint32), (b, i)
        _compare_batch(s, idx, q, 10, 40, 30)
        sc = idx.begin_scan()
        try:
            assert scan_rows(s, sc, q[1], None, 30, 20, 24) == 24
        finally:
            sc.end()


# ---- 3. the rerank kernel's shared-memory bound ---------------------------------------------------------------------

def smem_optin():
    if emulating():
        return 232448                 # the fake runtime's sharedMemPerBlockOptin
    import torch
    return torch.cuda.get_device_properties(0).shared_memory_per_block_optin


def rerank_smem(dim, k, rescore):
    """The dynamic shared memory of one dann_rerank_kernel CTA: query row, one f32 per streamed row (even count),
    the rescore window of 8-byte entries, 16 bytes, 128 bytes of slack."""
    c_target = k if rescore == 0 else rescore + k - 1
    return ((dim + 3) & ~3) * 4 + ((c_target + 1) & ~1) * 4 + rescore * 8 + 16 + 128


def rerank_k_max(dim, rescore, limit):
    c_max = ((limit - ((dim + 3) & ~3) * 4 - rescore * 8 - 16 - 128) // 4) & ~1
    k = c_max if rescore == 0 else c_max - rescore + 1
    assert rerank_smem(dim, k, rescore) <= limit < rerank_smem(dim, k + 1, rescore)
    return k


@pytest.mark.parametrize("dim", [64, 12289])
def test_rerank_shared_memory_bound_is_checked_before_the_launch(lib, env, dim):
    """The largest k the library accepts returns every live row (k > n) as the oracle does; one more is refused with
    DANN_ERR_INVALID_ARG, and the handle still answers a normal batch.

    The limit is the device's opt-in shared memory less the kernel's static shared memory (cudaFuncGetAttributes), a
    figure only the library can read; the refusal of a k far past it states it.  The test holds that figure to the
    device's opt-in limit (the static part is the staging mbarrier and the like: a few bytes on hardware, none under the
    emulator, which keeps static shared variables outside its window), then finds k_max from the launch's layout
    restated here.  A failed launch would poison the handle, so nothing here probes for the bound: k_max runs because
    it must fit, and k_max + 1 must be refused with the restated size."""
    import re
    s = case(50, dim, None, L2, "uniform", seed=dim + 71, R=12, L_build=24)
    q = _queries(s, 3, dim + 2, "uniform")
    optin = smem_optin()
    with lib.DiskAnnIndex(s) as idx:
        for rescore in (0, 1, 1000):
            with pytest.raises(lib.DiskAnnError) as e:
                idx.search_batch(q, k=1_000_000, search_list_size=50, rescore=rescore)
            assert e.value.code == -1, str(e.value)
            limit = int(re.search(r"\(limit (\d+)\)", str(e.value)).group(1))
            assert (limit == optin) if emulating() else (optin - 1024 <= limit < optin), (limit, optin)
            k = rerank_k_max(dim, rescore, limit)
            with pytest.raises(lib.DiskAnnError) as e:
                idx.search_batch(q, k=k + 1, search_list_size=50, rescore=rescore)
            assert e.value.code == -1, (rescore, str(e.value))
            assert f"need {rerank_smem(dim, k + 1, rescore)} B" in str(e.value), str(e.value)
            g = _compare_batch(s, idx, q, k, 50, rescore)
            assert (g["count"] == s.n).all(), rescore
            _compare_batch(s, idx, q, 10, 50, rescore)


# ---- 4. the stand-alone SBQ distance kernel at every instantiation ------------------------------------------------

# (dim, UNRs): NCH 1-3 take DANN_SBQ_UNR = 1, 2, 4 or 8; NCH 4 is built with UNR 2 only, NCH 8 with UNR 1
SBQ_SHAPES = [(37, (1, 2, 4, 8)), (100, (1, 2, 4, 8)), (768, (1, 2, 4, 8)), (6144, (1, 2, 4, 8)),
              (6145, (None,)), (8192, (None,)), (8200, (None,)), (16000, (None,))]


@pytest.mark.parametrize("dim,unrs", SBQ_SHAPES, ids=[f"{d}x2" for d, _ in SBQ_SHAPES])
def test_sbq_distance_at_every_instantiation(lib, env, dim, unrs):
    """dann_sbq_distance_kernel<NCH, UNR> against numpy's popcount of codes[node] ^ qcodes[query], for 1, 7 and
    2^17 + 3 pairs; one CTA per SM, so that the grid-stride loop turns many times over the long pair list."""
    import torch
    s = case(64, dim, 2, L2, "uniform", seed=dim + 3, R=8, L_build=16)
    words, cw, G, nch, _ = code_mapping(dim, 2)
    assert nch == {37: 1, 100: 2, 768: 3, 6144: 3, 6145: 4, 8192: 4, 8200: 8, 16000: 8}[dim]
    Q = 9
    rng = np.random.default_rng(dim)
    qcodes = rng.integers(0, 2**64, size=(Q, cw), dtype=np.uint64)
    qcodes[:, words:] = 0
    table = np.bitwise_count(qcodes[:, None, :words] ^ s.codes[None, :, :]).sum(axis=2).astype(np.int32)
    dev = buffer_device()
    with lib.DiskAnnIndex(s) as idx:
        assert idx.code_stride == cw
        d_q = torch.from_numpy(qcodes.view(np.int64)).to(dev)
        for npairs in (1, 7, 2**17 + 3):
            pq = rng.integers(0, Q, size=npairs, dtype=np.uint32)
            pn = rng.integers(0, s.n, size=npairs, dtype=np.uint32)
            d_pq = torch.from_numpy(pq.view(np.int32)).to(dev)
            d_pn = torch.from_numpy(pn.view(np.int32)).to(dev)
            for unr in unrs:
                env(SBQ_BLOCKS_PER_SM=1, **({} if unr is None else {"SBQ_UNR": unr}))
                d_out = torch.full((npairs + 1,), -1, dtype=torch.int32, device=dev)
                idx.sbq_distance(dptr(d_q), dptr(d_pq), dptr(d_pn), dptr(d_out[:npairs]))
                out = d_out.cpu().numpy()
                assert np.array_equal(out[:npairs], table[pq, pn]), (npairs, unr)
                assert out[npairs] == -1                      # nothing written past the last pair
