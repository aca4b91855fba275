"""LIMIT 10 under a selective post-filter, with the rows of a streaming scan fetched many per GPU step.

An amgettuple shim that reads ahead fills a buffer with dann_scan_fetch, asking for 1, 2, 4, ... rows (up to --cap) each
time the buffer runs dry, and hands the rows out one at a time.  This tool repeats tools/deep_scan.py's post-filter
experiment (a deterministic predicate on the TID passing 1/100, 1/1000 and 1/10000 of rows) three ways, alternating
query by query in one run: that read-ahead, dann_scan_gettuple one row at a time, and the CPU oracle on one thread.
Before anything is timed, the rows of both GPU ways equal the oracle's for every query.

Reports rows streamed per query and queries/s of each way, the p50 of one dann_scan_fetch(n) right after amrescan for
n = 1, 16, 256 and 4096, and the card's name and power limit from the same run.

    python tools/scan_fetch.py                               # 1M x 768, L = 100, rescore = 200
    python tools/scan_fetch.py --n 20000000 --L 600 --rescore 600

Writes one JSON line to stdout and profiles/h100_scan_fetch_<n>.json, n in millions when whole (or under --out-dir)."""
from __future__ import annotations

import argparse
import json
import os
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

from tools.deep_scan import FILTERS, LIMIT, passes  # noqa: E402
from tools.scan_many import _pct, card  # noqa: E402

FETCH_SIZES = [1, 16, 256, 4096]


def limit_read_ahead(sc, q, L, rescore, m, cap):
    """LIMIT 10 through a read-ahead buffer: fetch 1, 2, 4, ... rows (at most cap) whenever it runs dry"""
    sc.rescan(q, None, L, rescore)
    got, n, ask = [], 0, 1
    while len(got) < LIMIT:
        blk, off, _, _, _ = sc.fetch(ask)
        for b, o in zip(blk.tolist(), off.tolist()):
            n += 1
            tid = (b << 16) | o
            if passes(tid, m):
                got.append(tid)
                if len(got) == LIMIT:
                    break
        if len(blk) < ask:
            break
        ask = min(2 * ask, cap)
    return n, got


def limit_single(sc, q, L, rescore, m):
    """LIMIT 10 through dann_scan_gettuple, one row per call"""
    sc.rescan(q, None, L, rescore)
    got, n = [], 0
    while len(got) < LIMIT:
        r = sc.gettuple()
        if r is None:
            break
        n += 1
        tid = (r[0] << 16) | r[1]
        if passes(tid, m):
            got.append(tid)
    return n, got


def limit_oracle(oracle, snap, q, L, rescore, m, n):
    ref = oracle.scan(snap, q, None, L, rescore, n)
    return [int(t) for t in ref["tid"] if passes(int(t), m)][:LIMIT]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--n", type=int, default=1_000_000)
    ap.add_argument("--dim", type=int, default=768)
    ap.add_argument("--data", default="lowrank", choices=["lowrank", "gaussian"])
    ap.add_argument("--bits", type=int, default=0)
    ap.add_argument("--L", type=int, default=100)
    ap.add_argument("--rescore", type=int, default=200)
    ap.add_argument("--cap", type=int, default=4096, help="largest fetch of the read-ahead buffer")
    ap.add_argument("--queries", type=int, default=4, help="queries of each post-filter workload")
    ap.add_argument("--out-dir", default=os.path.join(ROOT, "profiles"))
    args = ap.parse_args()
    import torch
    from oracle import oracle
    from pgvectorscale_b200 import diskann
    from tools import fixture as fx
    if diskann.device_count() < 1:
        raise SystemExit("scan_fetch: no CUDA device visible")
    oracle.build_lib()
    device = torch.device("cuda", 0)
    info = card()
    n, dim, L, rescore = args.n, args.dim, args.L, args.rescore
    log = lambda *a: print(*a, file=sys.stderr, flush=True)
    snap, idx, _ = fx.codes_and_graph(n, dim, args.data, args.bits, device, log=log, download_nbrs=True)
    X = torch.empty((n, dim), dtype=torch.float32, device=device)
    fx.fill_rows(X, n, dim, args.data, device)
    idx.set_vectors_device(X.data_ptr())
    q = fx.gen_queries(args.queries + 1, 1, dim, args.data, device).cpu().numpy()
    sparse = fx.SparseRows(n, dim)                                # the heap rows the oracle's rerank reads
    snap.vectors = sparse.arr
    sc = idx.begin_scan()
    try:
        limit_read_ahead(sc, q[0], L, rescore, 100, args.cap)     # warm-up: module loads, workspace allocations
        limit_single(sc, q[0], L, rescore, 100)
        # one fetch(n) right after amrescan
        fetch_ms = {}
        for size in FETCH_SIZES:
            ms = []
            for rep in range(5):
                for qi in range(1, len(q)):
                    sc.rescan(q[qi], None, L, rescore)
                    t = time.perf_counter()
                    sc.fetch(size)
                    if rep:
                        ms.append((time.perf_counter() - t) * 1e3)
            fetch_ms[str(size)] = {"p50_ms": _pct(ms, 0.5), "calls": len(ms)}
        log(json.dumps({"fetch_after_rescan": fetch_ms}))
        post = []
        for m in FILTERS:
            # identical rows before anything is timed
            streamed = []
            for qq in q[1:]:
                na, rows_a = limit_read_ahead(sc, qq, L, rescore, m, args.cap)
                ns, rows_s = limit_single(sc, qq, L, rescore, m)
                assert rows_a == rows_s and na == ns, f"post-filter 1/{m}: read-ahead and gettuple differ"
                streamed.append(ns)
            need = fx.oracle_rerank_rows(oracle, snap, q[1:], L, rescore, max(streamed), fx.host_cores()["effective"])
            sparse.fill_from_device(need, X)
            for qq, ns in zip(q[1:], streamed):
                ref = limit_oracle(oracle, snap, qq, L, rescore, m, ns)
                assert limit_single(sc, qq, L, rescore, m)[1] == ref, f"post-filter 1/{m}: GPU rows differ from the oracle's"
            # timed: the three ways alternate query by query
            secs = {"read_ahead": 0.0, "gettuple": 0.0, "oracle": 0.0}
            for qq, ns in zip(q[1:], streamed):
                t = time.perf_counter()
                limit_read_ahead(sc, qq, L, rescore, m, args.cap)
                secs["read_ahead"] += time.perf_counter() - t
                t = time.perf_counter()
                limit_single(sc, qq, L, rescore, m)
                secs["gettuple"] += time.perf_counter() - t
                t = time.perf_counter()
                limit_oracle(oracle, snap, qq, L, rescore, m, ns)
                secs["oracle"] += time.perf_counter() - t
            nq = len(streamed)
            post.append({"passes_one_in": m, "limit": LIMIT, "queries": nq, "rows_streamed": streamed,
                         "read_ahead_queries_per_s": round(nq / secs["read_ahead"], 2),
                         "gettuple_queries_per_s": round(nq / secs["gettuple"], 2),
                         "oracle_1_thread_queries_per_s": round(nq / secs["oracle"], 2),
                         "rows_identical_to_oracle": True})
            log(json.dumps(post[-1]))
    finally:
        sc.end()
    line = {"metric": f"LIMIT {LIMIT} under a post-filter with read-ahead dann_scan_fetch, {n}x{dim}-d SBQ diskann index",
            "card": info,
            "config": {"n": n, "dim": dim, "search_list_size": L, "rescore": rescore, "data": args.data,
                       "read_ahead": f"fetch 1, 2, 4, ... up to {args.cap} rows whenever the buffer runs dry"},
            "fetch_after_rescan": fetch_ms, "post_filter": post,
            "timing": "host clock around each query (every call ends in a device synchronise); oracle: one thread"}
    os.makedirs(args.out_dir, exist_ok=True)
    size = f"{n // 1_000_000}m" if n % 1_000_000 == 0 else str(n)
    with open(os.path.join(args.out_dir, f"h100_scan_fetch_{size}.json"), "w") as f:
        json.dump(line, f, indent=1)
    print(json.dumps(line))
    idx.close()


if __name__ == "__main__":
    main()
