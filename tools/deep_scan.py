"""How a streaming scan behaves in depth: one scan of the index drained row by row, and LIMIT 10 under a selective
post-filter.  The scan regrows its planned workspace by replay until that can grow no further, then enters the deep
mode (dann_scan_gettuple in include/diskann_b200.h) and grows in place.

Reports
  - p50 / p99 time of one amgettuple (a host clock around dann_scan_gettuple, which ends in a device synchronise) in
    windows of streamed depth: rows 1-100, 101-1k, 1k-10k, 10k-100k, 100k-1M;
  - the row at which the scan entered the deep mode: where the parent commit's scan failed with DANN_ERR_CAPACITY
    (the handoff is exactly where scan_regrow or dann_make_plan used to return it), or null if it never did;
  - the time of every call that ran a replay regrow, and of every call that grew the deep workspace in place;
  - post-filter: LIMIT 10 under a deterministic predicate on the TID passing 1/100, 1/1000 and 1/10000 of rows: rows
    streamed per query and queries/s, against the CPU oracle streaming the same queries on one thread.  The GPU's rows
    equal the oracle's for every query before anything is timed.
Records the card's name and power limit from the same run.

    python tools/deep_scan.py                               # 1M x 768, L = 100, rescore = 200
    python tools/deep_scan.py --n 20000000 --L 600 --rescore 600

Writes one JSON line to stdout and profiles/h100_deep_scan_<n>.json, n in millions when whole (or under --out-dir)."""
from __future__ import annotations

import argparse
import json
import os
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

from tools.scan_many import _pct, card  # noqa: E402

WINDOWS = [(1, 100), (101, 1_000), (1_001, 10_000), (10_001, 100_000), (100_001, 1_000_000)]
FILTERS = [100, 1_000, 10_000]
LIMIT = 10


def passes(tid: int, m: int) -> bool:
    """the post-filter: a multiplicative hash of the TID, one row in m"""
    return ((tid * 0x9E3779B97F4A7C15) & 0xFFFFFFFFFFFFFFFF) >> 40 < (1 << 24) // m


def drain(idx, q, L, rescore, depth):
    """one scan, up to `depth` rows: the time of every call and the workspace after it"""
    sc = idx.begin_scan()
    ms, events, tids = [], [], []
    deep_at = None
    try:
        sc.rescan(q, None, L, rescore)
        last = sc.workspace()
        for i in range(1, depth + 1):
            t = time.perf_counter()
            r = sc.gettuple()
            dt = (time.perf_counter() - t) * 1e3
            if r is None:
                break
            ms.append(dt)
            tids.append((r[0] << 16) | r[1])
            ws = sc.workspace()
            if ws["regrows"] != last["regrows"]:
                events.append({"row": i, "kind": "replay regrow", "regrows": ws["regrows"], "ms": round(dt, 3)})
            if ws["mode"] == 1 and deep_at is None:
                deep_at = i
                events.append({"row": i, "kind": "deep mode entry", "ms": round(dt, 3), "device_bytes": ws["device_bytes"]})
            elif ws["growths"] != last["growths"]:
                events.append({"row": i, "kind": "in-place growth", "growths": ws["growths"], "ms": round(dt, 3),
                               "device_bytes": ws["device_bytes"]})
            last = ws
        final = sc.workspace()
    finally:
        sc.end()
    windows = []
    for lo, hi in WINDOWS:
        w = ms[lo - 1:hi]
        windows.append({"rows": f"{lo}-{hi}", "calls": len(w), **({"p50_ms": _pct(w, 0.5), "p99_ms": _pct(w, 0.99)}
                                                                 if w else {"not_reached": True})})
    return {"rows_streamed": len(ms), "deep_mode_entered_at_row": deep_at, "windows": windows, "events": events,
            "final_workspace": final, "total_s": round(sum(ms) / 1e3, 2)}, np.array(tids, np.uint64)


def post_filter_gpu(idx, queries, L, rescore, m):
    """LIMIT 10 under the predicate: rows streamed per query, matching TIDs, seconds"""
    sc = idx.begin_scan()
    streamed, rows = [], []
    try:
        t0 = time.perf_counter()
        for q in queries:
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
            streamed.append(n)
            rows.append(got)
        secs = time.perf_counter() - t0
    finally:
        sc.end()
    return streamed, rows, secs


def post_filter_oracle(oracle, snap, queries, L, rescore, m, streamed):
    """the oracle streaming the same queries on one thread, as far as the GPU streamed each"""
    rows = []
    t0 = time.perf_counter()
    for q, n in zip(queries, streamed):
        ref = oracle.scan(snap, q, None, L, rescore, n)
        rows.append([int(t) for t in ref["tid"] if passes(int(t), m)][:LIMIT])
    return rows, time.perf_counter() - t0


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--n", type=int, default=1_000_000)
    ap.add_argument("--dim", type=int, default=768)
    ap.add_argument("--data", default="lowrank", choices=["lowrank", "gaussian"])
    ap.add_argument("--bits", type=int, default=0)
    ap.add_argument("--L", type=int, default=100)
    ap.add_argument("--rescore", type=int, default=200)
    ap.add_argument("--depth", type=int, default=1_000_000, help="rows the depth drain streams at most")
    ap.add_argument("--queries", type=int, default=4, help="queries of each post-filter workload")
    ap.add_argument("--out-dir", default=os.path.join(ROOT, "profiles"))
    args = ap.parse_args()
    import torch
    from oracle import oracle
    from pgvectorscale_b200 import diskann
    from tools import fixture as fx
    if diskann.device_count() < 1:
        raise SystemExit("deep_scan: no CUDA device visible")
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
    post_filter_gpu(idx, q[1:3], L, rescore, 100)                 # warm-up: module loads, workspace allocations
    log("[deep_scan] depth drain")
    depth, _ = drain(idx, q[0], L, rescore, min(args.depth, n))
    log(json.dumps({k: v for k, v in depth.items() if k != "events"}))
    post = []
    sparse = fx.SparseRows(n, dim)                                # the heap rows the oracle's rerank reads
    snap.vectors = sparse.arr
    for m in FILTERS:
        streamed, rows, gpu_s = post_filter_gpu(idx, q[1:], L, rescore, m)
        # the oracle's scans on the rows they rerank: identical rows before any number is kept
        need = fx.oracle_rerank_rows(oracle, snap, q[1:], L, rescore, max(streamed), fx.host_cores()["effective"])
        sparse.fill_from_device(need, X)
        ref_rows, cpu_s = post_filter_oracle(oracle, snap, q[1:], L, rescore, m, streamed)
        assert rows == ref_rows, f"post-filter 1/{m}: GPU rows differ from the oracle's"
        streamed, rows, gpu_s = post_filter_gpu(idx, q[1:], L, rescore, m)   # timed run, after the check
        assert rows == ref_rows
        nq = len(rows)
        post.append({"passes_one_in": m, "limit": LIMIT, "queries": nq, "rows_streamed": streamed,
                     "gpu_queries_per_s": round(nq / gpu_s, 2), "oracle_1_thread_queries_per_s": round(nq / cpu_s, 2),
                     "rows_identical_to_oracle": True})
        log(json.dumps(post[-1]))
    line = {"metric": f"streaming scan in depth, {n}x{dim}-d SBQ diskann index", "card": info,
            "config": {"n": n, "dim": dim, "search_list_size": L, "rescore": rescore, "data": args.data,
                       "depth_limit": min(args.depth, n)},
            "depth": depth, "post_filter": post,
            "timing": "host clock around each dann_scan_gettuple (it ends in a device synchronise); oracle: one thread"}
    os.makedirs(args.out_dir, exist_ok=True)
    size = f"{n // 1_000_000}m" if n % 1_000_000 == 0 else str(n)
    with open(os.path.join(args.out_dir, f"h100_deep_scan_{size}.json"), "w") as f:
        json.dump(line, f, indent=1)
    print(json.dumps(line))
    idx.close()


if __name__ == "__main__":
    main()
