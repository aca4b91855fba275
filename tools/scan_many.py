"""Many streaming scans at once: N scans, each amrescan + 10 x amgettuple, through dann_scan_gettuple_many (one call per
row for all N scans) and, on the same scans, one by one through dann_scan_gettuple.  Reports, per N: scans/s and the
p50 / p95 latency of one _many call, the same N scans one by one, the dann_scan_rescan time, and how many scans one SM
holds at once under each scan's plan.  Asserts that both paths return the same rows, and the oracle's on a 16-scan
sample.  Records the card's name and power limit from the same run.

    python tools/scan_many.py                    # configs[1]: 1M x 768, L = 100, rescore = 200
    python tools/scan_many.py --n 20000000 --L 600 --rescore 600

Writes one JSON line to stdout and profiles/h100_scan_many_<n>.json, n in millions when whole (or under --out-dir)."""
from __future__ import annotations

import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

ROWS = 10
SMEM_PER_SM = 233472      # sm_90: 228 KB of shared memory per SM
SMEM_PER_CTA_RESERVED = 1024
STATIC_SMEM = 400         # dann_scan_search_many_kernel's static shared memory (its SearchArgs copy), -Xptxas -v
SLACK = 128               # DANN_SMEM_SLACK
REG_CTAS = 12             # __launch_bounds__(32, 12)


def _pct(v, p):
    v = sorted(v)
    return round(v[min(len(v) - 1, int(len(v) * p))], 4)


def card():
    r = subprocess.run(["nvidia-smi", "--id=0", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                       capture_output=True, text=True)
    name, power = (r.stdout.strip().split(", ") + ["?", "?"])[:2]
    return {"name": name, "power_limit": power}


def scans_per_sm(idx, q, L, rescore):
    """Resident scans per SM under the scan's plan: dann_scan_rescan plans make_plan(nq = 1, c_target = rescore + 64)
    of the single-warp kernel; a one-query DANN_SEARCH_KERNEL=1 batch plans the same when its c_target is equal.  A
    batch streams rescore + k - 1 rows (k with rescore = 0), so k = 65 (64 with rescore = 0)."""
    os.environ["DANN_SEARCH_KERNEL"] = "1"
    try:
        idx.search_batch(q[:1], k=65 if rescore else 64, search_list_size=L, rescore=rescore)
        p = idx.last_search_plan()
    finally:
        del os.environ["DANN_SEARCH_KERNEL"]
    per_cta = p["smem_per_slot"] + SLACK + STATIC_SMEM + SMEM_PER_CTA_RESERVED
    return {"smem_per_scan_bytes": p["smem_per_slot"], "heap_smem_entries": p["heap_smem"],
            "scans_per_sm": min(SMEM_PER_SM // per_cta, REG_CTAS, 32)}


def run_n(lib, idx, q, N, L, rescore):
    """N scans: rescan + ROWS rows through gettuple_many, then the same scans again one by one."""
    scans = [idx.begin_scan() for _ in range(N)]
    try:
        t0 = time.perf_counter()
        rescan_ms = []
        for i, sc in enumerate(scans):
            t = time.perf_counter()
            sc.rescan(q[i], None, L, rescore)
            rescan_ms.append((time.perf_counter() - t) * 1e3)
        call_ms, many_rows = [], []
        for _ in range(ROWS):
            t = time.perf_counter()
            out = lib.gettuple_many(scans)
            call_ms.append((time.perf_counter() - t) * 1e3)
            many_rows.append(out)
        many_s = time.perf_counter() - t0
        t0 = time.perf_counter()
        single_rows = [[] for _ in range(ROWS)]
        for i, sc in enumerate(scans):
            sc.rescan(q[i], None, L, rescore)
            for r in range(ROWS):
                single_rows[r].append(sc.gettuple())
        single_s = time.perf_counter() - t0
    finally:
        for sc in scans:
            sc.end()
    for r in range(ROWS):
        for a in many_rows[r]:
            assert not isinstance(a, Exception), a
    key = lambda x: None if x is None else x[:3] + (int(np.float32(x[3]).view(np.uint32)),)   # NaN-safe
    assert [[key(x) for x in row] for row in many_rows] == [[key(x) for x in row] for row in single_rows], \
        "gettuple_many and gettuple returned different rows"
    tids = np.array([[(x[0] << 16) | x[1] if x else 0xFFFFFFFFFFFFFFFF for x in row] for row in many_rows], np.uint64).T
    return {"scans": N,
            "many": {"scans_per_s": round(N / many_s, 1), "call_ms": {"p50": _pct(call_ms, 0.5), "p95": _pct(call_ms, 0.95)}},
            "one_by_one": {"scans_per_s": round(N / single_s, 1)},
            "rescan_ms": {"p50": _pct(rescan_ms, 0.5), "p95": _pct(rescan_ms, 0.95)}}, tids


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--n", type=int, default=1_000_000)
    ap.add_argument("--dim", type=int, default=768)
    ap.add_argument("--data", default="lowrank", choices=["lowrank", "gaussian"])
    ap.add_argument("--bits", type=int, default=0)
    ap.add_argument("--L", type=int, default=100)
    ap.add_argument("--rescore", type=int, default=200)
    ap.add_argument("--counts", default="1,16,132,528")
    ap.add_argument("--out-dir", default=os.path.join(ROOT, "profiles"))
    args = ap.parse_args()
    import torch
    from oracle import oracle
    from pgvectorscale_b200 import diskann
    from tools import fixture as fx
    if diskann.device_count() < 1:
        raise SystemExit("scan_many: no CUDA device visible")
    oracle.build_lib()
    device = torch.device("cuda", 0)
    info = card()
    n, dim, L, rescore = args.n, args.dim, args.L, args.rescore
    counts = [int(c) for c in args.counts.split(",")]
    log = lambda *a: print(*a, file=sys.stderr, flush=True)
    snap, idx, _ = fx.codes_and_graph(n, dim, args.data, args.bits, device, log=log, download_nbrs=True)
    X = torch.empty((n, dim), dtype=torch.float32, device=device)
    fx.fill_rows(X, n, dim, args.data, device)
    idx.set_vectors_device(X.data_ptr())
    q = fx.gen_queries(max(counts), 1, dim, args.data, device).cpu().numpy()
    plan = scans_per_sm(idx, q, L, rescore)
    run_n(diskann, idx, q, 16, L, rescore)                     # warm-up: module loads, workspace allocations
    runs, first16 = [], None
    for N in counts:
        try:
            r, tids = run_n(diskann, idx, q, N, L, rescore)
        except diskann.DiskAnnError as e:                        # HBM: the scans' workspaces beside the index
            runs.append({"scans": N, "error": str(e)})
            continue
        runs.append(r)
        if first16 is None and N >= 16:
            first16 = tids[:16]
        log(json.dumps(r))
    # the oracle on a 16-scan sample: the heap rows its rerank reads, then its scans
    rows = fx.SparseRows(n, dim)
    snap.vectors = rows.arr
    rows.fill_from_device(fx.oracle_rerank_rows(oracle, snap, q[:16], L, rescore, ROWS, fx.host_cores()["effective"]), X)
    ref = np.array([oracle.scan(snap, q[i], None, L, rescore, ROWS)["tid"] for i in range(16)], np.uint64)
    oracle_ok = first16 is not None and bool(np.array_equal(first16, ref))
    assert oracle_ok, "gettuple_many rows differ from the oracle's"
    line = {"metric": f"streaming scans through dann_scan_gettuple_many, {n}x{dim}-d SBQ diskann index",
            "unit": "scans/s", "card": info,
            "config": {"n": n, "dim": dim, "search_list_size": L, "rescore": rescore, "rows_per_scan": ROWS,
                       "data": args.data},
            "plan": plan, "runs": runs,
            "parity": {"many_equals_one_by_one": True, "oracle_sample_16": oracle_ok}}
    os.makedirs(args.out_dir, exist_ok=True)
    size = f"{n // 1_000_000}m" if n % 1_000_000 == 0 else str(n)
    with open(os.path.join(args.out_dir, f"h100_scan_many_{size}.json"), "w") as f:
        json.dump(line, f, indent=1)
    print(json.dumps(line))
    idx.close()


if __name__ == "__main__":
    main()
