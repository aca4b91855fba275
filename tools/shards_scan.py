"""Latency of the sharded streaming scan on the 20M x 768-d table (tools/shards.py's fixture and shard split) in 1, 2, 4
and 8 shards on one GPU -> profiles/h100_shards_scan_20m.json.

For each shard count, at its operating point (profiles/h100_shards_20m.json for 1, 2 and 4 shards; for 8 the first
point of bench.py's sweep with recall@10 >= 0.99 on the selection sample, the rule tools/shards.py applies), one query
at a time: amrescan + the first row, and amrescan + 10 rows, each timed two ways, alternating query by query in the
same run:
  (a) ShardedScan: one rescan of every shard, the first gettuple steps the shards together in one launch round, later
      calls one shard each;
  (b) one private IndexScan per shard, rescanned and stepped one after another and merged on the host by the same
      rule - what an executor's Merge Append over per-partition index scans does.
Checks: the rows of (a) equal those of (b), and the first 10 equal ShardedIndex.search_batch(k=10).  Host clock around
calls that each end in a device synchronisation.

    python tools/shards_scan.py [--n 20000000] [--shards 1,2,4,8] [--queries 200] [--out ...]
"""
from __future__ import annotations

import argparse
import json
import os
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
import numpy as np
import torch

import bench
from tools import shards as sd

K = sd.K


def merged_private(scans, q, L, rescore, rows):
    """(b): every shard's private scan rescanned, then stepped one after another for its head, merged on the host:
    each row is the head with the smallest (total_cmp key, shard), and only that shard steps again"""
    from shard_model import total_ukey
    for sc in scans:
        sc.rescan(q, search_list_size=L, rescore=rescore)
    heads = [sc.gettuple() for sc in scans]
    out = []
    while len(out) < rows:
        live = [(int(total_ukey(np.array([h[3]], np.float32))[0]), s) for s, h in enumerate(heads) if h is not None]
        if not live:
            break
        s = min(live)[1]
        out.append(heads[s] + (s,))
        if len(out) < rows:
            heads[s] = scans[s].gettuple()
    return out


def sharded(scan, q, L, rescore, rows):
    """(a)"""
    scan.rescan(q, search_list_size=L, rescore=rescore)
    out = []
    for _ in range(rows):
        r = scan.gettuple()
        if r is None:
            break
        out.append(r)
    return out


def pct(ts):
    return {"p50_ms": round(float(np.percentile(ts, 50)) * 1e3, 3), "p95_ms": round(float(np.percentile(ts, 95)) * 1e3, 3)}


def choose_point(sh, qh, truth):
    sweep = []
    for L, rescore in bench.SWEEP_LARGE:
        out = sh.search_batch(qh[:bench.SEL], k=K, search_list_size=L, rescore=rescore)
        rec = bench.recall_at_k(out["tid"], truth[:bench.SEL], K)
        sweep.append({"L": L, "rescore": rescore, "recall_selection_sample": round(rec, 4)})
        if rec >= 0.99:
            return sweep[-1], sweep
    return sweep[-1], sweep


def run(n, S, data, points, nq, warm):
    res = {"shards": S, "gpus": sd.gpu_info()}
    t0 = time.time()
    built = sd.build_sharded(n, S, [0] * S, data, res)
    if built is None:
        return res
    sh, snaps, gids, X, q, truth = built
    qh = q.cpu().numpy()
    res["fixture_s"] = round(time.time() - t0, 1)
    if S in points:
        L, rescore = points[S]
        res["operating_point"] = {"L": L, "rescore": rescore, "from": "profiles/h100_shards_20m.json"}
    else:
        pt, sweep = choose_point(sh, qh, truth)
        L, rescore = pt["L"], pt["rescore"]
        res["operating_point"] = dict(pt, sweep=sweep)
    sd.log(f"[shards_scan] S={S} L={L} rescore={rescore}")
    scan = sh.begin_scan()
    private = [sh.shard(i).begin_scan() for i in range(S)]
    batch = sh.search_batch(qh[:nq + warm], k=K, search_list_size=L, rescore=rescore)
    t = {(w, rows): [] for w in "ab" for rows in (1, 10)}
    mismatch = {"a_vs_b": 0, "a_vs_batch": 0}
    for j in range(nq + warm):
        for rows in (1, 10):
            order = (("a", sharded, scan), ("b", merged_private, private))
            for w, fn, obj in (order if j % 2 == 0 else order[::-1]):
                t1 = time.perf_counter()
                got = fn(obj, qh[j], L, rescore, rows)
                dt = time.perf_counter() - t1
                if j >= warm:
                    t[(w, rows)].append(dt)
                if w == "a":
                    ra = got
                else:
                    rb = got
            mismatch["a_vs_b"] += ra != rb
            if rows == 10:
                n_b = int(batch["count"][j])
                same = ([(r[0] << 16) | r[1] for r in ra] == batch["tid"][j, :n_b].tolist() and
                        [r[4] for r in ra] == batch["shard"][j, :n_b].tolist() and
                        np.array([r[3] for r in ra], np.float32).view(np.uint32).tolist() ==
                        batch["dist"][j, :n_b].view(np.uint32).tolist())
                mismatch["a_vs_batch"] += not same
    res["queries_timed"] = nq
    res["first_row"] = {"sharded_scan": pct(t[("a", 1)]), "one_after_another": pct(t[("b", 1)])}
    res["ten_rows"] = {"sharded_scan": pct(t[("a", 10)]), "one_after_another": pct(t[("b", 10)])}
    for key in ("first_row", "ten_rows"):
        r = res[key]
        r["p50_speedup"] = round(r["one_after_another"]["p50_ms"] / r["sharded_scan"]["p50_ms"], 2)
    res["checks"] = dict(mismatch, queries=nq + warm, ok=mismatch["a_vs_b"] == 0 and mismatch["a_vs_batch"] == 0)
    sd.log(f"[shards_scan] S={S} {res}")
    scan.end()
    for p in private:
        p.end()
    sh.close()
    del X
    torch.cuda.empty_cache()
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--n", type=int, default=20_000_000)
    ap.add_argument("--shards", default="1,2,4,8")
    ap.add_argument("--data", default="lowrank")
    ap.add_argument("--queries", type=int, default=200)
    ap.add_argument("--warmup", type=int, default=10)
    ap.add_argument("--points", default=os.path.join(ROOT, "profiles", "h100_shards_20m.json"))
    ap.add_argument("--out", default=os.path.join(ROOT, "profiles", "h100_shards_scan_20m.json"))
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("tools/shards_scan.py measures on a GPU; none is visible")
    points = {}
    if a.n == 20_000_000:       # the committed operating points belong to the 20M table only
        with open(a.points) as f:
            for r in json.load(f)["by_shards"]:
                if "operating_point" in r:
                    points[r["shards"]] = (r["operating_point"]["L"], r["operating_point"]["rescore"])
    doc = {"gpus_before": sd.gpu_info(),
           "table": f"{a.n} x {sd.DIM}-d {a.data}, 2-bit SBQ, chunk c -> shard c mod S, every shard on GPU 0",
           "timing": "host clock per call sequence, p50/p95 over the timed queries; (a) ShardedScan, (b) private "
                     "IndexScans one after another merged on the host; (a) and (b) alternate query by query",
           "by_shards": []}
    os.makedirs(os.path.dirname(a.out), exist_ok=True)
    for S in [int(x) for x in a.shards.split(",")]:
        doc["by_shards"].append(run(a.n, S, a.data, points, a.queries, a.warmup))
        doc["gpus_after"] = sd.gpu_info()
        with open(a.out, "w") as f:         # after every shard count: a partial run still leaves its results
            json.dump(doc, f, indent=1)
    print(json.dumps({"out": a.out, "checks": [r.get("checks", {}).get("ok") for r in doc["by_shards"]]}))


if __name__ == "__main__":
    main()
