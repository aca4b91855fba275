"""The 20M x 768-d config-3 table (tools/fixture.py chunks and seeds) split into 1, 2 and 4 shards on one GPU and served
through dann_shards (ShardedIndex) -> profiles/h100_shards_20m.json.

Chunk c of the table goes to shard c mod S.  Every shard gets its own SBQ means, its own graph (dann_build_graph, in
place through ShardedIndex.shard(i)) and its rows attached in place (set_vectors_device); heap TIDs stay global, so
recall is measured against the exact top-10 of the whole table (RunningTopK).  For each shard count: the bench.py
sweep over (L, rescore) on the host-buffer path up to the first point with recall@10 >= 0.99 on the selection sample,
parity there (a query sample against tests/shard_model.scan_shards, heap rows through SparseRows as bench.py takes
them), and at that point: queries/s, per-shard search and rerank times (dann_last_batch_timing) and the merge kernel's time
(torch.profiler, CUDA activities, in calls of their own).  A shard count that does not fit in HBM is recorded with
its error.  The 50M table needs at least three GPUs (one shard each); it is run only when that many are visible.

    python tools/shards.py [--n 20000000] [--shards 1,2,4] [--out profiles/h100_shards_20m.json]
"""
from __future__ import annotations

import argparse
import json
import os
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
import numpy as np
import torch

import bench
from tools import fixture as fx
from tools import synth_index as si

K, DIM, B = 10, 768, 4096


def log(*a):
    print(*a, file=sys.stderr, flush=True)


def gpu_info():
    r = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True)
    return [dict(zip(("name", "power_limit", "max_sm_clock"), l.split(", "))) for l in r.stdout.strip().splitlines()]


def shard_chunks(n, S):
    """chunk c -> shard c mod S: each shard's list of (chunk, global start, global end)"""
    out = [[] for _ in range(S)]
    for c, s, e in fx.chunks(n):
        out[c % S].append((c, s, e))
    return out


def shard_snapshot(n, parts, data, device):
    """means, SBQ codes and an empty 64-slot graph over one shard's chunks; heap TIDs of the rows' global positions"""
    from pgvectorscale_b200.snapshot import COSINE, INVALID_NODE, Snapshot, code_words, default_bits, make_heap_tids
    m = sum(e - s for _, s, e in parts)
    mean = torch.zeros(DIM, device=device, dtype=torch.float64)
    sq = torch.zeros(DIM, device=device, dtype=torch.float64)
    for c, s, e in parts:
        x = fx.gen_chunk(c, e - s, DIM, data, device).double()
        mean += x.sum(0)
        sq += (x * x).sum(0)
    mean /= m
    mean_h, m2_h = mean.float().cpu().numpy(), (sq - m * mean ** 2).float().cpu().numpy()
    bits = default_bits(DIM)
    codes = np.empty((m, code_words(DIM, bits)), np.uint64)
    gid = np.empty(m, np.int64)
    o = 0
    for c, s, e in parts:
        x = fx.gen_chunk(c, e - s, DIM, data, device)
        codes[o:o + e - s] = si.quantize_nodes(x, COSINE, bits, mean_h, m2_h, m)
        gid[o:o + e - s] = np.arange(s, e)
        o += e - s
    snap = Snapshot(n=m, dim=DIM, dim_index=DIM, bits=bits, words=codes.shape[1], R=64, distance_type=COSINE,
                    has_labels=False, count=m, mean=mean_h, m2=m2_h, codes=codes,
                    nbrs=np.full((m, 64), INVALID_NODE, np.uint32), heap_tid=make_heap_tids(n)[gid], vectors=None,
                    start_default=0)
    return snap, gid


def merge_ms(sh, q, L, rescore, calls=5):
    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(calls):
            sh.search_batch(q, k=K, search_list_size=L, rescore=rescore)
    ev = [e for e in prof.events() if "dann_shard_merge_kernel" in e.name]
    return round(sum(e.device_time for e in ev) / max(len(ev), 1) / 1e3, 4), len(ev)


def build_sharded(n, S, devices, data, res):
    """The table's S shards loaded, their graphs built and their rows attached, with B queries and the exact top-K of
    each over the whole table -> (ShardedIndex, snapshots, each shard's global row ids, each shard's device rows,
    queries on the first device, truth); None when it does not fit (res["error"] says why)."""
    from pgvectorscale_b200 import diskann
    dev0 = torch.device("cuda", devices[0])
    parts = shard_chunks(n, S)
    snaps, gids = [], []
    for i in range(S):
        s, g = shard_snapshot(n, parts[i], data, torch.device("cuda", devices[i]))
        snaps.append(s)
        gids.append(g)
    res["rows_per_shard"] = [s.n for s in snaps]
    q = fx.gen_queries(B, 1, DIM, data, dev0)
    topk = fx.RunningTopK(q, K)
    X = []
    sh = None
    try:
        sh = diskann.ShardedIndex(snaps, devices=devices)
        build = []
        for i in range(S):
            ix = sh.shard(i)
            st = ix.build_graph(50, 100, 1.2, 1 << 20)
            build.append(round(st["total_ms"] / 1e3, 1))
            snaps[i].nbrs = ix.download_nbrs()
            torch.cuda.empty_cache()
            x = torch.empty((snaps[i].n, DIM), dtype=torch.float32, device=torch.device("cuda", devices[i]))
            o = 0
            for c, s, e in parts[i]:
                y = fx.gen_chunk(c, e - s, DIM, data, x.device)
                x[o:o + e - s] = y
                topk.add(y.to(dev0), s)
                o += e - s
                del y
            ix.set_vectors_device(x.data_ptr())
            X.append(x)
        res["graph_build_s"] = build
    except (diskann.DiskAnnError, torch.OutOfMemoryError) as e:
        res["error"] = f"{type(e).__name__}: {e}"
        log(f"[shards] S={S}: {res['error']}")
        if sh is not None:
            sh.close()
        X.clear()
        torch.cuda.empty_cache()
        return None
    return sh, snaps, gids, X, q, topk.result()


def run(n, S, devices, data, parity_queries, reps):
    from oracle import oracle
    from shard_model import scan_shards
    res = {"shards": S, "devices": devices, "rows_per_shard": []}
    t0 = time.time()
    built = build_sharded(n, S, devices, data, res)
    if built is None:
        return res
    sh, snaps, gids, X, q, truth = built
    qh = q.cpu().numpy()
    res["fixture_s"] = round(time.time() - t0, 1)

    sweep, chosen = [], None
    for L, rescore in bench.SWEEP_LARGE:
        sh.search_batch(qh, k=K, search_list_size=L, rescore=rescore)
        ts = []
        for _ in range(reps):
            t = time.perf_counter()
            out = sh.search_batch(qh, k=K, search_list_size=L, rescore=rescore)
            ts.append(time.perf_counter() - t)
        rec = bench.recall_at_k(out["tid"], truth, K)
        rec_sel = bench.recall_at_k(out["tid"][:bench.SEL], truth[:bench.SEL], K)
        ms = float(np.median(ts)) * 1e3
        tim = [sh.shard(i).last_batch_timing() for i in range(S)]
        pt = {"L": L, "rescore": rescore, "recall": round(rec, 4), "recall_selection_sample": round(rec_sel, 4),
              "call_ms": round(ms, 2), "qps": round(B / ms * 1e3),
              "shard_search_ms": [round(t["search_ms"], 2) for t in tim],
              "shard_rerank_ms": [round(t["rerank_ms"], 2) for t in tim]}
        sweep.append(pt)
        log(f"[shards] S={S} {pt}")
        if rec_sel >= 0.99:
            chosen = pt
            break
    res["sweep"] = sweep
    if chosen is None:
        chosen = sweep[-1]
        res["warning"] = "recall 0.99 not reached; reported at the last sweep point"
    L, rescore = chosen["L"], chosen["rescore"]
    res["operating_point"] = chosen
    res["merge_kernel_ms"], res["merge_kernel_launches_profiled"] = merge_ms(sh, qh, L, rescore)

    # parity on a query sample: every shard's oracle scan over the heap rows it reranks, merged by the model
    ns = parity_queries
    for i in range(S):
        rows = fx.SparseRows(snaps[i].n, DIM)
        snaps[i].vectors = rows.arr
        need = fx.oracle_rerank_rows(oracle, snaps[i], qh[:ns], L, rescore, K, fx.host_cores()["effective"])
        rows.fill_from_device(np.searchsorted(gids[i], need), X[i])      # global node ids -> the shard's rows
    got = sh.search_batch(qh[:ns], k=K, search_list_size=L, rescore=rescore)
    tid, dist, shard, count, stats = scan_shards(snaps, qh[:ns], None, None, L, rescore, K)
    res["parity"] = {"queries": ns, "tids_identical": bool(np.array_equal(got["tid"], tid)),
                     "dist_bits_identical": bool(np.array_equal(got["dist"].view(np.uint32), dist.view(np.uint32))),
                     "shards_identical": bool(np.array_equal(got["shard"], shard)),
                     "counts_identical": bool(np.array_equal(got["count"], count)),
                     "counters_identical": all(bool(np.array_equal(got["stats"][f].astype(np.uint64), stats[f]))
                                               for f in ("visits", "d_quantized", "candidates", "d_full"))}
    res["parity"]["ok"] = all(res["parity"][k] for k in res["parity"] if k.endswith("identical"))
    log(f"[shards] S={S} parity {res['parity']}")
    sh.close()
    del X
    torch.cuda.empty_cache()
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--n", type=int, default=20_000_000)
    ap.add_argument("--shards", default="1,2,4")
    ap.add_argument("--data", default="lowrank")
    ap.add_argument("--parity-queries", type=int, default=64)
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--out", default=os.path.join(ROOT, "profiles", "h100_shards_20m.json"))
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("tools/shards.py measures on a GPU; none is visible")
    ndev = torch.cuda.device_count()
    doc = {"gpus": gpu_info(), "table": f"{a.n} x {DIM}-d {a.data}, 2-bit SBQ, batch {B}, k={K}, chunk c -> shard c mod S",
           "by_shards": []}
    for S in [int(x) for x in a.shards.split(",")]:
        doc["by_shards"].append(run(a.n, S, [0] * S, a.data, a.parity_queries, a.reps))
    if ndev >= 3:
        doc["n50m"] = run(50_000_000, ndev, list(range(ndev)), a.data, a.parity_queries, a.reps)
    else:
        doc["n50m"] = f"not measured: one shard per GPU needs at least three GPUs, {ndev} visible"
    os.makedirs(os.path.dirname(a.out), exist_ok=True)
    with open(a.out, "w") as f:
        json.dump(doc, f, indent=1)
    print(json.dumps({"out": a.out, "parity": [r.get("parity", {}).get("ok") for r in doc["by_shards"]]}))


if __name__ == "__main__":
    main()
