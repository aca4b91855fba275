"""Where the lean search kernel's time goes at the 20M x 768-d headline: its occupancy curve.

   python tools/visit_budget.py [--n 20000000 --batch 4096 --L 600 --rescore 600 --warps 8,12,16,32 --rounds 3]
   python tools/visit_budget.py --lib OTHER/libdiskann_b200.so --warps 16 ...   (the same with another build)

Builds the bench's index fixture (tools/fixture.py: same rows, same GPU-built graph, same queries), then times the
search kernel (dann_search3_kernel, CUDA events around it: dann_last_batch_timing.search_ms) at each number of resident
query slots per SM (DANN_SEARCH_WARPS, read on every call), the slot counts alternating round by round.  For each it
records the search time per launch and visits per microsecond per SM (visits from the per-query counters).  A curve
that stays flat as slots are added means the kernel is at a throughput wall (memory transactions), not bound by the
latency of one query's chain; a rising curve means more resident queries still hide latency.  The card's name and power
limit are read in the same run.  One JSON document on stdout (and in --out)."""
from __future__ import annotations

import argparse
import json
import os
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

import numpy as np  # noqa: E402


def card():
    q = "name,power.limit,clocks.max.sm"
    try:
        out = subprocess.run(["nvidia-smi", f"--query-gpu={q}", "--format=csv,noheader"], capture_output=True,
                             text=True, timeout=30).stdout.strip().splitlines()
        name, pl, clk = [x.strip() for x in out[0].split(",")]
        return {"name": name, "power_limit": pl, "max_sm_clock": clk}
    except Exception as e:  # the numbers are still device-timed; the card is then "not read"
        return {"error": f"nvidia-smi not read: {e}"}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--n", type=int, default=20_000_000)
    ap.add_argument("--dim", type=int, default=768)
    ap.add_argument("--batch", type=int, default=4096)
    ap.add_argument("--k", type=int, default=10)
    ap.add_argument("--L", type=int, default=600)
    ap.add_argument("--rescore", type=int, default=600)
    ap.add_argument("--warps", default="8,12,16,32")
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--steps", type=int, default=4, help="timed launches per slot count per round")
    ap.add_argument("--lib", default=None, help="library to time (default: the in-tree build)")
    ap.add_argument("--out", default=None)
    ap.add_argument("--dump", default=None, help="write the rows and counters of the first batch as DIR/rows.npz")
    a = ap.parse_args()

    import torch
    from pgvectorscale_b200 import diskann
    from tools import fixture as fx

    if a.lib:
        diskann._LIB = diskann.load_library(os.path.abspath(a.lib))
    device = torch.device("cuda", 0)
    log = lambda *x: print(*x, file=sys.stderr, flush=True)  # noqa: E731
    t0 = time.time()
    _, idx, _ = fx.codes_and_graph(a.n, a.dim, "lowrank", 0, device, log=log, download_nbrs=False)
    B = a.batch
    nb = 1 + a.steps
    q_all = fx.gen_queries(B, nb, a.dim, "lowrank", device)
    torch.cuda.empty_cache()
    X = torch.empty((a.n, a.dim), dtype=torch.float32, device=device)
    fx.fill_rows(X, a.n, a.dim, "lowrank", device)
    idx.set_vectors_device(X.data_ptr())
    torch.cuda.empty_cache()
    log(f"[visit_budget] fixture {time.time() - t0:.1f}s")

    stream = torch.cuda.Stream(device)
    d_tid = torch.empty((B, a.k), dtype=torch.int64, device=device)
    d_dist = torch.empty((B, a.k), dtype=torch.float32, device=device)
    d_cnt = torch.empty(B, dtype=torch.int32, device=device)
    d_stats = torch.empty((B, 6), dtype=torch.int32, device=device)
    sm_count = torch.cuda.get_device_properties(device).multi_processor_count

    def run(qb):
        idx.search_batch_device(qb, a.k, a.L, a.rescore, d_tid, d_dist, d_cnt, d_stats, stream=stream.cuda_stream)
        torch.cuda.synchronize(device)
        return idx.last_batch_timing()

    warps = [int(w) for w in a.warps.split(",")]
    res = {w: {"search_ms": [], "visits": 0.0, "candidates": 0.0, "plan": None} for w in warps}
    ref_rows = None
    for r in range(a.rounds):
        for w in (warps if r % 2 == 0 else warps[::-1]):
            os.environ["DANN_SEARCH_WARPS"] = str(w)
            run(q_all[:B])  # a changed plan pays for its workspace here
            for s in range(1, nb):
                t = run(q_all[s * B:(s + 1) * B])
                res[w]["search_ms"].append(round(t["search_ms"], 4))
                st = d_stats.cpu().numpy().astype(np.float64)
                res[w]["visits"] += st[:, 0].sum()
                res[w]["candidates"] += st[:, 2].sum()
            res[w]["plan"] = idx.last_search_plan()
            run(q_all[:B])
            rows = (d_tid.cpu().numpy(), d_dist.cpu().numpy().view(np.uint32), d_stats.cpu().numpy())
            if ref_rows is None:
                ref_rows = rows
            res[w]["rows_equal_first"] = all(np.array_equal(x, y) for x, y in zip(rows, ref_rows))
    os.environ.pop("DANN_SEARCH_WARPS", None)
    if a.dump:  # what another build must return for the same batch: TIDs, distance bits, counters
        os.makedirs(a.dump, exist_ok=True)
        np.savez(os.path.join(a.dump, "rows.npz"), tid=ref_rows[0], dist_bits=ref_rows[1], stats=ref_rows[2])

    curve = []
    for w in warps:
        ms = np.array(res[w]["search_ms"])
        launches = len(ms)
        vis_per_launch = res[w]["visits"] / launches
        curve.append({
            "slots_per_sm": res[w]["plan"]["slots_per_sm"], "requested": w, "heap_smem": res[w]["plan"]["heap_smem"],
            "search_ms_median": round(float(np.median(ms)), 3), "search_ms_min": round(float(ms.min()), 3),
            "search_ms_max": round(float(ms.max()), 3), "launches": launches, "search_ms": res[w]["search_ms"],
            "visits_per_query": round(vis_per_launch / B, 1),
            "candidates_per_visit": round(res[w]["candidates"] / res[w]["visits"], 2),
            "visits_per_us_per_sm": round(vis_per_launch / (float(np.median(ms)) * 1e3) / sm_count, 4),
            "rows_and_counters_equal_across_slot_counts": bool(res[w]["rows_equal_first"]),
        })
    doc = {"what": "lean search kernel occupancy curve: search time and visit throughput vs resident query slots per SM",
           "workload": f"{a.n}x{a.dim}-d lowrank SBQ 2-bit index (tools/fixture.py), batch {B}, k={a.k}, "
                       f"L={a.L}, rescore={a.rescore}",
           "card": card(), "sm_count": sm_count, "library": os.path.abspath(a.lib) if a.lib else "in-tree build",
           "rounds": a.rounds, "timing": "CUDA events around the search kernel (dann_last_batch_timing.search_ms); "
                                         "slot counts alternate round by round", "curve": curve}
    txt = json.dumps(doc, indent=1)
    print(txt)
    if a.out:
        with open(a.out, "w") as f:
            f.write(txt + "\n")
    idx.close()


if __name__ == "__main__":
    main()
