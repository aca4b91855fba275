"""Serving traffic whose queries differ in k, search_list_size, rescore and key, on a 1M x 768 labeled index.

(a) The same B queries of four parameter classes, run two ways in alternation: one dann_search_batch_mixed call, and one
    dann_search_batch per class back to back (what the coalescer dispatched while it only merged requests of equal
    parameters).  Per B: the median time per batch and queries/s of each way; the rows are asserted identical, and
    the mixed rows equal the oracle's on a 16-query sample.
(b) Coalescer.search from T threads, thread t in class t % 4: queries/s, dispatches and the largest dispatch.

Records the card's name and power limit from the same run.

    python tools/mixed_batch.py                  # 1M x 768 lowrank, 2 bits, cosine, labels

Writes one JSON line to stdout and profiles/h100_mixed_batch_1m.json (or under --out-dir)."""
from __future__ import annotations

import argparse
import json
import os
import subprocess
import sys
import threading
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

DATA_SEED = 0x5EED0050
QUERY_SEED = 0x5EED0051
LABELS_SEED = 0x5EED0052
# (k, search_list_size, rescore, key): LIMITs of 5 / 10 / 20, two session settings of L, unfiltered and filtered
CLASSES = [(10, 100, 50, None), (5, 200, 50, [3]), (20, 100, 100, None), (10, 200, 50, [2, 7])]


def card():
    r = subprocess.run(["nvidia-smi", "--id=0", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                       capture_output=True, text=True)
    name, power = (r.stdout.strip().split(", ") + ["?", "?"])[:2]
    return {"name": name, "power_limit": power}


def classes_of(B):
    c = np.arange(B) % len(CLASSES)
    k = np.array([CLASSES[i][0] for i in c])
    L = np.array([CLASSES[i][1] for i in c])
    r = np.array([CLASSES[i][2] for i in c])
    labels = [CLASSES[i][3] for i in c]
    return c, k, L, r, labels


def mixed(idx, q, B):
    _, k, L, r, labels = classes_of(B)
    return idx.search_batch(q[:B], labels=labels, k=k, search_list_size=L, rescore=r)


def per_class(idx, q, B):
    """one uniform batch per class, back to back -> rows scattered back into query order"""
    c, *_ = classes_of(B)
    out = []
    for j, (k, L, r, key) in enumerate(CLASSES):
        sel = np.nonzero(c == j)[0]
        labels = None if key is None else [key] * len(sel)
        out.append((sel, idx.search_batch(q[sel], labels=labels, k=k, search_list_size=L, rescore=r)))
    return out


def same_rows(m, parts):
    for sel, g in parts:
        k = g["tid"].shape[1]
        if not (np.array_equal(m["tid"][sel, :k], g["tid"]) and np.array_equal(m["count"][sel], g["count"])
                and np.array_equal(m["dist"][sel, :k].view(np.uint32), g["dist"].view(np.uint32))
                and np.array_equal(m["stats"][sel], g["stats"])):
            return False
    return True


def time_ab(idx, q, B, reps):
    mixed(idx, q, B)                 # warm-up of both ways: workspaces, module loads
    per_class(idx, q, B)
    tm, tp = [], []
    for _ in range(reps):
        t = time.perf_counter()
        m = mixed(idx, q, B)
        tm.append(time.perf_counter() - t)
        t = time.perf_counter()
        p = per_class(idx, q, B)
        tp.append(time.perf_counter() - t)
        assert same_rows(m, p), f"B={B}: the mixed batch and the per-class batches returned different rows"
    med = lambda v: float(np.median(v))      # noqa: E731
    return {"queries": B, "reps": reps,
            "mixed": {"ms_per_batch": round(med(tm) * 1e3, 3), "queries_per_s": round(B / med(tm), 1)},
            "per_class_back_to_back": {"launches": len(CLASSES), "ms_per_batch": round(med(tp) * 1e3, 3),
                                       "queries_per_s": round(B / med(tp), 1)},
            "speedup": round(med(tp) / med(tm), 3), "rows_identical": True}


def coalesced(lib, idx, q, threads, per_thread, max_batch, max_wait_us):
    errors = []
    with lib.Coalescer(idx, max_batch=max_batch, max_wait_us=max_wait_us) as co:
        start = threading.Barrier(threads + 1)

        def backend(t):
            try:
                k, L, r, key = CLASSES[t % len(CLASSES)]
                start.wait()
                for j in range(per_thread):
                    co.search(q[(t * per_thread + j) % q.shape[0]], labels=key, k=k, search_list_size=L, rescore=r)
            except Exception as e:      # noqa: BLE001
                errors.append(e)

        th = [threading.Thread(target=backend, args=(t,)) for t in range(threads)]
        for x in th:
            x.start()
        start.wait()
        t0 = time.perf_counter()
        for x in th:
            x.join()
        dt = time.perf_counter() - t0
        st = co.stats()
    assert not errors, errors[:3]
    return {"threads": threads, "queries": st["queries"], "queries_per_s": round(st["queries"] / dt, 1),
            "dispatches": st["batches"], "largest_batch": st["largest_batch"],
            "mean_batch": round(st["queries"] / max(st["batches"], 1), 1), "max_batch": max_batch,
            "max_wait_us": max_wait_us}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--n", type=int, default=1_000_000)
    ap.add_argument("--dim", type=int, default=768)
    ap.add_argument("--bits", type=int, default=2)
    ap.add_argument("--batches", default="4096,256")
    ap.add_argument("--reps", type=int, default=20)
    ap.add_argument("--threads", default="64,256")
    ap.add_argument("--per-thread", type=int, default=64)
    ap.add_argument("--out-dir", default=os.path.join(ROOT, "profiles"))
    args = ap.parse_args()
    import torch
    from oracle import oracle
    from pgvectorscale_b200 import diskann
    from pgvectorscale_b200.snapshot import COSINE
    from tools import synth_index as si
    if diskann.device_count() < 1:
        raise SystemExit("mixed_batch: no CUDA device visible")
    oracle.build_lib()
    info = card()
    log = lambda *a: print(*a, file=sys.stderr, flush=True)      # noqa: E731
    device = torch.device("cuda", 0)
    t0 = time.time()
    x = si.gen_dataset(args.n, args.dim, DATA_SEED, "lowrank", device=device)
    snap, idx, bst = si.build_index_vamana(x, COSINE, bits=args.bits, keep_index=True, labels_seed=LABELS_SEED, log=log)
    del x
    torch.cuda.empty_cache()
    log(f"index built in {time.time() - t0:.1f}s")
    batches = [int(b) for b in args.batches.split(",")]
    q = si.gen_dataset(max(batches), args.dim, QUERY_SEED, "lowrank", device=device).cpu().numpy()

    # the mixed rows against the oracle on a 16-query sample (every class four times)
    g = mixed(idx, q, 16)
    _, k, L, r, labels = classes_of(16)
    for b in range(16):
        ref = oracle.scan(snap, q[b], labels[b], int(L[b]), int(r[b]), int(k[b]))
        n = len(ref["tid"])
        assert int(g["count"][b]) == n and g["tid"][b, :n].tolist() == ref["tid"].tolist(), f"oracle parity, query {b}"
        assert g["dist"][b, :n].view(np.uint32).tolist() == ref["dist"].view(np.uint32).tolist(), f"oracle dist, query {b}"

    runs = []
    for B in batches:
        runs.append(time_ab(idx, q, B, args.reps))
        log(json.dumps(runs[-1]))
    co_runs = []
    for T in [int(t) for t in args.threads.split(",")]:
        co_runs.append(coalesced(diskann, idx, q, T, args.per_thread, max_batch=4096, max_wait_us=200))
        log(json.dumps(co_runs[-1]))
    line = {"metric": f"mixed-parameter batches, {args.n}x{args.dim}-d {args.bits}-bit SBQ diskann index with labels",
            "unit": "queries/s", "card": info,
            "config": {"n": args.n, "dim": args.dim, "bits": args.bits, "data": "lowrank", "distance": "cosine",
                       "classes": [{"k": c[0], "search_list_size": c[1], "rescore": c[2], "key": c[3]} for c in CLASSES],
                       "timing": "host clock around each call (each returns after its stream has drained), median"},
            "batch": runs, "coalescer": co_runs,
            "parity": {"mixed_equals_per_class": True, "oracle_sample_16": True}}
    os.makedirs(args.out_dir, exist_ok=True)
    size = f"{args.n // 1_000_000}m" if args.n % 1_000_000 == 0 else str(args.n)
    with open(os.path.join(args.out_dir, f"h100_mixed_batch_{size}.json"), "w") as f:
        json.dump(line, f, indent=1)
    print(json.dumps(line))
    idx.close()


if __name__ == "__main__":
    main()
