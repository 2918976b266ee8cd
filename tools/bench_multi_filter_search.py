"""Batches of queries that each carry their own candidates filter, on the C2 index.

Workload: C2 (1M x 768 Cosine, 50 trees, SEED, centre 0.5), built through Writer as tools/bench_filtered_search.py builds it.
1000 by_item queries, each with its own seeded random filter of 1 %, 0.1 % or 0.02 % of the ids, or of 10 ids (the shortcut),
and a mix of the four in one call. For each:
  - QPS of one Reader.nns_batch_by_item(filters=..., filter_of_query=...) call and its time split (filter upload + row masks,
    summaries, walk, sort, re-rank, from arroy_b200_search_breakdown), and the multi_filter_stats of the call;
  - the same queries as a loop of single QueryBuilder.candidates(..).by_item calls (what a caller without the batch API does);
  - the shared-filter batch (candidates=, one filter of the same size for every query), the ceiling, and the same shared
    filter through the multi-filter call;
  - every multi-filter row is asserted equal to the single-query result (ids and float32 bytes).
Writes DIR/multi_filter_search.json, with the GPU name, power limit and max SM clock read in the same run.

    python tools/bench_multi_filter_search.py --out DIR [--n 1000000] [--trees 50] [--queries 1000]
"""
import argparse
import ctypes as C
import json
import os
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))

from bench_filtered_search import SEED, gpu_info  # noqa: E402


def timed(fn, reps=3):
    fn()   # warm-up: shapes, scratch buffers
    best, out = None, None
    for _ in range(reps):
        t0 = time.perf_counter()
        out = fn()
        dt = time.perf_counter() - t0
        best = dt if best is None else min(best, dt)
    return out, best


def breakdown(ctx):
    out = (C.c_double * 8)()
    ctx._ck(ctx.lib.arroy_b200_search_breakdown(ctx.h, out))
    return dict(zip(["walk_ms", "sort_ms", "distance_ms", "topk_ms", "normalize_ms", "filter_upload_ms", "filter_summary_ms"], list(out)[:7]))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", required=True)
    ap.add_argument("--n", type=int, default=1_000_000)
    ap.add_argument("--d", type=int, default=768)
    ap.add_argument("--trees", type=int, default=50)
    ap.add_argument("--count", type=int, default=10)
    ap.add_argument("--queries", type=int, default=1000)
    ap.add_argument("--single", type=int, default=1000, help="single queries timed (and checked) per filter kind")
    args = ap.parse_args()
    os.makedirs(args.out, exist_ok=True)

    import torch
    import arroy_b200 as ab

    n, d, T, count, nq = args.n, args.d, args.trees, args.count, args.queries
    info = gpu_info()
    ctx = ab.Context(0)
    items = torch.empty((n, d), dtype=torch.float32, device="cuda")
    ctx.synth_device(SEED, d, 0, n, 0.5, items.data_ptr())
    host = items.cpu().numpy()
    del items
    ids = np.arange(n, dtype=np.uint32)
    env = ab.Env(0)
    env._ctx = ctx
    w = ab.Writer(env, 0, d, "cosine")
    w.add_items(ids, host)
    t0 = time.perf_counter()
    w.builder(ab.StdRng.from_seed(SEED)).n_trees(T).build()
    build_s = time.perf_counter() - t0
    del host
    reader = ab.Reader.open(env, 0, "cosine")
    reader.nns(count).by_item(0)   # stages the items and uploads the forest
    st = reader.stats()["tree_stats"]
    nodes = sum(t["split_nodes"] + t["descendants"] for t in st)
    group_bytes = 4 * ((n + 31) // 32 * 32 + (nodes + 31) // 32 * 32 + 32 * nodes) + 256

    rng = np.random.default_rng(4321)
    rand_filter = lambda m: np.unique(rng.integers(0, n, size=m)).astype(np.uint32)
    sizes = {"random 1%": n // 100, "random 0.1%": n // 1000, "random 0.02%": n // 5000, "random 10 items (shortcut)": 10}
    qitems = np.random.default_rng(99).choice(n, size=nq, replace=False).astype(np.uint32)
    kinds = [(name, [m] * nq) for name, m in sizes.items()] + [("mix of the four", [list(sizes.values())[i % 4] for i in range(nq)])]
    rows = []
    for name, ms in kinds:
        fl = [rand_filter(m) for m in ms]
        fq = np.arange(nq, dtype=np.uint32)
        s0, m0 = ctx.search_stats(), ctx.multi_filter_stats()
        (mi, md, ml, _), t_multi = timed(lambda: reader.nns_batch_by_item(qitems, count, filters=fl, filter_of_query=fq))
        s1, m1 = ctx.search_stats(), ctx.multi_filter_stats()
        split = breakdown(ctx)
        # the loop of single queries, and the identity check
        k = min(args.single, nq)
        lat = []
        for i in range(k):
            t0 = time.perf_counter()
            single = reader.nns(count).candidates(fl[i]).by_item(int(qitems[i]))
            lat.append(time.perf_counter() - t0)
            assert mi[i, :ml[i]].tolist() == [x[0] for x in single], (name, i)
            assert md[i, :ml[i]].tobytes() == np.array([x[1] for x in single], np.float32).tobytes(), (name, i)
        # one filter of this size for every query: the bitmap path (candidates=) and the same through the multi-filter call
        f0 = fl[0] if len(set(ms)) == 1 else rand_filter(n // 1000)
        (si, sd, sl, _), t_shared = timed(lambda: reader.nns_batch_by_item(qitems, count, candidates=f0))
        (ui, ud, ul, _), t_shared_multi = timed(lambda: reader.nns_batch_by_item(qitems, count, filters=[f0], filter_of_query=np.zeros(nq, np.uint32)))
        assert ul.tolist() == sl.tolist() and ui.tobytes() == si.tobytes() and ud.tobytes() == sd.tobytes(), name
        per_call = lambda a, b: {key: (b[key] - a[key]) // 4 for key in a}   # warm-up + 3 timed calls
        row = {"filters": name, "filter_items": int(np.mean([f.size for f in fl])), "queries": nq,
               "multi_qps": nq / t_multi, "multi_call_ms": t_multi * 1e3, "multi_last_call_split_ms": split,
               "multi_stats_per_call": per_call(m0, m1), "search_stats_per_call": per_call(s0, s1),
               "single_loop": {"queries": k, "p50_ms": float(np.percentile(lat, 50)) * 1e3, "qps": k / sum(lat)},
               "shared_filter_batch_qps": nq / t_shared, "shared_filter_via_multi_qps": nq / t_shared_multi,
               "shared_filter_items": int(f0.size), "multi_equals_single": True}
        rows.append(row)
        print(json.dumps(row), flush=True)
    rec = {"workload": {"n": n, "d": d, "trees": T, "metric": "cosine", "centre": 0.5, "count": count, "search_k": "default (count x trees)",
                        "forest_nodes": nodes, "summary_bytes_per_group_of_32": group_bytes},
           "gpu": info, "build_s": build_s, "rows": rows}
    with open(os.path.join(args.out, "multi_filter_search.json"), "w") as f:
        json.dump(rec, f, indent=1)
    env._ctx = None
    ctx.close()


if __name__ == "__main__":
    main()
