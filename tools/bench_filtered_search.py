"""Filtered queries (QueryBuilder::candidates) on the C2 index: device walk vs host walk.

Workload: C2 (1M x 768 Cosine, 50 trees, SEED, centre 0.5), built through Writer as bench.py's query section builds it.
Filters: seeded random subsets of the ids at 100 %, 10 %, 5 %, 1 %, 0.1 %, 0.02 %, one of 10 items (at most `count`: the
shortcut that skips the walk) and contiguous id ranges of 5 %, 1 %, 0.1 % and 0.02 %. For each filter:
  - single-query by_item latency (p50 / p99): QueryBuilder.by_item as a user calls it (the library takes the host walk where
    host.hpp filter_prefers_host_walk says it is faster, the device walk elsewhere), the device walk forced for every filter (a
    one-query Reader.nns_batch_by_item), the same through the batched walk kernel (ARROY_B200_NO_WALK1=1), and the host walk
    (ARROY_B200_HOST_WALK=1, a smaller sample, timed through both entry points): both sides of that choice at every filter;
  - batched QPS of 1000 by_item queries sharing the filter (Reader.nns_batch_by_item(candidates=...));
  - the search_stats counters of those calls;
  - device and host results are asserted identical (ids and float32 bytes).
Writes DIR/filtered_search.json, with the GPU name, power limit and max SM clock read in the same run.

    python tools/bench_filtered_search.py --out DIR [--n 1000000] [--trees 50]
"""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

SEED = bytes([42] * 32)


def gpu_info():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True, text=True, timeout=30).stdout
        name, power, clock = [x.strip() for x in out.strip().splitlines()[0].split(",")]
        return {"name": name, "power_limit": power, "sm_clock_max": clock}
    except Exception as e:   # the numbers are still written; the record says what could not be read
        return {"error": str(e)}


def pct(xs, p):
    xs = sorted(xs)
    return xs[min(len(xs) - 1, int(len(xs) * p))] * 1e3


def single_latency(reader, items, count, F):
    out, lat = [], []
    reader.nns(count).candidates(F).by_item(int(items[0]))   # warm-up: shapes, scratch buffers
    for it in items:
        t0 = time.perf_counter()
        out.append(reader.nns(count).candidates(F).by_item(int(it)))
        lat.append(time.perf_counter() - t0)
    return out, {"p50_ms": pct(lat, 0.5), "p99_ms": pct(lat, 0.99), "queries": len(lat)}


def one_query_batch_latency(reader, items, count, F):
    """A one-query Reader.nns_batch_by_item: the device walk whatever the filter (arroy_b200_search_batch_filtered), or with
    ARROY_B200_HOST_WALK=1 the host walk, through the same entry point."""
    out, lat = [], []
    reader.nns_batch_by_item(items[:1], count, candidates=F)
    for i in range(len(items)):
        t0 = time.perf_counter()
        ids_, dist, ln, _ = reader.nns_batch_by_item(items[i:i + 1], count, candidates=F)
        lat.append(time.perf_counter() - t0)
        out.append(list(zip(ids_[0, :ln[0]].tolist(), dist[0, :ln[0]].tolist())))
    return out, {"p50_ms": pct(lat, 0.5), "p99_ms": pct(lat, 0.99), "queries": len(lat)}


def with_env(name, fn):
    os.environ[name] = "1"
    try:
        return fn()
    finally:
        os.environ.pop(name)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", required=True)
    ap.add_argument("--n", type=int, default=1_000_000)
    ap.add_argument("--d", type=int, default=768)
    ap.add_argument("--trees", type=int, default=50)
    ap.add_argument("--count", type=int, default=10)
    ap.add_argument("--single", type=int, default=50, help="single queries per filter (device and QueryBuilder.by_item)")
    ap.add_argument("--host-single", type=int, default=5, help="host-walk single queries per filter")
    ap.add_argument("--batch", type=int, default=1000)
    args = ap.parse_args()
    os.makedirs(args.out, exist_ok=True)

    import torch
    import arroy_b200 as ab

    n, d, T, count = args.n, args.d, args.trees, args.count
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

    rng = np.random.default_rng(1234)
    pick = lambda m: np.sort(rng.choice(n, size=m, replace=False)).tolist()
    rng_ = lambda m: ("range %g%% (ids %d..%d)" % (100 * m / n, 400_000, 400_000 + m - 1), list(range(400_000, 400_000 + m)))
    grid = [("random 100%", ids.tolist()), ("random 10%", pick(n // 10)), ("random 5%", pick(n // 20)), ("random 1%", pick(n // 100)),
            ("random 0.1%", pick(n // 1000)), ("random 0.02%", pick(n // 5000)), ("random 10 items (shortcut)", pick(10)),
            rng_(n // 20), rng_(n // 100), rng_(n // 1000), rng_(n // 5000)]
    qitems = np.random.default_rng(99).choice(n, size=max(args.single, args.batch), replace=False).astype(np.uint32)
    rows = []
    for name, F in grid:
        s0 = ctx.search_stats()
        dev_out, dev_lat = single_latency(reader, qitems[:args.single], count, F)
        s1 = ctx.search_stats()
        breakdown = ctx.search_breakdown()
        f_out, f_lat = one_query_batch_latency(reader, qitems[:args.single], count, F)
        b_out, b_lat = with_env("ARROY_B200_NO_WALK1", lambda: single_latency(reader, qitems[:args.single], count, F))
        host_out, host_lat = with_env("ARROY_B200_HOST_WALK", lambda: single_latency(reader, qitems[:args.host_single], count, F))
        hb_out, hb_lat = with_env("ARROY_B200_HOST_WALK", lambda: one_query_batch_latency(reader, qitems[:args.host_single], count, F))
        assert all(hb_out[i] == f_out[i] for i in range(args.host_single)), name
        for i in range(args.host_single):
            assert [x[0] for x in dev_out[i]] == [x[0] for x in host_out[i]], (name, i)
            assert np.array([x[1] for x in dev_out[i]], np.float32).tobytes() == np.array([x[1] for x in host_out[i]], np.float32).tobytes(), (name, i)
        assert all(dev_out[i] == b_out[i] == f_out[i] for i in range(args.single)), name
        bq = qitems[:args.batch]
        reader.nns_batch_by_item(bq, count, candidates=F)   # warm-up
        s2 = ctx.search_stats()
        times = []
        for _ in range(3):
            t0 = time.perf_counter()
            bi, bd, bl, _ = reader.nns_batch_by_item(bq, count, candidates=F)
            times.append(time.perf_counter() - t0)
        s3 = ctx.search_stats()
        for i in range(args.single):
            assert bi[i, :bl[i]].tolist() == [x[0] for x in dev_out[i]], (name, i)
        row = {"filter": name, "filter_items": len(F), "single_by_item": dev_lat, "single_device_batched_walk": b_lat, "single_host_walk": host_lat,
               "single_device_forced": f_lat, "single_host_walk_same_entry": hb_lat, "single_stats": {k: s1[k] - s0[k] for k in s1}, "last_device_query_breakdown_ms": breakdown, "batch_qps": args.batch / min(times), "batch_queries": args.batch,
               "batch_stats_per_call": {k: (s3[k] - s2[k]) // 3 for k in s3}, "device_equals_host": True}
        rows.append(row)
        print(json.dumps(row), flush=True)
    rec = {"workload": {"n": n, "d": d, "trees": T, "metric": "cosine", "centre": 0.5, "count": count, "search_k": "default (count x trees)"},
           "gpu": info, "build_s": build_s, "filters": rows}
    with open(os.path.join(args.out, "filtered_search.json"), "w") as f:
        json.dump(rec, f, indent=1)
    env._ctx = None
    ctx.close()


if __name__ == "__main__":
    main()
