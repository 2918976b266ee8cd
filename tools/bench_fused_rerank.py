"""The fused re-rank (frerank.cuh) of device-placed indexes: batched queries and rerank_batch, per float metric, for comparing
two builds of the library (ARROY_B200_LIB) on the same seeded data.

Workloads, each staged and built through Writer as bench.py's query section builds C2 (SEED, centre 0.5):
  - 1M x 768, 50 trees, for each of Euclidean, Cosine, DotProduct and Manhattan;
  - two edge shapes (Cosine): 1M x 32, 50 trees (d < 64, where the build writes no planes) and 100k x 16384, 10 trees
    (d above the planes' range).
Per workload:
  - QPS of 1000-query batches (Reader.nns_batch_by_vector / nns_batch_by_item) at top-10 and top-100: median, min and max
    of `--reps` timed calls after one warm-up (host clock around calls that end in a device synchronise);
  - QPS of rerank_batch on walk-like candidate lists: for each of 200 queries its top-100 rows and 5000 random rows, sorted;
  - survivors re-scored and candidates estimated per query by the plane pre-filter (arroy_b200_plane_rerank_stats; zero where
    the batch took the bf16 kernel or the plain kernels), and the fused batches and fallbacks (arroy_b200_counters);
  - device bytes the context holds after the first batched query: torch.cuda.mem_get_info before the context is created
    minus after that query (f32 rows, planes, headers, forest and scratch).
Results (ids, distances, lengths of every call) go to DIR/<workload>.npz, so two builds (ARROY_B200_LIB) can be compared
byte for byte with --compare DIR_A DIR_B. One JSON line per workload on stdout, with the GPU name and power limit.

    python tools/bench_fused_rerank.py --out DIR [--reps 5] [--only NAME ...]
    python tools/bench_fused_rerank.py --compare DIR_A DIR_B
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
WORKLOADS = {
    "euclidean_768": ("euclidean", 1_000_000, 768, 50),
    "cosine_768": ("cosine", 1_000_000, 768, 50),
    "dot-product_768": ("dot-product", 1_000_000, 768, 50),
    "manhattan_768": ("manhattan", 1_000_000, 768, 50),
    "cosine_32": ("cosine", 1_000_000, 32, 50),
    "cosine_16384": ("cosine", 100_000, 16384, 10),
}


def gpu_info():
    out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True, text=True, timeout=30).stdout
    return out.strip().splitlines()[0]


def timed(fn, n, reps):
    """(result, [median, min, max] QPS over `reps` timed calls after one warm-up)"""
    res = fn()
    qps = []
    for _ in range(reps):
        t0 = time.perf_counter()
        res = fn()
        qps.append(n / (time.perf_counter() - t0))
    return res, [round(float(np.median(qps)), 1), round(min(qps), 1), round(max(qps), 1)]


def run(name, reps, out_dir):
    import torch

    import arroy_b200 as ab
    metric, n, d, T = WORKLOADS[name]
    torch.cuda.init()
    items = torch.empty((n, d), dtype=torch.float32, device="cuda:0")
    ctx = ab.Context(0)
    ctx.synth_device(SEED, d, 0, n, 0.5, items.data_ptr())
    host = items.cpu().numpy()
    del items
    torch.cuda.synchronize()
    torch.cuda.empty_cache()
    rng = np.random.default_rng(7)
    qv = (host[rng.choice(n, 1000)] + rng.standard_normal((1000, d)).astype(np.float32) * np.float32(0.05)).astype(np.float32)
    qitems = rng.choice(n, 1000).astype(np.uint32)
    ctx.close()

    free_before = torch.cuda.mem_get_info()[0]
    ctx = ab.Context(0)
    env = ab.Env(0)
    env._ctx = ctx
    w = ab.Writer(env, 0, d, metric)
    w.add_items(np.arange(n, dtype=np.uint32), host)
    w.builder(ab.StdRng.from_seed(SEED)).n_trees(T).build()
    reader = ab.Reader.open(env, 0, metric)
    res = {}
    res["vec10_first"] = reader.nns_batch_by_vector(qv, 10)[:3]
    torch.cuda.synchronize()
    held = free_before - torch.cuda.mem_get_info()[0]
    rec = {"workload": name, "metric": metric, "n": n, "d": d, "trees": T, "device_bytes_held": int(held)}
    for k in (10, 100):
        for by, fn in (("vector", lambda: reader.nns_batch_by_vector(qv, k)), ("item", lambda: reader.nns_batch_by_item(qitems, k))):
            s0, c0 = ctx.plane_rerank_stats(), ctx.counters()
            r, qps = timed(fn, len(qv), reps)
            s1, c1 = ctx.plane_rerank_stats(), ctx.counters()
            calls = reps + 1
            key = "%s_top%d" % (by, k)
            res[key] = r[:3]
            rec["qps_" + key] = qps
            rec["rescored_per_query_" + key] = round((s1["rows_rescored"] - s0["rows_rescored"]) / (calls * len(qv)), 2)
            rec["estimated_per_query_" + key] = round((s1["rows_estimated"] - s0["rows_estimated"]) / (calls * len(qv)), 1)
            rec["fused_batches_" + key] = int(c1["fused_rerank_batches"] - c0["fused_rerank_batches"])
            rec["fallbacks_" + key] = int(c1["fused_rerank_fallbacks"] - c0["fused_rerank_fallbacks"])
    # rerank_batch on walk-like lists: the query's top-100 rows plus 5000 random rows
    nq = 200
    top = res["vector_top100"][0][:nq]
    lists = [np.union1d(top[i][top[i] < n], rng.choice(n, 5000, replace=False)).astype(np.uint32) for i in range(nq)]
    offs = np.zeros(nq + 1, np.uint64)
    offs[1:] = np.cumsum([len(x) for x in lists])
    flat = np.concatenate(lists)
    qh = np.array([ab_header(metric, v) for v in qv[:nq]], np.float32)
    for k in (10, 100):
        s0 = ctx.plane_rerank_stats()
        r, qps = timed(lambda: ctx.rerank_batch(qv[:nq], qh, flat, offs, k), nq, reps)
        s1 = ctx.plane_rerank_stats()
        res["rerank_batch_top%d" % k] = r
        rec["qps_rerank_batch_top%d" % k] = qps
        rec["rescored_per_query_rerank_batch_top%d" % k] = round((s1["rows_rescored"] - s0["rows_rescored"]) / ((reps + 1) * nq), 2)
        rec["candidates_per_query_rerank_batch"] = round(len(flat) / nq, 1)
    del reader, w
    env._ctx = None
    env.close()
    ctx.close()
    flat_res = {}
    for key, arrs in res.items():
        for j, a in enumerate(arrs):
            flat_res["%s_%d" % (key, j)] = np.asarray(a)
    np.savez(os.path.join(out_dir, name + ".npz"), **flat_res)
    return rec


def ab_header(metric, v):
    if metric != "cosine":
        return 0.0
    import oracle
    return oracle.new_header(oracle.COSINE, v)[0]


def compare(a, b):
    ok = True
    for f in sorted(os.listdir(a)):
        if not f.endswith(".npz"):
            continue
        x, y = np.load(os.path.join(a, f)), np.load(os.path.join(b, f))
        same = sorted(x.files) == sorted(y.files) and all(x[k].dtype == y[k].dtype and x[k].tobytes() == y[k].tobytes() for k in x.files)
        print(json.dumps({"workload": f[:-4], "identical": bool(same)}), flush=True)
        ok &= same
    return ok


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out")
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--only", nargs="*", choices=sorted(WORKLOADS))
    ap.add_argument("--compare", nargs=2, metavar=("DIR_A", "DIR_B"))
    args = ap.parse_args()
    if args.compare:
        sys.exit(0 if compare(*args.compare) else 1)
    os.makedirs(args.out, exist_ok=True)
    card = gpu_info()
    for name in args.only or list(WORKLOADS):
        rec = run(name, args.reps, args.out)
        rec["card"] = card
        rec["lib"] = os.environ.get("ARROY_B200_LIB", "in-tree")
        print(json.dumps(rec), flush=True)


if __name__ == "__main__":
    main()
