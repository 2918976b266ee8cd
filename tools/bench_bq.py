"""Binary-quantized benchmark: device bytes of the staged items, forest-build throughput and (--search) batched top-10
QPS and single-query p50 latency by item of a BQ Cosine index.

Items are synthesized on the device and staged with stage_items_device (one f32 copy of the index on the device while it is
quantized). Prints one JSON line per run with the GPU's name, power limit and SM clock beside the numbers. Set ARROY_B200_LIB
to time another build of the library (e.g. the parent commit's) with the same script; run the two alternately.

    python tools/bench_bq.py --n 1000000 --d 1536 --trees 50 --repeats 2 --search

--search decodes the forest in Python to load it (a few seconds per 100k nodes), so it is meant for indexes of about 1M rows.
"""
import argparse
import json
import os
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))   # forest_arrays: NodeCodec bytes -> the arrays of load_forest


def gpu_info():
    q = "name,power.limit,clocks.max.sm,clocks.sm"
    out = subprocess.run(["nvidia-smi", "--query-gpu=" + q, "--format=csv,noheader"], capture_output=True, text=True).stdout
    return out.strip().splitlines()[0] if out.strip() else "unknown"


def time_search(ctx, seeds, a):
    import numpy as np
    import torch

    import oracle
    from test_gpu_filtered_search import forest_arrays
    nodes = ctx.build_trees(seeds, list(range(a.trees)), a.trees)
    dp = (a.d + 63) // 64 * 64
    ctx.load_forest(roots=np.arange(a.trees, dtype=np.uint32), **forest_arrays(nodes, oracle.BQ_COSINE, dp))
    del nodes
    items = np.random.default_rng(3).choice(a.n, size=a.queries, replace=False).astype(np.uint32)
    ctx.search_batch(10, query_rows=items)   # warm-up
    batch = []
    for _ in range(3):
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        _, _, _, status = ctx.search_batch(10, query_rows=items)
        batch.append(time.perf_counter() - t0)
        assert not status.any()
    single = []
    for it in items[:200]:
        t0 = time.perf_counter()
        ctx.search_batch(10, query_rows=np.array([it], dtype=np.uint32))
        single.append(time.perf_counter() - t0)
    return {"batched_top10_qps": round(a.queries / min(batch)), "single_query_p50_ms": round(1e3 * float(np.median(single[20:])), 4)}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--n", type=int, default=1_000_000)
    ap.add_argument("--d", type=int, default=1536)
    ap.add_argument("--trees", type=int, default=50)
    ap.add_argument("--repeats", type=int, default=2)
    ap.add_argument("--search", action="store_true")
    ap.add_argument("--queries", type=int, default=1000)
    a = ap.parse_args()
    import numpy as np
    import torch

    import arroy_b200 as ab
    ctx = ab.Context(0)
    seed = bytes([42] * 32)
    ids = np.arange(a.n, dtype=np.uint32)
    src = torch.empty((a.n, a.d), dtype=torch.float32, device="cuda:0")
    ctx.synth_device(seed, a.d, 0, a.n, 0.5, src.data_ptr())
    torch.cuda.synchronize()
    ctx.stage_items_device("binary quantized cosine", ids, a.d, src.data_ptr())
    torch.cuda.synchronize()
    del src
    torch.cuda.empty_cache()
    _, ld = ctx.device_ptrs()
    seeds = [bytes([(7 * t + i) & 255 for i in range(32)]) for t in range(a.trees)]
    times = []
    nodes = 0
    for _ in range(a.repeats + 1):   # the first build is the warm-up
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        nodes = ctx.build_trees(seeds, list(range(a.trees)), a.trees, collect=False)
        times.append(time.perf_counter() - t0)
    best = min(times[1:])
    search = {}
    if a.search:
        search = time_search(ctx, seeds, a)
    print(json.dumps({**search, "lib": os.environ.get("ARROY_B200_LIB", "tree"), "gpu": gpu_info(), "n": a.n, "d": a.d, "trees": a.trees,
                      "item_bytes_per_row": ld * 4, "item_bytes": ld * 4 * a.n, "nodes": nodes,
                      "build_s": [round(t, 4) for t in times[1:]], "build_vectors_per_s": round(a.n * a.trees / best)}))
    ctx.close()


if __name__ == "__main__":
    main()
