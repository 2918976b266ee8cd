"""What placing an index's f32 rows in host memory costs, and an index that only fits that way.

  C2: 1M x 768 Cosine, 50 trees, staged from host arrays (arroy_b200_stage_items_flat): the default placement (device) and the
      forced host placement (ARROY_B200_HOST_ITEMS=1), alternating, three runs each. Per run: stage ms and device build ms (both
      host clocks around calls that end in a device synchronise; the build is arroy_b200_build_trees_begin, NodeCodec encoding
      apart), the bytes a host-placed build reads from host memory as the counters give them (stage-3 rows of the pre-filter and
      12 rows per create_split call, 4 ld bytes each; reads of the same row by several trees are counted each time), 1000-query
      batched search QPS (by vector, 10 neighbours) and the p50 of single-query calls. The forests of both placements must be
      byte-identical, and so must the query results.
  Re-rank (--rerank): C2 staged once with forced host placement and built once; then the batched queries alternate between
      the plane pre-filter of the re-rank (default) and ARROY_B200_FRERANK=0 (every candidate row read from host memory), three
      runs each: 1000-query batched QPS by vector and by item at top-10 and top-100, the p50 of single-query calls (a path the
      switch does not touch), and rows read from host memory per query (arroy_b200_plane_rerank_stats out[3] / queries) against
      the candidates per query (out[2] / queries). Both sides' results must be byte-identical. One device-placed run of the
      same queries is printed for comparison.
  Out of core: 11M x 1536 Cosine, 10 trees, staged with the automatic choice: 67.6 GB of f32 rows and 33.8 GB of planes, so an
      80 GB card must choose host. It runs only if MemAvailable covers the caller's copy plus the library's (about 140 GB);
      otherwise it prints "not run: host memory".

Needs a GPU: there is no fallback. Data comes from synth_device with a fixed seed."""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import arroy_b200 as ab   # noqa: E402
import oracle            # noqa: E402  (NodeCodec decoding of the forest the searches load)

SEED = bytes([42] * 32)


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True, text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 and q.stdout.strip() else torch.cuda.get_device_name(0) + ", power limit not readable"


def synth_host(ctx, n, d, chunk_rows=1 << 20):
    """n x d f32 rows in (pageable) host memory, generated on the device chunk by chunk"""
    out = np.empty((n, d), dtype=np.float32)
    t = torch.empty((min(n, chunk_rows), d), dtype=torch.float32, device="cuda:0")
    for a in range(0, n, chunk_rows):
        b = min(n, a + chunk_rows)
        ctx.synth_device(SEED, d, a, b - a, 0.5, t.data_ptr())
        out[a:b] = t[:b - a].cpu().numpy()
    del t
    torch.cuda.empty_cache()
    return out


def tree_seeds(T):
    r1 = oracle.StdRng(oracle.StdRng(SEED).gen_seed())
    return [r1.gen_seed() for _ in range(T)]


def forest_arrays(nodes, d):
    nn = max(nodes) + 1
    kind = np.zeros(nn, np.uint8)
    left, right, nidx = np.zeros(nn, np.uint32), np.zeros(nn, np.uint32), np.full(nn, 0xffffffff, np.uint32)
    nh0, doff, dlen = np.zeros(nn, np.float32), np.zeros(nn, np.uint32), np.zeros(nn, np.uint32)
    normals, desc, n_desc = [], [], 0
    for i, b in nodes.items():
        nd = oracle.decode_node(b, oracle.COSINE, d)
        if nd["kind"] == "descendants":
            kind[i], doff[i], dlen[i] = 1, n_desc, len(nd["descendants"])
            desc.append(np.asarray(nd["descendants"], dtype=np.uint32))
            n_desc += dlen[i]
        else:
            kind[i], left[i], right[i] = 2, nd["left"], nd["right"]
            if nd["normal"] is not None:
                nidx[i], nh0[i] = len(normals), nd["header"][0]
                normals.append(nd["normal"])
    return dict(kind=kind, left=left, right=right, normal_idx=nidx, normal_hdr0=nh0, desc_off=doff, desc_len=dlen,
                normals=np.stack(normals), desc_rows=np.concatenate(desc))


def set_placement(host):
    if host:
        os.environ["ARROY_B200_HOST_ITEMS"] = "1"
    else:
        os.environ.pop("ARROY_B200_HOST_ITEMS", None)


def stage_and_build(ctx, rows, T, host):
    n, d = rows.shape
    set_placement(host)
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    ctx.stage_items_flat("cosine", np.arange(n, dtype=np.uint32), rows)
    stage_ms = (time.perf_counter() - t0) * 1e3
    set_placement(False)
    pl = ctx.item_placement()
    t0 = time.perf_counter()
    counts = ctx.build_trees_begin(tree_seeds(T))
    build_ms = (time.perf_counter() - t0) * 1e3
    st, pre = ctx.build_stats(), ctx.build_prefilter_stats()
    ld = (d + 31) // 32 * 32
    host_read = (pre["rows_rescored_f32"] + 12 * int(st["create_split_calls"])) * 4 * ld if pl["placement"] == "host" else 0
    return counts, {"placement": pl["placement"], "device_item_GB": round(pl["device_bytes"] / 1e9, 3), "pinned_GB": round(pl["host_bytes"] / 1e9, 3),
                    "stage_ms": round(stage_ms, 1), "build_ms": round(build_ms, 1), "device_build_ms": round(st["build_ms"], 1),
                    "stage3_rows": pre["rows_rescored_f32"], "create_split_calls": int(st["create_split_calls"]),
                    "host_read_GB": round(host_read / 1e9, 3)}


def emit(ctx, counts, T):
    base, c = np.zeros(T, dtype=np.uint64), T
    for t in range(T - 1, -1, -1):   # last tree first (arroy_b200_build_trees)
        base[t] = c
        c += int(counts[t]) - 1
    return ctx.build_trees_emit(np.arange(T, dtype=np.uint32), base)


def queries(ctx, qv, qh):
    ctx.search_batch(10, queries=qv, qhdr0=qh)   # warm-up
    torch.cuda.synchronize()
    reps = 3
    t0 = time.perf_counter()
    for _ in range(reps):
        res = ctx.search_batch(10, queries=qv, qhdr0=qh)
    qps = reps * len(qv) / (time.perf_counter() - t0)
    lat = []
    for i in range(200):
        t0 = time.perf_counter()
        ctx.search_batch(10, queries=qv[i:i + 1], qhdr0=qh[i:i + 1])
        lat.append((time.perf_counter() - t0) * 1e3)
    return res, round(qps, 1), round(float(np.percentile(lat, 50)), 3)


def c2(ctx, runs):
    n, d, T = 1_000_000, 768, 50
    rows = synth_host(ctx, n, d)
    rng = np.random.default_rng(3)
    qv = (rows[rng.choice(n, 1000)] + rng.standard_normal((1000, d)).astype(np.float32) * np.float32(0.05)).astype(np.float32)
    qh = np.array([oracle.new_header(oracle.COSINE, v)[0] for v in qv], dtype=np.float32)
    ref_nodes, ref_res, loaded = None, None, False
    for r in range(runs):
        for host in (False, True):
            counts, rec = stage_and_build(ctx, rows, T, host)
            nodes = emit(ctx, counts, T)
            if ref_nodes is None:
                ref_nodes = nodes
            rec["forest_identical"] = nodes == ref_nodes
            if not loaded:
                arrays = forest_arrays(ref_nodes, d)
                loaded = True
            ctx.load_forest(roots=np.arange(T, dtype=np.uint32), **arrays)
            res, qps, p50 = queries(ctx, qv, qh)
            if ref_res is None:
                ref_res = res
            rec["results_identical"] = all(np.asarray(a).tobytes() == np.asarray(b).tobytes() for a, b in zip(res, ref_res))
            rec.update({"run": r, "batched_qps_1000": qps, "single_query_p50_ms": p50})
            print(json.dumps({"workload": "C2 1Mx768 Cosine 50 trees", **rec}), flush=True)
            assert rec["forest_identical"] and rec["results_identical"], rec


def timed_qps(fn, nq, reps=3):
    fn()   # warm-up
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    for _ in range(reps):
        res = fn()
    return res, round(reps * nq / (time.perf_counter() - t0), 1)


def rerank_side(ctx, qv, qh, qrows, plane):
    if plane:
        os.environ.pop("ARROY_B200_FRERANK", None)
    else:
        os.environ["ARROY_B200_FRERANK"] = "0"
    rec, res = {}, {}
    for k in (10, 100):
        s0 = ctx.plane_rerank_stats()
        res["vec%d" % k], rec["qps_by_vector_top%d" % k] = timed_qps(lambda: ctx.search_batch(k, queries=qv, qhdr0=qh), len(qv))
        res["item%d" % k], rec["qps_by_item_top%d" % k] = timed_qps(lambda: ctx.search_batch(k, query_rows=qrows), len(qrows))
        s1 = ctx.plane_rerank_stats()
        nq = 2 * 4 * len(qv)   # (warm-up + 3 timed calls) x (by vector, by item)
        rec["top%d_rows_estimated_per_query" % k] = round((s1["rows_estimated"] - s0["rows_estimated"]) / nq, 1)
        rec["top%d_rows_from_host_per_query" % k] = round((s1["rows_rescored"] - s0["rows_rescored"]) / nq, 2)
        rec["top%d_fallback_batches" % k] = s1["fallbacks"] - s0["fallbacks"]
    lat = []
    for i in range(200):
        t0 = time.perf_counter()
        ctx.search_batch(10, queries=qv[i:i + 1], qhdr0=qh[i:i + 1])
        lat.append((time.perf_counter() - t0) * 1e3)
    rec["single_query_p50_ms"] = round(float(np.percentile(lat, 50)), 3)
    os.environ.pop("ARROY_B200_FRERANK", None)
    return res, rec


def host_rerank(ctx, runs):
    n, d, T = 1_000_000, 768, 50
    rows = synth_host(ctx, n, d)
    rng = np.random.default_rng(3)
    qv = (rows[rng.choice(n, 1000)] + rng.standard_normal((1000, d)).astype(np.float32) * np.float32(0.05)).astype(np.float32)
    qh = np.array([oracle.new_header(oracle.COSINE, v)[0] for v in qv], dtype=np.float32)
    qrows = rng.choice(n, 1000).astype(np.uint32)
    counts, rec = stage_and_build(ctx, rows, T, host=False)
    nodes = emit(ctx, counts, T)
    arrays = forest_arrays(nodes, d)
    ctx.load_forest(roots=np.arange(T, dtype=np.uint32), **arrays)
    dev_res, dev_rec = rerank_side(ctx, qv, qh, qrows, plane=True)
    print(json.dumps({"workload": "C2 re-rank", "placement": rec["placement"], **dev_rec}), flush=True)
    counts, rec = stage_and_build(ctx, rows, T, host=True)
    assert rec["placement"] == "host", rec
    assert emit(ctx, counts, T) == nodes
    ctx.load_forest(roots=np.arange(T, dtype=np.uint32), **arrays)
    for r in range(runs):
        for plane in (True, False):
            res, side = rerank_side(ctx, qv, qh, qrows, plane)
            same = all(np.asarray(a).tobytes() == np.asarray(b).tobytes() for key in res for a, b in zip(res[key], dev_res[key]))
            print(json.dumps({"workload": "C2 re-rank", "placement": "host", "path": "planes" if plane else "ARROY_B200_FRERANK=0", "run": r,
                              **side, "results_identical_to_device_placement": same}), flush=True)
            assert same


def mem_available():
    with open("/proc/meminfo") as f:
        for line in f:
            if line.startswith("MemAvailable:"):
                return int(line.split()[1]) * 1024
    return 0


def out_of_core(ctx):
    n, d, T = 11_000_000, 1536, 10
    need = 2 * n * d * 4 + (4 << 30)
    avail = mem_available()
    if avail < need:
        print(json.dumps({"workload": "out of core 11Mx1536 Cosine 10 trees", "result": "not run: host memory",
                          "mem_available_GB": round(avail / 1e9, 1), "needed_GB": round(need / 1e9, 1)}), flush=True)
        return
    t0 = time.perf_counter()
    rows = synth_host(ctx, n, d)
    gen_s = time.perf_counter() - t0
    free0 = torch.cuda.mem_get_info()[0]
    plan = ab.item_placement_plan("cosine", d, n, free0)
    counts, rec = stage_and_build(ctx, rows, T, host=False)   # the automatic choice
    rec.update({"workload": "out of core 11Mx1536 Cosine 10 trees", "plan": plan, "free_GB_before": round(free0 / 1e9, 1),
                "nodes": int(np.sum(counts)), "generate_s": round(gen_s, 1)})
    print(json.dumps(rec), flush=True)
    assert rec["placement"] == "host", rec


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--runs", type=int, default=3)
    ap.add_argument("--skip-out-of-core", action="store_true")
    ap.add_argument("--rerank", action="store_true", help="only the host-placed re-rank comparison")
    args = ap.parse_args()
    print(json.dumps({"card": card()}), flush=True)
    ctx = ab.Context(0)
    if args.rerank:
        host_rerank(ctx, args.runs)
        ctx.close()
        return
    c2(ctx, args.runs)
    if not args.skip_out_of_core:
        out_of_core(ctx)
    ctx.close()


if __name__ == "__main__":
    main()
