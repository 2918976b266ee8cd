"""What keeping the items resident saves: builds and first queries with ARROY_B200_FULL_RESTAGE=1 (every staging is full) and
with the default (delta staging, readers adopt the rows a build left), alternating, in fresh Envs on one context.

  C2: 1M x 768 Cosine, 50 trees through the host mirror: fresh build, then updates of +100, +10 000 / -1 000 and +100 000
      items; for each the wall time of build() (it ends in a device synchronise), build_timings(), stage_stats() and the time
      from Reader.open to the first answered query.
  BQ: 1M x 1536 binary-quantized Cosine at the C ABI (the host mirror's Writers store f32 vectors): the same updates as
      staging calls, full against delta.
  The move: a delta staging call that moves every row by one place, under CUDA events, against 2 x moved_rows x row_bytes over
  the data-sheet 3.35 TB/s of the H100 SXM. The interval is the whole call (plan, header decode, scratch allocation, the two
  copy launches per window, header upload), so the share is the call's, not the kernels'; the two-launch move reads and writes
  every moved row twice, so half of the data-sheet figure is the kernels' ceiling.

Needs a GPU: there is no fallback. Data comes from synth_device with a fixed seed."""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import arroy_b200 as ab   # noqa: E402

SEED = bytes([42] * 32)
HBM_DATASHEET = 3.35e12


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True, text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 and q.stdout.strip() else torch.cuda.get_device_name(0) + ", power limit not readable"


def synth(ctx, n, d):
    t = torch.empty((n, d), dtype=torch.float32, device="cuda:0")
    ctx.synth_device(SEED, d, 0, n, 0.5, t.data_ptr())
    return t.cpu().numpy()


def c2_round(ctx, host, n, d, trees, full):
    if full:
        os.environ["ARROY_B200_FULL_RESTAGE"] = "1"
    else:
        os.environ.pop("ARROY_B200_FULL_RESTAGE", None)
    env = ab.Env(0)
    env._ctx = ctx
    w = ab.Writer(env, 0, d, "cosine")
    rng = ab.StdRng.from_seed(SEED)
    out = []
    nxt = n

    def build(name):
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        w.builder(rng).n_trees(trees).build()
        dt = (time.perf_counter() - t0) * 1e3
        bt, st = w.build_timings(), ctx.stage_stats()
        t0 = time.perf_counter()
        r = ab.Reader.open(env, 0, "cosine")
        r.nns(10).by_item(5)
        q = (time.perf_counter() - t0) * 1e3
        del r
        out.append({"step": name, "mode": "full" if full else "resident", "build_ms": round(dt, 1), "stage_ms": round(bt["stage_ms"], 1),
                    "device_build_ms": round(bt["build_ms"], 1), "total_ms": round(bt["total_ms"], 1), "h2d_MB": round(st["h2d_bytes"] / 1e6, 2),
                    "uploaded_rows": st["uploaded_rows"], "moved_rows": st["moved_rows"], "delta": st["delta"], "open_to_first_answer_ms": round(q, 1)})
        print(json.dumps(out[-1]), flush=True)

    w.add_items(np.arange(n, dtype=np.uint32), host[:n])
    build("fresh")
    for name, add, dele in (("+100", 100, 0), ("+10000/-1000", 10_000, 1_000), ("+100000", 100_000, 0)):
        w.add_items(np.arange(nxt, nxt + add, dtype=np.uint32), host[nxt:nxt + add])
        nxt += add
        for i in range(dele):
            w.del_item(i * 7 + 1)
        build(name)
    env._ctx = None
    env.close()
    return out


def bq_leg(ctx, n, d, rounds):
    metric, ll = "binary quantized cosine", 5 + (d + 63) // 64 * 8
    rng = np.random.default_rng(1)
    total = n + 110_100
    pool = np.frombuffer(rng.bytes(total * ll), np.uint8).reshape(total, ll).copy()
    pool[:, 0] = 0
    base = np.uint64(pool.ctypes.data)
    out = []
    for rnd in range(rounds):
        for full in (True, False):
            ids = np.arange(n, dtype=np.uint32)
            ctx.stage_items_ptrs(metric, d, ids, base + ids.astype(np.uint64) * np.uint64(ll))
            nxt = n
            for name, add, dele in (("+100", 100, 0), ("+10000/-1000", 10_000, 1_000), ("+100000", 100_000, 0)):
                new = np.arange(nxt, nxt + add, dtype=np.uint32)
                gone = np.arange(dele, dtype=np.uint32) * 7 + 1
                ids = np.union1d(np.setdiff1d(ids, gone), new).astype(np.uint32)
                nxt += add
                ptrs = base + ids.astype(np.uint64) * np.uint64(ll)
                torch.cuda.synchronize()
                t0 = time.perf_counter()
                if full:
                    ctx.stage_items_ptrs(metric, d, ids, ptrs)
                else:
                    ctx.stage_items_delta(metric, d, ids, ptrs, np.union1d(gone, new).astype(np.uint32))
                dt = (time.perf_counter() - t0) * 1e3
                st = ctx.stage_stats()
                out.append({"leg": "bq", "round": rnd, "step": name, "mode": "full" if full else "resident", "stage_ms": round(dt, 2),
                            "h2d_MB": round(st["h2d_bytes"] / 1e6, 2), "uploaded_rows": st["uploaded_rows"], "moved_rows": st["moved_rows"], "delta": st["delta"]})
                print(json.dumps(out[-1]), flush=True)
    return out


def move_alone(ctx, metric, d, n, iters=10):
    """a delta staging that moves (nearly) every row by one place, up then down again, under CUDA events around the whole call"""
    m = ab.METRICS[metric]
    ll = 5 + ((d + 63) // 64 * 8 if m >= 4 else 4 * d)
    rb = 16 * ((d + 127) // 128) if m >= 4 else 4 * ((d + 31) // 32 * 32)
    pool = np.zeros((n + 1, ll), np.uint8)
    base = np.uint64(pool.ctypes.data)
    a, b = np.arange(1, n + 1, dtype=np.uint32), np.arange(0, n, dtype=np.uint32)   # dropping id n and adding id 0 moves n - 1 rows up
    ptr = lambda ids: base + ids.astype(np.uint64) * np.uint64(ll)   # noqa: E731
    ctx.stage_items_ptrs(metric, d, a, ptr(a))
    ms = []
    for it in range(iters + 2):
        cur, chg = (b, [0, n]) if it % 2 == 0 else (a, [0, n])
        ctx.timer_start()
        ctx.stage_items_delta(metric, d, cur, ptr(cur), np.array(chg, dtype=np.uint32))
        t = ctx.timer_stop()
        st = ctx.stage_stats()
        assert st["delta"] == 1 and st["moved_rows"] == n - 1, st
        if it >= 2:
            ms.append(t)
    med = float(np.median(ms))
    algo = 2.0 * (n - 1) * rb
    res = {"leg": "move", "metric": metric, "n": n, "row_bytes": rb, "moved_rows": n - 1, "median_ms": round(med, 3), "min_ms": round(min(ms), 3),
           "algorithmic_GB": round(algo / 1e9, 3), "call_share_of_datasheet_3.35TBps": round(algo / (med * 1e-3) / HBM_DATASHEET, 3)}
    print(json.dumps(res), flush=True)
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--n", type=int, default=1_000_000)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--trees", type=int, default=50)
    ap.add_argument("--out", default=None, help="write the JSON results here as well")
    a = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("bench_resident_items needs a CUDA device: there is no fallback")
    print("card:", card(), flush=True)
    ctx = ab.Context(0)
    results = {"card": card(), "c2": [], "bq": [], "move": []}
    results["move"].append(move_alone(ctx, "cosine", 768, a.n))
    results["move"].append(move_alone(ctx, "binary quantized cosine", 1536, a.n))
    results["bq"] = bq_leg(ctx, a.n, 1536, a.rounds)
    host = synth(ctx, a.n + 110_100, 768)
    for rnd in range(a.rounds):
        for full in (True, False):
            for row in c2_round(ctx, host, a.n, 768, a.trees, full):
                row["round"] = rnd
                results["c2"].append(row)
    os.environ.pop("ARROY_B200_FULL_RESTAGE", None)
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as f:
            json.dump(results, f, indent=1)
    ctx.close()


if __name__ == "__main__":
    main()
