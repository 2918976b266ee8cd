"""Micro-benchmark of the side()/margin scan kernel (the roofline kernel of SURVEY.md §8d):
synthetic N x d matrix generated on the device, contiguous and gathered row lists."""
import argparse
import json
import os
import sys

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import arroy_b200  # noqa: E402


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--n", type=int, default=1_000_000)
    ap.add_argument("--d", type=int, default=768)
    ap.add_argument("--iters", type=int, default=10)
    ap.add_argument("--metric", default="cosine")
    ap.add_argument("--variants", default="0")
    args = ap.parse_args()
    peaks = {"hbm_gbs": 6592.9}
    pk = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "MEASURED_PEAKS.json")
    if os.path.exists(pk):
        peaks = json.load(open(pk))
    ctx = arroy_b200.Context(0)
    t = torch.empty((args.n, args.d), dtype=torch.float32, device="cuda:0")
    ctx.synth_device(bytes([42] * 32), args.d, 0, args.n, 0.5, t.data_ptr())
    ctx.stage_items_device(args.metric, np.arange(args.n, dtype=np.uint32), args.d, t.data_ptr())
    del t
    torch.cuda.empty_cache()
    r = np.random.default_rng(0)
    normal = (r.standard_normal(args.d) / np.sqrt(args.d)).astype(np.float32)
    out = []
    # the same row lists for every variant, so that their Left counts can be compared
    cases = (("contiguous", None), ("gathered_half", np.sort(r.choice(args.n, size=args.n // 2, replace=False)).astype(np.uint32)),
             ("gathered_4k", np.sort(r.choice(args.n, size=4096, replace=False)).astype(np.uint32)))
    for variant in [int(v) for v in args.variants.split(",")]:
        for name, rows in cases:
            n_rows = args.n if rows is None else rows.size
            ms, left = ctx.time_scan(normal, (0.0, 0.0), n_rows, rows=rows, iters=args.iters, flush_l2=True, variant=variant)
            rec = {"variant": variant, "rows": name, "n_rows": n_rows, "d": args.d, "ms": round(ms, 4)}
            if variant == 1:
                # the pre-filter reads the hi plane of every row, the lo plane of stage 2's rows and the f32 row of stage 3's
                st = ctx.build_prefilter_stats()
                nbytes = n_rows * args.d + st["rows_stage2"] * args.d + st["rows_rescored_f32"] * args.d * 4
                rec.update(stage2_frac=round(st["rows_stage2"] / n_rows, 5), stage3_frac=round(st["rows_rescored_f32"] / n_rows, 6))
            else:
                nbytes = n_rows * args.d * 4
            gbs = nbytes / (ms * 1e-3) / 1e9
            rec.update(GBps=round(gbs, 1), frac_of_measured_hbm=round(gbs / peaks["hbm_gbs"], 3), left=left)
            print(json.dumps(rec), flush=True)
            out.append(rec)
    return out


if __name__ == "__main__":
    main()
