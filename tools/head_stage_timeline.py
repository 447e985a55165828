"""Where the head stage of the filtered sweep spends its time (filter_head_kernel, DESIGN.md section 3.5).

Builds C2 as bench.py does (256 x 256 pendulum grid, two M=500 GPs, two factors), flushes L2 with the
same 256 MiB write before every sweep and reads the %globaltimer marks of slb_debug_head_timing: per
head CTA the time its last warp passed entry, tables landed, the bound of factor 0, the bound of every
factor, the screened decision, the round's fp64 means, the final decision and exit, and the time the last
stage-1 warp left.  Prints, as the median over the sweeps, the launch gap and each span, both for the
median CTA and for the slowest.

    python tools/head_stage_timeline.py [--sweeps N] [--profile]

--profile instead times the default step (update_safe_set, L2 flushed before each) under torch.profiler
and prints the per-kernel device times.
"""
import argparse
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np
import torch

import bench
import bench_workloads as W
from safe_learning_b200 import _native as nat

MARKS = ["entry", "tables landed", "bound factor 0", "bound all factors", "screened decision",
         "round means", "final decision", "exit"]
CTAS = 132


def build():
    par = W.make_pendulum(num_points=bench.GRID, M=bench.M_TRAIN, shared_hypers=False)
    lyap = W.build_product(par)
    for _ in range(3):
        lyap.update_safe_set()
    torch.cuda.synchronize()
    return lyap


def timeline(lyap, sweeps):
    lib = nat.load()
    flush = torch.empty(256 << 20, dtype=torch.uint8, device="cuda")
    buf = torch.zeros((CTAS + 1, 8), dtype=torch.int64, device="cuda")
    rows = []
    for _ in range(sweeps):
        flush.fill_(1)
        buf.zero_()
        nat.check(lib.slb_debug_head_timing(buf.data_ptr()), "slb_debug_head_timing")
        lyap.compute_negative()
        torch.cuda.synchronize()
        nat.check(lib.slb_debug_head_timing(None), "slb_debug_head_timing")
        rows.append(buf.cpu().numpy().astype(np.float64))
    print("device:", torch.cuda.get_device_name(0), "| sweeps:", sweeps)
    gap, span, per_cta_median, worst = [], [], [], []
    for t in rows:
        head, s1_exit = t[:CTAS], t[CTAS, 0]
        t0 = head[:, 0]
        gap.append((t0.min() - s1_exit) * 1e-3)
        span.append((head[:, 7].max() - s1_exit) * 1e-3)
        working = head[:, 2] > 0                      # CTAs that had a group
        rel = np.where(head > 0, head - t0[:, None], np.nan)[working] * 1e-3
        per_cta_median.append(np.nanmedian(rel, axis=0))
        worst.append(np.nanmax(rel, axis=0))
    print("launch gap (first head CTA entry - last stage-1 warp exit): %.2f us" % np.median(gap))
    print("stage-1 exit -> last head CTA exit: %.2f us" % np.median(span))
    print("working CTAs: %d of %d" % (int((rows[-1][:CTAS, 2] > 0).sum()), CTAS))
    med, mx = np.nanmedian(np.array(per_cta_median), axis=0), np.nanmedian(np.array(worst), axis=0)
    print("%-20s %12s %12s" % ("mark (us after entry)", "median CTA", "slowest CTA"))
    for i, name in enumerate(MARKS):
        print("%-20s %12.2f %12.2f" % (name, med[i], mx[i]))


def profile(lyap, steps):
    from torch.profiler import ProfilerActivity, profile as tprofile
    flush = torch.empty(256 << 20, dtype=torch.uint8, device="cuda")
    with tprofile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(steps):
            flush.fill_(1)
            lyap.update_safe_set()
        torch.cuda.synchronize()
    print("device:", torch.cuda.get_device_name(0), "| steps:", steps)
    print(prof.key_averages().table(sort_by="self_device_time_total", row_limit=25, max_name_column_width=60))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--sweeps", type=int, default=50)
    ap.add_argument("--profile", action="store_true")
    args = ap.parse_args()
    lyap = build()
    if args.profile:
        profile(lyap, args.sweeps)
    else:
        timeline(lyap, args.sweeps)


if __name__ == "__main__":
    main()
