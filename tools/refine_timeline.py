"""Where the refine pass of the filtered sweep spends its time (gp_tile_kernel on list B, DESIGN.md section 3.1).

Builds C2 as bench.py does (256 x 256 pendulum grid, two M=500 GPs, two factors), flushes L2 with the same
256 MiB write before every sweep and reads the %globaltimer marks of slb_debug_refine_timing: per CTA of the
row-split refine launch the time its last warp passed entry, prologue, each j-panel's generation and
contraction, partial sums written, ticket taken, factor epilogues, decision and fold, and exit.  The head
stage's marks (slb_debug_head_timing) give the origin: every time is counted from the last head CTA's exit.
Prints, as the median over the sweeps, each mark for the median CTA and for the CTA that finished last.

    python tools/refine_timeline.py [--sweeps N]
"""
import argparse
import os
import sys
import warnings

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np
import torch

import bench
import bench_workloads as W
from safe_learning_b200 import _native as nat

MARKS = ["entry", "prologue done", "j-panel 0 generated", "j-panel 1 generated", "j-panel 2 generated",
         "j-panel 3+ generated", "j-panel 0 contracted", "j-panel 1 contracted", "j-panel 2 contracted",
         "j-panel 3+ contracted", "partial sums written", "ticket taken", "factor epilogues done",
         "decision and fold done", "exit"]
HEAD_CTAS = 132
ROWS, SLOTS = 512, 16


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
    head = torch.zeros((HEAD_CTAS + 1, 8), dtype=torch.int64, device="cuda")
    marks = torch.zeros((ROWS, SLOTS), dtype=torch.int64, device="cuda")
    runs = []
    for _ in range(sweeps):
        flush.fill_(1)
        head.zero_()
        marks.zero_()
        nat.check(lib.slb_debug_head_timing(head.data_ptr()), "slb_debug_head_timing")
        nat.check(lib.slb_debug_refine_timing(marks.data_ptr()), "slb_debug_refine_timing")
        lyap.compute_negative()
        torch.cuda.synchronize()
        nat.check(lib.slb_debug_head_timing(None), "slb_debug_head_timing")
        nat.check(lib.slb_debug_refine_timing(None), "slb_debug_refine_timing")
        runs.append((head.cpu().numpy().astype(np.float64), marks.cpu().numpy().astype(np.float64)))
    print("device:", torch.cuda.get_device_name(0), "| sweeps:", sweeps)
    warnings.simplefilter("ignore", RuntimeWarning)          # marks no CTA passed (j-panels beyond M) are NaN
    median_cta, last_cta, span, ctas, finishers = [], [], [], [], []
    for h, m in runs:
        origin = h[:HEAD_CTAS, 7].max()                   # the last head CTA's exit
        working = m[:, 0] > 0
        rel = np.where(m[:, :len(MARKS)] > 0, m[:, :len(MARKS)] - origin, np.nan)[working] * 1e-3
        fin = m[working, 15] == 1
        median_cta.append(np.nanmedian(rel, axis=0))
        last_cta.append(rel[fin][np.nanargmax(rel[fin, -1])])
        span.append(np.nanmax(rel[:, -1]))
        ctas.append(int(working.sum()))
        finishers.append(int(fin.sum()))
    print("refine CTAs: %d, of which finish a tile: %d" % (ctas[-1], finishers[-1]))
    print("last head CTA exit -> last refine CTA exit: %.2f us" % np.median(span))
    med = np.nanmedian(np.array(median_cta), axis=0)
    last = np.nanmedian(np.array(last_cta), axis=0)
    print("%-26s %12s %14s" % ("mark (us after head exit)", "median CTA", "last finisher"))
    for i, name in enumerate(MARKS):
        print("%-26s %12.2f %14.2f" % (name, med[i], last[i]))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--sweeps", type=int, default=50)
    args = ap.parse_args()
    timeline(build(), args.sweeps)


if __name__ == "__main__":
    main()
