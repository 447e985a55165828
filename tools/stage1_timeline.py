"""Where stage 1 of the filtered sweep spends its time on the factored grid mean (filter_grid_mean_kernel,
DESIGN.md section 3.5).

Builds C2 as bench.py does (256 x 256 pendulum grid, two M=500 GPs, two factors), flushes L2 with the
same 256 MiB write before every sweep and reads the %globaltimer marks of slb_debug_stage1_timing: per
tile the time its last warp passed entry, the prologue (z, V(x), threshold and regime of every point),
each work item (factor, regime), the means and exit.  Prints, as the median over the sweeps, each mark
after the CTA's entry for the median CTA, the slowest single-regime CTA (two items at C2) and the slowest
mixed CTA (more), and the spread of the CTAs' entry times.

    python tools/stage1_timeline.py [--sweeps N]
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

MARKS = ["entry", "prologue", "item 0", "item 1", "item 2", "item 3+", "means", "exit"]
TILE = 16


def build():
    par = W.make_pendulum(num_points=bench.GRID, M=bench.M_TRAIN, shared_hypers=False)
    lyap = W.build_product(par)
    for _ in range(3):
        lyap.update_safe_set()
    torch.cuda.synchronize()
    return lyap


def timeline(lyap, sweeps):
    lib = nat.load()
    desc = lyap.sweep_descriptor()
    assert lib.slb_filter_mean_scheme(desc) == nat.MEAN_GRID_FACTORED
    n0, n1 = desc.grid.num_points[0], desc.grid.num_points[1]
    tiles = -(-n0 // TILE) * -(-n1 // TILE)
    flush = torch.empty(256 << 20, dtype=torch.uint8, device="cuda")
    buf = torch.zeros((tiles, 8), dtype=torch.int64, device="cuda")
    rows = []
    for _ in range(sweeps):
        flush.fill_(1)
        buf.zero_()
        nat.check(lib.slb_debug_stage1_timing(buf.data_ptr()), "slb_debug_stage1_timing")
        lyap.compute_negative()
        torch.cuda.synchronize()
        nat.check(lib.slb_debug_stage1_timing(None), "slb_debug_stage1_timing")
        rows.append(buf.cpu().numpy().astype(np.float64))
    print("device:", torch.cuda.get_device_name(0), "| sweeps:", sweeps, "| tiles:", tiles)
    items = (rows[0][:, 2:6] > 0).sum(axis=1)
    single, mixed = items <= 2, items > 2
    print("tiles by work items: %s" % {int(k): int((items == k).sum()) for k in np.unique(items)})
    spread, total, groups = [], [], {"median CTA": [], "slowest single-regime": [], "slowest mixed": []}
    for t in rows:
        t0 = t[:, 0]
        spread.append((t0.max() - t0.min()) * 1e-3)
        total.append((t[:, 7].max() - t0.min()) * 1e-3)
        rel = np.where(t > 0, t - t0[:, None], np.nan) * 1e-3
        groups["median CTA"].append(np.nanmedian(rel, axis=0))
        for name, sel in (("slowest single-regime", single), ("slowest mixed", mixed)):
            if sel.any():
                worst = np.nanargmax(np.where(sel, rel[:, 7], np.nan))
                groups[name].append(rel[worst])
    print("CTA entry spread (last - first entry): %.2f us" % np.median(spread))
    print("first CTA entry -> last CTA exit: %.2f us" % np.median(total))
    names = [k for k in groups if groups[k]]
    print("%-22s" % "mark (us after entry)" + "".join("%24s" % k for k in names))
    with np.errstate(all="ignore"):
        med = {k: np.nanmedian(np.array(groups[k]), axis=0) for k in names}
    for i, name in enumerate(MARKS):
        print("%-22s" % name + "".join("%24.2f" % med[k][i] for k in names))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--sweeps", type=int, default=50)
    args = ap.parse_args()
    timeline(build(), args.sweeps)


if __name__ == "__main__":
    main()
