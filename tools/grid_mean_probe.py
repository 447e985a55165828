"""Stage 1 of the filtered sweep on the C2 grid (256 x 256, two M = 500 GPs on distinct factors): the
factored grid mean (filter_grid_mean_kernel) against the fp32 screening kernel that bit 5 of
slb_debug_filter_stages forces in its place.  Prints one JSON line per scheme: the stage timed alone
(CUDA events, median), the kernel's own time from a torch.profiler run (by name), its algorithmic fp64
FLOP/s against the DMMA peak, the table exponentials, the tile counts per policy regime, and the filter
fractions of the whole sweep (decided in stage 1 / by the head bound / refined)."""
import json
import os
import sys

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import bench_workloads as W  # noqa: E402
from safe_learning_b200 import _native as nat  # noqa: E402

GR, GC = 16, 16                 # tile of filter_grid_mean_kernel (its constants: csrc/gp_mean_grid.cuh)
DMMA_PEAK = 33.2e12             # fp64 FLOP/s measured on H100 80GB HBM3 (DESIGN.md section 6)

lib = nat.load()


def timed(fn, steps=50, warm=10):
    for _ in range(warm):
        fn()
    torch.cuda.synchronize()
    ev = []
    for _ in range(steps):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record(); fn(); b.record(); ev.append((a, b))
    torch.cuda.synchronize()
    return float(np.median([x.elapsed_time(y) for x, y in ev]))


def kernel_ms(fn, name, steps=20):
    from torch.profiler import profile, ProfilerActivity
    fn(); torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(steps):
            fn()
        torch.cuda.synchronize()
    tot, cnt = 0.0, 0
    for e in prof.key_averages():
        if name in e.key:
            tot += e.device_time_total if hasattr(e, "device_time_total") else e.cuda_time_total
            cnt += e.count
    return (tot / cnt / 1e3) if cnt else float("nan")


def regimes(par):
    """Tiles of the grid by the set of policy regimes their points are in."""
    n0, n1 = par["num_points"]
    lo = par["limits"][:, 0]
    unit = (par["limits"][:, 1] - lo) / (np.asarray(par["num_points"]) - 1)
    x0 = np.arange(n0) * unit[0] + lo[0]
    x1 = np.arange(n1) * unit[1] + lo[1]
    K = -np.asarray(par["K"]).reshape(-1)
    y = x0[:, None] * K[0] + x1[None, :] * K[1]
    reg = np.where(y <= -1.0, 0, np.where(y >= 1.0, 1, 2))
    counts, kinds = {}, []
    for r in range(0, n0, GR):
        for c in range(0, n1, GC):
            s = tuple(sorted(set(reg[r:r + GR, c:c + GC].ravel().tolist())))
            key = "+".join({0: "low", 1: "high", 2: "affine"}[v] for v in s)
            counts[key] = counts.get(key, 0) + 1
            kinds.append(len(s))
    return counts, kinds


par = W.make_pendulum(num_points=256, M=500)
lyap = W.build_product(par)
lyap.filter = True
n = 256 * 256
Mp = (500 + 7) // 8 * 8
counts, kinds = regimes(par)
for label, mask, kname in (("grid factored", 0, "filter_grid_mean_kernel"),
                           ("fp32 screening", 32, "filter_mean32_kernel")):
    lib.slb_debug_filter_stages(mask)
    scheme = lib.slb_filter_mean_scheme(lyap.sweep_descriptor())
    stage_ms = timed(lyap.compute_negative)
    k_ms = kernel_ms(lyap.compute_negative, kname)
    lib.slb_debug_filter_stages(3 | mask)
    lyap.reset_filter_stats()
    lyap.compute_negative()
    st = dict(lyap.filter_stats)
    lib.slb_debug_filter_stages(3)
    out = {"scheme": label, "mean_scheme": scheme, "stage1_ms": stage_ms, "kernel": kname, "kernel_ms": k_ms,
           "stats": st, "decided_stage1": st["prior"] / st["points"], "refined": st["refined"]}
    if mask == 0:
        flop = 2.0 * 2 * sum(k * GR * GC * Mp for k in kinds)        # two factors, every regime of a tile
        out.update({"algorithmic_flop": flop, "tflops": flop / (k_ms * 1e-3) / 1e12,
                    "of_dmma_peak": flop / (k_ms * 1e-3) / DMMA_PEAK,
                    "table_exps": 2 * sum(k * 5 * Mp for k in kinds),   # two per table column, one weight
                    "tiles": len(kinds), "tiles_per_regime_set": counts})
    print(json.dumps(out))
print(json.dumps({"gpu": torch.cuda.get_device_name(0)}))
