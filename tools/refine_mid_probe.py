"""Refine pass on mid-size lists (between ~600 and 4736 points: fewer spare CTAs per 32-point tile): stage time
of the refine pass for a few discretisation constants of the C2 workload."""
import json, os, sys
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch
import bench_workloads as W
from safe_learning_b200 import _native as nat
lib = nat.load()
flush = torch.empty(256 << 20, dtype=torch.uint8, device="cuda")


def timed(fn, steps=20):
    ev = []
    for _ in range(steps):
        flush.fill_(1)
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record(); fn(); e1.record(); ev.append((e0, e1))
    torch.cuda.synchronize()
    per = sorted(a.elapsed_time(b) for a, b in ev)
    return per[len(per) // 2]


for ts in (1 / 8., 1 / 16., 1 / 24., 1 / 32., 1 / 48.):
    par = W.make_pendulum(num_points=256, M=500, shared_hypers=False, tau_scale=ts)
    lyap = W.build_product(par)
    lyap.reset_filter_stats(); lyap.compute_negative(); st = lyap.filter_stats
    out = {"tau_scale": ts, "refined": st["refined"], "tiles32": -(-st["refined"] // 32)}
    for stage, mask in (("mean_head", 1), ("all", 3)):
        lib.slb_debug_filter_stages(mask)
        for _ in range(3):
            lyap.compute_negative()
        out[stage + "_ms"] = timed(lyap.compute_negative)
    lib.slb_debug_filter_stages(3)
    out["refine_us"] = round(1e3 * (out["all_ms"] - out["mean_head_ms"]), 1)
    print(json.dumps(out), flush=True)
