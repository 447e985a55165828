"""Where the flagship step spends its time after the last decision (DESIGN.md section 6).

Builds C2 as bench.py does (256 x 256 pendulum grid, two M=500 GPs, two factors), warms the step up until
it replays as one CUDA graph, then records `--steps` replays of update_safe_set under torch.profiler with
CUDA activities, L2 flushed (the same 256 MiB write) before each.  Prints the card and its power limit,
then, as medians over the steps, the start and end of every kernel and memset of one step relative to the
step's first node, and the tail: from the end of the refine pass (the last gp_tile_kernel) to the end of
apply_prefix_kernel, with and without apply_prefix_kernel's own duration.

    python tools/step_tail_trace.py [--steps N] [--trace PATH]
"""
import argparse
import json
import os
import subprocess
import sys
import tempfile

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np
import torch

import bench
import bench_workloads as W


def card():
    name = torch.cuda.get_device_name(0)
    try:
        limit = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader", "-i",
                                str(torch.cuda.current_device())], capture_output=True, text=True,
                               timeout=30).stdout.strip()
    except (OSError, subprocess.SubprocessError):
        limit = "unknown"
    return "%s, power limit %s" % (name, limit or "unknown")


def short(name):
    if name.startswith("Memset"):
        return "memset"
    base = name[5:] if name.startswith("void ") else name
    base = base.replace("(anonymous namespace)::", "")
    args = base.split("<", 1)[1].split(">")[0].split(",") if "<" in base.split("(")[0] else []
    base = base.split("<")[0].split("(")[0].strip()
    if base == "gp_tile_kernel" and len(args) == 4:
        # the two refine launches differ in the tile size (last template argument)
        return "gp_tile_kernel tp=%s" % args[3].strip()
    return base


def record(lyap, steps, path):
    from torch.profiler import ProfilerActivity, profile
    flush = torch.empty(256 << 20, dtype=torch.uint8, device="cuda")
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(steps):
            flush.fill_(1)
            lyap.update_safe_set()
        torch.cuda.synchronize()
    prof.export_chrome_trace(path)
    with open(path) as f:
        events = json.load(f)["traceEvents"]
    dev = [e for e in events if e.get("cat") in ("kernel", "gpu_memset") and "ts" in e]
    dev.sort(key=lambda e: e["ts"])
    # one step: everything between two flushes (the flush is torch's fill kernel)
    rows, cur = [], None
    for e in dev:
        if "FillFunctor" in e["name"]:
            if cur:
                rows.append(cur)
            cur = []
        elif cur is not None:
            cur.append((short(e["name"]), float(e["ts"]), float(e["ts"]) + float(e.get("dur", 0.0))))
    if cur:
        rows.append(cur)
    return rows


def report(rows):
    shapes = {}
    for r in rows:
        shapes.setdefault(tuple(n for n, _, _ in r), []).append(r)
    names, same = max(shapes.items(), key=lambda kv: len(kv[1]))
    print("steps: %d (%d with this node sequence)" % (len(rows), len(same)))
    print("nodes per step: %d" % len(names))
    t = np.array([[[s, e] for _, s, e in r] for r in same])        # [steps, nodes, 2]
    t0 = t[:, :1, 0:1]
    rel = t - t0
    print("%-3s %-34s %10s %10s %10s" % ("#", "node", "start us", "end us", "dur us"))
    for i, n in enumerate(names):
        print("%-3d %-34s %10.2f %10.2f %10.2f" % (i + 1, n, np.median(rel[:, i, 0]), np.median(rel[:, i, 1]),
                                                 np.median(t[:, i, 1] - t[:, i, 0])))
    print("first node start -> last node end: %.2f us" % np.median(rel[:, -1, 1]))
    refine = [i for i, n in enumerate(names) if n.startswith("gp_tile_kernel")]
    prefix = [i for i, n in enumerate(names) if n.startswith("apply_prefix_kernel")]
    if refine and prefix:
        r, p = refine[-1], prefix[-1]
        tail = t[:, p, 1] - t[:, r, 1]
        own = t[:, p, 1] - t[:, p, 0]
        print("end of refine pass -> end of apply_prefix_kernel: %.2f us" % np.median(tail))
        print("  minus apply_prefix_kernel's own duration: %.2f us" % np.median(tail - own))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=100)
    ap.add_argument("--trace", default=None, help="where to keep the chrome trace (default: a temporary file)")
    args = ap.parse_args()
    par = W.make_pendulum(num_points=bench.GRID, M=bench.M_TRAIN, shared_hypers=False)
    lyap = W.build_product(par)
    for _ in range(5):
        lyap.update_safe_set()
    torch.cuda.synchronize()
    print("device:", card())
    with tempfile.TemporaryDirectory() as tmp:
        rows = record(lyap, args.steps, args.trace or os.path.join(tmp, "step.pt.trace.json"))
    report(rows)


if __name__ == "__main__":
    main()
