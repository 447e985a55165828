"""Time the rollouts of the GP mean model against the Bellman sweep on the same GP: C2's pendulum
(``bench_workloads.make_pendulum``, two RBF factors of M = 500 rows) under the saturated LQR policy.

    python tools/gp_mean_rollout_timing.py [--reps 5] [--out gp_mean_timing.json]

Workloads: ``compute_roa`` from 256^2 grid starts with horizon 500, ``reward_rollout`` from 101^2 starts
with horizon 1000 (tol 0: no early stop, every step runs), and one ``value_iteration`` sweep on a 256^2
grid.  Each is warmed up once, then timed with CUDA events over `reps` repetitions; the median, the spread
and the kernel values per second (points x steps x factors x M) are printed with the card's name and
power limit, read in the same run.  The CPU figure runs the numpy oracle's mean on 1/64 of the
``compute_roa`` starts.
"""
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

import bench_workloads as W  # noqa: E402
import oracle as O  # noqa: E402
import safe_learning_b200 as sl  # noqa: E402


def card():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                             capture_output=True, text=True, check=True).stdout.strip().splitlines()[0]
    except (OSError, subprocess.CalledProcessError, IndexError):
        out = torch.cuda.get_device_name(0) + ", power limit not read"
    return out


def timed(fn, reps):
    """CUDA-event times (s) of `reps` calls after one warm-up."""
    fn()
    times = []
    for _ in range(reps):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        torch.cuda.synchronize()
        a.record()
        fn()
        b.record()
        torch.cuda.synchronize()
        times.append(a.elapsed_time(b) / 1e3)
    return times


def row(name, times, kvals):
    med = float(np.median(times))
    return dict(workload=name, median_ms=1e3 * med, min_ms=1e3 * min(times), max_ms=1e3 * max(times),
                kernel_values=float(kvals), kernel_values_per_s=float(kvals) / med)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    par = W.make_pendulum(num_points=8, M=500)
    _, dynamics = W._build(sl, par, "product")
    policy = sl.Saturation(sl.LinearSystem(-par["K"]), -1., 1.)
    cl = sl.ClosedLoop(dynamics.to_mean_function(), policy)
    rw = sl.ClosedLoop(sl.QuadraticFunction(-np.diag([1., 2., 1.2])), policy)
    factors, M = 2, 500
    print("card:", card())
    rows = []

    grid = sl.GridWorld(par["limits"], 256)
    t = timed(lambda: sl.compute_roa(grid, cl, 500, 0.01), args.reps)
    rows.append(row("compute_roa 256^2 h=500", t, grid.nindex * 499 * factors * M))

    grid_r = sl.GridWorld(par["limits"], 101)
    with open(os.devnull, "w") as null:
        stdout, sys.stdout = sys.stdout, null
        try:
            t = timed(lambda: sl.reward_rollout(grid_r, cl, rw, 0.99, 1000, 0.0), args.reps)
        finally:
            sys.stdout = stdout
    rows.append(row("reward_rollout 101^2 h=1000", t, grid_r.nindex * 1000 * factors * M))

    value = sl.Triangulation(grid, -np.sum(grid.all_points ** 2, axis=1, keepdims=True), project=True)
    rl = sl.PolicyIteration(policy, dynamics, sl.QuadraticFunction(-np.diag([1., 2., 1.2])), value, gamma=0.98)
    t = timed(rl.value_iteration, args.reps)
    rows.append(row("value_iteration 256^2", t, grid.nindex * factors * M))

    # CPU: the numpy oracle's mean on every 64th start, the reference's loop
    _, o_dyn = W._build(O, par, "oracle")
    o_pol = O.Saturation(O.LinearSystem(-par["K"]), -1., 1.)
    starts = grid.all_points[::64]
    t0 = time.perf_counter()
    x = starts
    for _ in range(1, 500):
        x = np.asarray(o_dyn(np.hstack((x, o_pol(x))))[0])
    cpu = time.perf_counter() - t0
    kv = starts.shape[0] * 499 * factors * M
    rows.append(dict(workload="compute_roa numpy oracle, 1/64 of the starts", median_ms=1e3 * cpu,
                     kernel_values=float(kv), kernel_values_per_s=kv / cpu))
    for r in rows:
        print(json.dumps(r))
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as f:
            json.dump(dict(card=card(), rows=rows), f, indent=1)


if __name__ == "__main__":
    main()
