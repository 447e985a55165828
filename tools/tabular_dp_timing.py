"""Time tabular dynamic programming on a 512 x 512 grid: ``value_iteration``,
``discrete_policy_optimization`` (101 actions) and ``optimize_value_function`` with ``PiecewiseConstant``
value and policy tables, against the same calls on ``Triangulation`` tables, with the C3 GP dynamics (two
RBF factors of M = 500 rows) and with the deterministic inverted pendulum.

    python tools/tabular_dp_timing.py [--reps 5] [--out tabular_dp.json]

Each call is warmed up once, then timed with a device synchronise around every repetition (every
``optimize_value_function`` starts from the same table, reset outside the timed region); the median and
the spread are printed with the card's name and power limit (read in the same run).
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
import safe_learning_b200 as sl  # noqa: E402


def card():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                             capture_output=True, text=True, check=True).stdout.strip().splitlines()[0]
    except (OSError, subprocess.CalledProcessError, IndexError):
        out = torch.cuda.get_device_name(0) + ", power limit not read"
    return out


def setup(kind, dynamics):
    par = W.make_pendulum(num_points=8, M=500)
    grid = sl.GridWorld(par["limits"], 512)
    if dynamics == "gp":
        _, dyn = W._build(sl, par, "product")
    else:
        pl = par["plant"]
        dyn = sl.InvertedPendulum(normalization=[pl["state_norm"], pl["action_norm"]], **pl["true"])
    reward = sl.QuadraticFunction(-np.diag([1., 2., 1.2]))
    pts = grid.all_points
    v0 = -np.sum(pts ** 2, axis=1, keepdims=True)
    p0 = np.clip(pts.dot(np.array([[-0.6], [-0.3]])), -1, 1)
    if kind == "table":
        value, policy = sl.PiecewiseConstant(grid, v0), sl.PiecewiseConstant(grid, p0)
    else:
        value, policy = sl.Triangulation(grid, v0, project=True), sl.Triangulation(grid, p0, project=True)
    return sl.PolicyIteration(policy, dyn, reward, value, gamma=0.98)


def timed(fn, reps, prepare=None):
    """Wall times of `reps` calls after one warm-up; `prepare` (untimed) runs before every call."""
    times = []
    for r in range(reps + 1):
        if prepare is not None:
            prepare()
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        fn()
        torch.cuda.synchronize()
        if r:
            times.append(time.perf_counter() - t0)
    return times


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    actions = np.linspace(-1, 1, 101)[:, None]
    rows = []
    print("card:", card())
    for dynamics in ("gp", "pendulum"):
        for kind in ("table", "triangulation"):
            rl = setup(kind, dynamics)
            p0 = rl.policy.parameters if kind == "table" else rl.policy.parameters[0]
            v0 = rl.value_function.parameters if kind == "table" else rl.value_function.parameters[0]
            calls = {"value_iteration": rl.value_iteration,
                     "discrete_policy_optimization": lambda: rl.discrete_policy_optimization(actions)}
            for name, fn in calls.items():
                t = timed(fn, args.reps)
                rows.append(dict(dynamics=dynamics, value=kind, call=name, median_ms=1e3 * float(np.median(t)),
                                 min_ms=1e3 * min(t), max_ms=1e3 * max(t)))
            rl.policy.parameters = p0

            def reset():                  # every solve starts from the same table
                rl.value_function.parameters = v0
            try:
                t = timed(lambda: rl.optimize_value_function(max_iters=20000), args.reps, reset)
                extra = dict(iterations=rl.last_solve["iterations"], tier=rl.last_solve["tier"])
            except sl.OptimizationError as e:
                t, extra = [float("nan")], dict(error=str(e)[:80])
            rows.append(dict(dynamics=dynamics, value=kind, call="optimize_value_function",
                             median_ms=1e3 * float(np.median(t)), min_ms=1e3 * min(t), max_ms=1e3 * max(t), **extra))
            for r in rows[-3:]:
                print(json.dumps(r))
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as f:
            json.dump(dict(card=card(), rows=rows), f, indent=1)


if __name__ == "__main__":
    main()
