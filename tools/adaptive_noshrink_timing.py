"""Time cell 25 of the reference's ``examples/adaptive_safety_verification.ipynb`` at the notebook's own size:
``update_safe_set(can_shrink=False, N_max=16, safety_factor=1.)`` on a 501 x 501 grid with GP dynamics of the
cell 9 kernel ``Linear(3, ARD) + Matern32(1, active_dims=[0]) * Linear(1)``, after every 10 measurements
chosen by ``get_safe_sample(positive=True)`` (cell 23), for 12 rounds.

Each update is timed with a host clock that ends in a device synchronise.  Its split is measured in the same
call, with a synchronise around each phase: the sweep with details (``compute_negative``), the refined mesh
checks (``_refined_mesh_check``), and the rest -- V sort, ``slb_no_shrink_scan``, ``slb_no_shrink_resolve``
and the read-back.  Prints one JSON line with the card's name and power limit.

    python tools/adaptive_noshrink_timing.py [--points 501] [--rounds 12] [--per-round 10]
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


def notebook_lyapunov(points):
    """Cells 7-17: true and "wrong" pendulum, the cell 9 GPs on one zero data point, LQR policy, P, L_V."""
    theta_max, omega_max = np.deg2rad(30), np.sqrt(9.81 / 0.5)
    u_max = 9.81 * 0.15 * 0.5 * np.sin(theta_max)
    norm = [(theta_max, omega_max), (u_max,)]
    true_pendulum = sl.InvertedPendulum(0.15, 0.5, 0.1, 0.01, normalization=norm)
    A_true, B_true = true_pendulum.linearize()
    A, B = sl.InvertedPendulum(0.1, 0.4, 0.0, 0.01, normalization=norm).linearize()
    prior_variances = np.clip((np.hstack((A_true, B_true)) - np.hstack((A, B))) ** 2, 1e-3, None)
    gps = []
    for j, spec in enumerate(W.notebook_pendulum_kernels(prior_variances)):
        gp = sl.GPRCached(np.zeros((1, 3)), np.zeros((1, 1)), W.build_kernel(sl, spec),
                          mean_function=sl.LinearSystem(np.hstack((A, B))[[j]]), noise_variance=0.001 ** 2)
        gps.append(sl.GaussianProcess(gp, beta=2.))
    grid = sl.GridWorld(np.array([[-1., 1.]] * 2), points)
    tau = float(np.sum(grid.unit_maxes) / 2)
    initial = np.linalg.norm(grid.all_points, ord=2, axis=1) <= 0.2
    K, P = W._dlqr(A_true, B_true, np.diag([1., 2.]), 1.2 * np.eye(1))
    P = P / np.abs(P).max()
    L_dyn = np.linalg.norm(A_true, 1) + np.linalg.norm(B_true, 1) * np.linalg.norm(-K, 1)
    policy = sl.Saturation(sl.LinearSystem(-K), -1., 1.)
    l_v = sl.AbsFunction(sl.LinearSystem((2 * P,)))
    lyap = sl.Lyapunov(grid, sl.QuadraticFunction(P), sl.FunctionStack(gps), float(L_dyn), l_v, tau, policy,
                       initial, adaptive=True)
    return lyap, true_pendulum


def timed(fn, bucket, key):
    def wrapper(*args, **kwargs):
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        out = fn(*args, **kwargs)
        torch.cuda.synchronize()
        bucket[key] += time.perf_counter() - t0
        return out
    return wrapper


def _card():
    q = subprocess.run(["nvidia-smi", "-i", str(torch.cuda.current_device()), "--query-gpu=power.limit",
                        "--format=csv,noheader,nounits"], stdout=subprocess.PIPE, text=True)
    return {"gpu": torch.cuda.get_device_name(), "power_limit_w": q.stdout.strip() or None}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--points", type=int, default=501)
    ap.add_argument("--rounds", type=int, default=12)
    ap.add_argument("--per-round", type=int, default=10)
    ap.add_argument("--n-max", type=int, default=16)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("adaptive_noshrink_timing: no CUDA device")
    np.random.seed(0)
    lyap, true_pendulum = notebook_lyapunov(args.points)
    lyap.update_safe_set()                                           # cell 17
    bucket = {"sweep": 0.0, "mesh": 0.0}
    lyap.compute_negative = timed(lyap.compute_negative, bucket, "sweep")
    lyap._refined_mesh_check = timed(lyap._refined_mesh_check, bucket, "mesh")
    rounds = []
    for _ in range(args.rounds):
        for _ in range(args.per_round):                              # cell 23: update_gp()
            sa, _ = sl.get_safe_sample(lyap, np.array([[0.]]), np.array([[-1., 1.]]), positive=True,
                                       num_samples=1000)
            lyap.dynamics.add_data_point(sa, true_pendulum(sa))
        bucket["sweep"] = bucket["mesh"] = 0.0
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        lyap.update_safe_set(False, args.n_max, 1., 4)              # cell 25
        torch.cuda.synchronize()
        total = time.perf_counter() - t0
        rounds.append({"total_ms": round(1e3 * total, 3), "sweep_ms": round(1e3 * bucket["sweep"], 3),
                       "mesh_ms": round(1e3 * bucket["mesh"], 3),
                       "scan_resolve_ms": round(1e3 * (total - bucket["sweep"] - bucket["mesh"]), 3),
                       "safe_fraction": round(float(lyap.safe_set.mean()), 5),
                       "refined_cells": int((np.asarray(lyap._refinement) > 1).sum()),
                       "c_max": float(lyap.feed_dict[lyap.c_max])})
    med = {k: float(np.median([r[k] for r in rounds[1:] or rounds]))
           for k in ("total_ms", "sweep_ms", "mesh_ms", "scan_resolve_ms")}
    out = {"tool": "adaptive_noshrink_timing", "points": lyap.discretization.nindex, "n_max": args.n_max,
           "rounds": rounds, "median_after_first": med}
    out.update(_card())
    print(json.dumps(out))


if __name__ == "__main__":
    main()
