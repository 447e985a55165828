"""Time ``compute_roa`` of the reverse-time Van der Pol plant and of the normalised inverted pendulum on the
same 1001 x 1001 grid and horizon, both as fused closed loops (one CUDA pass per chunk of steps).  Prints
one JSON line: per plant the median time of a call (CUDA events, after warm-up), the rate in point-steps
per second and the size of the region of attraction found; with the card's name and power limit.

    python tools/vanderpol_roa.py [--points 1001] [--horizon 1000] [--repeats 5]
"""
import argparse
import json
import os
import subprocess
import sys

import numpy as np
import scipy.linalg
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import safe_learning_b200 as sl  # noqa: E402


def _loops():
    """(name, ClosedLoop) of each plant: Van der Pol with the zero policy it needs for its action column,
    the pendulum with the saturated LQR of reinforcement_learning_pendulum.ipynb cells 7-14."""
    vdp = sl.VanDerPol(damping=1, dt=0.01, normalization=(2.5, 3.0))
    theta_max, omega_max = np.deg2rad(30), np.sqrt(9.81 / 0.5)
    u_max = 9.81 * 0.15 * 0.5 * np.sin(theta_max)
    pend = sl.InvertedPendulum(0.15, 0.5, 0.1, 0.01, normalization=[(theta_max, omega_max), (u_max,)])
    A, B = pend.linearize()
    Q, R = 0.1 * np.eye(2), 0.1 * np.eye(1)
    P = scipy.linalg.solve_discrete_are(A, B, Q, R)
    K = np.linalg.solve(B.T.dot(P).dot(B) + R, B.T.dot(P).dot(A))
    return [("vanderpol", sl.ClosedLoop(vdp, sl.LinearSystem(np.zeros((1, 2))))),
            ("pendulum", sl.ClosedLoop(pend, sl.Saturation(sl.LinearSystem((-K,)), -1., 1.)))]


def _card():
    q = subprocess.run(["nvidia-smi", "-i", str(torch.cuda.current_device()), "--query-gpu=power.limit",
                        "--format=csv,noheader,nounits"], stdout=subprocess.PIPE, text=True)
    return {"gpu": torch.cuda.get_device_name(), "power_limit_w": q.stdout.strip() or None}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--points", type=int, default=1001)
    ap.add_argument("--horizon", type=int, default=1000)
    ap.add_argument("--tol", type=float, default=0.05)
    ap.add_argument("--repeats", type=int, default=5)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("vanderpol_roa: no CUDA device")
    grid = sl.GridWorld([[-1.2, 1.2], [-1.2, 1.2]], args.points)
    out = {"tool": "vanderpol_roa", "points": grid.nindex, "horizon": args.horizon}
    for name, cl in _loops():
        roa = sl.compute_roa(grid, cl, args.horizon, args.tol)            # warm-up
        times = []
        for _ in range(args.repeats):
            start, stop = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            start.record()
            roa = sl.compute_roa(grid, cl, args.horizon, args.tol)
            stop.record()
            torch.cuda.synchronize()
            times.append(start.elapsed_time(stop) / 1e3)
        t = float(np.median(times))
        out[name] = {"seconds": round(t, 6), "point_steps_per_s": float("%.4g" % (grid.nindex * (args.horizon - 1) / t)),
                     "roa_points": int(roa.sum())}
    out.update(_card())
    print(json.dumps(out))


if __name__ == "__main__":
    main()
