"""Secondary measurements (not the bench.py headline): one JSON line each.

  bellman   C3: PolicyIteration.value_iteration on a 512x512 grid, GP-mean dynamics M=500
  det       deterministic-dynamics Lyapunov sweep (true pendulum plant) on large grids: the
            HBM-side variant of the path (SURVEY.md section 8d)
  c5        resolution x M sweep of the GP Lyapunov sweep kernel (C5), single GPU
  shared    C2 with shared hyper-parameters (one Cholesky factor for both outputs)
  det_linear  deterministic LinearSystem dynamics on 4096^2 / 8192^2 (closest to the HBM roofline)
  c4        cart-pole 32^4 grid, M=2000, four factors, LyapunovNetwork V (C4 at 1-GPU size)
  nb        the reference's 2001x1501 pendulum experiment with its own covariance expressions

    python tools/bench_extra.py [bellman] [det] [c5] [shared]
"""
import json
import os
import sys

import numpy as np
import scipy.linalg

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import torch  # noqa: E402

import bench_workloads as W  # noqa: E402
import safe_learning_b200 as sl  # noqa: E402
from bench import algorithmic_flops_per_point  # noqa: E402
from bench import DMMA_PEAK_TFLOPS as PEAK_TF, HBM_PEAK_GBS as HBM_GBS  # noqa: E402


def timed(fn, steps=10, warmup=3):
    for _ in range(warmup):
        fn()
    torch.cuda.synchronize()
    ev = []
    for _ in range(steps):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        fn()
        e1.record()
        ev.append((e0, e1))
    torch.cuda.synchronize()
    return float(np.median([a.elapsed_time(b) for a, b in ev]))


def bellman():
    par = W.make_pendulum(num_points=8, M=500)
    grid = sl.GridWorld(par["limits"], 512)
    _, dyn = W._build(sl, par, "product")
    policy = sl.Saturation(sl.LinearSystem(-par["K"]), -1., 1.)
    reward = sl.QuadraticFunction(-scipy.linalg.block_diag(np.diag([1., 2.]), 1.2 * np.eye(1)))
    value = sl.Triangulation(grid, np.zeros((grid.nindex, 1)), project=True)
    rl = sl.PolicyIteration(policy, dyn, reward, value, gamma=0.98)
    ms = timed(rl.value_iteration, steps=10)
    n = grid.nindex
    exps = 2 * 500
    print(json.dumps({"bench": "bellman_value_iteration", "grid": "512x512", "M": 500,
                      "ms_per_sweep": ms, "state_updates_per_s": n / (ms * 1e-3),
                      "exp_per_s": n * exps / (ms * 1e-3),
                      "note": "mean-only GP dynamics (2 x 500 fp64 exp per state), Triangulation V "
                              "gather, Jacobi; includes max|dV| reduction and table swap"}))


def det():
    for num in (1024, 4096):
        par = W.make_pendulum(num_points=num, M=8)
        lyap = W.build_product(par, deterministic=True)
        ms = timed(lyap.compute_negative, steps=10)
        n = lyap.discretization.nindex
        ms_full = timed(lyap.update_safe_set, steps=5)
        print(json.dumps({"bench": "deterministic_sweep", "grid": "%dx%d" % (num, num),
                          "kernel_ms": ms, "points_per_s": n / (ms * 1e-3),
                          "hbm_algorithmic_gbs": n * 17 / (ms * 1e-3) * 1e-9,
                          "hbm_frac_of_measured": n * 17 / (ms * 1e-3) * 1e-9 / HBM_GBS,
                          "update_safe_set_ms": ms_full,
                          "update_safe_set_points_per_s": n / (ms_full * 1e-3),
                          "note": "pendulum plant: 10 Euler sub-steps with fp64 sin per point -> "
                                  "fp64-CUDA-core bound, not HBM bound; 17 algorithmic B/pt"}))


def det_linear():
    """Cheapest deterministic variant: LinearSystem dynamics, quadratic V, |2Px| Lipschitz term --
    ~10^2 fp64 operations per point against 17 algorithmic HBM bytes."""
    for num in (4096, 8192):
        par = W.make_pendulum(num_points=num, M=8)
        grid = sl.GridWorld(par["limits"], par["num_points"])
        policy = sl.Saturation(sl.LinearSystem(-par["K"]), -1., 1.)
        dyn = sl.LinearSystem((par["A_true"], par["B_true"]))
        lyap = sl.Lyapunov(grid, sl.QuadraticFunction(par["P"]), dyn, par["L_dyn"],
                           abs(sl.LinearSystem((2 * par["P"],))), par["tau"], policy)
        from safe_learning_b200 import _native as nat
        lib = nat.load()
        n = grid.nindex
        for fast in (1, 0):
            lib.slb_debug_det_fast(fast)
            ms = timed(lyap.compute_negative, steps=10)
            print(json.dumps({"bench": "deterministic_linear_sweep", "grid": "%dx%d" % (num, num),
                              "kernel": "det_sweep_fast_kernel (specialised)" if fast else
                                        "det_sweep_kernel (generic interpreter)",
                              "kernel_ms": ms, "points_per_s": n / (ms * 1e-3),
                              "hbm_algorithmic_gbs": n * 17 / (ms * 1e-3) * 1e-9,
                              "hbm_frac_of_measured": n * 17 / (ms * 1e-3) * 1e-9 / HBM_GBS,
                              "note": "writes 1 B flag per point (V not written); coordinates "
                                      "generated; 17 algorithmic B/pt"}))
        lib.slb_debug_det_fast(1)
        del lyap
        torch.cuda.empty_cache()


def c4():
    """C4 at single-GPU size: 4-D cart-pole grid 32^4, four RBF GPs on 5-D inputs (M=2000, four
    Cholesky factors), V = LyapunovNetwork(4, [64, 64, 64], tanh)."""
    par = W.make_cartpole(num_points=32, M=2000)
    lyap = W.build_product(par)
    ms = timed(lyap.update_safe_set, steps=2, warmup=1)
    n = lyap.discretization.nindex
    fl = algorithmic_flops_per_point(2000, 5, 4, 4)
    print(json.dumps({"bench": "c4_cartpole_update_safe_set", "grid": "32^4", "M": 2000,
                      "factors": 4, "ms_per_sweep": ms, "points_per_s": n / (ms * 1e-3),
                      "tflops": fl * n / (ms * 1e-3) * 1e-12,
                      "frac_of_fp64_peak": fl * n / (ms * 1e-3) * 1e-12 / PEAK_TF}))


def c5():
    """Resolution x M points of the pendulum sweep on one GPU: the default (filtered) decision pass
    and the full posterior for every point (the kernel the algorithmic FLOP count describes)."""
    for num, M in ((128, 100), (256, 100), (256, 200), (256, 500), (512, 500), (1024, 500),
                   (2048, 500), (256, 1000), (256, 2000), (128, 5000)):
        par = W.make_pendulum(num_points=num, M=M)
        lyap = W.build_product(par)
        lyap.reset_filter_stats()
        lyap.compute_negative()
        fs = lyap.filter_stats
        ms = timed(lyap.compute_negative, steps=5, warmup=2)
        ms_step = timed(lyap.update_safe_set, steps=5, warmup=2)
        lyap.filter = False
        ms_full = timed(lyap.compute_negative, steps=3, warmup=1)
        n = lyap.discretization.nindex
        fl = algorithmic_flops_per_point(M, 3, 2, 2)
        print(json.dumps({"bench": "c5_gp_sweep", "grid": "%dx%d" % (num, num), "M": M,
                          "decision_ms": ms, "update_safe_set_ms": ms_step,
                          "points_per_s": n / (ms_step * 1e-3),
                          "refined_frac": fs["refined"] / max(fs["points"], 1),
                          "full_posterior_kernel_ms": ms_full,
                          "full_posterior_points_per_s": n / (ms_full * 1e-3),
                          "full_posterior_tflops": fl * n / (ms_full * 1e-3) * 1e-12,
                          "full_posterior_frac_of_fp64_peak": fl * n / (ms_full * 1e-3) * 1e-12 / PEAK_TF}))
        del lyap
        torch.cuda.empty_cache()


def nb():
    """The reference's own pendulum experiment (examples/inverted_pendulum.ipynb cells 4-6): 2001 x
    1501 grid, per-output kernel Linear(3, ARD) + Matern32(1, active_dims=[0]) * Linear(1), linear
    prior mean, two factors; M as it grows during the learning loop."""
    for M in (50, 200, 500):
        par = W.make_pendulum(num_points=[2001, 1501], M=M, with_prior_mean=True)
        par["kernel_specs"] = W.notebook_pendulum_kernels([[2e-3, 6e-3, 1.5e-3], [2.5e-2, 8e-3, 1.2e-2]])
        lyap = W.build_product(par)
        ms = timed(lyap.compute_negative, steps=3, warmup=1)
        ms_full = timed(lyap.update_safe_set, steps=3, warmup=1)
        n = lyap.discretization.nindex
        fl = algorithmic_flops_per_point(M, 3, 2, 2)
        print(json.dumps({"bench": "notebook_pendulum_kernels", "grid": "2001x1501", "M": M,
                          "kernel": "Linear(3,ARD) + Matern32(1,[0]) * Linear(1)",
                          "kernel_ms": ms, "update_safe_set_ms": ms_full,
                          "points_per_s": n / (ms_full * 1e-3),
                          "tflops_rbf_equivalent": fl * n / (ms * 1e-3) * 1e-12,
                          "frac_of_fp64_peak_rbf_equivalent": fl * n / (ms * 1e-3) * 1e-12 / PEAK_TF}))
        del lyap
        torch.cuda.empty_cache()


def shared():
    par = W.make_pendulum(num_points=256, M=500, shared_hypers=True)
    lyap = W.build_product(par)
    ms = timed(lyap.compute_negative, steps=10)
    ms_full = timed(lyap.update_safe_set, steps=10)
    n = lyap.discretization.nindex
    fl = algorithmic_flops_per_point(500, 3, 1, 2)
    print(json.dumps({"bench": "c2_shared_factor", "grid": "256x256", "M": 500, "factors": 1,
                      "kernel_ms": ms, "points_per_s_kernel": n / (ms * 1e-3),
                      "update_safe_set_ms": ms_full, "points_per_s": n / (ms_full * 1e-3),
                      "tflops": fl * n / (ms * 1e-3) * 1e-12,
                      "frac_of_fp64_peak": fl * n / (ms * 1e-3) * 1e-12 / PEAK_TF}))


def argmax():
    """discrete_policy_optimization at C3 size: 512 x 512 states, |A| = 101, GP-mean dynamics M=500;
    the factored tensor-core path (csrc/bellman_tile.cu) against one sweep per action."""
    par = W.make_pendulum(num_points=8, M=500)
    grid = sl.GridWorld(par["limits"], 512)
    _, dyn = W._build(sl, par, "product")
    reward = sl.QuadraticFunction(-scipy.linalg.block_diag(np.diag([1., 2.]), 1.2 * np.eye(1)))
    value = sl.Triangulation(grid, np.random.default_rng(0).normal(size=(grid.nindex, 1)), project=True)
    policy = sl.Triangulation(grid, np.zeros((grid.nindex, 1)), project=True)
    rl = sl.PolicyIteration(policy, dyn, reward, value, gamma=0.98)
    actions = np.linspace(-1, 1, 101).reshape(-1, 1)
    out = {}
    for name, flag in (("factored", True), ("per_action_sweeps", False)):
        rl.factor_actions = flag
        ms = timed(lambda: rl.discrete_policy_optimization(actions), steps=3, warmup=1)
        out[name] = {"ms": ms, "policy": policy.parameters[0].copy()}
    same = float(np.mean(out["factored"]["policy"] == out["per_action_sweeps"]["policy"]))
    n = grid.nindex
    flops = 2.0 * n * 101 * 500 * 2
    print(json.dumps({"bench": "discrete_policy_optimization", "grid": "512x512", "actions": 101,
                      "M": 500, "factored_ms": out["factored"]["ms"],
                      "per_action_sweeps_ms": out["per_action_sweeps"]["ms"],
                      "speedup": out["per_action_sweeps"]["ms"] / out["factored"]["ms"],
                      "factored_tflops": flops / (out["factored"]["ms"] * 1e-3) * 1e-12,
                      "same_greedy_action_frac": same}))


if __name__ == "__main__":
    which = sys.argv[1:] or ["bellman", "det", "det_linear", "c5", "shared", "c4", "nb", "argmax"]
    for name in which:
        globals()[name]()
