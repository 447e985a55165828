"""Secondary measurements (not the bench.py headline): one JSON line each.

  bellman   C3: PolicyIteration.value_iteration on a 512x512 grid, GP-mean dynamics M=500
  det       deterministic-dynamics Lyapunov sweep (true pendulum plant) on large grids: the
            HBM-side variant of the path (SURVEY.md section 8d)
  c5        resolution x M sweep of the GP Lyapunov sweep kernel (C5), single GPU
  shared    C2 with shared hyper-parameters (one Cholesky factor for both outputs)
  det_linear  deterministic LinearSystem dynamics on 4096^2 / 8192^2 (closest to the HBM roofline)
  c4        cart-pole 32^4 grid, M=2000, four factors, LyapunovNetwork V (C4 at 1-GPU size)
  nb        the reference's 2001x1501 pendulum experiment with its own covariance expressions
  roa       compute_roa of the saturated-LQR closed loops: pendulum 2001x1501 (horizon 500),
            pendulum 101^2 with trajectories, cart-pole 51^4 (horizon 2000)
  reward_rollout  reward_rollout of the pendulum loop on 2001x1501 (discount 0.95, horizon 1000,
            tol 1e-2), reporting the stopping step T*
  value_opt PolicyIteration.optimize_value_function (gamma 0.98, tol 1e-10) with RBF GP-mean dynamics
            (bench_workloads.make_pendulum) on 55x55 (M=50, the one-CTA solver) and on C3's 512x512
            (M=500, the cooperative solver):
            operator assembly, the whole call, iterations; against scipy spsolve on the host and
            against value_iteration sweeps to the same bound
  train     slb_function_vjp (gradients of the points and of every parameter) for
            LyapunovNetwork(2, [64, 64, 64], tanh) and the 2-64-64-1 ReLU MLP on 100, 1000 and 251^2
            points, against torch's autograd of the same network on the same GPU (fp64 cuBLAS), and the
            per-step time of three notebook training loops (value net, policy net, Lyapunov pre-training)
  nn_lv     L_V = |dV/dx|_1 of a LyapunovNetwork fused into the sweeps (Norm1Function(V.gradient_function())):
            the notebook's 251^2 update_safe_set fused against composed, a 256^2 GP sweep (M = 500) and the
            C4 shape against a constant L_V, and the gradient evaluation against slb_function_vjp
  gp_vjp    reverse mode of the GP posterior (slb_gp_vjp): inverted_pendulum.ipynb cell 17's policy step
            (batch 1000, notebook-kernel FunctionStack at M = 0, 50, 200) through the GP node against
            torch_predict as a plain dynamics callable, and the VJP alone on C2's GPs (plain RBF, M = 500,
            two factors) for 10^3, 10^4 and 65536 points against the forward and torch autograd
  gp_fit    GPRCached hyper-parameter fit at M = 500, 2000, 5000 (notebook kernel and ARD RBF, d_in = 3): the
            fused gradient kernel alone, one value + gradient, torch autograd of the same, optimize(maxiter=50)

    python tools/bench_extra.py [bellman] [det] [c5] [shared] [roa] [reward_rollout] [value_opt] [train] [nn_lv] [gp_vjp]
                                [gp_fit]
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


def _rollout_parts(plant):
    """Saturated-LQR closed loop of reinforcement_learning_{pendulum,cartpole}.ipynb (cells 7-14):
    (product ClosedLoop dynamics / reward, oracle callables)."""
    sys.path.insert(0, os.path.join(ROOT, "tests"))
    import oracle as O
    import rollout_oracle as R
    if plant == "pendulum":
        norm = [np.array([np.deg2rad(30), np.sqrt(9.81 / 0.5)]), np.array([9.81 * 0.15 * 0.5 * np.sin(np.deg2rad(30))])]
        args = (0.15, 0.5, 0.1, 0.01)
        dyn, odyn = sl.InvertedPendulum(*args, normalization=norm), O.InvertedPendulum(*args, normalization=norm)
    else:
        m, M = 0.175, 1.732
        norm = [np.array([0.5, np.deg2rad(30), 2., np.deg2rad(30)]), np.array([(m + M) * 4 / 0.5])]
        args = (m, M, 0.28, 0.01, 0.01)
        dyn, odyn = sl.CartPole(*args, normalization=norm), O.CartPole(*args, normalization=norm)
    A, B = dyn.linearize()
    d = A.shape[0]
    Q, Rm = 0.1 * np.eye(d), 0.1 * np.eye(1)
    K, _ = O.dlqr(A, B, Q, Rm)
    rew = scipy.linalg.block_diag(-Q, -Rm)
    pol = sl.Saturation(sl.LinearSystem((-K,)), -1., 1.)
    opol = O.Saturation(O.LinearSystem((-K,)), -1., 1.)
    return (sl.ClosedLoop(dyn, pol), sl.ClosedLoop(sl.QuadraticFunction(rew), pol),
            R.closed_loop(odyn, opol), R.closed_loop(O.QuadraticFunction(rew), opol), R)


def _gpu_info(fn):
    """GPU name, power limit and SM clock while `fn` runs."""
    from bench import ClockSampler
    cs = ClockSampler(torch.cuda.current_device())
    cs.start()
    fn()
    torch.cuda.synchronize()
    c = cs.stop()
    return {"gpu": torch.cuda.get_device_name(), "power_limit_w": c["power_limit_w"], "sm_mhz": c["sm_mhz"]}


def _subset(grid, count=4096, seed=0):
    idx = np.sort(np.random.default_rng(seed).choice(grid.nindex, count, replace=False))
    return grid.index_to_state(idx)


def roa():
    """compute_roa of the saturated-LQR closed loops at the notebooks' sizes.  Per step and point:
    pendulum = policy (2 DMUL + 1 DADD + clamp) + 10 Euler sub-steps (one fp64 sin, ~6 DMUL/DADD);
    cart-pole = policy (4 DMUL + 3 DADD) + 10 sub-steps (3 fp64 sin/cos, ~40 DMUL/DADD/DFMA, 2 DDIV).
    CUDA's fp64 sin is a range reduction plus a polynomial on the fp64 FMA pipe (~30 fp64 ops),
    so both plants are fp64-pipe bound; trajectories add 8 d B per point-step of HBM writes."""
    import time
    for plant, num, horizon, tol, no_traj in (("pendulum", [2001, 1501], 500, 1e-2, True),
                                              ("pendulum", [101, 101], 500, 1e-2, False),
                                              ("cartpole", [51] * 4, 2000, 0.1, True)):
        cl, _, ocl, _, R = _rollout_parts(plant)
        d = 2 if plant == "pendulum" else 4
        grid = sl.GridWorld([[-1., 1.]] * d, num)
        n = grid.nindex
        steps = 3 if n > 10 ** 6 else 10
        info = _gpu_info(lambda: sl.compute_roa(grid, cl, horizon, tol, no_traj=no_traj))
        ms = timed(lambda: sl.compute_roa(grid, cl, horizon, tol, no_traj=no_traj), steps=steps, warmup=1)
        # parity and the numpy oracle's rate on a seeded subset of 4096 start states
        sub = _subset(grid)
        t0 = time.perf_counter()
        want = R.compute_roa(sub, ocl, horizon, tol)
        cpu_s = time.perf_counter() - t0
        got = sl.compute_roa(sub, cl, horizon, tol)
        full = sl.compute_roa(grid, cl, horizon, tol)
        idx = np.sort(np.random.default_rng(0).choice(n, 4096, replace=False))
        point_steps = n * max(horizon - 1, 0)
        line = {"bench": "compute_roa", "plant": plant, "grid": "x".join(map(str, num)), "points": n,
                "horizon": horizon, "no_traj": no_traj, "ms": ms,
                "point_steps_per_s": point_steps / (ms * 1e-3),
                "oracle_point_steps_per_s": 4096 * (horizon - 1) / cpu_s,
                "oracle_subset": "4096 seeded start states (numpy, one process)",
                "roa_points": int(full.sum()),
                "parity": {"subset_flags_equal": int((got == want).sum()), "subset": 4096,
                           "full_vs_subset_equal": bool(np.array_equal(full[idx], got))}}
        if not no_traj:
            traj_bytes = n * d * horizon * 8
            line["traj_bytes_per_s"] = traj_bytes / (ms * 1e-3)
            line["traj_frac_of_hbm_datasheet"] = traj_bytes / (ms * 1e-3) / (HBM_GBS * 1e9)
            line["note"] = ("latency-bound: %d sequential chains in %d blocks of 64 threads, 1-2 warps "
                            "per SM of 132; the time includes the host copy of the trajectory array"
                            % (n, -(-n // 64)))
        line.update(info)
        print(json.dumps(line))
        torch.cuda.empty_cache()


def reward_rollout():
    """reward_rollout of the pendulum's saturated-LQR loop on 2001 x 1501, discount 0.95,
    horizon 1000, tol 1e-2: chunks of 32 steps, grid-wide early stop decided on the device."""
    import contextlib
    import io
    import time
    cl, rw, ocl, orw, R = _rollout_parts("pendulum")
    grid = sl.GridWorld([[-1., 1.]] * 2, [2001, 1501])
    n = grid.nindex
    quiet = contextlib.redirect_stdout(io.StringIO())
    with quiet:
        info = _gpu_info(lambda: sl.reward_rollout(grid, cl, rw, 0.95, 1000, 1e-2))
        ms = timed(lambda: sl.reward_rollout(grid, cl, rw, 0.95, 1000, 1e-2), steps=5, warmup=1)
    buf = io.StringIO()
    with contextlib.redirect_stdout(buf):
        sums = sl.reward_rollout(grid, cl, rw, 0.95, 1000, 1e-2)
    msg = buf.getvalue().strip()
    stop = int(msg.split("after ")[1].split(" ")[0]) - 1 if "after" in msg else -1
    idx = np.sort(np.random.default_rng(0).choice(n, 4096, replace=False))
    sub = grid.index_to_state(idx)
    # the oracle on the subset, summed over the same steps 0..T* (tol 0: no early stop of its own)
    t0 = time.perf_counter()
    o_sums, _ = R.reward_rollout(sub, ocl, orw, 0.95, (stop + 1) if stop >= 0 else 1000, 0.0)
    cpu_s = time.perf_counter() - t0
    # T* of the subset alone, product against oracle
    with contextlib.redirect_stdout(io.StringIO()) as b2:
        sl.reward_rollout(sub, cl, rw, 0.95, 1000, 1e-2)
    sub_msg = b2.getvalue()
    sub_stop = int(sub_msg.split("after ")[1].split(" ")[0]) - 1 if "after" in sub_msg else -1
    o_sub_stop = R.reward_rollout(sub, ocl, orw, 0.95, 1000, 1e-2)[1]
    rel = np.abs(sums[idx] - o_sums) / np.maximum(np.abs(o_sums), 1e-300)
    executed = (stop + 1) if stop >= 0 else 1000
    print(json.dumps({"bench": "reward_rollout", "plant": "pendulum", "grid": "2001x1501", "points": n,
                      "discount": 0.95, "horizon": 1000, "tol": 1e-2, "T_star": stop, "ms": ms,
                      "point_steps_per_s": n * executed / (ms * 1e-3),
                      "oracle_point_steps_per_s": 4096 * executed / cpu_s,
                      "oracle_subset": "4096 seeded start states (numpy, one process)",
                      "parity": {"subset_T_star": sub_stop, "oracle_subset_T_star": o_sub_stop,
                                 "sums_max_rel_diff": float(rel.max()),
                                 "sums_finite_equal": bool(np.array_equal(np.isfinite(sums[idx]),
                                                                          np.isfinite(o_sums)))},
                      "note": "point-steps counted up to T*; the chunk holding T* runs twice "
                              "(at most 32 extra steps)", **info}))


def value_opt():
    import time
    from safe_learning_b200 import _device as dev, _native as nat
    lib = nat.load()
    for num, M in ((55, 50), (512, 500)):
        par = W.make_pendulum(num_points=8, M=M)
        grid = sl.GridWorld(par["limits"], num)
        _, dyn = W._build(sl, par, "product")
        policy = sl.Saturation(sl.LinearSystem(-par["K"]), -1., 1.)
        reward = sl.QuadraticFunction(-scipy.linalg.block_diag(np.diag([1., 2.]), 1.2 * np.eye(1)))
        value = sl.Triangulation(grid, np.zeros((grid.nindex, 1)), project=True)
        rl = sl.PolicyIteration(policy, dyn, reward, value, gamma=0.98)
        n = grid.nindex
        cols, w = dev.empty((n, 3), torch.int32), dev.empty((n, 3))
        r, stats = dev.empty((n,)), dev.zeros((nat.VALUE_STATS,), torch.int64)
        cfg = rl.bellman_descriptor()

        def assemble():
            nat.check(lib.slb_value_operator(dev.stream(), cfg, 0, n, cols.data_ptr(), w.data_ptr(),
                                             r.data_ptr(), stats.data_ptr()), "slb_value_operator")

        ms_assembly = timed(assemble, steps=10)
        v = dev.empty((n,))
        need = int(lib.slb_value_solve_workspace(n, 3))
        work = dev.empty((need // 8,)) if need else None

        def solve():                     # the solver launch alone, from a zero table
            v.zero_()
            nat.check(lib.slb_value_solve(dev.stream(), n, 3, cols.data_ptr(), w.data_ptr(),
                                          r.data_ptr(), 0.98, 1e-10, 200000, v.data_ptr(),
                                          dev.ptr(work), stats.data_ptr()), "slb_value_solve")

        assemble()
        ms_solve = timed(solve, steps=5, warmup=1)

        def cold_call():
            value.parameters = np.zeros((n, 1))
            rl.optimize_value_function()

        info = _gpu_info(cold_call)
        ms_call = timed(cold_call, steps=5, warmup=1)
        it = rl.last_solve["iterations"]
        ms_warm = timed(rl.optimize_value_function, steps=5, warmup=1)
        warm_iters = rl.last_solve["iterations"]
        ms_sweep = timed(rl.value_iteration, steps=10)
        # host reference: the same operator, scipy's sparse LU
        assemble()
        c, wt, rw = cols.cpu().numpy(), w.cpu().numpy(), r.cpu().numpy()
        t0 = time.perf_counter()
        import scipy.sparse as sps
        import scipy.sparse.linalg as spla
        T = sps.csr_matrix((wt.ravel(), (np.repeat(np.arange(n), 3), c.ravel())), shape=(n, n))
        exact = spla.spsolve((sps.identity(n) - 0.98 * T).tocsc(), rw)
        ms_spsolve = (time.perf_counter() - t0) * 1e3
        value.parameters = np.zeros((n, 1))
        got = rl.optimize_value_function().ravel()
        print(json.dumps({"bench": "value_opt", "grid": "%dx%d" % (num, num), "M": M,
                          "tier": rl.last_solve["tier"], "iterations": it,
                          "ms_assembly": ms_assembly, "ms_call_cold": ms_call,
                          "ms_solve": ms_solve, "us_per_iteration": ms_solve * 1e3 / it,
                          "ms_call_warm": ms_warm, "warm_iterations": warm_iters,
                          "ms_spsolve_host": ms_spsolve,
                          "max_abs_diff_vs_spsolve": float(np.max(np.abs(got - exact))),
                          "bound": rl.last_solve["bound"],
                          "ms_value_iteration_sweep": ms_sweep,
                          "ms_value_iteration_same_bound": ms_sweep * it,
                          "note": "median of CUDA events; ms_solve is the solver launch alone (plus a "
                                  "table reset), the call includes assembly, solve, the host-side work "
                                  "and the one device-to-host copy; value iteration to the same bound takes "
                                  "the same number of sweeps (the same map), timed per sweep",
                          **info}))


def _torch_mlp(x, params, use_bias=True):
    """The 2-64-64-1 ReLU MLP as plain torch operations (autograd through cuBLAS fp64)."""
    k = params[0:-1:2] if use_bias else params[:-1]
    b = params[1:-1:2] if use_bias else []
    net = x
    for i, w in enumerate(k):
        net = torch.relu(net @ w + b[i] if use_bias else net @ w)
    return net @ params[-1]


def _torch_lnn(x, params, net_obj):
    it, din, net = iter(params), net_obj.input_dim, x
    for dout in net_obj.output_dims:
        w0 = next(it)
        k = w0.T @ w0 + net_obj.eps * torch.eye(din, dtype=torch.float64, device=x.device)
        if dout > din:
            k = torch.cat([k, next(it)], dim=0)
        net = torch.tanh(net @ k.T)
        din = dout
    return torch.sum(net * net, dim=1, keepdim=True)


def train():
    """Gradient kernel against torch autograd, and per-step times of three notebook loops.  FLOPs per
    point of one VJP: 6 sum_l in_l out_l (forward, weight gradient and input gradient, 2 each)."""
    rng = np.random.default_rng(0)
    lnn = sl.LyapunovNetwork(2, [64, 64, 64], ["tanh"] * 3, seed=1)
    mlp = sl.NeuralNetwork([2, 64, 64, 1], ["relu", "relu", None], seed=1)
    info = _gpu_info(lambda: mlp.vjp(torch.zeros((1000, 2), dtype=torch.float64, device="cuda"),
                                     torch.ones((1000, 1), dtype=torch.float64, device="cuda")))
    for name, net, ref in (("lyapunov_2x64x64x64_tanh", lnn, lambda x, p: _torch_lnn(x, p, lnn)),
                           ("mlp_2x64x64x1_relu", mlp, _torch_mlp)):
        if isinstance(net, sl.LyapunovNetwork):
            dims = [2, 64, 64, 64]
        else:
            dims = [2, 64, 64, 1]
        flops_pt = 6 * sum(a * b for a, b in zip(dims[:-1], dims[1:]))
        for n in (100, 1000, 251 ** 2):
            x = torch.tensor(rng.uniform(-1, 1, (n, 2)), device="cuda")
            cot = torch.ones((n, 1), dtype=torch.float64, device="cuda")
            ms_vjp = timed(lambda: net.vjp(x, cot), steps=50, warmup=5)
            params = [p.detach().clone().requires_grad_(True) for p in net.parameters]
            xr = x.clone().requires_grad_(True)

            def torch_grad():
                torch.autograd.grad(ref(xr, params).sum(), [xr] + params)
            ms_torch = timed(torch_grad, steps=50, warmup=5)
            print(json.dumps({"bench": "train_vjp", "network": name, "points": n,
                              "ms_slb_function_vjp": ms_vjp, "ms_torch_autograd": ms_torch,
                              "flops_per_point": flops_pt,
                              "gflops_slb": flops_pt * n / ms_vjp / 1e6, **info}))
    # the three loops of test_gpu_network_grad.py, one SGD step each
    pend = sl.InvertedPendulum(0.15, 0.5, 0.1, 0.01, [(np.deg2rad(30), np.sqrt(9.81 / 0.5)),
                                                      (9.81 * 0.15 * 0.5 * 0.5,)])
    lqr, reward = sl.LinearSystem(np.array([[-0.7, -0.4]])), sl.QuadraticFunction(-0.1 * np.eye(3))
    vf = sl.NeuralNetwork([64, 64, 1], ["relu", "relu", None], seed=2)
    pol = sl.NeuralNetwork([64, 64, 1], ["relu", "relu", None], use_bias=False, seed=3)
    xb = torch.tensor(rng.uniform(-1, 1, (100, 2)), device="cuda")
    vf.torch(xb), pol.torch(xb)
    opt_v, opt_p = torch.optim.SGD(vf.parameters, lr=0.005), torch.optim.SGD(pol.parameters, lr=0.6)
    opt_l = torch.optim.SGD(lnn.parameters, lr=0.1)
    xl = torch.tensor(rng.uniform(-0.07, 0.07, (1000, 2)), device="cuda")

    def value_step():
        z = torch.cat([xb, lqr.torch(xb)], dim=1)
        target = (reward.torch(z) + 0.95 * vf.torch(pend.torch(z))).detach()
        obj = torch.mean(torch.abs(vf.torch(xb) - target)) / 0.3
        opt_v.zero_grad()
        obj.backward()
        opt_v.step()

    def policy_step():
        z = torch.cat([xb, pol.torch(xb)], dim=1)
        obj = -0.25 * torch.mean(reward.torch(z) + 0.95 * vf.torch(pend.torch(z)))
        opt_p.zero_grad()
        obj.backward()
        opt_p.step()

    def pretrain_step():
        obj = torch.mean(torch.abs(lnn.torch(xl) - 0.1 * torch.sum(xl * xl, dim=1, keepdim=True)))
        opt_l.zero_grad()
        obj.backward()
        opt_l.step()

    for name, step in (("value_net_batch100", value_step), ("policy_net_batch100", policy_step),
                       ("lyapunov_pretrain_batch1000", pretrain_step)):
        print(json.dumps({"bench": "train_loop", "loop": name, "ms_per_step": timed(step, steps=50),
                          "note": "median of CUDA events around one SGD step (forward, backward, "
                                  "update; the LyapunovNetwork forms its kernels on the host each step)",
                          **info}))


def tri_train():
    """Triangulation vertex gradient (slb_function_vjp, deterministic) against torch.index_add_ (atomic
    scatter, not deterministic) and torch.sparse.mm of parameter_derivative^T, and one SGD step of the
    two Triangulation training loops of test_gpu_triangulation_grad.py.  Bytes per point of the VJP:
    rows (d + 1) x (8 B key + 8 B weight written), sort (~4 passes of 16 B per key), sum (key, weight
    and cotangent read once more)."""
    rng = np.random.default_rng(0)
    cases = (("55x55", [[-1, 1], [-1, 1]], [55, 55]), ("512x512", [[-1, 1], [-1, 1]], [512, 512]),
             ("21^4", [[-1, 1]] * 4, [21] * 4))
    info = None
    for name, limits, num in cases:
        grid = sl.GridWorld(limits, num)
        tri = sl.Triangulation(grid, rng.normal(size=(grid.nindex, 1)), project=True)
        d = grid.ndim
        for n in (10 ** 3, 10 ** 5, 10 ** 6):
            x = torch.tensor(rng.uniform(-1.1, 1.1, (n, d)), device="cuda")
            g = torch.tensor(rng.normal(size=(n, 1)), device="cuda")
            if info is None:
                info = _gpu_info(lambda: tri._param_vjp(x, g))
            ms_vjp = timed(lambda: tri._param_vjp(x, g), steps=20, warmup=3)
            pd = tri.tri.parameter_derivative(x.cpu().numpy())
            cols = torch.tensor(pd.col, device="cuda")
            w = torch.tensor(pd.data, device="cuda")
            rows = torch.tensor(pd.row, device="cuda")
            out = torch.zeros((grid.nindex, 1), dtype=torch.float64, device="cuda")

            def index_add():
                out.zero_()
                out.index_add_(0, cols, (w * g[rows, 0])[:, None])
            ms_index_add = timed(index_add, steps=20, warmup=3)
            spt = torch.sparse_coo_tensor(torch.stack([cols, rows]), w, (grid.nindex, n)).coalesce()
            ms_sparse = timed(lambda: torch.sparse.mm(spt, g), steps=20, warmup=3)
            ref = tri._param_vjp(x, g)[0]
            index_add()
            print(json.dumps({"bench": "tri_vjp", "grid": name, "vertices": grid.nindex, "points": n,
                              "ms_slb_function_vjp": ms_vjp, "ms_torch_index_add": ms_index_add,
                              "ms_torch_sparse_mm_coalesced": ms_sparse,
                              "max_abs_diff_index_add": float((out - ref).abs().max()),
                              "note": "median of CUDA events; index_add_ and sparse.mm start from rows "
                                      "already built (parameter_derivative), the VJP builds its own",
                              **info}))
    # one SGD step of tests/test_rl.py:29-77 and of the mountain-car loop
    a, b = np.array([[1.2]]), np.array([[0.9]])
    disc = sl.GridWorld([[-1, 1]], 19)
    pdisc = sl.GridWorld([-1, 1], 5)
    policy = sl.Triangulation(pdisc, -0.3 * pdisc.all_points)
    rl = sl.PolicyIteration(policy, sl.LinearSystem((a, b)),
                            sl.QuadraticFunction(-scipy.linalg.block_diag([[1.]], [[0.1]])),
                            sl.Triangulation(disc, 0. * disc.all_points, project=True))
    opt = torch.optim.SGD([policy.vertex_values], lr=0.01)
    st = torch.tensor(rl.state_space, device="cuda")

    def rl_step():
        loss = -torch.sum(rl.future_values(st))
        opt.zero_grad()
        loss.backward()
        opt.step()

    mc = sl.GridWorld([[-1.2, 0.7], [-.07, .07]], [20, 20])
    ptri = sl.Triangulation(mc, np.zeros(mc.nindex), project=True)

    def dyn(s, u):
        return torch.stack((s[:, 0] + s[:, 1], s[:, 1] + 0.001 * u[:, 0] - 0.0025 * torch.cos(3 * s[:, 0])), 1)

    def rew(s, u):
        return torch.where(s[:, :1] > 0.6, 0.01 * torch.ones_like(s[:, :1]), torch.zeros_like(s[:, :1]))
    mrl = sl.PolicyIteration(sl.Saturation(ptri, -1., 1.), dyn, rew,
                             sl.Triangulation(mc, np.linspace(0, 1, mc.nindex), project=True), gamma=0.99)
    mopt = torch.optim.SGD([ptri.vertex_values], lr=1.)
    ms = torch.tensor(mrl.state_space, device="cuda")

    def mc_step():
        loss = -100. * torch.mean(mrl.future_values(ms))
        mopt.zero_grad()
        loss.backward()
        mopt.step()

    for name, step in (("test_rl_integration_19pts", rl_step), ("mountain_car_20x20", mc_step)):
        print(json.dumps({"bench": "tri_train_loop", "loop": name, "ms_per_step": timed(step, steps=50),
                          "note": "median of CUDA events around one SGD step (forward, backward, update)",
                          **info}))


def nn_lv():
    """L_V = |dV/dx|_1 of a LyapunovNetwork fused as Norm1Function(V.gradient_function()):
    (1) lyapunov_function_learning.ipynb's 251^2 update_safe_set (pendulum plant, saturated LQR, V =
        LyapunovNetwork(2, [64, 64, 64], tanh), tau = sum(unit) / 2), fused against the composed path
        through V.gradient;
    (2) a 256^2 pendulum GP sweep (M = 500) with the same V: filtered update_safe_set and the share of points
        each stage decides, with L_V = |dV/dx|_1 against a constant L_V;
    (3) the C4 shape (make_cartpole 16^4, M = 200): L_V = |dV/dx|_1 against L_v = 1.0;
    (4) slb_eval_function with the gradient flag against slb_function_vjp (cotangent 1) at 251^2 points."""
    from safe_learning_b200 import functions as F
    par = W.make_pendulum(num_points=251, M=8)
    pl = par["plant"]
    plant = sl.InvertedPendulum(normalization=[pl["state_norm"], pl["action_norm"]], **pl["true"])
    policy = sl.Saturation(sl.LinearSystem(-par["K"]), -1., 1.)
    V = sl.LyapunovNetwork(2, [64, 64, 64], ["tanh"] * 3, eps=1e-8, seed=21)
    grid = sl.GridWorld(par["limits"], par["num_points"])
    fused = sl.Lyapunov(grid, V, plant, par["L_dyn"], sl.Norm1Function(V.gradient_function()), par["tau"],
                        policy, par["initial"])
    composed = sl.Lyapunov(grid, V, plant, par["L_dyn"], lambda x: np.abs(V.gradient(x)).sum(1, keepdims=True),
                           par["tau"], policy, par["initial"])
    info = _gpu_info(fused.update_safe_set)
    ms_f = timed(lambda: (fused.update_safe_set(), fused.safe_set), steps=20)
    ms_c = timed(lambda: (composed.update_safe_set(), composed.safe_set), steps=5, warmup=1)
    same = bool(np.array_equal(fused.safe_set, composed.safe_set)
                and fused.feed_dict[fused.c_max] == composed.feed_dict[composed.c_max])
    print(json.dumps({"bench": "nn_lv_notebook_update_safe_set", "grid": "251x251", "ms_fused": ms_f,
                      "ms_composed": ms_c, "speedup": ms_c / ms_f, "same_safe_set_and_c_max": same,
                      "note": "median of CUDA events around update_safe_set + the safe_set read-back", **info}))

    gpar = W.make_pendulum(num_points=256, M=500)
    base = W.build_product(gpar)
    for name, lv in (("norm1_grad", sl.Norm1Function(V.gradient_function())), ("constant", 1.0)):
        lyap = sl.Lyapunov(base.discretization, V, base.dynamics, gpar["L_dyn"], lv, gpar["tau"], base.policy,
                           initial_set=gpar["initial"])
        lyap.filter = True
        ms = timed(lambda: (lyap.update_safe_set(), lyap.safe_set), steps=10)
        lyap.reset_filter_stats()
        lyap.compute_negative()
        st = lyap.filter_stats
        pts = max(st["points"], 1)
        print(json.dumps({"bench": "nn_lv_gp_filtered_sweep", "grid": "256x256", "M": 500, "L_V": name,
                          "ms_update_safe_set": ms,
                          "stage1": "fp%d" % _stage1(lyap),
                          "frac_prior": st["prior"] / pts, "frac_head": st["head"] / pts,
                          "frac_refined": st["refined"] / pts, **info}))

    cpar = W.make_cartpole(num_points=16, M=200)
    cbase = W.build_product(cpar)
    CV = cbase.lyapunov_function
    for name, lv in (("norm1_grad", sl.Norm1Function(CV.gradient_function())), ("L_v=1.0", 1.0)):
        lyap = sl.Lyapunov(cbase.discretization, CV, cbase.dynamics, cpar["L_dyn"], lv, cpar["tau"],
                           cbase.policy, initial_set=cpar["initial"])
        ms = timed(lambda: (lyap.update_safe_set(), lyap.safe_set), steps=10)
        print(json.dumps({"bench": "nn_lv_c4_update_safe_set", "grid": "16^4", "M": 200, "L_V": name,
                          "ms_update_safe_set": ms, **info}))

    x = torch.tensor(grid.all_points, device="cuda")
    g = V.gradient_function()
    ones = torch.ones((x.shape[0], 1), dtype=torch.float64, device="cuda")
    ms_eval = timed(lambda: g.evaluate_device(x), steps=50)
    ms_vjp = timed(lambda: F._function_vjp(V, x, ones), steps=50)
    print(json.dumps({"bench": "nn_lv_gradient_eval", "points": int(x.shape[0]),
                      "ms_eval_function_gradient_flag": ms_eval, "ms_function_vjp": ms_vjp,
                      "bit_identical": bool(torch.equal(g.evaluate_device(x), F._function_vjp(V, x, ones)[0])),
                      **info}))


def gp_vjp():
    """(1) examples/inverted_pendulum.ipynb cell 17: one SGD step on -mean(future_values(states, lyapunov=...))
    for a NeuralNetwork([32, 32, 1]) policy, 1000 states, the notebook-kernel FunctionStack at M = 0, 50, 200, a
    55x55 Triangulation value function and L_V = MaxAbsFunction(V.gradient_function())
    (bench_workloads.notebook_policy_case), with GaussianProcess.torch's node against torch_predict;
    (2) slb_gp_vjp alone on C2's stack (make_pendulum, plain RBF, M = 500, two factors): both cotangents and
    mean only, against slb_gp_predict and torch autograd through torch_predict.  FLOPs: the algorithmic
    count of the forward-mode err term, (1 + d_in) M (M + 1) per point and factor (one FMA per L^-1 entry
    and right-hand side), over the DMMA peak of DESIGN.md section 6."""
    info = None
    for M in (0, 50, 200):
        ms = {}
        for label, torch_dynamics in (("node", False), ("torch_predict", True)):
            case = W.notebook_policy_case(sl, M, torch_dynamics=torch_dynamics)
            net = case["policy"]
            net._build(2)
            opt = torch.optim.SGD(net.parameters, lr=1e-3)
            if info is None:
                info = _gpu_info(lambda: case["step"](opt))
            ms[label] = timed(lambda: case["step"](opt), steps=20, warmup=3)
        print(json.dumps({"bench": "gp_vjp_cell17_policy_step", "batch": 1000, "M": M,
                          "ms_node": ms["node"], "ms_torch_predict": ms["torch_predict"],
                          "speedup": ms["torch_predict"] / ms["node"],
                          "note": "median of CUDA events around zero_grad + forward + backward + SGD step", **info}))

    par = W.make_pendulum(num_points=64, M=500)
    stack = W.build_product(par).dynamics
    din, M, nf = 3, 500, stack.gp_stack().num_factors
    for n in (1000, 10000, 65536):
        rng = np.random.default_rng(n)
        x = torch.tensor(rng.uniform(-1, 1, (n, din)), device="cuda")
        g = torch.tensor(rng.normal(size=(n, 2)), device="cuda")
        ms_both = timed(lambda: stack.vjp_device(x, g, g), steps=20)
        ms_mean = timed(lambda: stack.vjp_device(x, g, None), steps=20)
        ms_fwd = timed(lambda: stack.predict_device(x), steps=20)

        def autograd():
            xg = x.clone().requires_grad_(True)
            mean, err = stack._torch_expression(xg)
            torch.autograd.grad((mean * g).sum() + (err * g).sum(), xg)

        ms_torch = timed(autograd, steps=10)
        flops = float(n) * nf * (1 + din) * M * (M + 1)
        print(json.dumps({"bench": "gp_vjp_c2", "points": n, "M": M, "factors": nf, "ms_vjp": ms_both,
                          "ms_vjp_mean_only": ms_mean, "ms_forward": ms_fwd, "ms_torch_autograd": ms_torch,
                          "gflop_err_term": flops / 1e9, "tflops": flops / ms_both / 1e9,
                          "share_of_dmma_peak": flops / ms_both / 1e9 / PEAK_TF, **info}))


def _gp_fit_kernel(kind, din, K):
    """(product kernel, hyper-parameter tensors, torch expression of K(X) in them) of a gp_fit workload."""
    if kind == "notebook":
        kern = K.Linear(din, variance=np.linspace(0.2, 0.5, din), ARD=True) + \
            K.Matern32(1, variance=0.8, lengthscales=0.7, active_dims=[0]) * K.Linear(1, variance=0.6)

        def expr(X, t):
            x0 = X[:, :1] / t["kern.kern_list[1].kern_list[0].lengthscales"]
            sq = (x0 * x0).sum(1)
            r = torch.sqrt(-2 * x0 @ x0.T + sq[:, None] + sq[None, :] + 1e-12)
            m32 = t["kern.kern_list[1].kern_list[0].variance"] * (1 + np.sqrt(3) * r) * torch.exp(-np.sqrt(3) * r)
            return (X * t["kern.kern_list[0].variance"]) @ X.T + \
                m32 * ((X[:, :1] * t["kern.kern_list[1].kern_list[1].variance"]) @ X[:, :1].T)
    else:
        kern = K.RBF(din, variance=1.3, lengthscales=np.linspace(0.7, 1.2, din), ARD=True)

        def expr(X, t):
            xs = X / t["kern.lengthscales"]
            sq = (xs * xs).sum(1)
            return t["kern.variance"] * torch.exp(-0.5 * (-2 * xs @ xs.T + sq[:, None] + sq[None, :]))
    return kern, expr


def gp_fit():
    """GPRCached hyper-parameter fit (d_in = 3, noise 0.01): the notebook kernel Linear(3, ARD) + Matern32(1,
    active_dims=[0]) * Linear(1) and an ARD RBF at M = 500, 2000, 5000.  Reported: the fused gradient kernel
    alone (slb_gp_lml_grad on a given K^-1 and alpha; it reads the lower triangle of K^-1 once, M (M + 1) / 2
    doubles); one log_likelihood_and_gradient (K, Cholesky, K^-1, alpha, kernel, host copy); the same LML and
    gradient by torch autograd through the tensor expression of K; optimize(maxiter=50) wall time."""
    import time
    from safe_learning_b200 import _native as nat
    lib = nat.load()
    info = None
    din = 3
    for kind in ("notebook", "rbf_ard"):
        for M in (500, 2000, 5000):
            rng = np.random.default_rng(M)
            X = rng.uniform(-1, 1, (M, din))
            Y = np.sin(2 * X).sum(axis=1, keepdims=True) + 0.1 * rng.standard_normal((M, 1))
            kern, expr = _gp_fit_kernel(kind, din, sl.kernels)
            gp = sl.GPR(X, Y, kern, noise_variance=0.01)
            Xd = torch.tensor(X, device="cuda")
            Yd = torch.tensor(Y, device="cuda")
            Kn = kern.K_device(Xd) + 0.01 * torch.eye(M, dtype=torch.float64, device="cuda")
            L = torch.linalg.cholesky(Kn)
            kinv = torch.cholesky_inverse(L).contiguous()
            alpha = torch.cholesky_solve(Yd, L)[:, 0].contiguous()
            ks = nat.SlbKernel()
            kern.fill(ks, din)
            work = torch.empty(int(lib.slb_gp_lml_grad_workspace(M)) // 8, dtype=torch.float64, device="cuda")
            grad = torch.empty(nat.SLB_GP_HYPER_SLOTS, dtype=torch.float64, device="cuda")
            stream = torch.cuda.current_stream().cuda_stream

            def fused():
                nat.check(lib.slb_gp_lml_grad(stream, Xd.data_ptr(), M, din, ks, kinv.data_ptr(), alpha.data_ptr(),
                                              grad.data_ptr(), work.data_ptr()), "slb_gp_lml_grad")

            if info is None:
                info = _gpu_info(lambda: [fused() for _ in range(200)])
            ms_kernel = timed(fused, steps=50, warmup=5)
            ms_value_grad = timed(gp.log_likelihood_and_gradient, steps=10)

            def autograd():
                t = {p: torch.tensor(np.asarray(v, dtype=np.float64), device="cuda", requires_grad=True)
                     for p, v in gp.hyperparameters().items()}
                Lt = torch.linalg.cholesky(expr(Xd, t) + t["likelihood.variance"]
                                           * torch.eye(M, dtype=torch.float64, device="cuda"))
                a = torch.linalg.solve_triangular(Lt, Yd, upper=False)
                lml = -0.5 * M * np.log(2 * np.pi) - torch.log(torch.diagonal(Lt)).sum() - 0.5 * (a * a).sum()
                torch.autograd.grad(lml, list(t.values()))

            ms_autograd = timed(autograd, steps=10)
            start = gp.hyperparameters()
            fits = []
            for _ in range(3):
                gp._set_hyperparameters(start)
                torch.cuda.synchronize()
                t0 = time.perf_counter()
                res = gp.optimize(maxiter=50, fixed=("likelihood.variance",))
                torch.cuda.synchronize()
                fits.append(time.perf_counter() - t0)
            nbytes = M * (M + 1) / 2 * 8
            print(json.dumps({"bench": "gp_fit", "kernel": kind, "d_in": din, "M": M, "ms_fused_kernel": ms_kernel,
                              "kinv_gbs": nbytes / ms_kernel / 1e6, "ms_value_and_gradient": ms_value_grad,
                              "ms_torch_autograd": ms_autograd, "autograd_over_value_and_gradient":
                              ms_autograd / ms_value_grad, "s_optimize_maxiter50": float(np.median(fits)),
                              "optimize_nfev": int(res.nfev), "optimize_nit": int(res.nit),
                              "note": "median of CUDA events (kernel: 50, calls: 10); optimize: median of 3 "
                                      "wall-clock fits from the same start", **info}))


def _stage1(lyap):
    from safe_learning_b200 import _native as nat
    return nat.load().slb_filter_stage1(lyap.sweep_descriptor())


if __name__ == "__main__":
    which = sys.argv[1:] or ["bellman", "det", "det_linear", "c5", "shared", "c4", "nb", "argmax"]
    for name in which:
        globals()[name]()
