"""Time multi-output GPs: one ``GPRCached`` with a Y of k columns against the models users would otherwise
write.

    python tools/multi_output_gp_timing.py [--reps 5] [--out multi_output_timing.json]

1. ``update_safe_set`` on C2's pendulum (``bench_workloads.make_pendulum``, 256^2 grid, M = 500, one kernel
   for both columns): ONE k = 2 GP, a ``FunctionStack`` of two one-column GPs that share their factor (the
   same work: the same kernels run on the same tables), and a stack of two GPs with separate factors (the
   second GP's lengthscales differ by one part in 10^12, so the factors are distinct).  Each safe set is
   checked equal to the k = 2 GP's.
2. ``log_likelihood_and_gradient`` at M in {500, 1000} for k = 1..6 target columns (the notebooks' kernel
   expression): one call on the k-column model (one fused pass, ``slb_gp_lml_grad_cols``) against k calls on
   one-column models.  Also the fused gradient kernel alone (``slb_gp_lml_grad_cols`` on a given K^-1 and
   alpha) against k one-column kernel calls.

Everything is warmed up once and timed with CUDA events (median, min, max): `reps` repetitions of each
likelihood workload, and 5 alternating rounds of 10 x `reps` sweeps of each ``update_safe_set`` model.  The
card's name, power limit and maximum SM clock are read in the same run.
"""
import argparse
import json
import os
import subprocess
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import bench_workloads as W  # noqa: E402
import safe_learning_b200 as sl  # noqa: E402
from safe_learning_b200 import _device as dev  # noqa: E402
from safe_learning_b200 import _native as nat  # noqa: E402


def card():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                             capture_output=True, text=True, check=True).stdout.strip().splitlines()[0]
    except (OSError, subprocess.CalledProcessError, IndexError):
        out = torch.cuda.get_device_name(0) + ", power limit not read"
    return out


def timed(fn, reps):
    """CUDA-event times (ms) of `reps` calls after one warm-up."""
    fn()
    times = []
    for _ in range(reps):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        torch.cuda.synchronize()
        a.record()
        fn()
        b.record()
        torch.cuda.synchronize()
        times.append(a.elapsed_time(b))
    return times


def row(name, times, **extra):
    out = dict(workload=name, median_ms=float(np.median(times)), min_ms=float(min(times)), max_ms=float(max(times)))
    out.update(extra)
    print(json.dumps(out))
    return out


ROUNDS = 5


def safe_set_rows(reps):
    par = W.make_pendulum(num_points=256, M=500, shared_hypers=True)
    ls = np.asarray(par["lengthscales"][0], dtype=np.float64)

    def gp(cols, lengthscales):
        Y = par["Y"][:, cols]
        mean = sl.LinearSystem(par["prior_rows"][cols])
        kern = sl.RBF(3, variance=par["variances"][0], lengthscales=lengthscales)
        return sl.GaussianProcess(sl.GPRCached(par["X"], Y, kern, mean_function=mean,
                                               noise_variance=par["noise_variance"], scale=par["scale"]),
                                  beta=par["beta"])
    models = [("one k = 2 GP", gp([0, 1], ls)),
              ("stack of 2 GPs, shared factor", sl.FunctionStack([gp([0], ls), gp([1], ls)])),
              ("stack of 2 GPs, separate factors", sl.FunctionStack([gp([0], ls), gp([1], ls * (1 + 1e-12))]))]
    lyaps, first = [], None
    for name, dyn in models:
        lyap = sl.Lyapunov(sl.GridWorld(par["limits"], par["num_points"]), sl.QuadraticFunction(par["P"]), dyn,
                           par["L_dyn"], sl.AbsFunction(sl.LinearSystem((2 * par["P"],))), par["tau"],
                           sl.Saturation(sl.LinearSystem(-par["K"]), -1., 1.), initial_set=par["initial"])
        lyap.update_safe_set()
        if first is None:
            first = lyap.safe_set.copy()
        lyaps.append((name, dyn, lyap, bool(np.array_equal(lyap.safe_set, first))))
    # the three models alternate, ROUNDS rounds of 10 reps each, so that drift hits them alike
    times = {name: [] for name, _, _, _ in lyaps}
    for _ in range(ROUNDS):
        for name, _, lyap, _ in lyaps:
            times[name] += timed(lyap.update_safe_set, 10 * reps)
    return [row("update_safe_set 256^2 M=500: " + name, times[name], factors=int(dyn.gp_stack().num_factors),
                safe_set_equal=same) for name, dyn, _, same in lyaps]


def lml_rows(reps):
    rows = []
    lib = nat.load()
    for M in (500, 1000):
        rng = np.random.default_rng(M)
        X = rng.uniform(-1, 1, (M, 3))
        Y = np.sin(X @ rng.uniform(-1, 1, (3, 6))) + 0.05 * rng.standard_normal((M, 6))
        spec = W.notebook_pendulum_kernels([[0.2, 0.35, 0.5]])[0]
        for k in range(1, 7):
            multi = sl.GPRCached(X, Y[:, :k], W.build_kernel(sl, spec), noise_variance=0.05)
            singles = [sl.GPRCached(X, Y[:, [c]], W.build_kernel(sl, spec), noise_variance=0.05) for c in range(k)]
            t_multi = timed(multi.log_likelihood_and_gradient, reps)
            t_single = timed(lambda: [s.log_likelihood_and_gradient() for s in singles], reps)
            rows.append(row("log_likelihood_and_gradient M=%d k=%d: one k-column call" % (M, k), t_multi))
            rows.append(row("log_likelihood_and_gradient M=%d k=%d: k one-column calls" % (M, k), t_single))
            # the fused gradient kernel alone
            kstruct = nat.SlbKernel()
            multi.kern.fill(kstruct, 3)
            Xd = dev.to_device(X)
            K = multi.kern.K_device(Xd) + 0.05 * torch.eye(M, dtype=torch.float64, device=Xd.device)
            kinv = torch.cholesky_inverse(torch.linalg.cholesky(K)).contiguous()
            alpha = dev.to_device(rng.standard_normal((M, k)))
            cols = [alpha[:, c].contiguous() for c in range(k)]
            work = dev.empty((int(lib.slb_gp_lml_grad_workspace(M)) // 8,))
            grad = dev.empty((nat.SLB_GP_HYPER_SLOTS,))
            stream = dev.stream()

            def fused():
                nat.check(lib.slb_gp_lml_grad_cols(stream, Xd.data_ptr(), M, 3, kstruct, kinv.data_ptr(),
                                                   alpha.data_ptr(), k, grad.data_ptr(), work.data_ptr()),
                          "slb_gp_lml_grad_cols")

            def separate():
                for a in cols:
                    nat.check(lib.slb_gp_lml_grad_cols(stream, Xd.data_ptr(), M, 3, kstruct, kinv.data_ptr(),
                                                       a.data_ptr(), 1, grad.data_ptr(), work.data_ptr()),
                              "slb_gp_lml_grad_cols")
            rows.append(row("slb_gp_lml_grad_cols kernel M=%d k=%d: fused" % (M, k), timed(fused, reps)))
            rows.append(row("slb_gp_lml_grad_cols kernel M=%d k=%d: k calls of k=1" % (M, k), timed(separate, reps)))
    return rows


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    print("card:", card())
    rows = safe_set_rows(args.reps) + lml_rows(args.reps)
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as f:
            json.dump(dict(card=card(), rows=rows), f, indent=1)


if __name__ == "__main__":
    main()
