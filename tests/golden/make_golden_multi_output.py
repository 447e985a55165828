"""Generate ``tests/golden/multi_output_gp.npz`` by running the UNMODIFIED reference's ``GPRCached`` and
``GaussianProcess`` (``functions.py:357-546``) with a ``Y`` of several columns, on the numpy-backed TF1 /
gpflow shims.

    SAFE_LEARNING_REFERENCE=<checkout> python tests/golden/make_golden_multi_output.py

One kernel and noise for all columns; ``build_predict`` solves every column and tiles the one variance
(``functions.py:438-456``).  Cases, for Y of 2 and 3 columns: an ARD RBF and the notebooks' ``Linear +
Matern32 * Linear`` expression, a linear prior mean with one row per column, ``scale != 1``; predictions at
seeded points before and after ``add_data_point`` of two rows; and the empty (0, 2) data set before and
after its first points.  Then ``Lyapunov.update_safe_set`` on a small pendulum grid with ONE two-column
GP as the dynamics (the pendulum of ``bench_workloads.make_pendulum`` with one kernel for both columns):
V on the grid, the safe set and ``c_max``.
"""
import json
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, HERE)
sys.path.insert(0, ROOT)

from make_golden import sl  # noqa: E402  (loads the reference on the shims)
from reference_loader import REFERENCE  # noqa: E402
import gpflow  # noqa: E402  (shim)
import tensorflow as tf  # noqa: E402  (shim)

import bench_workloads as W  # noqa: E402

assert os.path.abspath(sl.__file__).startswith(os.path.abspath(REFERENCE))

KERNELS = {
    "rbf": json.dumps(["rbf", 3, {"variance": 0.6, "lengthscales": [0.9, 1.05, 1.2], "ARD": True}]),
    "expr": json.dumps(["add", ["linear", 3, {"variance": [0.2, 0.35, 0.5], "ARD": True}],
                        ["prod", ["matern32", 1, {"lengthscales": 1.0, "active_dims": [0]}],
                         ["linear", 1, {"variance": 0.3}]]]),
}
NOISE = 1e-2
SCALE = 1.7
BETA = 2.0


def data(M, k, seed):
    rng = np.random.default_rng(seed)
    X = rng.uniform(-1, 1, (M, 3))
    mix = rng.uniform(-0.4, 0.4, (3, k))
    mix[:k, :k] += 0.7 * np.eye(k)
    Y = np.sin(X @ mix) + 0.3 * X @ mix + 1e-2 * rng.standard_normal((M, k))
    rows = rng.uniform(-0.5, 0.5, (k, 3))
    rows += 0.6 * np.eye(k, 3)
    return X, Y, rows


def ref_gp(X, Y, kernel, rows, scale):
    kern = W.build_kernel(gpflow.kernels, kernel)
    gp = sl.GPRCached(X, Y, kern, sl.LinearSystem((rows,), name="prior"), scale)
    gp.likelihood.variance = NOISE
    gp.update_cache()
    return sl.GaussianProcess(gp, beta=BETA)


def predict(fun, points):
    ph = tf.placeholder(tf.float64, [None, 3])
    mean, err = fun(ph)
    fd = dict(fun.feed_dict)
    fd[ph] = points
    return mean.eval(fd), err.eval(fd)


def main():
    res = {"noise": np.array(NOISE), "scale": np.array(SCALE), "beta": np.array(BETA)}
    points = np.random.default_rng(5).uniform(-1.2, 1.2, (150, 3))
    res["points"] = points
    with tf.Session():
        for kind, spec in KERNELS.items():
            res["kernel_" + kind] = np.array(spec)
            for k, M in ((2, 40), (3, 33), (2, 0)):
                tag = "%s_k%d_M%d" % (kind, k, M)
                X, Y, rows = data(M, k, seed=10 * k + M)
                fun = ref_gp(X, Y, spec, rows, SCALE)
                res[tag + "_X"], res[tag + "_Y"], res[tag + "_rows"] = X, Y, rows
                res[tag + "_mean"], res[tag + "_err"] = predict(fun, points)
                rng = np.random.default_rng(M + k)
                xnew, ynew = rng.uniform(-1, 1, (2, 3)), rng.standard_normal((2, k))
                fun.add_data_point(xnew, ynew)
                res[tag + "_xnew"], res[tag + "_ynew"] = xnew, ynew
                res[tag + "_mean_after"], res[tag + "_err_after"] = predict(fun, points)
                print(tag, res[tag + "_mean"].shape, float(np.abs(res[tag + "_err"]).max()))

        # the pendulum with ONE two-column GP as dynamics
        par = W.make_pendulum(num_points=[26, 21], M=90, tau_scale=1 / 150., shared_hypers=True, seed=4)
        kern = gpflow.kernels.RBF(3, variance=par["variances"][0], lengthscales=np.asarray(par["lengthscales"][0]),
                                  ARD=True)
        gp = sl.GPRCached(par["X"], par["Y"], kern, sl.LinearSystem((par["prior_rows"],), name="prior"),
                          par["scale"])
        gp.likelihood.variance = par["noise_variance"]
        gp.update_cache()
        dynamics = sl.GaussianProcess(gp, beta=par["beta"])
        grid = sl.GridWorld(par["limits"], par["num_points"])
        policy = sl.Saturation(sl.LinearSystem((-par["K"],), name="policy"), -1., 1.)
        grad = sl.LinearSystem((2 * par["P"],), name="grad_v")
        lyap = sl.Lyapunov(grid, sl.QuadraticFunction(par["P"]), dynamics, par["L_dyn"],
                           lambda x: tf.abs(grad(x)), par["tau"], policy, par["initial"].copy())
        res["lyap_values"] = lyap.values.copy()
        lyap.update_safe_set()
        for key in ("X", "Y", "variances", "lengthscales", "noise_variance", "beta", "scale", "prior_rows",
                    "K", "P", "L_dyn", "tau", "limits", "num_points", "initial"):
            res["lyap_par_" + key] = np.asarray(par[key])
        res["lyap_safe_set"] = lyap.safe_set.copy()
        res["lyap_c_max"] = np.array(lyap.feed_dict[lyap.c_max])
        print("pendulum, one k = 2 GP: safe", res["lyap_safe_set"].sum(), "/", res["lyap_safe_set"].size,
              "c_max", res["lyap_c_max"])
    np.savez_compressed(os.path.join(HERE, "multi_output_gp.npz"), **res)


if __name__ == "__main__":
    main()
