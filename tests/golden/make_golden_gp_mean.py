"""Generate ``tests/golden/gp_mean.npz`` by running the UNMODIFIED reference's rollout helpers
(``examples/utilities.py`` ``compute_roa`` / ``reward_rollout``) on the learned model
``GaussianProcess(...).to_mean_function()`` (``functions.py:209-230``), on the numpy-backed TF1 / gpflow
shims.

    SAFE_LEARNING_REFERENCE=<checkout> python tests/golden/make_golden_gp_mean.py

The model is C2's pendulum (``bench_workloads.make_pendulum``) fitted on a few dozen samples: two RBF GPs on
``[x, u]`` with the linear prior mean of the wrong plant, one with ``scale = 1`` and one with
``scale = 2`` (the prior mean enters scaled).  The closed loop follows the notebooks
(``inverted_pendulum.ipynb`` cell 11): one placeholder, the saturated LQR policy feeding the mean of each
GP of a ``FunctionStack``.  Cases: ``compute_roa`` on a 25 x 21 grid, on a seeded state array and on its
states near the origin (flags, end states and the trajectories of a seeded subsample), and
``reward_rollout`` with its stop step, for two horizons each (from the grid and the whole array the sums
diverge and never stop; near the origin they stop).  One-step means at seeded points are stored too.
"""
import os
import sys

import numpy as np
from scipy.linalg import block_diag

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, HERE)
sys.path.insert(0, ROOT)

from make_golden import ref_gp_stack  # noqa: E402  (loads the reference on the shims)
from reference_loader import REFERENCE  # noqa: E402
import make_golden_rollout  # noqa: E402

import bench_workloads as W  # noqa: E402

sl = make_golden_rollout.sl
ex = make_golden_rollout.ex
import tensorflow as tf  # noqa: E402  (shim)

assert os.path.abspath(ex.__file__).startswith(os.path.abspath(REFERENCE))

M = 36


def model(scale):
    """The pendulum's two GPs, fitted on M seeded samples."""
    par = W.make_pendulum(num_points=8, M=M, seed=21, scale=scale, noise_std=1e-3)
    return par, ref_gp_stack(par)


def closed_loops(stack, policy, reward_function):
    """states -> mean f(states, policy(states)) and the reward, through to_mean_function()."""
    states = tf.placeholder(tf.float64, [None, 2])
    actions = policy(states)
    mean_fns = [gp.to_mean_function() for gp in stack.functions]
    future = tf.concat([fn(states, actions) for fn in mean_fns], axis=1)
    rewards = reward_function(states, actions)
    feed = dict(stack.feed_dict)

    def run(tensor, x):
        fd = dict(feed)
        fd[states] = x
        return tensor.eval(fd)
    return (lambda x: run(future, x)), (lambda x: run(rewards, x))


def main():
    res = {"M": np.array(M)}
    reward = sl.QuadraticFunction(block_diag(-np.diag([1., 2.]), -1.2 * np.eye(1)), name="reward_function")
    res["reward"] = block_diag(-np.diag([1., 2.]), -1.2 * np.eye(1))
    with tf.Session():
        for scale in (1.0, 2.0):
            tag = "s%d" % int(scale)
            par, stack = model(scale)
            policy = sl.Saturation(sl.LinearSystem((-par["K"],), name="policy"), -1., 1.)
            cl, rw = closed_loops(stack, policy, reward)
            res.update({tag + "_" + k: np.asarray(par[k]) for k in
                        ("X", "Y", "variances", "lengthscales", "noise_variance", "beta", "scale",
                         "prior_rows", "K", "limits")})
            # one-step means of the learned model at seeded points (states and actions)
            pts = np.random.default_rng(3).uniform(-1.2, 1.2, (200, 3))
            ph = tf.placeholder(tf.float64, [None, 3])
            mean = tf.concat([gp.to_mean_function()(ph) for gp in stack.functions], axis=1)
            fd = dict(stack.feed_dict)
            fd[ph] = pts
            res[tag + "_points"] = pts
            res[tag + "_mean"] = mean.eval(fd)
            grid = sl.GridWorld(par["limits"], [25, 21])
            states = np.random.default_rng(9).uniform(-1, 1, (300, 2))
            res[tag + "_grid_num_points"] = grid.num_points
            inner = states[np.linalg.norm(states, axis=1) < 0.4]       # the reward sums converge here
            res[tag + "_states"] = states
            res[tag + "_inner"] = inner
            for name, start in (("grid", grid), ("states", states), ("inner", inner)):
                for horizon, tol in ((40, 0.05), (120, 0.02)):
                    key = "%s_%s_h%d" % (tag, name, horizon)
                    roa, traj = ex.compute_roa(start, cl, horizon, tol, no_traj=False)
                    assert np.array_equal(roa, ex.compute_roa(start, cl, horizon, tol))
                    pick = np.sort(np.random.default_rng(horizon).choice(traj.shape[0], min(16, traj.shape[0]),
                                                                          replace=False))
                    res.update({key + "_horizon": horizon, key + "_tol": tol, key + "_roa": roa,
                                key + "_end": traj[:, :, -1], key + "_traj_index": pick,
                                key + "_traj": traj[pick]})
                    print("%s: %d states, %d in the ROA" % (key, roa.size, roa.sum()))
                for horizon, tol, discount in ((60, 1e-3, 0.95), (400, 1e-3, 0.98)):
                    key = "%s_%s_r%d" % (tag, name, horizon)
                    sums = ex.reward_rollout(start, cl, rw, discount, horizon, tol)
                    # T*: the reference only prints it; recover it from the same loop's stopping rule
                    current, stop = (start.all_points if not isinstance(start, np.ndarray) else start), -1
                    for t in range(horizon):
                        temp = (discount ** t) * rw(current).ravel()
                        if np.max(np.abs(temp)) < tol:
                            stop = t
                            break
                        current = cl(current)
                    res.update({key + "_horizon": horizon, key + "_tol": tol, key + "_discount": discount,
                                key + "_sums": sums, key + "_stop": stop})
                    print("%s: T* = %d" % (key, stop))
    np.savez_compressed(os.path.join(HERE, "gp_mean.npz"), **res)


if __name__ == "__main__":
    main()
