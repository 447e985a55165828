"""Generate ``tests/golden/value_optimization.npz`` by running the UNMODIFIED reference's
``PolicyIteration.optimize_value_function`` (``reinforcement_learning.py:142-211``) on the numpy-backed
TF1 shim, with the shim's cvxpy (``tf1_shim/cvxpy``: the LP on scipy's HiGHS ``linprog``).

    SAFE_LEARNING_REFERENCE=<checkout> python tests/golden/make_golden_value_opt.py

Cases:
  ``matrix``  the transition matrix of the reference's own test (``tests/test_rl.py:83-127``);
  ``lqr24``   a saturated linear closed loop on a projected 24 x 20 Triangulation of [-1, 1]^2 (the LP
              is bounded, its optimum is stored);
  ``lqr25``   the same loop on 25 x 21, where next states on grid lines (the origin among them) get
              rows with a weight of -1 (DESIGN.md §3.2 Q6) and the LP is unbounded: the status and
              the reference's ``parameter_derivative`` rows are stored;
  ``gp1d``    ``1d_example.ipynb`` cell 15 shaped: 51 vertices, a GaussianProcess with a Matern32 x
              Linear kernel on 10 data points and a linear prior mean, a Triangulation policy; three
              rounds of optimize_value_function -> discrete_policy_optimization (values and policy
              after every round);
  ``gp55``    ``inverted_pendulum.ipynb`` cells 6-9 shaped: 55 x 55, a FunctionStack of two GPs with
              the notebook kernel Linear(3, ARD) + Matern32(1) x Linear(1) on 12 data points, the
              saturated LQR policy; one optimize_value_function.
"""
import os
import sys
from unittest import mock

import json

import numpy as np
from scipy.linalg import block_diag

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)

from reference_loader import load_reference  # noqa: E402

sl = load_reference()
import gpflow  # noqa: E402  (shim)
import tensorflow as tf  # noqa: E402  (shim)
import cvxpy  # noqa: E402  (shim)

sys.path.insert(0, os.path.dirname(os.path.dirname(HERE)))
import bench_workloads as W  # noqa: E402

assert os.path.abspath(cvxpy.__file__).startswith(os.path.join(HERE, "tf1_shim"))
from safe_learning.reinforcement_learning import OptimizationError  # noqa: E402

A = np.array([[1., .05], [-.2, .97]])
B = np.array([[0.], [.05]])
K = np.array([[.8, 1.1]])
REWARD = block_diag(-np.eye(2), -0.1 * np.eye(1))
GAMMA = 0.98


def matrix_case(res):
    trans = np.array([[0, .5, .5, 0], [.2, .1, .3, .5], [.3, .2, .4, .1], [0, 0, 0, 1]])
    rewards = np.arange(4, dtype=np.float64)[:, None]
    value_function = mock.Mock()
    value_function.tri.parameter_derivative.return_value = trans
    value_function.nindex = 4
    value_function.parameters = [tf.Variable(np.zeros((4, 1)))]
    value_function.discretization.all_points = np.arange(4, dtype=np.float64)[:, None]
    rl = sl.PolicyIteration(mock.Mock(return_value="actions"), mock.Mock(return_value=rewards),
                            mock.Mock(return_value=rewards), value_function)
    with tf.Session() as sess:
        sess.run(tf.variables_initializer(value_function.parameters))
        sess.run(rl.optimize_value_function())
        values = value_function.parameters[0].eval()
    res.update(matrix_T=trans, matrix_rewards=rewards, matrix_gamma=rl.gamma, matrix_values=values)
    print("matrix: values", values.ravel())


def lqr_case(res, name, num_points):
    grid = sl.GridWorld(np.array([[-1., 1.], [-1., 1.]]), num_points)
    value_function = sl.Triangulation(grid, np.zeros(grid.nindex), project=True)
    policy = sl.Saturation(sl.LinearSystem((-K,)), -1., 1.)
    rl = sl.PolicyIteration(policy, sl.LinearSystem((A, B)), sl.QuadraticFunction(REWARD),
                            value_function, gamma=GAMMA)
    states = grid.all_points
    with tf.Session():
        actions = policy(states).eval()
        next_states = sl.LinearSystem((A, B))(states, actions).eval()
        rewards = sl.QuadraticFunction(REWARD)(states, actions).eval()
    T = value_function.tri.parameter_derivative(next_states).tocoo()
    res.update({name + "_num_points": np.array(num_points), name + "_next_states": next_states,
                name + "_rewards": rewards, name + "_T_rows": T.row, name + "_T_cols": T.col,
                name + "_T_data": T.data, name + "_gamma": GAMMA})
    try:
        with tf.Session():
            values = rl.optimize_value_function().eval()
        status = cvxpy.OPTIMAL
    except OptimizationError as err:
        values, status = np.full((grid.nindex, 1), np.nan), str(err)
    res.update({name + "_values": values, name + "_status": status})
    print("%s: %d rows with a negative weight, %s" % (name, np.sum(T.data < -1e-12), status))


GP1D_KERNEL = json.dumps(["prod", ["matern32", 1, {"lengthscales": 0.5, "variance": 0.04,
                                                  "active_dims": [0]}],
                          ["linear", 1, {"active_dims": [0]}]])
GP1D_PRIOR = np.array([[1.0, 0.1]])
GP1D_REWARD = np.diag([-1.0, -0.2])
GP1D_ACTIONS = np.linspace(-0.5, 0.5, 11)[:, None]


def gp1d_data():
    rng = np.random.default_rng(11)
    X = np.column_stack((rng.uniform(-1, 1, 10), rng.uniform(-0.5, 0.5, 10)))
    Y = (X[:, :1] + 0.1 * X[:, 1:] - 0.05 * np.sin(3 * X[:, :1]) + 1e-3 * rng.standard_normal((10, 1)))
    return X, Y


def ref_gp(X, Y, spec, prior_row, noise):
    kern = W.build_kernel(gpflow.kernels, spec)
    gp = sl.GPRCached(X, Y, kern, sl.LinearSystem((prior_row[None, :],)), 1.0)
    gp.likelihood.variance = noise
    gp.update_cache()
    return sl.GaussianProcess(gp, beta=2.0)


def gp1d_case(res):
    X, Y = gp1d_data()
    grid = sl.GridWorld(np.array([[-1., 1.]]), 51)
    dynamics = ref_gp(X, Y, GP1D_KERNEL, GP1D_PRIOR[0], 1e-6)
    policy = sl.Triangulation(grid, -0.3 * grid.all_points, name="policy")
    value = sl.Triangulation(grid, np.zeros(grid.nindex), project=True, name="value")
    rl = sl.PolicyIteration(policy, dynamics, sl.QuadraticFunction(GP1D_REWARD), value, gamma=0.98)
    values, policies = [], []
    with tf.Session() as sess:
        sess.run(tf.variables_initializer(policy.parameters + value.parameters))
        for _ in range(3):
            values.append(rl.optimize_value_function().eval())
            rl.discrete_policy_optimization(GP1D_ACTIONS)
            policies.append(policy.parameters[0].eval())
    res.update(gp1d_X=X, gp1d_Y=Y, gp1d_values=np.stack(values), gp1d_policies=np.stack(policies))
    print("gp1d: values", [float(v.min()) for v in values])


def gp55_par():
    par = W.make_pendulum(num_points=55, M=12, with_prior_mean=True, seed=3)
    par["kernel_specs"] = W.notebook_pendulum_kernels([[2e-3, 6e-3, 1.5e-3], [2.5e-2, 8e-3, 1.2e-2]])
    return par


def gp55_case(res):
    par = gp55_par()
    grid = sl.GridWorld(par["limits"], par["num_points"])
    dynamics = sl.FunctionStack([ref_gp(par["X"], par["Y"][:, [j]], par["kernel_specs"][j],
                                        par["prior_rows"][j], par["noise_variance"]) for j in range(2)])
    policy = sl.Saturation(sl.LinearSystem((-par["K"],)), -1., 1.)
    reward = sl.QuadraticFunction(block_diag(-np.diag([1., 2.]), -1.2 * np.eye(1)))
    value = sl.Triangulation(grid, np.zeros(grid.nindex), project=True)
    rl = sl.PolicyIteration(policy, dynamics, reward, value, gamma=0.98)
    states = grid.all_points
    with tf.Session():
        actions = policy(states).eval()
        mean = dynamics(states, actions)[0].eval()
        values = rl.optimize_value_function().eval()
    T = value.tri.parameter_derivative(mean).tocoo()
    res.update(gp55_next_states=mean, gp55_values=values, gp55_T_rows=T.row, gp55_T_cols=T.col,
               gp55_T_data=T.data)
    print("gp55: %d rows with a negative weight, values in [%g, %g]"
          % (np.sum(T.data < -1e-12), values.min(), values.max()))


def main():
    res = {"A": A, "B": B, "K": K, "reward": REWARD}
    matrix_case(res)
    lqr_case(res, "lqr24", [24, 20])
    lqr_case(res, "lqr25", [25, 21])
    gp1d_case(res)
    gp55_case(res)
    np.savez_compressed(os.path.join(HERE, "value_optimization.npz"), **res)


if __name__ == "__main__":
    main()
