"""Generate ``tests/golden/rollout.npz`` by running the UNMODIFIED reference's rollout helpers
(``examples/utilities.py`` ``compute_roa`` / ``reward_rollout``, plants ``InvertedPendulum`` /
``CartPole``) on the numpy-backed TF1 shim, with closed loops built from the reference's own objects
the way its notebooks build them (``reinforcement_learning_pendulum.ipynb`` cells 7-24,
``reinforcement_learning_cartpole.ipynb`` cells 7-24).

    SAFE_LEARNING_REFERENCE=<checkout> python tests/golden/make_golden_rollout.py

Cases: a saturated-LQR linear closed loop on a ragged 41 x 37 grid, the normalised pendulum with the
same policy, and the cart-pole on a 2-D plane of a 4-D grid passed as a state array.  Trajectories
are stored for a seeded subsample of start states only.
"""
import os
import sys

import numpy as np
from scipy.linalg import block_diag

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)

from reference_loader import REFERENCE, load_reference  # noqa: E402

sl = load_reference()
import tensorflow as tf  # noqa: E402  (shim)

sys.path.insert(0, os.path.join(REFERENCE, "examples"))
import utilities as ex  # noqa: E402  (the reference's examples/utilities.py)

assert os.path.abspath(ex.__file__).startswith(os.path.abspath(REFERENCE))


def closed_loops(dynamics, policy, reward_function, state_dim):
    """The notebooks' graph: one placeholder, one policy node feeding the dynamics and the reward."""
    states = tf.placeholder(tf.float64, [None, state_dim])
    actions = policy(states)
    future_states = dynamics(states, actions)
    rewards = reward_function(states, actions)
    return (lambda x: future_states.eval({states: x}),
            lambda x: rewards.eval({states: x}))


def run_case(res, name, start, dynamics, policy, reward_function, d, horizon, tol, discount,
             reward_horizon, reward_tol, n_traj=24):
    cl, rw = closed_loops(dynamics, policy, reward_function, d)
    roa, traj = ex.compute_roa(start, cl, horizon, tol, no_traj=False)
    assert np.array_equal(roa, ex.compute_roa(start, cl, horizon, tol))
    n = traj.shape[0]
    inside = np.flatnonzero(roa)
    outside = np.flatnonzero(~roa)
    rng = np.random.default_rng(len(name))
    pick = np.concatenate([rng.choice(inside, min(n_traj // 2, inside.size), replace=False),
                           rng.choice(outside, min(n_traj // 2, outside.size), replace=False)])
    pick = np.sort(pick)
    sums = ex.reward_rollout(start, cl, rw, discount, reward_horizon, reward_tol)
    # T*: the reference only prints it; recover it from the same loop's stopping rule
    current, stop = (start.all_points if not isinstance(start, np.ndarray) else start), -1
    for t in range(reward_horizon):
        temp = (discount ** t) * rw(current).ravel()
        if np.max(np.abs(temp)) < reward_tol:
            stop = t
            break
        current = cl(current)
    res.update({name + "_horizon": horizon, name + "_tol": tol, name + "_roa": roa,
                name + "_traj_index": pick, name + "_traj": traj[pick],
                name + "_discount": discount, name + "_reward_horizon": reward_horizon,
                name + "_reward_tol": reward_tol, name + "_sums": sums, name + "_stop": stop})
    print("%s: %d states, %d in the ROA, T* = %d" % (name, n, roa.sum(), stop))


def main():
    res = {}
    Q, R = 0.1 * np.eye(2), 0.1 * np.eye(1)
    # ---- pendulum (reinforcement_learning_pendulum.ipynb cell 7)
    dt, g, m, L, b = 0.01, 9.81, 0.15, 0.5, 0.1
    theta_max = np.deg2rad(30)
    omega_max = np.sqrt(g / L)
    u_max = g * m * L * np.sin(theta_max)
    Tx, Tu = np.array([theta_max, omega_max]), np.array([u_max])
    pendulum = ex.InvertedPendulum(m, L, b, dt, [(theta_max, omega_max), (u_max,)])
    A, B = pendulum.linearize()
    K, _ = sl.utilities.dlqr(A, B, Q, R)
    policy = sl.Saturation(sl.LinearSystem((-K,), name="policy_lqr"), -1, 1)
    reward = sl.QuadraticFunction(block_diag(-Q, -R), name="reward_function")
    for name in ("linear", "pendulum"):
        res.update({name + "_K": K, name + "_reward": block_diag(-Q, -R), name + "_kind": name,
                    name + "_A": A, name + "_B": B, name + "_plant": np.array([m, L, b, dt]),
                    name + "_Tx": Tx, name + "_Tu": Tu})
    # 1. saturated LQR on the linearisation: ragged grid, wider than the ROA of the saturated loop
    grid = sl.GridWorld(np.array([[-6., 6.], [-6., 6.]]), [41, 37])
    res.update({"linear_limits": grid.limits, "linear_num_points": grid.num_points})
    run_case(res, "linear", grid, sl.LinearSystem((A, B), name="dynamics"), policy, reward, 2,
             horizon=120, tol=1e-2, discount=0.98, reward_horizon=400, reward_tol=1e-2)
    # 2. the normalised pendulum plant
    grid = sl.GridWorld(np.array([[-4., 4.], [-4., 4.]]), [45, 39])
    res.update({"pendulum_limits": grid.limits, "pendulum_num_points": grid.num_points})
    run_case(res, "pendulum", grid, pendulum.__call__, policy, reward, 2,
             horizon=300, tol=1e-2, discount=0.98, reward_horizon=600, reward_tol=1e-2)
    # 3. cart-pole (reinforcement_learning_cartpole.ipynb cell 7), plane theta vs omega of a 4-D grid
    dt, m, M, L, b = 0.01, 0.175, 1.732, 0.28, 0.01
    x_max, theta_max, x_dot_max, theta_dot_max = 0.5, np.deg2rad(30), 2, np.deg2rad(30)
    u_max = (m + M) * (x_dot_max ** 2) / x_max
    cartpole = ex.CartPole(m, M, L, b, dt, [(x_max, theta_max, x_dot_max, theta_dot_max), (u_max,)])
    A, B = cartpole.linearize()
    Q4 = 0.1 * np.eye(4)
    K, _ = sl.utilities.dlqr(A, B, Q4, R)
    policy = sl.Saturation(sl.LinearSystem((-K,), name="policy_lqr"), -1, 1)
    reward = sl.QuadraticFunction(block_diag(-Q4, -R), name="reward_function")
    grid4 = sl.GridWorld(np.array([[-4., 4.]] * 4), 25)
    pts = grid4.all_points
    mask = np.logical_and(pts[:, 0] == 0.0, pts[:, 2] == 0.0)
    states = pts[mask]
    res.update({"cartpole_K": K, "cartpole_reward": block_diag(-Q4, -R), "cartpole_kind": "cartpole",
                "cartpole_plant": np.array([m, M, L, b, dt]),
                "cartpole_Tx": np.array([x_max, theta_max, x_dot_max, theta_dot_max]),
                "cartpole_Tu": np.array([u_max]), "cartpole_states": states})
    run_case(res, "cartpole", states, cartpole.__call__, policy, reward, 4,
             horizon=300, tol=0.1, discount=0.98, reward_horizon=300, reward_tol=1e-2)
    np.savez_compressed(os.path.join(HERE, "rollout.npz"), **res)


if __name__ == "__main__":
    main()
