"""Generate ``tests/golden/vanderpol.npz`` by running the UNMODIFIED reference's reverse-time Van der Pol
plant (``examples/utilities.py:440-519``), its rollout helpers ``compute_roa`` / ``reward_rollout`` and
``Lyapunov.update_safe_set`` on the numpy-backed TF1 shim.

    SAFE_LEARNING_REFERENCE=<checkout> python tests/golden/make_golden_vanderpol.py

Cases: one step of the plant with and without normalisation on states that include overflowing and
non-finite rows; ``linearize()``; ``compute_roa`` on a 41 x 37 grid whose corners lie outside the
limit cycle (their trajectories overflow to inf and NaN), given as a ``GridWorld`` and as a seeded
state array; reward sums and their stop step; the safe set of ``V = x^T P x`` with ``P`` from
``solve_discrete_lyapunov(Ad^T, Q)``.  The closed loop is the plant fed by the zero policy
``LinearSystem(zeros((1, 2)))``, whose one column the plant's ``tf.split(state_action, [2, 1])`` needs.
"""
import os
import sys

import numpy as np
import scipy.linalg
from scipy.linalg import block_diag

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)

from make_golden_rollout import closed_loops  # noqa: E402
from reference_loader import REFERENCE  # noqa: E402
import make_golden_rollout  # noqa: E402  (loads the reference on the shim)

sl = make_golden_rollout.sl
ex = make_golden_rollout.ex
import tensorflow as tf  # noqa: E402  (shim)

# the plant's ODE squares with `x ** 2` (utilities.py:517), an operator the shim's Tensor lacks
if not hasattr(tf.Tensor, "__pow__"):
    tf.Tensor.__pow__ = lambda self, o: tf._binary(np.power, self, o)

assert os.path.abspath(ex.__file__).startswith(os.path.abspath(REFERENCE))

DAMPING, DT, TX = 1, 0.01, (2.5, 3.0)


def one_step_inputs():
    """Seeded states in and around the limit cycle, then rows that overflow inside the sub-steps and
    rows with inf / NaN components (the action column is ignored by the plant)."""
    rng = np.random.default_rng(11)
    x = rng.uniform(-1.5, 1.5, (64, 2))
    big = np.array([[1e100, 0.5], [0.5, 1e100], [-1e160, 1.], [1e154, 1e154], [3e102, -2e102],
                    [1e300, 1e300], [-1e300, 2.], [0., 0.], [-0., 0.], [1., -0.]])
    inf, nan = np.inf, np.nan
    bad = np.array([[inf, 1.], [1., inf], [-inf, 0.], [0., -inf], [inf, inf], [inf, -inf], [nan, 1.],
                    [1., nan], [nan, nan], [nan, inf]])
    states = np.vstack([x, big, bad])
    actions = rng.uniform(-1, 1, (states.shape[0], 1))
    return np.hstack([states, actions])


def main():
    res = {"damping": np.array(DAMPING, dtype=np.float64), "dt": np.array(DT), "Tx": np.array(TX)}
    plants = {"plain": ex.VanDerPol(DAMPING, DT), "norm": ex.VanDerPol(DAMPING, DT, TX)}
    sa = one_step_inputs()
    res["step_inputs"] = sa
    ph = tf.placeholder(tf.float64, [None, 3])
    with np.errstate(over="ignore", invalid="ignore"):
        for name, plant in plants.items():
            res["step_%s" % name] = plant(ph).eval({ph: sa})
            res["linearize_%s" % name] = plant.linearize()
    vdp = plants["norm"]
    policy = sl.LinearSystem((np.zeros((1, 2)),), name="zero_policy")
    Q, R = 0.1 * np.eye(2), 0.1 * np.eye(1)
    reward = sl.QuadraticFunction(block_diag(-Q, -R), name="reward_function")
    res["reward"] = block_diag(-Q, -R)
    cl, rw = closed_loops(vdp, policy, reward, 2)

    def roa_case(name, start, horizon, tol, n_traj=24):
        with np.errstate(over="ignore", invalid="ignore"):
            roa, traj = ex.compute_roa(start, cl, horizon, tol, no_traj=False)
            assert np.array_equal(roa, ex.compute_roa(start, cl, horizon, tol))
        rng = np.random.default_rng(len(name))
        inside, outside = np.flatnonzero(roa), np.flatnonzero(~roa)
        escaped = np.flatnonzero(~np.isfinite(traj[:, :, -1]).all(axis=1))
        pick = np.concatenate([rng.choice(inside, n_traj // 3, replace=False),
                               rng.choice(np.setdiff1d(outside, escaped), n_traj // 3, replace=False),
                               rng.choice(escaped, n_traj // 3, replace=False)])
        pick = np.sort(pick)
        res.update({name + "_horizon": horizon, name + "_tol": tol, name + "_roa": roa,
                    name + "_traj_index": pick, name + "_traj": traj[pick]})
        print("%s: %d states, %d in the ROA, %d escape to inf / NaN" % (name, roa.size, roa.sum(),
                                                                       escaped.size))

    def reward_case(name, start, discount, horizon, tol):
        with np.errstate(over="ignore", invalid="ignore"):
            sums = ex.reward_rollout(start, cl, rw, discount, horizon, tol)
            # T*: the reference only prints it; recover it from the same loop's stopping rule
            current, stop = (start.all_points if not isinstance(start, np.ndarray) else start), -1
            for t in range(horizon):
                temp = (discount ** t) * rw(current).ravel()
                if np.max(np.abs(temp)) < tol:
                    stop = t
                    break
                current = cl(current)
        res.update({name + "_discount": discount, name + "_reward_horizon": horizon,
                    name + "_reward_tol": tol, name + "_sums": sums, name + "_stop": stop})
        print("%s: T* = %d, %d non-finite sums" % (name, stop, (~np.isfinite(sums)).sum()))

    # compute_roa: the grid, then a seeded state array over the same square
    grid = sl.GridWorld(np.array([[-1.2, 1.2], [-1.2, 1.2]]), [41, 37])
    res.update({"grid_limits": grid.limits, "grid_num_points": grid.num_points})
    roa_case("grid", grid, horizon=600, tol=0.05)
    reward_case("grid", grid, discount=0.98, horizon=300, tol=1e-2)
    states = np.random.default_rng(5).uniform(-1.2, 1.2, (700, 2))
    res["states"] = states
    roa_case("states", states, horizon=600, tol=0.05)
    inner = states[np.linalg.norm(states, axis=1) < 0.5]
    res["inner_states"] = inner
    reward_case("inner", inner, discount=0.98, horizon=600, tol=1e-2)

    # update_safe_set with V = x^T P x, the discrete Lyapunov function of the linearisation
    Ad = vdp.linearize()
    P = scipy.linalg.solve_discrete_lyapunov(Ad.T, Q)
    lgrid = sl.GridWorld(np.array([[-1., 1.], [-1., 1.]]), 41)
    initial = np.linalg.norm(lgrid.all_points, axis=1) < 0.1
    L_f, L_v, tau = 1.0, 1.0, 1e-4
    with tf.Session():
        lyap = sl.Lyapunov(lgrid, sl.QuadraticFunction(P), vdp, L_f, L_v, tau, policy, initial.copy())
        lyap.update_safe_set()
        res.update({"lyap_limits": lgrid.limits, "lyap_num_points": lgrid.num_points, "lyap_P": P,
                    "lyap_initial": initial, "lyap_L_f": L_f, "lyap_L_v": L_v, "lyap_tau": tau,
                    "lyap_values": lyap.values.copy(), "lyap_safe_set": lyap.safe_set.copy(),
                    "lyap_c_max": np.array(lyap.feed_dict[lyap.c_max])})
        print("safe set: %d / %d, c_max %r" % (lyap.safe_set.sum(), lyap.safe_set.size,
                                               float(lyap.feed_dict[lyap.c_max])))
    np.savez_compressed(os.path.join(HERE, "vanderpol.npz"), **res)


if __name__ == "__main__":
    main()
