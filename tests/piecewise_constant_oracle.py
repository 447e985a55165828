"""numpy restatement of ``PiecewiseConstant`` (``functions.py:820-932``) and of tabular dynamic programming
on it, the yardstick of the host and GPU tests.

``nearest_index`` is ``GridWorld.state_to_index`` (``:733-752``) with the pinned NaN rule (DESIGN.md
§3.15): a row with a NaN coordinate has index -1 and evaluates to NaN in every column, where the reference
raises from ``ravel_multi_index``.
"""
import numpy as np


def nearest_index(limits, num_points, points):
    limits = np.asarray(limits, dtype=np.float64)
    num_points = np.asarray(num_points, dtype=np.int64)
    points = np.atleast_2d(np.asarray(points, dtype=np.float64))
    offset = limits[:, 0]
    inv = 1. / ((limits[:, 1] - offset) / (num_points - 1))
    nan = np.isnan(points).any(axis=1)
    ijk = np.rint((np.clip(points, limits[:, 0], limits[:, 1]) - offset) * inv)
    ijk[nan] = 0
    idx = np.ravel_multi_index(ijk.astype(np.int64).T, num_points)
    idx[nan] = -1
    return idx


def evaluate(limits, num_points, table, points):
    table = np.asarray(table, dtype=np.float64).reshape(int(np.prod(num_points)), -1)
    idx = nearest_index(limits, num_points, points)
    out = table[np.maximum(idx, 0)].copy()
    out[idx < 0] = np.nan
    return out


def table_vjp(limits, num_points, points, grad_out, ncols):
    """The vertex-table gradient: np.add.at in ascending point order; NaN points add nothing."""
    idx = nearest_index(limits, num_points, points)
    grad = np.zeros((int(np.prod(num_points)), ncols))
    keep = idx >= 0
    np.add.at(grad, idx[keep], np.asarray(grad_out, dtype=np.float64).reshape(-1, ncols)[keep])
    return grad


# ---- tabular dynamic programming on one grid: next states and rewards are given per (state, action)
def bellman_sweep(limits, num_points, values, next_states, rewards, gamma):
    """One Jacobi sweep r + gamma V(x+) (reinforcement_learning.py:65-140), V a one-column table."""
    v = evaluate(limits, num_points, values, next_states)[:, 0]
    return np.asarray(rewards, dtype=np.float64).reshape(-1) + gamma * v


def greedy(limits, num_points, values, next_states_per_action, rewards_per_action, gamma):
    """np.argmax over actions of r + gamma V(x+) (:213-279); NaN counts as the maximum."""
    q = np.stack([bellman_sweep(limits, num_points, values, nxt, rew, gamma)
                  for nxt, rew in zip(next_states_per_action, rewards_per_action)], axis=0)
    return np.argmax(q, axis=0), q


def evaluate_policy(limits, num_points, next_states, rewards, gamma):
    """Exact policy evaluation (:142-211): solve (I - gamma T) v = r with T's one-hot rows."""
    n = int(np.prod(num_points))
    idx = nearest_index(limits, num_points, next_states)
    T = np.zeros((n, n))
    T[np.arange(n), idx] = 1.0
    return np.linalg.solve(np.eye(n) - gamma * T, np.asarray(rewards, dtype=np.float64).reshape(n))
