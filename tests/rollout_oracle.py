"""CPU restatement of the reference's rollout helpers (``examples/utilities.py:522-545``
``reward_rollout`` and ``:654-686`` ``compute_roa``), the checker of ``safe_learning_b200.rollout``.

The closed loops are plain callables built from ``oracle`` function objects
(``closed_loop(dynamics, policy)`` is the notebooks' ``dynamics(x, policy(x))``).  The two helpers
return what the reference returns, plus the step ``T*`` at which the reward sums stopped (-1: they
did not converge) so tests can compare it.  ``chunked_reward_rollout`` emulates in numpy the
device's chunked early-stop rule (``csrc/rollout.cu``) on a precomputed reward sequence.
"""
import numpy as np


def closed_loop(fun, policy):
    """``x -> fun(x, policy(x))`` (the notebooks' closed-loop lambdas)."""
    return lambda x: fun(x, policy(x))


def compute_roa(grid, closed_loop_dynamics, horizon=100, tol=1e-3, equilibrium=None, no_traj=True):
    """``examples/utilities.py:654-686``."""
    if isinstance(grid, np.ndarray):
        all_points = grid
        nindex = grid.shape[0]
        ndim = grid.shape[1]
    else:
        all_points = grid.all_points
        nindex = grid.nindex
        ndim = grid.ndim
    if no_traj:
        end_states = all_points
        for t in range(1, horizon):
            end_states = closed_loop_dynamics(end_states)
    else:
        trajectories = np.empty((nindex, ndim, horizon))
        trajectories[:, :, 0] = all_points
        for t in range(1, horizon):
            trajectories[:, :, t] = closed_loop_dynamics(trajectories[:, :, t - 1])
        end_states = trajectories[:, :, -1]
    if equilibrium is None:
        equilibrium = np.zeros((1, ndim))
    dists = np.linalg.norm(end_states - equilibrium, ord=2, axis=1, keepdims=True).ravel()
    roa = (dists <= tol)
    if no_traj:
        return roa
    return roa, trajectories


def reward_rollout(grid, closed_loop_dynamics, reward_function, discount, horizon=250, tol=1e-3):
    """``examples/utilities.py:522-545`` -> (sums, T*) with T* = -1 when not converged."""
    if isinstance(grid, np.ndarray):
        all_points = grid
        nindex = grid.shape[0]
    else:
        all_points = grid.all_points
        nindex = grid.nindex
    stop = -1
    rollout = np.zeros(nindex)
    current_states = all_points
    for t in range(horizon):
        temp = (discount ** t) * reward_function(current_states).ravel()
        rollout += temp
        if np.max(np.abs(temp)) < tol:
            stop = t
            break
        current_states = closed_loop_dynamics(current_states)
    return rollout, stop


def row_norm_sequential(x):
    """``np.linalg.norm(x, 2, axis=1)`` as the kernels compute it: sqrt of the left-to-right sum of
    squares."""
    x = np.asarray(x, dtype=np.float64)
    acc = x[:, 0] * x[:, 0]
    for c in range(1, x.shape[1]):
        acc = acc + x[:, c] * x[:, c]
    return np.sqrt(acc)


def _bits(values):
    return np.abs(values).view(np.uint64)


def chunked_reward_rollout(rewards, discount_table, tol, chunk):
    """The device algorithm on rewards [horizon, n] (reward of every state at every step): chunks
    of `chunk` steps each write per-step maxima of |temp| (as bit patterns), the finish step finds
    the first step below tol, and that chunk is re-run from its saved start sum up to T*.
    Returns (sums, T*)."""
    horizon, n = rewards.shape
    tol_bits = np.array([tol], dtype=np.float64).view(np.uint64)[0] if tol > 0 else np.uint64(0)
    sums = np.zeros(n)
    if horizon == 0:
        return sums, -1
    nchunks = -(-horizon // chunk)
    for c in range(nchunks):
        start = sums.copy()                           # the chunk's saved input
        t0, t1 = c * chunk, min((c + 1) * chunk, horizon)
        maxima = []
        for t in range(t0, t1):
            temp = discount_table[t] * rewards[t]
            sums = sums + temp
            maxima.append(_bits(temp).max() if n else np.uint64(0))
        below = [s for s, m in enumerate(maxima) if m < tol_bits]
        if below:
            stop = t0 + below[0]
            sums = start
            for t in range(t0, stop + 1):
                sums = sums + discount_table[t] * rewards[t]
            return sums, stop
    return sums, -1
