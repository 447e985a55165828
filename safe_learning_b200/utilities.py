"""Host helpers kept from ``safe_learning/utilities.py``: ``batchify`` (``:224-249``, defines the
reference's batch semantics), ``dlqr`` / ``lqr`` (``:300-356``), and the small array builders the
callers of the path use: ``combinations`` / ``linearly_spaced_combinations`` (``:252-296``, the
action set of ``discrete_policy_optimization``), ``unique_rows`` (``:496-516``) and
``compute_trajectory`` (``:519-583``)."""

import numpy as np
import scipy.linalg

__all__ = ["batchify", "dlqr", "lqr", "concatenate_inputs", "combinations",
           "linearly_spaced_combinations", "unique_rows", "compute_trajectory"]

from .functions import concatenate_inputs  # noqa: E402,F401


def batchify(arrays, batch_size):
    """Yield ``(start, [views])`` in order; the last batch may be short."""
    if not isinstance(arrays, (list, tuple)):
        arrays = (arrays,)
    start = 0
    while True:
        views = [arr[start:start + batch_size] for arr in arrays]
        if views[0].size == 0:
            return
        yield start, views
        start += batch_size


def dlqr(a, b, q, r):
    """Discrete-time LQR: returns (k, p) with u = -k x."""
    a, b, q, r = (np.atleast_2d(m) for m in (a, b, q, r))
    p = scipy.linalg.solve_discrete_are(a, b, q, r)
    btp = b.T.dot(p)
    return np.linalg.solve(btp.dot(b) + r, btp.dot(a)), p


def lqr(a, b, q, r):
    """Continuous-time LQR: returns (k, p)."""
    a, b, q, r = (np.atleast_2d(m) for m in (a, b, q, r))
    p = scipy.linalg.solve_continuous_are(a, b, q, r)
    return np.linalg.solve(r, b.T.dot(p)), p


def combinations(arrays):
    """All combinations of the entries of ``arrays`` as rows (last array varies fastest)."""
    return np.array(np.meshgrid(*arrays)).T.reshape(-1, len(arrays))


def linearly_spaced_combinations(bounds, num_samples):
    """Rows of all combinations of ``num_samples`` linearly spaced values within ``bounds``
    (``[(lo, hi), ...]``; ``num_samples`` an integer or one per variable)."""
    bounds = np.atleast_2d(bounds)
    num_samples = np.broadcast_to(num_samples, len(bounds))
    return combinations([np.linspace(b[0], b[1], n) for b, n in zip(bounds, num_samples)])


def unique_rows(array):
    """Unique rows in the order of ``np.unique`` on the raw row bytes (what
    ``perturb_actions`` relies on, ``lyapunov.py:645-649``)."""
    array = np.ascontiguousarray(array)
    dtype = np.dtype((np.void, array.dtype.itemsize * array.shape[1]))
    _, idx = np.unique(array.view(dtype=dtype), return_index=True)
    return array[idx]


def compute_trajectory(dynamics, policy, initial_state, num_steps):
    """The trajectory of ``x_{t+1} = dynamics(x_t, policy(x_t))`` from one initial state
    (``utilities.py:519-583``): returns ``states [num_steps, d]`` and ``actions [num_steps - 1, m]``
    with ``actions[t] = policy(states[t])``, as float64 arrays.

    When dynamics and policy form a fused ``ClosedLoop`` (fusable function objects, the dynamics
    possibly a GP's ``PosteriorMean``) the states come from one rollout on the GPU and the actions
    from one batched policy evaluation, bit-identical to the step-by-step loop; any other callables
    run the reference's loop on the host, one call of each per step."""
    from .functions import Function, FunctionStack, GaussianProcess
    from .rollout import ClosedLoop, compute_roa

    initial_state = np.atleast_2d(initial_state)
    state_dim = initial_state.shape[1]
    states = np.empty((num_steps, state_dim), dtype=np.float64)
    actions = np.empty((num_steps - 1, policy.output_dim), dtype=np.float64)
    states[0, :] = initial_state
    loop = None
    if isinstance(dynamics, Function) and not isinstance(dynamics, (GaussianProcess, FunctionStack)):
        loop = ClosedLoop(dynamics, policy)
    if loop is not None and loop.fused:
        if num_steps > 1:
            _, traj = compute_roa(states[:1], loop, horizon=num_steps, no_traj=False)
            states[:] = traj[0].T
            actions[:] = policy.evaluate_device(states[:-1]).cpu().numpy()
        return states, actions
    for i in range(num_steps - 1):
        action = policy(states[[i], :])
        states[i + 1, :], actions[i, :] = dynamics(states[[i], :], action), action
    return states, actions
