"""Closed-loop rollouts: the ground truth the certified safe set and the learned values are judged
against (``examples/utilities.py:654-686`` ``compute_roa``, ``:522-545`` ``reward_rollout``).

``ClosedLoop(fun, policy)`` is the function ``x -> fun(x, policy(x))`` the reference's notebooks
build as a TF lambda.  When both ``fun`` and ``policy`` are fused function objects (they have
descriptors) and ``fun`` is deterministic, ``compute_roa`` / ``reward_rollout`` run the whole
rollout in one CUDA pass per chunk of steps (``csrc/rollout.cu``): one thread per start state,
the state in registers, start states generated from the grid index.  The posterior mean of a GP
(``gp.to_mean_function()``, a ``PosteriorMean``) is fused as dynamics too: the rollout kernels
evaluate it on the Bellman sweep's staged pipeline (DESIGN.md §3.16).  Any other callable runs the
reference's algorithm on the host, calling it once per step.
"""

from __future__ import annotations

import numpy as np
import torch

from . import _device as dev
from . import _native as nat
from .functions import (DeterministicFunction, Function, FunctionStack, GaussianProcess, GridWorld,
                        PosteriorMean, UncertainFunction, _PostOp, concatenate_inputs)

__all__ = ["ClosedLoop", "compute_roa", "reward_rollout"]

# device bytes of one slab of trajectories (compute_roa with no_traj=False); the host array is
# filled slab by slab
TRAJECTORY_SLAB_BYTES = 2 << 30


def _fusable(fun):
    """True when ``fun`` describes itself to the kernels (without touching the device)."""
    if not isinstance(fun, Function) or isinstance(fun, UncertainFunction):
        return False
    if isinstance(fun, _PostOp):
        return _fusable(fun.fun)
    return type(fun).descriptor is not Function.descriptor


class ClosedLoop(DeterministicFunction):
    """``x -> fun(x, policy(x))``: the closed-loop dynamics ``dynamics(x, policy(x))`` or the
    closed-loop reward ``reward_function(x, policy(x))`` of the notebooks.  Called on numpy
    states it evaluates one step (on the GPU when both parts are fused function objects)."""

    def __init__(self, fun, policy, name="closed_loop"):
        super().__init__(name)
        if isinstance(fun, (GaussianProcess, FunctionStack)):
            raise TypeError("ClosedLoop: GP dynamics return (mean, error) and have no closed loop "
                            "to roll out")
        self.fun, self.policy = fun, policy
        self.input_dim = getattr(policy, "input_dim", None)
        self.output_dim = getattr(fun, "output_dim", None)

    @property
    def fused(self):
        """Both parts run inside the rollout kernels (a ``PosteriorMean`` as the dynamics only: a
        closed-loop reward on one is not fused, ``reward_rollout`` checks that)."""
        return (_fusable(self.fun) or self.gp_mean) and _fusable(self.policy)

    @property
    def gp_mean(self):
        """The dynamics are a GP's posterior mean (the rollouts' ``_gp_mean`` entry points)."""
        return isinstance(self.fun, PosteriorMean)

    def __call__(self, *inputs):
        states = concatenate_inputs(inputs)
        if self.fused:
            return self.evaluate_device(states).cpu().numpy()
        return np.asarray(self.fun(states, self.policy(states)))

    def evaluate_device(self, points):
        """One step from the library's one-step evaluations: ``fun([x, policy(x)])``."""
        pts = dev.to_device(points)
        return self.fun.evaluate_device(torch.cat((pts, self.policy.evaluate_device(pts)), dim=1))


def _states_of(grid):
    """(GridWorld or None, device states or None, n, d) -- the two forms the reference accepts."""
    if isinstance(grid, GridWorld):
        return grid, None, grid.nindex, grid.ndim
    states = np.asarray(grid, dtype=np.float64)
    if states.ndim != 2:
        raise ValueError("grid must be a GridWorld or an [n, d] state array, got shape %s"
                         % (states.shape,))
    return None, states, states.shape[0], states.shape[1]


def _host_points(grid):
    return grid.all_points if isinstance(grid, GridWorld) else np.asarray(grid)


def _descriptor(grid_world, d, closed_loop, reward=None):
    cfg = nat.SlbBellman()
    if grid_world is not None:
        cfg.grid = grid_world.descriptor()
    else:
        cfg.grid.ndim = d
    cfg.policy = closed_loop.policy.descriptor()
    if closed_loop.gp_mean:
        cfg.gp = closed_loop.fun.gp_stack()
    else:
        cfg.dynamics = closed_loop.fun.descriptor()
    if reward is not None:
        cfg.reward = reward.fun.descriptor()
    return cfg


def _source(states, d):
    """Device start states (kept alive by the caller) or None for grid indices."""
    if states is None:
        return None
    return dev.to_device(states.reshape(-1, d) if states.size else np.zeros((0, d)))


def compute_roa(grid, closed_loop_dynamics, horizon=100, tol=1e-3, equilibrium=None, no_traj=True):
    """The states whose closed-loop trajectory ends within ``tol`` of the equilibrium after
    ``horizon - 1`` steps (``examples/utilities.py:654-686``).  Returns the boolean flags, and with
    ``no_traj=False`` also the trajectories ``[n, d, horizon]`` (float64).

    ``grid``: a ``GridWorld`` (coordinates are generated on the device, ``all_points`` is never
    built) or an ``[n, d]`` state array.  ``closed_loop_dynamics``: a fused ``ClosedLoop`` runs on
    the GPU; any other callable ``x -> x_next`` runs the reference's loop on the host."""
    grid_world, states, n, d = _states_of(grid)
    horizon = int(horizon)
    eq = np.zeros(d) if equilibrium is None else np.asarray(equilibrium, dtype=np.float64)
    if eq.size != d:
        raise ValueError("equilibrium must have %d entries, got shape %s" % (d, eq.shape))
    traj_host = None
    if not no_traj:
        traj_host = np.empty((n, d, horizon))        # the reference's array (ValueError if < 0)
        if horizon < 1:
            raise IndexError("index 0 is out of bounds for axis 2 with size %d" % horizon)
    if not (isinstance(closed_loop_dynamics, ClosedLoop) and closed_loop_dynamics.fused):
        return _compute_roa_host(_host_points(grid), closed_loop_dynamics, horizon, tol, eq.reshape(1, d),
                                 traj_host)
    if n == 0:
        roa = np.zeros(0, dtype=bool)
        return roa if no_traj else (roa, traj_host)
    lib = nat.load()
    cfg = _descriptor(grid_world, d, closed_loop_dynamics)
    entry = "slb_rollout_gp_mean" if closed_loop_dynamics.gp_mean else "slb_rollout"
    src = _source(states, d)
    eq_host = np.ascontiguousarray(eq.ravel())
    h = max(horizon, 0)
    roa = dev.empty((n,), torch.uint8)
    if no_traj:
        slabs = [(0, n)]
    else:
        per = max(1, int(TRAJECTORY_SLAB_BYTES // (d * horizon * 8)))
        slabs = [(p, min(p + per, n)) for p in range(0, n, per)]
        traj_dev = dev.empty((min(per, n), d, horizon))
    for p0, p1 in slabs:
        cnt = p1 - p0
        need = int(lib.slb_rollout_workspace(cfg, cnt, 0))
        work = dev.empty((need // 8 + 1,)) if need else None
        nat.check(getattr(lib, entry)(dev.stream(), cfg,
                                      None if src is None else src[p0:p1].data_ptr(), p0, cnt, h,
                                      eq_host.ctypes.data, float(tol), roa[p0:p1].data_ptr(), None,
                                      None if no_traj else traj_dev.data_ptr(), dev.ptr(work)),
                  entry)
        if not no_traj:
            torch.from_numpy(traj_host[p0:p1]).copy_(traj_dev[:cnt])
    flags = roa.cpu().numpy().astype(bool)
    return flags if no_traj else (flags, traj_host)


def _compute_roa_host(all_points, closed_loop_dynamics, horizon, tol, equilibrium, trajectories):
    """``examples/utilities.py:665-686`` for callables the kernels cannot fuse."""
    if trajectories is None:
        end_states = all_points
        for _ in range(1, horizon):
            end_states = closed_loop_dynamics(end_states)
    else:
        trajectories[:, :, 0] = all_points
        for t in range(1, horizon):
            trajectories[:, :, t] = closed_loop_dynamics(trajectories[:, :, t - 1])
        end_states = trajectories[:, :, -1]
    dists = np.linalg.norm(end_states - equilibrium, ord=2, axis=1, keepdims=True).ravel()
    roa = dists <= tol
    return roa if trajectories is None else (roa, trajectories)


def discount_table(discount, horizon):
    """``[discount ** t for t in range(horizon)]`` as float64, computed the way the reference's
    loop computes each factor (Python's float pow for a float discount), so the kernels multiply by
    bit-identical numbers."""
    return np.array([float(discount ** t) for t in range(max(int(horizon), 0))], dtype=np.float64)


def _report(stop):
    if stop >= 0:
        print('Reward sums converged after {} steps!'.format(stop + 1))
    else:
        print('Reward sums did not converge!')


def reward_rollout(grid, closed_loop_dynamics, reward_function, discount, horizon=250, tol=1e-3):
    """Discounted reward sums along the closed-loop trajectories from every start state, stopped
    after the first step at which ``max |discount^t r|`` over all states is below ``tol``
    (``examples/utilities.py:522-545``), with the reference's two messages.

    Runs fused on the GPU when both arguments are fused ``ClosedLoop`` objects around the SAME
    policy object (one policy evaluation per step feeds the reward and the dynamics); the dynamics
    may be a ``PosteriorMean``, the reward may not."""
    grid_world, states, n, d = _states_of(grid)
    horizon = int(horizon)
    fused = (isinstance(closed_loop_dynamics, ClosedLoop) and closed_loop_dynamics.fused
             and isinstance(reward_function, ClosedLoop) and reward_function.fused
             and not reward_function.gp_mean
             and reward_function.policy is closed_loop_dynamics.policy)
    if not fused:
        return _reward_rollout_host(_host_points(grid), n, closed_loop_dynamics, reward_function,
                                    discount, horizon, tol)
    if n == 0 and horizon > 0:
        np.max(np.abs(np.zeros(0)))                  # the reference's np.max on no states raises
    if horizon <= 0 or n == 0:
        _report(-1)
        return np.zeros(n)
    lib = nat.load()
    cfg = _descriptor(grid_world, d, closed_loop_dynamics, reward_function)
    src = _source(states, d)
    table = dev.to_device(discount_table(discount, horizon))
    sums = dev.empty((n,))
    stop = dev.empty((1,), torch.int64)
    need = int(lib.slb_rollout_workspace(cfg, n, 1))
    work = dev.empty((need // 8 + 1,))
    entry = "slb_reward_rollout_gp_mean" if closed_loop_dynamics.gp_mean else "slb_reward_rollout"
    nat.check(getattr(lib, entry)(dev.stream(), cfg, dev.ptr(src), 0, n, horizon,
                                  table.data_ptr(), float(tol), sums.data_ptr(),
                                  stop.data_ptr(), work.data_ptr()), entry)
    out = sums.cpu().numpy()
    _report(int(stop.item()))
    return out


def _reward_rollout_host(all_points, nindex, closed_loop_dynamics, reward_function, discount,
                         horizon, tol):
    """``examples/utilities.py:531-545`` for callables the kernels cannot fuse."""
    converged = False
    rollout = np.zeros(nindex)
    current_states = all_points
    t = -1
    for t in range(horizon):
        temp = (discount ** t) * np.asarray(reward_function(current_states)).ravel()
        rollout += temp
        if np.max(np.abs(temp)) < tol:
            converged = True
            break
        current_states = closed_loop_dynamics(current_states)
    _report(t if converged else -1)
    return rollout
