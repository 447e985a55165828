"""``PolicyIteration`` (``safe_learning/reinforcement_learning.py:26-279``): the Bellman sweep.

``value_iteration`` and ``discrete_policy_optimization`` run as fused CUDA sweeps over the
value function's grid (``slb_bellman_sweep`` / ``slb_bellman_argmax``); ``future_values`` on
arbitrary state arrays is composed from the eager GPU evaluations of the function objects.
``optimize_value_function`` (``:142-211``) solves the reference's LP as what it is for a
policy, exact policy evaluation: the fixed point of ``v = r + gamma T v``, assembled and iterated
to a certified error bound on the GPU (``csrc/value_opt.cu``, DESIGN.md §3.9).
``bellmann_error`` (``:116-133``, autodiff) is outside this build's hot path.
"""

from __future__ import annotations

import numpy as np
import torch

from . import _device as dev
from . import _native as nat
from .functions import (Function, FunctionStack, GaussianProcess, PiecewiseConstant, PosteriorMean,
                        ScaledFunction, Triangulation, TriangulationGradient, UncertainFunction, _PostOp)

__all__ = ["PolicyIteration", "OptimizationError"]


class OptimizationError(Exception):
    """``reinforcement_learning.py:22-23``."""


# cvxpy options of the reference's call (``prob.solve(**solver_options)``) that have no meaning for
# the fixed-point solve; accepted so that notebook calls run unchanged
_IGNORED_SOLVER_OPTIONS = ("solver", "verbose", "eps", "warm_start")


def _fusable(fn):
    """True when ``fn`` has a descriptor the CUDA kernels can evaluate."""
    if not isinstance(fn, Function) or isinstance(fn, UncertainFunction):
        return False
    try:
        fn.descriptor()
    except (NotImplementedError, TypeError, ValueError):
        return False
    return True


def _on_triangulation_gradient(fn):
    """True when ``fn`` is a ``TriangulationGradient`` under post-op wrappers."""
    while isinstance(fn, _PostOp):
        fn = fn.fun
    return isinstance(fn, TriangulationGradient)


def _table_of(value_function):
    """The vertex table (Triangulation or PiecewiseConstant) under an optional ``-V`` / ``c * V``
    wrapper."""
    base = value_function
    while isinstance(base, ScaledFunction):
        base = base.fun
    if not isinstance(base, (Triangulation, PiecewiseConstant)):
        raise TypeError("value_function must be a Triangulation or a PiecewiseConstant (possibly scaled)")
    return base


def min_weight_of_stats(slot):
    """The smallest operator weight from slot 0 of the value statistics (slb200.h ``SLB_VALUE_STATS``): the
    complement of the weight's order-preserving key (``value_key``, value_opt.cu)."""
    key = ~np.uint64(slot)
    bits = (key & np.uint64(0x7fffffffffffffff)) if key >> np.uint64(63) else ~key
    return float(np.array([bits], dtype=np.uint64).view(np.float64)[0])


class PolicyIteration(object):
    """See ``reinforcement_learning.py:26-63`` for the parameters."""

    def __init__(self, policy, dynamics, reward_function, value_function, gamma=0.98):
        self.dynamics = dynamics
        self.reward_function = reward_function
        self.value_function = value_function
        self.gamma = gamma
        self.policy = policy
        self.feed_dict = {}
        self._storage = {}
        self.factor_actions = True        # discrete_policy_optimization: see csrc/bellman_tile.cu
        self._grid = _table_of(value_function).discretization
        self._begin, self._end = dev.shard_range(self._grid.nindex)

    @property
    def state_space(self):
        """``value_function.discretization.all_points`` (``:58-59``)."""
        return self._grid.all_points

    # ------------------------------------------------------------------ generic path
    def future_values(self, states, policy=None, actions=None, lyapunov=None,
                      lagrange_multiplier=1.):
        """``r(x, u) + gamma V(mean f(x, u))`` [``- lambda (decrease - threshold)``]
        (``:65-114``); numpy in, numpy [n, 1] out."""
        if isinstance(states, torch.Tensor) or isinstance(actions, torch.Tensor):
            return self._future_values_torch(states, policy, actions, lyapunov, lagrange_multiplier)
        states = np.atleast_2d(np.asarray(states, dtype=np.float64))
        if actions is None:
            actions = (policy or self.policy)(states)
        actions = np.broadcast_to(np.atleast_2d(actions), (states.shape[0],
                                                           np.atleast_2d(actions).shape[1]))
        next_states = self.dynamics(states, actions)
        rewards = self.reward_function(states, actions)
        var = None
        if isinstance(next_states, tuple):
            next_states, var = next_states
        updated = rewards + self.gamma * self.value_function(next_states)
        if lyapunov is not None:
            decrease = lyapunov.v_decrease_bound(states, (next_states, var))
            updated = updated - lagrange_multiplier * (decrease - lyapunov.threshold(states))
        return updated

    def _future_values_torch(self, states, policy, actions, lyapunov, lagrange_multiplier):
        """``future_values`` on device tensors as a differentiable torch expression (the reference
        differentiates this graph with ``tf.gradients`` to optimise a parametric policy under the
        Lyapunov penalty, ``examples/inverted_pendulum.ipynb`` cell 17): every fused function
        object is one autograd node (CUDA evaluation forward, its device Jacobian backward,
        ``Function.torch``), and so is the GP posterior (``slb_gp_predict`` forward, ``slb_gp_vjp``
        backward).  A Lipschitz term built on a ``TriangulationGradient`` (``MaxAbsFunction(
        V.gradient_function())``, cell 14) passes no gradient, as in the reference.  ``policy`` may
        be any callable on tensors (e.g. a ``torch.nn.Module``), and
        ``dynamics`` / ``reward_function`` any callable ``fn(states, actions)`` on tensors, as in the
        reference; gradients flow to ``actions`` / the policy's parameters (network weights,
        Triangulation ``vertex_values``) and to ``states`` if they require them."""
        states = dev.to_device(states) if not isinstance(states, torch.Tensor) else states
        if actions is None:
            fn = policy or self.policy
            actions = fn.torch(states) if isinstance(fn, Function) else fn(states)
        elif not isinstance(actions, torch.Tensor):
            actions = dev.to_device(np.atleast_2d(np.asarray(actions, dtype=np.float64)))
        actions = actions.expand(states.shape[0], actions.shape[1])
        z = torch.cat((states, actions), dim=1)
        err = None
        if isinstance(self.dynamics, (FunctionStack, GaussianProcess)):
            mean, err = self.dynamics.torch(z)                                   # :92, :98-99
        elif isinstance(self.dynamics, Function):
            mean = self.dynamics.torch(z)
        else:
            mean = self.dynamics(states, actions)
            if isinstance(mean, tuple):
                mean, err = mean
        reward = self.reward_function
        rewards = reward.torch(z) if isinstance(reward, Function) else reward(states, actions)
        updated = rewards + self.gamma * self.value_function.torch(mean)
        if lyapunov is not None:                                                 # :107-112
            v_fn, lv = lyapunov.lyapunov_function, lyapunov._lipschitz_lyapunov
            decrease = v_fn.torch(mean) - v_fn.torch(states)
            if err is not None:
                if _on_triangulation_gradient(lv):
                    # the reference's Triangulation.gradient is a py_func without a gradient
                    # (functions.py:1501-1510): the factor is a constant of the next states
                    lv_mu = lv.evaluate_device(mean.detach())
                elif isinstance(lv, Function):
                    lv_mu = lv.torch(mean)
                else:
                    lv_mu = float(lv)
                decrease = decrease + (lv_mu * err).sum(dim=1, keepdim=True)
            threshold = dev.to_device(np.broadcast_to(
                lyapunov.threshold(states.detach().cpu().numpy()), (states.shape[0], 1)).copy())
            updated = updated - lagrange_multiplier * (decrease - threshold)
        return updated

    # ------------------------------------------------------------------ fused sweeps
    def bellman_descriptor(self, fixed_action=None):
        cfg = nat.SlbBellman()
        cfg.grid = self._grid.descriptor()
        if fixed_action is None:
            cfg.policy = self.policy.descriptor()
        else:
            action = np.atleast_1d(np.asarray(fixed_action, dtype=np.float64))
            cfg.fixed_action = 1
            cfg.policy.out_dim = len(action)
            for i, a in enumerate(action):
                cfg.action[i] = float(a)
        if isinstance(self.dynamics, (FunctionStack, GaussianProcess, PosteriorMean)):
            cfg.gp = self.dynamics.gp_stack()           # the sweeps use the mean only
        elif isinstance(self.dynamics, UncertainFunction) or not isinstance(self.dynamics, Function):
            raise TypeError("dynamics must be a fusable Function, GaussianProcess, FunctionStack or "
                            "PosteriorMean")
        else:
            cfg.dynamics = self.dynamics.descriptor()
        cfg.reward = self.reward_function.descriptor()
        cfg.value = self.value_function.descriptor()
        cfg.gamma = float(self.gamma)
        return cfg

    def _sweep_device(self):
        """One Jacobi sweep over this rank's slab -> full new vertex table on the device."""
        lib = nat.load()
        cfg = self.bellman_descriptor()
        n = self._end - self._begin
        slab = dev.empty((n,))
        nat.check(lib.slb_bellman_sweep(dev.stream(), cfg, self._begin, self._end,
                                        slab.data_ptr()), "slb_bellman_sweep")
        return self._gather(slab)

    def _gather(self, slab):
        rank, world = dev.dist_info()
        if world == 1:
            return slab
        import torch.distributed as dist
        n = self._grid.nindex
        per = -(-n // world)
        padded = torch.zeros(per, dtype=slab.dtype, device=slab.device)
        padded[:slab.numel()] = slab
        out = torch.empty(per * world, dtype=slab.dtype, device=slab.device)
        dist.all_gather_into_tensor(out, padded)      # the one collective per sweep
        return out[:n]

    def value_iteration(self):
        """One synchronous value-iteration sweep (``:135-140``): every vertex is updated from
        the OLD table, then the table is replaced.  Returns ``max |V_new - V_old|`` (the
        convergence test user code applies, ``tests/test_rl.py:66-69``)."""
        lib = nat.load()
        tri = _table_of(self.value_function)
        scale = 1.0
        base = self.value_function
        while isinstance(base, ScaledFunction):
            scale *= base.factor
            base = base.fun
        new = self._sweep_device()
        if scale != 1.0:
            new = new / scale            # the table stores the un-scaled vertex values
        old = tri._param_dev
        if old.shape[1] != 1:
            raise ValueError("value function must have one output")
        residual = dev.zeros((1,))
        nat.check(lib.slb_max_abs_diff(dev.stream(), new.data_ptr(), old.data_ptr(),
                                       new.numel(), residual.data_ptr()), "slb_max_abs_diff")
        tri._store(new.reshape(-1, 1).contiguous())
        return float(residual.item())

    def discrete_policy_optimization(self, action_space, constraint=None):
        """Greedy policy over a discrete action set (``:213-279``): the vertex values of the
        piecewise-linear (Triangulation) or tabular (PiecewiseConstant) policy become
        ``action_space[argmax_a future_values(x, a)]``."""
        lib = nat.load()
        policy_tri = _table_of(self.policy)
        grid = policy_tri.discretization
        if grid.nindex != self._grid.nindex or np.any(grid.num_points != self._grid.num_points) \
                or np.any(grid.limits != self._grid.limits):
            raise NotImplementedError("policy and value function must share one discretization")
        actions = np.atleast_2d(np.asarray(action_space, dtype=np.float64))
        n_opt, m = actions.shape
        cfg = self.bellman_descriptor(fixed_action=actions[0])
        n = self._end - self._begin
        cons_dev = None
        if constraint is not None:
            n_states = grid.nindex
            rows = []
            for action in actions:
                arr = np.broadcast_to(action, (n_states, m))
                rows.append(np.asarray(constraint(arr), dtype=np.float64).reshape(-1)
                            [self._begin:self._end])
            cons_dev = dev.to_device(np.stack(rows))
        actions_dev = dev.to_device(actions)
        best = dev.empty((n,), torch.int32)
        # factored path (csrc/bellman_tile.cu): one kernel row per state + a tensor-core contraction
        # against the per-action table, when the library says it applies (workspace > 0)
        need = int(lib.slb_bellman_argmax_workspace(cfg, n_opt)) if self.factor_actions else 0
        scratch = dev.empty((need // 8 + 1,)) if need else None
        nat.check(lib.slb_bellman_argmax(dev.stream(), cfg, self._begin, self._end,
                                         actions_dev.data_ptr(), n_opt, dev.ptr(cons_dev),
                                         best.data_ptr(), None, dev.ptr(scratch)),
                  "slb_bellman_argmax")
        chosen = actions_dev[best.to(torch.int64)]            # [n, m]
        if m != 1 and dev.dist_info()[1] > 1:
            raise NotImplementedError("multi-GPU policy optimisation supports m == 1")
        full = self._gather(chosen[:, 0].contiguous()).reshape(-1, 1) if m == 1 else chosen
        policy_tri.parameters = full
        return full

    # ------------------------------------------------------------------ exact policy evaluation
    def optimize_value_function(self, **solver_options):
        """Evaluate the current policy exactly (``:180-211``) and store the values in the value
        function; returns them as a numpy array ``[N, 1]``.

        The reference maximises ``sum(v)`` subject to ``v <= r + gamma T v`` with cvxpy, T the value
        Triangulation's barycentric rows at the mean next states.  For nonnegative rows and
        ``gamma < 1`` the optimum is the fixed point ``v = r + gamma T v``; it is computed here by
        iterating that map from the current values until the certified error
        ``gamma rho / (1 - gamma rho) ||v_k - v_{k-1}||_inf`` is at most ``tol * max(1, ||v||_inf)``.

        Options: ``tol`` (1e-10) and ``max_iters`` (200000); the cvxpy options ``solver``,
        ``verbose``, ``eps`` and ``warm_start`` are accepted and ignored.  ``last_solve`` holds
        ``iterations``, ``bound``, ``rho``, ``repaired_rows`` and ``tier`` of the call.

        Raises ``OptimizationError`` when a row extrapolates (a weight < -1e-12: an unprojected
        next state outside the grid), when ``gamma * rho >= 1``, when a reward, a next state or a
        value of the current table (the start point) is NaN,
        or when ``max_iters`` iterations do not reach the bound; ``TypeError`` when the value
        function is not a plain one-output ``Triangulation`` or ``PiecewiseConstant``.  A
        ``PiecewiseConstant`` gives one-hot rows (the next state's nearest vertex, weight 1; DESIGN.md
        §3.15), so rho = 1.  Next states on a grid line are looked
        up in the simplex that contains them (DESIGN.md §3.2 Q6; the reference's lookup can pick a
        simplex of the wrong side of the cell there, which makes its LP unbounded).
        """
        tol = float(solver_options.pop("tol", 1e-10))
        max_iters = int(solver_options.pop("max_iters", 200000))
        unknown = set(solver_options) - set(_IGNORED_SOLVER_OPTIONS)
        if unknown:
            raise TypeError("optimize_value_function got unexpected options %s" % sorted(unknown))
        if not 0.0 <= self.gamma < 1.0:
            raise OptimizationError("Optimization problem is not a contraction: gamma = %r is "
                                    "outside [0, 1)" % (self.gamma,))
        values, stats = self._evaluate_policy(tol, max_iters)
        status = stats["status"]
        if status == nat.VALUE_NEGATIVE_WEIGHT:
            raise OptimizationError("Optimization problem is unbounded: the value function "
                                    "extrapolates (smallest interpolation weight %.3g); use a "
                                    "projected Triangulation" % stats["min_weight"])
        if status == nat.VALUE_NOT_CONTRACTIVE:
            raise OptimizationError("Optimization problem is not a contraction: gamma * rho = %.17g "
                                    ">= 1" % (self.gamma * stats["rho"]))
        if status == nat.VALUE_NAN:
            raise OptimizationError("Optimization problem is infeasible: NaN in the rewards, the "
                                    "next states or the value function's current table")
        if status == nat.VALUE_MAX_ITERS:
            raise OptimizationError("Optimization problem is not solved after %d iterations "
                                    "(certified error %.3g)" % (stats["iterations"], stats["bound"]))
        return values

    def _evaluate_policy(self, tol, max_iters):
        """Assemble the operator and iterate; the table is replaced when the iteration converged.
        Returns (the last iterate [N, 1] numpy, statistics); the statistics come back with the
        values in one device-to-host copy."""
        lib = nat.load()
        tri = self.value_function
        if type(tri) not in (Triangulation, PiecewiseConstant):
            raise TypeError("optimize_value_function needs a plain Triangulation or PiecewiseConstant value "
                            "function (the reference reaches value_function.tri), got %s" % type(tri).__name__)
        if tri._param_dev is None or tri._param_dev.shape[1] != 1:
            raise TypeError("optimize_value_function needs a one-output %s" % type(tri).__name__)
        n, d = self._grid.nindex, self._grid.ndim
        ncols = 2 if type(tri) is PiecewiseConstant else d + 1         # value_opt.cu: operator_cols
        idx = torch.int64 if n > 0x7fffffff else torch.int32
        cols = dev.empty((n, ncols), idx)
        weights = dev.empty((n, ncols))
        stats = dev.zeros((nat.VALUE_STATS,), torch.int64)
        if all(_fusable(f) for f in (self.policy, self.reward_function)) and (
                isinstance(self.dynamics, (FunctionStack, GaussianProcess, PosteriorMean))
                or _fusable(self.dynamics)):
            # every rank assembles and solves the whole system: no collective, identical tables
            rewards = dev.empty((n,))
            nat.check(lib.slb_value_operator(dev.stream(), self.bellman_descriptor(), 0, n,
                                             cols.data_ptr(), weights.data_ptr(), rewards.data_ptr(),
                                             stats.data_ptr()), "slb_value_operator")
        else:                                                                 # :197-205 on the host
            states = self.state_space
            actions = self.policy(states)
            next_states = self.dynamics(states, actions)
            if isinstance(next_states, tuple):
                next_states = next_states[0]
            rewards = dev.to_device(np.asarray(self.reward_function(states, actions),
                                               dtype=np.float64).reshape(n))
            nxt = dev.to_device(np.asarray(next_states, dtype=np.float64).reshape(n, d))
            nat.check(lib.slb_value_operator_points(dev.stream(), tri.descriptor(), nxt.data_ptr(), n,
                                                    cols.data_ptr(), weights.data_ptr(),
                                                    stats.data_ptr()), "slb_value_operator_points")
        values = tri._param_dev.detach().reshape(-1).clone()                  # warm start
        need = int(lib.slb_value_solve_workspace(n, ncols))
        work = dev.empty((need // 8,)) if need else None
        nat.check(lib.slb_value_solve(dev.stream(), n, ncols, cols.data_ptr(), weights.data_ptr(),
                                      rewards.data_ptr(), float(self.gamma), tol, max_iters,
                                      values.data_ptr(), dev.ptr(work), stats.data_ptr()),
                  "slb_value_solve")
        host = torch.cat((values, stats.view(torch.float64))).cpu().numpy()  # the one sync
        raw = host[n:].view(np.uint64)
        info = {"status": int(raw[7]), "iterations": int(raw[4]),
                "delta": float(host[n + 5]), "bound": float(host[n + 6]),
                "rho": float(host[n + 1]), "repaired_rows": int(raw[2]), "tier": int(raw[8]),
                "min_weight": min_weight_of_stats(raw[0])}
        self.last_solve = info
        out = host[:n].reshape(n, 1).copy()
        if info["status"] == nat.VALUE_CONVERGED:
            tri._store(values.reshape(-1, 1))
        return out, info
