"""Region-of-attraction estimation: the ``Lyapunov`` class of ``safe_learning/lyapunov.py:142-606``.

Same constructor, attributes and methods as the reference; the work is one fused CUDA sweep
(``slb_lyapunov_sweep``) + a sort-free prefix reduction (``slb_first_fail`` /
``slb_apply_prefix``) instead of a Python loop of 10 000-point ``Session.run`` calls.
With GP dynamics the sweep runs behind a certified decision filter (``slb_lyapunov_sweep_filtered``,
csrc/filter.cu): identical flags, the O(M^2) posterior only where the outcome depends on it.
With ``torch.distributed`` initialised, the grid is sharded by contiguous flat-index range
(one process per GPU) and the ranks exchange one 32-byte key per sweep -- through peer memory
inside the reduction kernels (``slb_exchange``), without a collective call or a host round trip;
``c_max`` and the statistics are resolved lazily when they are read.
"""

from __future__ import annotations

import zlib

import numpy as np
import torch

from . import _device as dev
from . import _native as nat
from .functions import Function, FunctionStack, GaussianProcess, PosteriorMean, UncertainFunction, config

__all__ = ["Lyapunov", "get_safe_sample", "perturb_actions", "smallest_boundary_value",
           "combine_fail_keys", "combine_prefix_stats", "adaptive_as_written"]


def _unique_rows(array):
    """Unique rows in byte order (``utilities.py:496-516``)."""
    array = np.ascontiguousarray(array)
    dtype = np.dtype((np.void, array.dtype.itemsize * array.shape[1]))
    _, idx = np.unique(array.view(dtype=dtype), return_index=True)
    return array[idx]


def smallest_boundary_value(fun, discretization):
    """Smallest value of ``fun`` on the faces of the grid (``lyapunov.py:22-56``): the level up to
    which a Lyapunov candidate's sub-level sets stay inside the discretisation.  ``fun`` is a
    fusable Function object (evaluated on the GPU) or any callable on numpy arrays."""
    min_value = np.inf
    for i in range(discretization.ndim):
        tmp = list(discretization.discrete_points)
        tmp[i] = discretization.discrete_points[i][[0, -1]]
        columns = [x.ravel() for x in np.meshgrid(*tmp, indexing="ij")]
        points = np.column_stack(columns)
        if isinstance(fun, Function):
            smallest = float(fun.evaluate_device(points).min().item())
        else:
            smallest = float(np.min(fun(points)))
        min_value = min(min_value, smallest)
    return min_value


def perturb_actions(states, actions, perturbations, limits=None):
    """State-action pairs from perturbed baseline actions (``lyapunov.py:609-651``)."""
    num_states, state_dim = states.shape
    states_new = np.repeat(states, len(perturbations), axis=0)
    actions_new = (np.repeat(actions, len(perturbations), axis=0)
                   + np.tile(perturbations, (num_states, 1)))
    state_actions = np.column_stack((states_new, actions_new))
    if limits is not None:
        limits = np.asarray(limits)
        acts = state_actions[:, state_dim:]
        np.clip(acts, limits[:, 0], limits[:, 1], out=acts)
        state_actions = _unique_rows(state_actions)
    return state_actions


def get_safe_sample(lyapunov, perturbations=None, limits=None, positive=False, num_samples=None,
                    actions=None):
    """Most uncertain safe state-action pair near the current policy (``lyapunov.py:657-797``).

    The candidate evaluation -- GP mean / beta*sigma at every (safe state, perturbed action),
    ``V(mean) + sum(L_V(mean) * sigma) < c_max`` and, unless ``positive``, membership of the mean
    in the safe set -- runs on the GPU (``slb_gp_predict`` + fused function evaluations); the
    candidate list itself (<= num_samples x perturbations rows) is assembled on the host like
    the reference does.
    """
    import warnings
    disc = lyapunov.discretization
    safe_idx = np.where(lyapunov.safe_set)[0]
    safe_states = disc.index_to_state(safe_idx)
    if num_samples is not None and len(safe_states) > num_samples:
        idx = np.random.choice(len(safe_states), num_samples, replace=True)
        safe_states = safe_states[idx]
    safe_actions = None
    if perturbations is None:
        arrays = [arr.ravel() for arr in np.meshgrid(safe_states, actions, indexing="ij")]
        state_actions = np.column_stack(arrays)
    else:
        safe_actions = lyapunov.policy(safe_states)
        state_actions = perturb_actions(safe_states, safe_actions, perturbations, limits)

    c_max = lyapunov.feed_dict[lyapunov.c_max]

    def evaluate(sa):
        mean, std = lyapunov.dynamics.predict_device(sa)
        bound = std.sum(dim=1, keepdim=True)
        def on_mean(fn):
            # fusable objects on the device; plain callables on the host (composed path)
            if isinstance(fn, Function):
                return fn.evaluate_device(mean)
            if callable(fn):
                out = np.asarray(fn(mean.cpu().numpy()), dtype=np.float64)
                return dev.to_device(out.reshape(mean.shape[0], -1))
            return float(fn)
        lv = on_mean(lyapunov._lipschitz_lyapunov)
        error = (lv * std).sum(dim=1, keepdim=True)
        future = on_mean(lyapunov.lyapunov_function) + error
        return (future < c_max)[:, 0].cpu().numpy(), mean.cpu().numpy(), bound.cpu().numpy()

    maps_inside, mean, bound = evaluate(state_actions)
    if not positive:
        maps_inside &= lyapunov.safe_set[disc.state_to_index(mean)]
    bound_safe = bound[maps_inside]
    if len(bound_safe) == 0:
        warnings.warn("No safe state-action pairs found! Using backup policy ...", RuntimeWarning)
        if safe_actions is None:
            safe_actions = lyapunov.policy(safe_states)
        state_actions = perturb_actions(safe_states, safe_actions, np.array([[0.]]), limits)
        _, _, bound = evaluate(state_actions)
        max_id = int(np.argmax(bound))
        return state_actions[[max_id]], bound[max_id].squeeze()
    max_id = int(np.argmax(bound_safe))
    return state_actions[maps_inside, :][[max_id]], bound_safe[max_id].squeeze()


class _CMax(object):
    """Hashable stand-in for the reference's ``c_max`` placeholder: the value lives in
    ``lyapunov.feed_dict[lyapunov.c_max]`` (``lyapunov.py:210-211, 595``)."""

    def __repr__(self):
        return "<c_max>"


class _FeedDict(dict):
    """``lyapunov.feed_dict``: a dict whose ``c_max`` entry is resolved from the device when it is
    read (the sweep itself never waits for the host)."""

    def __init__(self, owner):
        super().__init__()
        self._owner = owner

    def _sync(self):
        self._owner._resolve_pending()

    def __getitem__(self, key):
        self._sync()
        return dict.__getitem__(self, key)

    def get(self, key, default=None):
        self._sync()
        return dict.get(self, key, default)

    def items(self):
        self._sync()
        return dict.items(self)

    def values(self):
        self._sync()
        return dict.values(self)

    def copy(self):
        self._sync()
        return dict(self)


def _as_function(obj, what):
    if isinstance(obj, Function):
        return obj
    raise TypeError(
        "%s must be a safe_learning_b200 Function object (LinearSystem, QuadraticFunction, "
        "Saturation, Triangulation, abs(fun), ...) so it can be fused into the CUDA sweep; "
        "got %r. Arbitrary Python callables are not supported (no CPU fallback)." % (what, obj))


def combine_fail_keys(rows):
    """rows: int64 [world, 4] of per-rank ``slb_fail_key`` -> (winning rank, (key_value,
    key_index, total n_ok)).  Lexicographic min on (uint64 value key, flat index)."""
    rows = np.ascontiguousarray(rows, dtype=np.int64)
    kv = rows[:, 0].copy().view(np.uint64)
    best = min(range(rows.shape[0]), key=lambda r: (int(kv[r]), int(rows[r, 1])))
    return best, (int(kv[best]), int(rows[best, 1]), int(rows[:, 2].sum()))


def combine_prefix_stats(rows):
    """rows: int64 [world, 4] of per-rank ``slb_prefix_stats`` -> (n_safe, n_below, max_below,
    max_all) over all ranks."""
    rows = np.ascontiguousarray(rows, dtype=np.int64)
    u = rows.copy().view(np.uint64)
    return (int(rows[:, 0].sum()), int(rows[:, 1].sum()), int(u[:, 2].max()), int(u[:, 3].max()))


def _key_to_value(bits):
    """Inverse of the kernels' order-preserving uint64 key."""
    bits = int(bits)
    raw = (bits & 0x7fffffffffffffff) if bits & 0x8000000000000000 else (~bits) & 0xffffffffffffffff
    return float(np.array([raw], dtype=np.uint64).view(np.float64)[0])


def adaptive_as_written(values, negative, decrease, threshold, coef, initial, tau, batch,
                        max_refinement, safety_factor, safe_set=None, refinement=None):
    """Host loop of the reference's adaptive branch, as written (``lyapunov.py:497-606`` with
    ``:540-582``), over per-point quantities of the whole grid: ``negative``, ``decrease``,
    ``threshold`` (at ``tau``) and ``coef = -L_V(x)(1 + L_f)`` so that ``threshold(x, tau / n) =
    coef * (tau / n)``.  ``refined_safety_check`` (``:457-481``) compares the decrease of EVERY
    state fed in the slice with the cell's own refined threshold, i.e. a cell passes iff the
    largest decrease of the slice is below it.  Returns (safe [N] bool, refinement [N] int,
    sorted position of c_max).  ``safe_set`` / ``refinement`` are the previous safe set and
    refinement the loop starts from (``can_shrink=False``, ``:507-510``); by default the initial
    set with refinement 1 (``can_shrink=True``)."""
    n_total = len(values)
    order = np.argsort(values, kind="stable")
    safe_s = (initial if safe_set is None else np.asarray(safe_set, dtype=bool))[order].copy()
    refine_s = (initial if refinement is None else np.asarray(refinement))[order].astype(int)
    start = bound = refine_bound = 0
    for start in range(0, n_total, batch):
        sel = order[start:start + batch]
        neg_b = negative[sel]
        safe_b = safe_s[start:start + batch]            # views: edited in place
        refine_b = refine_s[start:start + batch]
        safe_b |= neg_b
        refine_b[neg_b] = 1
        bound = int(np.argmin(safe_b))
        refine_bound = 0
        if bound > 0 or not safe_b[0]:
            with np.errstate(divide="ignore", invalid="ignore"):
                ratio = safety_factor * threshold[sel[bound:]] / decrease[sel[bound:]]
            ratio = np.where(np.isnan(ratio), 0.0, ratio)
            refine_b[bound:] = np.ceil(np.maximum(ratio, 0))            # :445-455, :542-546
            idx_safe = neg_b | initial[sel]
            refine_b[idx_safe] = 1                                      # :548-551
            to_check = ((refine_b >= 1) & (refine_b <= max_refinement))[bound:]
            stop = len(to_check) if to_check.all() else int(np.argmin(to_check))
            if stop > 0:
                fed = sel[bound:bound + stop]
                dec = decrease[fed]
                worst = np.nan if np.isnan(dec).any() else dec.max()
                with np.errstate(invalid="ignore"):
                    thr = coef[fed] * (tau / refine_b[bound:bound + stop])
                    refined = worst < thr                               # :474-478
                refine_bound = len(refined) if refined.all() else int(np.argmin(refined))
                safe_b[bound:bound + refine_bound] = True
            if stop < len(to_check) or refine_bound < stop:
                safe_b[bound + refine_bound:] = False
                refine_b[bound + refine_bound:] = 0
                break
    position = start + bound + refine_bound - 1
    safe = np.zeros(n_total, dtype=bool)
    safe[order[safe_s]] = True
    refinement = np.zeros(n_total, dtype=int)
    refinement[order] = refine_s
    safe[initial] = True
    refinement[initial] = 1
    return safe, refinement, position


class Lyapunov(object):
    """See ``lyapunov.py:142-225`` for the parameters.

    ``lipschitz_lyapunov`` may be a float or a fusable Function (e.g. ``abs(LinearSystem(2P))``);
    ``lipschitz_dynamics`` a float, a fusable Function or any callable of the states.  With
    ``adaptive=True``, ``update_safe_set(max_refinement=R)`` re-checks failing cells on a locally
    refined mesh (``lyapunov.py:445-487, 540-582``, see ``_adaptive_ok``).

    ``policy``, ``lyapunov_function``, ``lipschitz_lyapunov`` (and deterministic ``dynamics``) may
    also be ARBITRARY Python callables on numpy arrays, as the reference allows
    (``lyapunov.py:227-263``, ``lyapunov_function_learning.ipynb`` cell 19).  A Python lambda
    cannot be fused into a CUDA kernel, so such a sweep takes the *composed* path
    (``_compute_negative_composed``): the GP posterior of every grid point still runs on the GPU
    (``slb_gp_predict``), the user's callables are evaluated on the host on the arrays the
    reference's graph would feed them, and the flags go back to the device for the first-fail
    reduction / prefix rule.  Orders of magnitude slower than the fused sweep -- use the Function
    objects where they exist.
    """

    def __init__(self, discretization, lyapunov_function, dynamics, lipschitz_dynamics,
                 lipschitz_lyapunov, tau, policy, initial_set=None, adaptive=False):
        self.discretization = discretization
        self.policy = policy
        self.tau = tau
        self.dynamics = dynamics
        self.lyapunov_function = lyapunov_function
        self._lipschitz_dynamics = lipschitz_dynamics
        self._lipschitz_lyapunov = lipschitz_lyapunov
        self.adaptive = adaptive
        self._pending = None              # sweep enqueued, c_max / statistics not read back yet
        self._last_sweep = {}
        self.feed_dict = _FeedDict(self)
        self.c_max = _CMax()
        dict.__setitem__(self.feed_dict, self.c_max, 0.)
        # decision filter in front of the O(M^2) posterior: "auto" (on when every GP's certified
        # variance floor is far above fp64 rounding), True, or False
        self.filter = "auto"
        self.refinement_mode = "mesh"     # or "reference": lyapunov.py:474-478 as written

        n = discretization.nindex
        self._begin, self._end = dev.shard_range(n)
        self._safe_host = np.zeros(n, dtype=bool)
        self._safe_dirty = False          # device slab newer than _safe_host
        self.initial_safe_set = initial_set
        if initial_set is not None:
            self._safe_host[initial_set] = True
        self._refinement = np.zeros(n, dtype=int)
        if initial_set is not None:
            self._refinement[initial_set] = 1

        self._values_host = None
        self._values_dev = None           # slab [end - begin]
        self._safe_dev = None
        self._negative_dev = None
        self._initial_dev = None
        self._initial_token = None
        self._workspace = None
        self._filter_ws = None
        self._filter_stats = None
        self._lf_cache = None
        self.update_values()

    # ------------------------------------------------------------------ attributes
    @property
    def safe_set(self):
        """Boolean numpy array over the whole grid (gathers the device slabs on demand)."""
        if self._safe_dirty:
            rank, world = dev.dist_info()
            if world == 1:
                # one synchronisation for both read-backs of a sweep: the safe set and the 64 bytes of
                # key + statistics that c_max / last_sweep are resolved from
                host = self._host_buffers()
                host[0].copy_(self._safe_dev, non_blocking=True)
                if self._pending is not None:
                    host[1].copy_(self._ks_dev, non_blocking=True)
                torch.cuda.current_stream().synchronize()
                self._safe_host = host[0].numpy().astype(bool)
                if self._pending is not None:
                    self._resolve_pending(host[1].numpy()[None, :].copy())
            else:
                slab = self._safe_dev.to(torch.bool)
                self._safe_host = self._gather(slab).cpu().numpy()
            self._safe_dirty = False
        return self._safe_host

    @safe_set.setter
    def safe_set(self, value):
        self._safe_host = np.asarray(value, dtype=bool).copy()
        self._safe_dirty = False

    @property
    def values(self):
        if self._values_host is None and self._values_dev is not None:
            self._values_host = self._gather(self._values_dev).cpu().numpy()
        return self._values_host

    @values.setter
    def values(self, value):
        self._values_host = None if value is None else np.asarray(value, dtype=np.float64)
        if value is not None:
            self._values_dev = dev.to_device(self._values_host[self._begin:self._end])

    def _gather(self, slab):
        rank, world = dev.dist_info()
        if world == 1:
            return slab
        import torch.distributed as dist
        n = self.discretization.nindex
        per = -(-n // world)
        padded = torch.zeros(per, dtype=slab.dtype, device=slab.device)
        padded[:slab.numel()] = slab
        out = torch.empty(per * world, dtype=slab.dtype, device=slab.device)
        if slab.dtype == torch.bool:
            dist.all_gather_into_tensor(out.view(torch.uint8), padded.view(torch.uint8))
        else:
            dist.all_gather_into_tensor(out, padded)
        return out[:n]

    # ------------------------------------------------------------------ Lipschitz helpers
    def lipschitz_dynamics(self, states):
        """``lyapunov.py:227-244``."""
        f = self._lipschitz_dynamics
        return f(states) if callable(f) else f

    def lipschitz_lyapunov(self, states):
        """``lyapunov.py:246-263``."""
        f = self._lipschitz_lyapunov
        return f(states) if callable(f) else f

    def threshold(self, states, tau=None):
        """``-lv * (1 + lf) * tau`` (``lyapunov.py:265-288``); numpy in, numpy out."""
        if tau is None:
            tau = self.tau
        lv = self.lipschitz_lyapunov(states)
        if callable(self._lipschitz_lyapunov) and lv.shape[1] > 1:
            lv = np.abs(lv).sum(axis=1, keepdims=True)
        lf = self.lipschitz_dynamics(states)
        return -lv * (1. + lf) * tau

    def is_safe(self, state):
        """``lyapunov.py:290-303``."""
        return self.safe_set[self.discretization.state_to_index(state)]

    def v_decrease_confidence(self, states, next_states):
        """``lyapunov.py:324-354`` on explicit arrays (eager GPU evaluation of V and L_V)."""
        if isinstance(next_states, (tuple, list)):
            next_states, error_bounds = next_states
            lv = self.lipschitz_lyapunov(next_states)
            bound = np.sum(lv * error_bounds, axis=1, keepdims=True)
        else:
            bound = 0.
        v_decrease = self.lyapunov_function(next_states) - self.lyapunov_function(states)
        return v_decrease, bound

    def v_decrease_bound(self, states, next_states):
        """``lyapunov.py:356-376``."""
        v_dot, v_dot_error = self.v_decrease_confidence(states, next_states)
        return v_dot + v_dot_error

    # ------------------------------------------------------------------ composed (callable) path
    def _is_composed(self):
        """True if a member is a plain Python callable, i.e. the sweep cannot be fused.  A GP's
        ``PosteriorMean`` as the dynamics is composed too: its decrease is nominal (no error term),
        as the reference computes it for deterministic dynamics, with the mean on the device."""
        def plain(obj):
            return callable(obj) and not isinstance(obj, Function)
        return (plain(self.policy) or plain(self.lyapunov_function)
                or plain(self._lipschitz_lyapunov) or plain(self.dynamics)
                or isinstance(self.dynamics, PosteriorMean))

    def _negative_composed(self, states, tau=None, want_details=False):
        """The graph of ``lyapunov.py:433-441`` on a numpy array of states with the members
        called as the reference calls them: ``dynamics(states, policy(states))``,
        ``v_decrease_bound``, ``threshold``, strict ``<`` (NaN compares false)."""
        actions = np.asarray(self.policy(states), dtype=np.float64)
        if actions.ndim == 1:
            actions = actions.reshape(len(states), -1)
        next_states = self.dynamics(states, actions)
        decrease = self.v_decrease_bound(states, next_states)
        threshold = self.threshold(states, tau)
        with np.errstate(invalid="ignore"):
            negative = np.squeeze(decrease < threshold, axis=1)
        if not want_details:
            return negative
        mean, err = next_states if isinstance(next_states, (tuple, list)) else (next_states, None)
        return negative, {"decrease": decrease[:, 0],
                          "threshold": np.broadcast_to(threshold, decrease.shape)[:, 0],
                          "mean": mean, "err": err}

    def _compute_negative_composed(self, want_details=False):
        grid = self.discretization
        n = self._end - self._begin
        flags = np.empty(n, dtype=bool)
        parts = {}
        chunk = 1 << 18
        for start in range(0, n, chunk):
            stop = min(start + chunk, n)
            states = grid.index_to_state(np.arange(self._begin + start, self._begin + stop))
            out = self._negative_composed(states, want_details=want_details)
            if want_details:
                out, det = out
                for k, v in det.items():
                    if v is not None:
                        parts.setdefault(k, []).append(v)
            flags[start:stop] = out
        if self._negative_dev is None or self._negative_dev.numel() != n:
            self._negative_dev = dev.empty((n,), torch.uint8)
        self._negative_dev.copy_(dev.to_device(flags.astype(np.uint8), torch.uint8))
        if not want_details:
            return self._negative_dev
        details = {k: dev.to_device(np.concatenate(v)) for k, v in parts.items()}
        details["values"] = self._values_dev
        return self._negative_dev, details

    # ------------------------------------------------------------------ descriptor
    def _descriptor_token(self):
        def tok(obj):
            return (id(obj), obj.version) if isinstance(obj, Function) else obj
        return (id(self.discretization), tok(self.policy), tok(self.dynamics),
                tok(self.lyapunov_function), tok(self._lipschitz_lyapunov),
                self._lipschitz_dynamics if not callable(self._lipschitz_dynamics) else id(
                    self._lipschitz_dynamics), self.tau)

    def sweep_descriptor(self):
        """The ``slb_sweep`` describing the graph of ``lyapunov.py:433-441`` (cached until a
        function object, the GP data / hyper-parameters or a scalar changes)."""
        token = self._descriptor_token()
        cached = self.__dict__.get("_cfg_cache")
        if cached is not None and cached[0] == token:
            return cached[1]
        cfg = self._build_descriptor()
        self.__dict__["_cfg_cache"] = (token, cfg)
        return cfg

    def _build_descriptor(self):
        cfg = nat.SlbSweep()
        cfg.grid = self.discretization.descriptor()
        cfg.policy = _as_function(self.policy, "policy").descriptor()
        cfg.lyapunov = _as_function(self.lyapunov_function, "lyapunov_function").descriptor()
        if isinstance(self.dynamics, (FunctionStack, GaussianProcess)):
            cfg.gp = self.dynamics.gp_stack()
        elif isinstance(self.dynamics, UncertainFunction):
            raise TypeError("uncertain dynamics must be a GaussianProcess or FunctionStack")
        else:
            cfg.dynamics = _as_function(self.dynamics, "dynamics").descriptor()
        lv = self._lipschitz_lyapunov
        if isinstance(lv, Function):
            cfg.lipschitz_v = lv.descriptor()
        elif callable(lv):
            _as_function(lv, "lipschitz_lyapunov")
        else:
            cfg.lv_const = float(lv)
        lf = self._lipschitz_dynamics
        if isinstance(lf, Function):
            cfg.lipschitz_f = lf.descriptor()              # state-dependent, fused
        elif callable(lf):
            # any Python callable (lyapunov.py:227-244; the notebooks pass lambdas, e.g.
            # lyapunov_function_learning.ipynb cell 13): tabulated once on EVERY point of this
            # rank's slab; a table that turns out constant collapses to the scalar
            table = self._tabulate_lipschitz_dynamics(lf)
            if table is None:
                lf = self._lf_cache[2]
                cfg.lf_const = float(lf)
            else:
                cfg.lf_values = table.data_ptr()
                cfg.lf_index_base = self._begin
        else:
            cfg.lf_const = float(lf)
        cfg.tau = float(self.tau)
        return cfg

    def _tabulate_lipschitz_dynamics(self, fn):
        """L_f(x) of a Python callable on this rank's grid points -> device table [n_local], or
        None if it is the same number everywhere (then ``_lf_cache[2]`` holds it)."""
        token = (id(fn), self._begin, self._end)
        if self._lf_cache is not None and self._lf_cache[0] == token:
            return self._lf_cache[1]
        grid = self.discretization
        parts = []
        for start in range(self._begin, self._end, 1 << 20):
            idx = np.arange(start, min(start + (1 << 20), self._end))
            vals = np.asarray(fn(grid.index_to_state(idx)), dtype=np.float64)
            if vals.ndim == 2 and vals.shape[1] > 1:
                raise ValueError("lipschitz_dynamics must return one value per state")
            parts.append(np.broadcast_to(vals.reshape(-1) if vals.size > 1 else vals.reshape(1),
                                         (len(idx),)).copy())
        table = np.concatenate(parts) if parts else np.zeros(0)
        constant = table.size == 0 or bool(np.all(table == table[0]))
        rank, world = dev.dist_info()
        if world > 1:                      # every rank must build the same kind of descriptor
            import torch.distributed as dist
            first = float(table[0]) if table.size else 0.0
            pair = torch.tensor([first, -first, 0.0 if constant else 1.0], dtype=torch.float64,
                                device=dev.device())
            dist.all_reduce(pair, op=dist.ReduceOp.MAX)
            lo, hi, varying = -float(pair[1]), float(pair[0]), float(pair[2])
            constant = varying == 0.0 and lo == hi
        if constant:
            self._lf_cache = (token, None, float(table[0]) if table.size else 0.0)
            return None
        self._lf_cache = (token, dev.to_device(table), None)
        return self._lf_cache[1]

    # ------------------------------------------------------------------ values
    def update_values(self):
        """``values = V(all grid points)`` (``lyapunov.py:305-322``), computed on the device
        from flat indices in chunks (coordinates are never materialised for the full grid)."""
        lib = nat.load()
        n = self._end - self._begin
        if not isinstance(self.lyapunov_function, Function) and callable(self.lyapunov_function):
            grid = self.discretization
            parts = [np.asarray(self.lyapunov_function(grid.index_to_state(
                np.arange(s0, min(s0 + (1 << 20), self._end)))), dtype=np.float64).reshape(-1)
                for s0 in range(self._begin, self._end, 1 << 20)]
            self._values_dev = dev.to_device(np.concatenate(parts) if parts else np.zeros(0))
            self._values_host = None
            return
        fn = _as_function(self.lyapunov_function, "lyapunov_function")
        out = dev.empty((n,))
        grid = self.discretization.descriptor()
        chunk = 1 << 22
        d = self.discretization.ndim
        for start in range(0, n, chunk):
            stop = min(start + chunk, n)
            pts = dev.empty((stop - start, d))
            nat.check(lib.slb_index_to_state(dev.stream(), grid, self._begin + start,
                                             self._begin + stop, pts.data_ptr()),
                      "slb_index_to_state")
            out[start:stop] = fn.evaluate_device(pts)[:, 0]
        self._values_dev = out
        self._values_host = None

    # ------------------------------------------------------------------ the sweep
    def _initial_device(self):
        """uint8 slab of the initial safe set (re-uploaded when the attribute changes)."""
        init = self.initial_safe_set
        if init is None:
            self._initial_dev = self._initial_token = None
            return None
        arr = np.ascontiguousarray(init)
        # keyed on the CONTENT (the reference re-reads the array on every update_safe_set,
        # lyapunov.py:504-506; callers do edit it in place)
        token = (arr.shape, arr.dtype.str, zlib.crc32(arr.view(np.uint8).reshape(-1)))
        if self._initial_dev is None or self._initial_token != token:
            mask = np.zeros(self.discretization.nindex, dtype=bool)
            mask[arr] = True
            self._initial_dev = dev.to_device(mask[self._begin:self._end].astype(np.uint8),
                                              torch.uint8)
            self._initial_token = token
        return self._initial_dev

    def _filter_enabled(self, cfg):
        """Whether the sweep goes through the decision filter (csrc/filter.cu)."""
        if cfg.gp.num_outputs == 0 or self.filter is False:
            return False
        if self.filter == "auto":
            return self.dynamics.variance_floor() >= 1e-9
        return True

    def compute_negative(self, want_details=False):
        """Run the fused sweep over this rank's index range.  Returns the device uint8 slab
        ``negative`` (and, if asked, a dict of device tensors: values, decrease, threshold,
        mean, err -- the details always come from the full posterior)."""
        n = self._end - self._begin
        if self._is_composed():
            return self._compute_negative_composed(want_details)
        if self._negative_dev is None or self._negative_dev.numel() != n:
            self._negative_dev = dev.empty((n,), torch.uint8)
        if not want_details:
            return self.compute_negative_range(self._begin, self._end, out=self._negative_dev)
        lib = nat.load()
        cfg = self.sweep_descriptor()
        details = {}
        d = self.discretization.ndim
        details["values"] = dev.empty((n,))
        details["decrease"] = dev.empty((n,))
        details["threshold"] = dev.empty((n,))
        details["mean"] = dev.empty((n, d))
        ptrs = [details[k].data_ptr() for k in ("values", "decrease", "threshold", "mean")]
        if cfg.gp.num_outputs > 0:
            details["err"] = dev.empty((n, d))
            ptrs.append(details["err"].data_ptr())
        else:
            ptrs.append(None)
        nat.check(lib.slb_lyapunov_sweep(dev.stream(), cfg, self._begin, self._end,
                                         self._negative_dev.data_ptr(), *ptrs),
                  "slb_lyapunov_sweep")
        return self._negative_dev, details

    def _filter_buffers(self, n):
        """Workspace of a filtered sweep of ``n`` points and the filter's statistics (device)."""
        lib = nat.load()
        need = int(lib.slb_filter_workspace(n)) // 8 + 1
        if self._filter_ws is None or self._filter_ws.numel() < need:
            self._filter_ws = dev.empty((need,), torch.int64)
        if self._filter_stats is None:
            self._filter_stats = dev.zeros((4,), torch.int64)
        return self._filter_ws, self._filter_stats

    def compute_negative_range(self, begin, end, out=None):
        """``negative`` for the flat grid indices ``[begin, end)`` on the default path (filtered
        when the dynamics are a GP, see ``filter``) -> device uint8 tensor."""
        lib = nat.load()
        cfg = self.sweep_descriptor()
        n = end - begin
        if out is None:
            out = dev.empty((n,), torch.uint8)
        if self._filter_enabled(cfg):
            ws, stats = self._filter_buffers(n)
            nat.check(lib.slb_lyapunov_sweep_filtered(dev.stream(), cfg, begin, end,
                                                      out.data_ptr(), None, ws.data_ptr(),
                                                      stats.data_ptr()),
                      "slb_lyapunov_sweep_filtered")
        else:
            nat.check(lib.slb_lyapunov_sweep(dev.stream(), cfg, begin, end, out.data_ptr(),
                                             None, None, None, None, None), "slb_lyapunov_sweep")
        return out

    @property
    def filter_stats(self):
        """Counts since the last ``reset_filter_stats()`` (this rank): points decided by the mean
        and the prior bound, by the head-rank variance bound, refined by the full posterior, and
        all points that went through the filter."""
        if self._filter_stats is None:
            return {"prior": 0, "head": 0, "refined": 0, "points": 0}
        a, b, c, n = (int(v) for v in self._filter_stats.cpu().numpy())
        return {"prior": a, "head": b, "refined": c, "points": n}

    def reset_filter_stats(self):
        if self._filter_stats is not None:
            self._filter_stats.zero_()

    def negative_at_points(self, points, tau=None):
        """The decision of ``lyapunov.py:436-441`` on an explicit device point list ``[n, d]``
        (``slb_lyapunov_points``), optionally with another discretisation constant."""
        if self._is_composed():
            flags = self._negative_composed(points.cpu().numpy(), tau=tau)
            return dev.to_device(flags.astype(np.uint8), torch.uint8)
        lib = nat.load()
        cfg = self.sweep_descriptor()
        if tau is not None and float(tau) != float(self.tau):
            cfg = nat.SlbSweep.from_buffer_copy(cfg)
            cfg.tau = float(tau)
        points = points.contiguous()
        n = points.shape[0]
        neg = dev.empty((n,), torch.uint8)
        if n:
            nat.check(lib.slb_lyapunov_points(dev.stream(), cfg, points.data_ptr(), n,
                                              neg.data_ptr(), None, None, None, None, None),
                      "slb_lyapunov_points")
        return neg

    def _refinement_offsets(self, n):
        """Mesh of ``lyapunov.py:459-472`` relative to the cell centre: ``0.5 (1 - 1/n) unit_maxes
        linspace(-1, 1, n)`` per dimension, ``indexing='ij'`` -> ``[n^d, d]``."""
        lengths = self.discretization.unit_maxes.reshape((-1, 1))
        spacing = np.linspace(-1., 1., n).reshape(1, -1)
        border = 0.5 * (1 - 1 / n) * lengths * np.tile(spacing, [len(lengths), 1])
        mesh = np.meshgrid(*border, indexing="ij")
        return np.stack([col.reshape(-1) for col in mesh], axis=1)

    @staticmethod
    def _required_refinement(details, safety_factor):
        """``n_req = ceil(max(safety_factor * threshold / decrease, 0))``, NaN -> 0 (``:447-455``),
        as a float64 slab."""
        ratio = float(safety_factor) * details["threshold"] / details["decrease"]
        ratio = torch.where(torch.isnan(ratio), torch.zeros_like(ratio), ratio)
        return torch.ceil(torch.clamp(ratio, min=0.0))

    def _refined_mesh_check(self, cand, n_req, max_refinement, ok):
        """The refined check of ``lyapunov.py:459-472`` at the candidates (bool slab ``cand``): the
        decrease condition with ``tau / n_req`` on all ``n_req^d`` mesh points of the cell.  Writes
        the verdict into ``ok`` at the candidates; one host synchronisation per mesh size."""
        values = self._values_dev
        grid = self.discretization
        d = grid.ndim
        num = torch.as_tensor(np.asarray(grid.num_points, dtype=np.int64), device=values.device)
        unit = dev.to_device(np.asarray(grid.unit_maxes, dtype=np.float64))
        offset = dev.to_device(np.asarray(grid.offset, dtype=np.float64))
        for n in range(2, int(max_refinement) + 1):
            idx = torch.nonzero(cand & (n_req == n))[:, 0]
            if idx.numel() == 0:
                continue
            offsets = dev.to_device(self._refinement_offsets(n))          # [n^d, d]
            chunk = max(1, (1 << 21) // offsets.shape[0])
            for c0 in range(0, idx.numel(), chunk):
                part = idx[c0:c0 + chunk]
                flat = part + self._begin
                ijk = torch.empty((part.numel(), d), dtype=torch.int64, device=values.device)
                for c in range(d - 1, -1, -1):
                    ijk[:, c] = flat % num[c]
                    flat = flat // num[c]
                centers = ijk.to(torch.float64) * unit + offset            # functions.py:714-731
                points = (offsets[None, :, :] + centers[:, None, :]).reshape(-1, d)
                fine = self.negative_at_points(points, self.tau / n)
                ok[part] = fine.view(part.numel(), -1).to(torch.bool).all(dim=1)

    def _adaptive_ok(self, max_refinement, safety_factor, initial):
        """Adaptive discretisation (``lyapunov.py:445-487, 540-582``) in closed form.

        ``n_req = ceil(max(safety_factor * threshold / decrease, 0))`` (NaN -> 0, ``:447-455``).  A
        point counts as verified if ``negative``, or if ``2 <= n_req <= max_refinement`` and the
        decrease condition holds with ``tau / n_req`` on all ``n_req^d`` mesh points of its cell
        (``:459-472``).  The reference's graph builds that mesh but compares the outer
        ``decrease`` tensor (``:474-478``, dead code); this implements the evident intent, the
        same as ``oracle.Lyapunov.update_safe_set(refinement_mode="mesh")``.  The V-sorted prefix
        rule then runs on the verified flags; refined candidates are only evaluated up to the
        first point that cannot be verified at all.  Returns (flags uint8, n_req int64) slabs.
        """
        neg, det = self.compute_negative(want_details=True)
        negb = neg.to(torch.bool)
        n_req = self._required_refinement(det, safety_factor)
        known = negb if initial is None else negb | initial.to(torch.bool)
        cand = ~known & (n_req >= 2) & (n_req <= max_refinement)
        hopeless = ~known & ~cand
        values = self._values_dev
        if bool(hopeless.any()):
            cand &= values <= values[hopeless].min()
        ok = negb.clone()
        self._refined_mesh_check(cand, n_req, max_refinement, ok)
        return ok.to(torch.uint8), n_req.to(torch.int64), negb

    def update_safe_set(self, can_shrink=True, max_refinement=1, safety_factor=1.,
                        parallel_iterations=1):
        """Compute and update the safe set (``lyapunov.py:407-606``).

        The call only ENQUEUES the sweep (fused decision kernel(s), first-fail reduction with the
        inter-rank key exchange, prefix application); ``safe_set``, ``c_max`` (through
        ``feed_dict``), ``_refinement`` and ``last_sweep`` synchronise when they are read.

        ``can_shrink=False`` keeps the previous safe set and refinement as the starting point and
        resolves the reference's V-sorted batch loop on the device (``_update_no_shrink``); it is
        complete when the call returns.  ``parallel_iterations`` (the reference's ``tf.map_fn``
        parallelism) is accepted and ignored."""
        adaptive = bool(self.adaptive and max_refinement > 1)
        if not can_shrink:
            if adaptive and self.initial_safe_set is None:
                raise NotImplementedError(
                    "adaptive refinement with can_shrink=False needs an initial safe set: the "
                    "reference's branch indexes initial_safe_set[indices] (lyapunov.py:547-548)")
            if dev.dist_info()[1] > 1:
                raise NotImplementedError("can_shrink=False needs global ranks: replicas only")
        safety_factor = max(float(safety_factor), 1.)
        self._pending = None
        if adaptive and self.refinement_mode == "reference":
            return self._update_adaptive_as_written(max_refinement, safety_factor, can_shrink)
        lib = nat.load()
        n_local = self._end - self._begin
        initial = self._initial_device()
        if not can_shrink:
            return self._update_no_shrink(int(max_refinement) if adaptive else 1, safety_factor,
                                          initial)

        rank, world = dev.dist_info()
        if self._workspace is None:
            self._workspace = dev.empty((int(lib.slb_first_fail_workspace(n_local)) // 8 + 16,))
            # [0:4] slb_fail_key, [4:8] slb_prefix_stats of this rank
            self._ks_dev = dev.zeros((8,), torch.int64)
            self._key_dev, self._stats_dev = self._ks_dev[0:4], self._ks_dev[4:8]
        if self._safe_dev is None or self._safe_dev.numel() != n_local:
            self._safe_dev = dev.empty((n_local,), torch.uint8)

        self.__dict__["_adaptive_state"] = None
        negb = None
        if adaptive:
            flags, n_req, negb = self._adaptive_ok(max_refinement, safety_factor, initial)
            self.__dict__["_adaptive_state"] = (n_req, negb)
        xchg = dev.get_exchange() if world > 1 else None

        def enqueue():
            st = dev.stream()
            if not adaptive and world == 1 and not self._is_composed():
                cfg = self.sweep_descriptor()
                if self._filter_enabled(cfg):
                    # the filter's decision kernels fold the first-fail key as they decide: one memset,
                    # the three stages and the prefix kernel (slb_safe_set_step)
                    if self._negative_dev is None or self._negative_dev.numel() != n_local:
                        self._negative_dev = dev.empty((n_local,), torch.uint8)
                    ws, stats = self._filter_buffers(n_local)
                    nat.check(lib.slb_safe_set_step(st, cfg, self._begin, self._end,
                                                    self._negative_dev.data_ptr(),
                                                    self._values_dev.data_ptr(), dev.ptr(initial),
                                                    ws.data_ptr(), stats.data_ptr(),
                                                    self._key_dev.data_ptr(), self._safe_dev.data_ptr(),
                                                    self._stats_dev.data_ptr()), "slb_safe_set_step")
                    return
            neg = flags if adaptive else self.compute_negative()
            args = (st, self._values_dev.data_ptr(), neg.data_ptr(), dev.ptr(initial), n_local,
                    self._begin, self._workspace.data_ptr(), self._key_dev.data_ptr())
            if xchg is not None:
                # the one exchange of the sweep: 32 bytes per rank stored into every peer's slot
                # by the reduction kernel itself; the prefix kernel waits for them (light.cu)
                nat.check(lib.slb_first_fail_x(*args, xchg), "slb_first_fail_x")
                nat.check(lib.slb_apply_prefix_x(st, self._values_dev.data_ptr(), dev.ptr(initial),
                                                 n_local, self._begin, self._key_dev.data_ptr(),
                                                 self._safe_dev.data_ptr(),
                                                 self._workspace.data_ptr(),
                                                 self._stats_dev.data_ptr(), xchg),
                          "slb_apply_prefix_x")
                return
            nat.check(lib.slb_first_fail(*args), "slb_first_fail")
            if world > 1:
                # fallback without peer memory: NCCL all-gather of the keys, reduced on device
                gathered = dev.allgather_rows(self._key_dev)
                nat.check(lib.slb_combine_fail_keys(st, gathered.data_ptr(), world,
                                                    self._key_dev.data_ptr()),
                          "slb_combine_fail_keys")
            nat.check(lib.slb_apply_prefix(st, self._values_dev.data_ptr(), dev.ptr(initial),
                                           n_local, self._begin, self._key_dev.data_ptr(),
                                           self._safe_dev.data_ptr(), self._workspace.data_ptr(),
                                           self._stats_dev.data_ptr()), "slb_apply_prefix")

        # CUDA-graph replay of the launches of a sweep (one memset + 5 kernels on the filtered single-process
        # path, memsets + 8 kernels otherwise; no collective call
        # inside when the keys travel through peer memory) while nothing they depend on changes:
        # the second sweep with an unchanged descriptor is captured, later ones replay it.  It saves
        # device time between the launches and the host enqueue time per sweep, which is what
        # bounds the end-to-end step.
        token = None
        if (not adaptive and not self._is_composed()
                and (world == 1 or xchg is not None)):
            token = (self._descriptor_token(), self._values_dev.data_ptr(),
                     0 if initial is None else initial.data_ptr(), n_local,
                     self._filter_enabled(self.sweep_descriptor()), dev.factor_dependency_epoch())
        cached = self.__dict__.get("_sweep_graph")
        if token is not None and cached is not None and cached[0] == token:
            cached[1].replay()
            lib.slb_note_graph_replay(cached[2])
        elif token is not None and self.__dict__.get("_sweep_graph_seen") == token:
            before = nat.launch_count()
            graph = torch.cuda.CUDAGraph()
            with torch.cuda.graph(graph):
                enqueue()
            self.__dict__["_sweep_graph"] = (token, graph, nat.launch_count() - before)
            graph.replay()
        else:
            self.__dict__["_sweep_graph_seen"] = token
            self.__dict__["_sweep_graph"] = None
            enqueue()
        self._pending = {"adaptive": adaptive, "negb": negb, "initial": initial}
        self._safe_dirty = True
        self._refinement = None      # materialised lazily from safe_set (0/1 in this branch)

    def _host_buffers(self):
        """Page-locked landing buffers of the read-backs (safe slab, key + statistics)."""
        n_local = self._end - self._begin
        bufs = self.__dict__.get("_host_bufs")
        if bufs is None or bufs[0].numel() != n_local:
            bufs = (torch.empty(n_local, dtype=torch.uint8).pin_memory(),
                    torch.empty(8, dtype=torch.int64).pin_memory())
            self.__dict__["_host_bufs"] = bufs
        return bufs

    def _resolve_pending(self, host=None):
        """The single host read-back of a sweep (key + statistics, 64 bytes per rank), deferred
        until ``c_max`` / ``last_sweep`` is read.  With several ranks this is a collective (like
        reading ``safe_set``): every rank must read at the same point of the program."""
        pending = self._pending
        if pending is None:
            return
        self._pending = None
        rank, world = dev.dist_info()
        n_total = self.discretization.nindex
        if host is not None:
            pass                            # already on the host (read together with the safe set)
        elif world > 1:
            host = dev.allgather_rows(self._ks_dev).cpu().numpy()
        else:
            host = self._ks_dev.cpu().numpy()[None, :]
        if int(host[0, 3]) == -1:
            raise RuntimeError("peer-memory key exchange timed out: a rank did not take part in "
                               "the sweep (set SLB200_EXCHANGE=nccl to use NCCL instead)")
        key = (int(host[0, 0:1].view(np.uint64)[0]), int(host[0, 1]), int(host[0, 2]))
        n_safe, n_below, max_below, max_all = combine_prefix_stats(host[:, 4:8])
        failed = key[1] != nat.INT64_MAX
        adaptive, negb, initial = pending["adaptive"], pending["negb"], pending["initial"]
        # c_max with the reference's index arithmetic (lyapunov.py:590-595, SURVEY.md Q4)
        if failed:
            position = n_below - 1
        else:
            batch = int(config.gp_batch_size)
            position = ((n_total - 1) // batch) * batch - 1
            if adaptive:
                # lyapunov.py:586-590 with refine_bound: if the last batch holds a cell that only
                # the refinement verified, the index is that of the largest V (rare path: needs ranks)
                values = self._gather(self._values_dev)
                known = negb if initial is None else negb | initial.to(torch.bool)
                known = self._gather(known.to(torch.uint8)).to(torch.bool)
                order = torch.sort(values, stable=True).indices
                if bool((~known[order[position + 1:]]).any()):
                    position = n_total - 1
        if position < 0:
            c_max = _key_to_value(max_all)                  # index -1: largest V on the grid
        elif failed:
            c_max = _key_to_value(max_below)
        else:
            c_max = self._kth_value(position)
        dict.__setitem__(self.feed_dict, self.c_max, c_max)
        self._last_sweep = {"n_safe": n_safe, "first_fail_position": n_below if failed else None,
                            "first_fail_index": key[1] if failed else None, "c_max": c_max}

    @property
    def last_sweep(self):
        self._resolve_pending()
        return self._last_sweep

    @last_sweep.setter
    def last_sweep(self, value):
        self._last_sweep = value

    def _update_adaptive_as_written(self, max_refinement, safety_factor, can_shrink=True):
        """``refinement_mode="reference"``: the adaptive branch exactly as the reference's graph and
        host loop evaluate it (``lyapunov.py:457-481, 540-582``) -- ``refined_safety_check`` builds
        the mesh but compares the OUTER ``decrease`` tensor of every state fed in the slice with
        ``threshold(center, tau / n)``, so a cell counts as verified iff the LARGEST decrease of the
        fed slice is below its own refined threshold, and initial-safe states are re-checked with
        n = 1.  The per-point quantities (``negative``, ``decrease``, the threshold coefficient
        ``-L_V(x)(1 + L_f)``) come from the fused sweep; the batch loop, which depends on
        ``config.gp_batch_size`` and on sorted ranks, is replayed on the host over them, from the
        previous safe set and refinement when ``can_shrink`` is False."""
        lib = nat.load()
        neg, det = self.compute_negative(want_details=True)
        # threshold(x, tau / n) = (-L_V(x) (1 + L_f)) * (tau / n): the coefficient is the sweep's
        # threshold output for tau = 1 (a multiplication by 1.0 is exact)
        n_local = self._end - self._begin
        if self._is_composed():
            grid = self.discretization
            parts = [np.broadcast_to(self.threshold(grid.index_to_state(
                np.arange(s0, min(s0 + (1 << 18), self._end))), 1.0),
                (min(s0 + (1 << 18), self._end) - s0, 1))[:, 0]
                for s0 in range(self._begin, self._end, 1 << 18)]
            coef = dev.to_device(np.concatenate(parts) if parts else np.zeros(0))
        else:
            cfg1 = nat.SlbSweep.from_buffer_copy(self.sweep_descriptor())
            cfg1.tau = 1.0
            coef = dev.empty((n_local,))
            scratch = dev.empty((n_local,), torch.uint8)
            nat.check(lib.slb_lyapunov_sweep(dev.stream(), cfg1, self._begin, self._end,
                                             scratch.data_ptr(), None, None, coef.data_ptr(),
                                             None, None), "slb_lyapunov_sweep")
        values = self._gather(self._values_dev).cpu().numpy()
        negative = self._gather(neg).cpu().numpy().astype(bool)
        decrease = self._gather(det["decrease"]).cpu().numpy()
        threshold = self._gather(det["threshold"]).cpu().numpy()
        coef = self._gather(coef).cpu().numpy()
        n_total = self.discretization.nindex
        initial = np.zeros(n_total, dtype=bool)
        if self.initial_safe_set is not None:
            initial[self.initial_safe_set] = True
        previous = {} if can_shrink else {"safe_set": self.safe_set,
                                          "refinement": np.asarray(self._refinement)}
        safe, refinement, position = adaptive_as_written(
            values, negative, decrease, threshold, coef, initial, self.tau,
            int(config.gp_batch_size), max_refinement, safety_factor, **previous)
        c_max = float(values[np.argsort(values, kind="stable")[position]])
        self._safe_host = safe
        self._safe_dirty = False
        self._safe_dev = dev.to_device(safe[self._begin:self._end].astype(np.uint8), torch.uint8)
        self._refinement = refinement
        self.__dict__["_adaptive_state"] = None
        dict.__setitem__(self.feed_dict, self.c_max, c_max)
        self._last_sweep = {"n_safe": int(safe.sum()), "c_max": c_max,
                            "first_fail_position": position + 1, "first_fail_index": None}

    # _refinement mirrors lyapunov.py:223-225, 531, 586, 601-606; without adaptive refinement
    # it is 1 exactly where the state is safe.
    @property
    def _refinement(self):
        if self.__dict__.get("_refinement_host") is None:
            safe = self.safe_set
            refinement = safe.astype(int)
            state = self.__dict__.get("_adaptive_state")
            if state is not None:     # N(x) = n_req where the refined mesh verified the cell
                n_req = self._gather(state[0]).cpu().numpy()
                negative = self._gather(state[1].to(torch.uint8)).cpu().numpy().astype(bool)
                refinement = np.where(safe & ~negative, n_req, refinement)
                if self.initial_safe_set is not None:
                    refinement[self.initial_safe_set] = 1
            self.__dict__["_refinement_host"] = refinement
        return self.__dict__["_refinement_host"]

    @_refinement.setter
    def _refinement(self, value):
        self.__dict__["_refinement_host"] = value

    def _kth_value(self, position):
        """V at sorted position `position` (only reached when no point fails)."""
        values = self._gather(self._values_dev)
        return float(torch.kthvalue(values, position + 1).values.item())

    def _update_no_shrink(self, max_refinement, safety_factor, initial):
        """``can_shrink=False`` (``lyapunov.py:497-606`` with ``:507-510, :540-587``; SURVEY.md Q3):
        the previous safe set and refinement seed the result and the batch size decides which
        trailing states keep their old label, so this mode needs sorted ranks -- a stable device
        sort (torch), single GPU.  ``slb_no_shrink_scan`` finds each batch's first unverified
        position and marks the cells whose refined check can still matter; the mesh checks run on
        those only (``max_refinement > 1``); ``slb_no_shrink_resolve`` replays the loop's outcome
        in grid order.  One read-back at the end; no host loop over batches."""
        lib = nat.load()
        n = self._end - self._begin
        batch = int(config.gp_batch_size)
        if max_refinement > 1:
            neg, det = self.compute_negative(want_details=True)
            n_req = self._required_refinement(det, safety_factor)
        else:
            neg, n_req = self.compute_negative(), None
        values = self._values_dev
        order = torch.sort(values, stable=True).indices
        prev = dev.to_device(self.safe_set.astype(np.uint8), torch.uint8)
        refine_prev = dev.to_device(np.asarray(self._refinement, dtype=np.int64), torch.int64)
        workspace = dev.empty((int(lib.slb_no_shrink_workspace(n, batch)) // 8,), torch.int64)
        cand = dev.empty((n,), torch.bool)
        refined = dev.zeros((n,), torch.bool)
        nat.check(lib.slb_no_shrink_scan(dev.stream(), order.data_ptr(), neg.data_ptr(),
                                         prev.data_ptr(), dev.ptr(initial), dev.ptr(n_req), n,
                                         batch, max_refinement, workspace.data_ptr(),
                                         cand.data_ptr()), "slb_no_shrink_scan")
        if max_refinement > 1:
            self._refined_mesh_check(cand, n_req, max_refinement, refined)
        # written in place: a captured sweep graph of can_shrink=True holds this buffer's address
        if self._safe_dev is None or self._safe_dev.numel() != n:
            self._safe_dev = dev.empty((n,), torch.uint8)
        safe = self._safe_dev
        refinement = dev.empty((n,), torch.int64)
        result = dev.empty((2,), torch.int64)          # [c_max position, c_max bits]
        nat.check(lib.slb_no_shrink_resolve(dev.stream(), order.data_ptr(), values.data_ptr(),
                                            neg.data_ptr(), prev.data_ptr(),
                                            refine_prev.data_ptr(), dev.ptr(initial),
                                            dev.ptr(n_req), refined.data_ptr(), n, batch,
                                            max_refinement, workspace.data_ptr(),
                                            safe.data_ptr(), refinement.data_ptr(),
                                            result[0:1].data_ptr(), result[1:2].data_ptr()),
                  "slb_no_shrink_resolve")
        host = self.__dict__.get("_no_shrink_bufs")
        if host is None or host[0].numel() != n:
            host = (torch.empty((n,), dtype=torch.uint8).pin_memory(),
                    torch.empty((n,), dtype=torch.int64).pin_memory(),
                    torch.empty((2,), dtype=torch.int64).pin_memory())
            self.__dict__["_no_shrink_bufs"] = host
        for dst, src in zip(host, (safe, refinement, result)):
            dst.copy_(src, non_blocking=True)
        torch.cuda.current_stream().synchronize()
        self._safe_host = host[0].numpy().astype(bool)
        self._safe_dirty = False
        self._refinement = host[1].numpy().astype(int)
        self.__dict__["_adaptive_state"] = None
        c_max = float(host[2].numpy()[1:2].view(np.float64)[0])
        dict.__setitem__(self.feed_dict, self.c_max, c_max)
