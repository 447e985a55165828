"""CPU tests of the GP posterior mean as a deterministic function (``PosteriorMean``,
``gp.to_mean_function()``): the reference's ``to_mean_function`` semantics, the object's dimensions and
version, which closed loops the rollout kernels fuse, ``Lyapunov`` choosing the composed path, the host
checks of ``slb_gp_mean`` / ``slb_rollout_gp_mean`` / ``slb_reward_rollout_gp_mean`` (fake, never
dereferenced device pointers), and ``compute_trajectory``'s host loop against the reference's."""
import ctypes as C
import os
import sys

import numpy as np
import pytest

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)

import safe_learning_b200 as sl  # noqa: E402
from safe_learning_b200 import _native as nat  # noqa: E402
from safe_learning_b200.utilities import compute_trajectory  # noqa: E402


def _has_gpu():
    try:
        import torch
        return torch.cuda.is_available()
    except Exception:  # pragma: no cover
        return False


def _gp(din=3, M=5, seed=0):
    rng = np.random.default_rng(seed)
    kern = sl.RBF(din, variance=1.0, lengthscales=[1.0] * din)
    return sl.GaussianProcess(sl.GPRCached(rng.uniform(-1, 1, (M, din)), rng.standard_normal((M, 1)),
                                           kern, noise_variance=1e-2))


# ---------------------------------------------------------------- the object
def test_mean_function_of_any_uncertain_function():
    """The reference's test_mean_function (tests/test_functions.py:142-147): the first output."""
    class Pair(sl.UncertainFunction):
        def __call__(self, *points):
            return 1, 2
    fd = Pair().to_mean_function()
    assert fd(None) == 1
    assert not isinstance(fd, sl.PosteriorMean)


def test_posterior_mean_dimensions_and_type():
    gp = _gp()
    pm = gp.to_mean_function()
    assert isinstance(pm, sl.PosteriorMean) and isinstance(pm, sl.DeterministicFunction)
    assert pm.input_dim == 3 and pm.output_dim == 1
    assert pm.gaussian_process is gp
    stack = sl.FunctionStack([_gp(seed=1), _gp(seed=2)])
    pms = stack.to_mean_function()
    assert isinstance(pms, sl.PosteriorMean)
    assert pms.input_dim == 3 and pms.output_dim == 2
    with pytest.raises(NotImplementedError):
        pm.descriptor()                      # fused as dynamics only, never through a descriptor
    with pytest.raises(TypeError):
        sl.PosteriorMean(sl.LinearSystem(np.eye(2)))


def test_posterior_mean_version_follows_the_gp():
    gp = _gp()
    model = gp.gaussian_process
    model._ensure = lambda: None             # no factorisation (no device): the version counter only
    pm = gp.to_mean_function()
    v0 = pm.version
    assert v0 == gp.version
    model._version += 1                      # what add_data_point's refactorisation does
    assert pm.version != v0 and pm.version == gp.version


# ---------------------------------------------------------------- fusion rules
def _policy():
    return sl.Saturation(sl.LinearSystem((-np.array([[0.5, 0.2]]),)), -1., 1.)


def test_closed_loop_fusion_rules():
    stack = sl.FunctionStack([_gp(seed=1), _gp(seed=2)])
    policy = _policy()
    cl = sl.ClosedLoop(stack.to_mean_function(), policy)
    assert cl.fused and cl.gp_mean
    with pytest.raises(TypeError):
        sl.ClosedLoop(stack, policy)                         # (mean, error): no closed loop
    assert not sl.ClosedLoop(stack.to_mean_function(), lambda x: x[:, :1]).fused
    # the mean as a policy: not fused
    pol_gp = sl.GaussianProcess(sl.GPRCached(np.zeros((2, 2)), np.zeros((2, 1)), sl.RBF(2)))
    assert not sl.ClosedLoop(sl.LinearSystem((np.eye(2), np.ones((2, 1)))), pol_gp.to_mean_function()).fused
    # the mean as a reward: the ClosedLoop is fused, reward_rollout still takes the host loop
    rw = sl.ClosedLoop(_gp(seed=3).to_mean_function(), policy)
    assert rw.gp_mean


def test_reward_on_posterior_mean_takes_the_host_loop(monkeypatch):
    """A PosteriorMean as the reward sends reward_rollout to the host loop (no kernel is called)."""
    import safe_learning_b200.rollout as ro
    calls = []
    monkeypatch.setattr(ro, "_reward_rollout_host", lambda *a: calls.append(a) or np.zeros(a[1]))
    policy = _policy()
    cl = sl.ClosedLoop(sl.LinearSystem((np.eye(2), np.ones((2, 1)))), policy)
    rw = sl.ClosedLoop(_gp(seed=3).to_mean_function(), policy)
    sl.reward_rollout(np.zeros((4, 2)), cl, rw, 0.9, 5)
    assert len(calls) == 1


def test_lyapunov_with_posterior_mean_is_composed():
    stack = sl.FunctionStack([_gp(seed=1), _gp(seed=2)])
    lyap = sl.Lyapunov.__new__(sl.Lyapunov)          # the members only: no sweep is built
    lyap.policy, lyap.lyapunov_function = _policy(), sl.QuadraticFunction(np.eye(2))
    lyap._lipschitz_lyapunov = 1.0
    lyap.dynamics = stack.to_mean_function()
    assert lyap._is_composed()
    lyap.dynamics = stack
    assert not lyap._is_composed()


# ---------------------------------------------------------------- C entry points
def test_new_symbols_exported():
    lib = nat.load()
    for name in ("slb_gp_mean", "slb_rollout_gp_mean", "slb_reward_rollout_gp_mean"):
        assert name in nat.SIGNATURES
        assert getattr(lib, name) is not None


def _gp_cfg(d=2, m=1, M=9):
    """A closed loop on the GP mean with fake (never dereferenced) device pointers."""
    cfg = nat.SlbBellman()
    cfg.grid.ndim, cfg.grid.nindex = d, 9 ** d
    for c in range(d):
        cfg.grid.num_points[c], cfg.grid.unit_maxes[c] = 9, 0.25
    cfg.policy.kind, cfg.policy.in_dim, cfg.policy.out_dim = nat.FN_LINEAR, d, m
    cfg.policy.matrix = 0x1000
    cfg.reward.kind, cfg.reward.in_dim, cfg.reward.out_dim = nat.FN_QUADRATIC, d + m, 1
    cfg.reward.matrix = 0x3000
    gp = cfg.gp
    gp.num_outputs, gp.num_factors, gp.input_dim = d, 1, d + m
    F = gp.factors[0]
    F.M, F.nrb, F.Xs, F.Wpack, F.Xf = M, (M + 7) // 8, 0x10000, 0x20000, 0x30000
    F.scale, F.variance = 1.0, 1.0
    for c in range(nat.SLB_MAX_IN):
        F.lengthscales[c] = 1.0
    for o in range(d):
        gp.outputs[o].factor = 0
        gp.outputs[o].alpha = 0x40000 + 0x1000 * o
        gp.outputs[o].gamma_f = 0x50000 + 0x1000 * o
    return cfg


def _call_reward(lib, cfg, horizon=10, n=81):
    return lib.slb_reward_rollout_gp_mean(None, cfg, None, 0, n, horizon, C.c_void_p(0x4000), 1e-3,
                                          C.c_void_p(0x5000), C.c_void_p(0x6000), C.c_void_p(0x7000))


def _call_roa(lib, cfg, horizon=10, n=81):
    eq = (C.c_double * cfg.grid.ndim)()
    return lib.slb_rollout_gp_mean(None, cfg, None, 0, n, horizon, eq, 1e-3, C.c_void_p(0x10), None, None,
                                   C.c_void_p(0x8000))


def _d_in_7(c):
    c.grid.ndim, c.grid.nindex = 6, 9 ** 6
    for k in range(6):
        c.grid.num_points[k], c.grid.unit_maxes[k] = 9, 0.25
    c.policy.in_dim = 6
    c.reward.in_dim = 7
    c.gp.num_outputs, c.gp.input_dim = 6, 7
    for o in range(6):
        c.gp.outputs[o].factor = 0
        c.gp.outputs[o].alpha = 0x40000 + 0x1000 * o
        c.gp.outputs[o].gamma_f = 0x50000 + 0x1000 * o


@pytest.mark.parametrize("mutate, message", [
    (lambda c: setattr(c.gp, "num_outputs", 1), "outputs but the state has"),
    (lambda c: setattr(c.gp, "num_outputs", 0), "outputs but the state has"),
    (lambda c: setattr(c.gp, "input_dim", 4), "GP input_dim 4 != state 2 + action 1"),
    (lambda c: setattr(c.dynamics, "kind", nat.FN_LINEAR) or setattr(c.dynamics, "in_dim", 3)
     or setattr(c.dynamics, "out_dim", 2), "dynamics.kind must be SLB_FN_NONE"),
    (lambda c: setattr(c.gp.factors[0], "Xf", None), "staged table Xf"),
    (lambda c: setattr(c.gp.factors[0], "Xf", 0x30008), "staged table Xf"),
    (lambda c: setattr(c.gp.outputs[1], "gamma_f", None), "staged table gamma_f"),
    (lambda c: setattr(c, "fixed_action", 1), "fixed_action"),
    (_d_in_7, "GP input_dim 7 not compiled"),
])
@pytest.mark.parametrize("which", ["roa", "reward"])
def test_gp_mean_rollouts_reject_malformed_descriptors(mutate, message, which):
    """Rejected by host-side checks before any launch (no device needed), the reason in slb_last_error."""
    lib = nat.load()
    cfg = _gp_cfg()
    mutate(cfg)
    rc = _call_roa(lib, cfg) if which == "roa" else _call_reward(lib, cfg)
    assert rc == 1 and message in nat.last_error(), nat.last_error()


def test_gp_mean_rollouts_reject_a_negative_horizon():
    lib = nat.load()
    cfg = _gp_cfg()
    for rc in (_call_roa(lib, cfg, horizon=-1), _call_reward(lib, cfg, horizon=-1)):
        assert rc == 1 and "negative horizon" in nat.last_error()


def test_existing_rollouts_still_reject_gp_stacks():
    lib = nat.load()
    cfg = _gp_cfg()
    eq = (C.c_double * 2)()
    rc = lib.slb_rollout(None, cfg, None, 0, 81, 10, eq, 1e-3, C.c_void_p(0x10), None, None, C.c_void_p(0x8000))
    assert rc == 1 and "GP dynamics cannot be rolled out" in nat.last_error()


def test_gp_mean_rollouts_workspace_and_empty_calls():
    lib = nat.load()
    cfg = _gp_cfg()
    assert lib.slb_rollout_workspace(cfg, 1000, 0) >= 2 * 1000 * 2 * 8
    eq = (C.c_double * 2)()
    assert lib.slb_rollout_gp_mean(None, cfg, None, 0, 0, 5, eq, 1e-3, None, None, None, None) == 0


def test_slb_gp_mean_host_checks():
    lib = nat.load()
    cfg = _gp_cfg()
    gp = cfg.gp
    rc = lib.slb_gp_mean(None, gp, C.c_void_p(0x10), -1, C.c_void_p(0x20))
    assert rc == 1 and "negative n" in nat.last_error()
    rc = lib.slb_gp_mean(None, gp, None, 5, C.c_void_p(0x20))
    assert rc == 1 and "null buffer" in nat.last_error()
    rc = lib.slb_gp_mean(None, gp, C.c_void_p(0x10), 5, None)
    assert rc == 1 and "null buffer" in nat.last_error()
    gp.factors[0].Xf = None
    rc = lib.slb_gp_mean(None, gp, C.c_void_p(0x10), 5, C.c_void_p(0x20))
    assert rc == 1 and "staged table Xf" in nat.last_error()
    gp.factors[0].Xf = 0x30000
    gp.input_dim = 7
    rc = lib.slb_gp_mean(None, gp, C.c_void_p(0x10), 5, C.c_void_p(0x20))
    assert rc == 1 and "not compiled" in nat.last_error()
    gp.input_dim = 3
    gp.num_outputs = 0
    rc = lib.slb_gp_mean(None, gp, C.c_void_p(0x10), 5, C.c_void_p(0x20))
    assert rc == 1 and "no outputs" in nat.last_error()
    gp.num_outputs = 2
    assert lib.slb_gp_mean(None, gp, None, 0, None) == 0            # n = 0: nothing to do


@pytest.mark.skipif(_has_gpu(), reason="checks the no-device error")
def test_no_device_raises():
    gp = _gp()
    pm = gp.to_mean_function()
    with pytest.raises(nat.NativeLibraryError):
        pm(np.zeros((4, 3)))
    with pytest.raises(nat.NativeLibraryError):
        sl.compute_roa(np.zeros((3, 2)), sl.ClosedLoop(sl.FunctionStack([_gp(seed=1), _gp(seed=2)])
                                                       .to_mean_function(), _policy()), 10)


# ---------------------------------------------------------------- compute_trajectory, host loop
def _reference_trajectory(dynamics, policy, initial_state, num_steps, action_dim):
    """utilities.py:519-583 with numpy callables in place of the session."""
    initial_state = np.atleast_2d(initial_state)
    states = np.empty((num_steps, initial_state.shape[1]))
    actions = np.empty((num_steps - 1, action_dim))
    states[0, :] = initial_state
    for i in range(num_steps - 1):
        a = policy(states[[i], :])
        states[i + 1, :], actions[i, :] = dynamics(states[[i], :], a), a
    return states, actions


class _Callable(object):
    def __init__(self, fun, output_dim):
        self.fun, self.output_dim = fun, output_dim

    def __call__(self, *args):
        return self.fun(*args)


@pytest.mark.parametrize("num_steps", [1, 2, 3, 20])
def test_compute_trajectory_host_loop(num_steps):
    A = np.array([[1., 0.1], [0., 1.]])
    B = np.array([[0.01], [0.1]])
    K = np.array([[0.8, 1.1]])
    dyn = _Callable(lambda x, u: x.dot(A.T) + np.atleast_2d(u).dot(B.T), 2)
    pol = _Callable(lambda x: np.tanh(-x.dot(K.T)), 1)
    x0 = np.array([[0.1, -0.05]])
    states, actions = compute_trajectory(dyn, pol, x0, num_steps)
    ref_s, ref_a = _reference_trajectory(dyn, pol, x0, num_steps, 1)
    assert states.shape == (num_steps, 2) and actions.shape == (num_steps - 1, 1)
    assert np.array_equal(states, ref_s) and np.array_equal(actions, ref_a)
    assert np.array_equal(states[0], x0[0])
    assert sl.compute_trajectory is compute_trajectory


def test_compute_trajectory_zero_steps_raises_like_the_reference():
    """num_steps = 0: the reference's np.empty((num_steps - 1, m)) raises ValueError."""
    dyn = _Callable(lambda x, u: x, 2)
    pol = _Callable(lambda x: x[:, :1], 1)
    with pytest.raises(ValueError):
        _reference_trajectory(dyn, pol, np.zeros(2), 0, 1)
    with pytest.raises(ValueError):
        compute_trajectory(dyn, pol, np.zeros(2), 0)


# ---------------------------------------------------------------- the reference's fixture, numpy oracle
@pytest.mark.parametrize("tag", ["s1", "s2"])
def test_fixture_against_the_numpy_oracle(tag):
    """tests/golden/gp_mean.npz (the unmodified reference's to_mean_function() rollouts): the numpy
    oracle's GP, rebuilt from the fixture's samples and hyper-parameters, reproduces the one-step means and,
    through the reference's loop, the 40-step end states -- the parameters round-trip and the fixture
    means what the GPU test takes it to mean."""
    import oracle as O
    sys.path.insert(0, os.path.dirname(HERE))
    import bench_workloads as W
    g = np.load(os.path.join(HERE, "golden", "gp_mean.npz"))
    keys = ("X", "Y", "variances", "lengthscales", "noise_variance", "beta", "scale", "prior_rows", "K",
            "limits")
    par = {k: g[tag + "_" + k] for k in keys}
    for k in ("noise_variance", "beta", "scale"):
        par[k] = float(par[k])
    par["num_points"] = [2, 2]                       # the builder's grid, unused here
    _, stack = W._build(O, par, "oracle")
    mean = np.asarray(stack(g[tag + "_points"])[0])
    np.testing.assert_allclose(mean, g[tag + "_mean"], rtol=1e-12, atol=1e-14)
    policy = O.Saturation(O.LinearSystem(-par["K"]), -1., 1.)
    x = g[tag + "_states"]
    for _ in range(1, 40):
        x = np.asarray(stack(np.hstack((x, policy(x))))[0])
    np.testing.assert_allclose(x, g[tag + "_states_h40_end"], rtol=1e-9, atol=1e-12)
