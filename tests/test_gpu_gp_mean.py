"""GPU tests of the GP posterior mean as a deterministic function (``gp.to_mean_function()``,
``PosteriorMean``): the one-step mean ``slb_gp_mean`` against an extended-precision reference of its
own form with a computed bound (tests/gp_mean_reference.py), the rollouts of the mean model against h
compositions of one-step evaluations (bit for bit), ``PolicyIteration`` and ``Lyapunov`` with mean-model
dynamics, the autograd node, ``compute_trajectory`` and data updates."""
import os
import sys

import numpy as np
import pytest
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
sys.path.insert(0, os.path.dirname(HERE))

import bench_workloads as W  # noqa: E402
import gp_mean_reference as GM  # noqa: E402
import oracle as O  # noqa: E402
import gp_posterior_reference as GR  # noqa: E402
import safe_learning_b200 as sl  # noqa: E402
from safe_learning_b200 import _device as dev  # noqa: E402
from safe_learning_b200 import _native as nat  # noqa: E402

pytestmark = pytest.mark.gpu


# ---------------------------------------------------------------- models
def _stack(din, Ms, kind="rbf", prior=True, shared=False, seed=0):
    """A FunctionStack of len(Ms) one-output GPs on d_in inputs; `shared`: the first two members share
    their data and hyper-parameters (one factor)."""
    rng = np.random.default_rng(seed)
    gps = []
    X0 = None
    for o, M in enumerate(Ms):
        X = rng.uniform(-1, 1, (M, din))
        if shared and o == 1:
            X = X0
        X0 = X if o == 0 else X0
        Y = np.sin(2 * X.sum(axis=1, keepdims=True) + o) + 0.01 * rng.standard_normal((X.shape[0], 1))
        if kind == "rbf":
            ls = [1.0 + 0.1 * c for c in range(din)]
            var = 0.7 if (shared and o <= 1) else 0.5 + 0.1 * o
            kern = sl.RBF(din, variance=var, lengthscales=ls)
        else:                                              # the notebooks' expression (d_in = 3)
            var = np.abs(rng.uniform(0.1, 1.0, din))
            kern = W.build_kernel(sl, W.notebook_pendulum_kernels([var])[0])
        mean = sl.LinearSystem(rng.uniform(-0.5, 0.5, (1, din))) if prior else None
        gps.append(sl.GaussianProcess(sl.GPRCached(X, Y, kern, mean_function=mean, noise_variance=1e-2)))
    return sl.FunctionStack(gps)


def _query(din, n, rng):
    return rng.uniform(-1.3, 1.3, (n, din))


# ---------------------------------------------------------------- 1. one-step accuracy
CASES = [(din, Ms, kind, prior, shared)
         for din in (2, 3, 4, 5, 6)
         for (Ms, kind, prior, shared) in [
             ((0,), "rbf", True, False), ((1,), "rbf", False, False), ((7, 8), "rbf", True, False),
             ((9, 255, 0), "rbf", True, False), ((256, 256, 257), "rbf", False, True),
             ((513,), "rbf", True, False), ((40, 40, 12, 7, 1, 9), "rbf", True, True)]]
CASES += [(3, Ms, "expr", prior, False) for Ms, prior in [((8, 9), True), ((255,), False), ((257, 0), True),
                                                           ((513, 40), False)]]


@pytest.mark.parametrize("din, Ms, kind, prior, shared", CASES)
def test_one_step_mean_within_its_bound(din, Ms, kind, prior, shared):
    stack = _stack(din, Ms, kind, prior, shared, seed=din * 100 + len(Ms))
    pm = stack.to_mean_function()
    z = _query(din, 300, np.random.default_rng(din))
    got = pm(z)
    assert got.shape == (300, len(Ms))
    assert np.array_equal(pm.evaluate_device(z).cpu().numpy(), got)
    tables = GM.staged_tables(stack)
    mean, bound = GM.reference(tables, z)
    assert GM.ratio(got, mean, bound) <= 1.0
    # mutations: a dropped row, two outputs' weights swapped -- each far outside the bound
    if Ms[0] >= 1:
        m_mean, _ = GM.reference(tables, z, "drop_row")
        assert GM.ratio(got, m_mean, bound) >= 10.0
    if len(Ms) >= 2 and Ms[0] == Ms[1] and Ms[0] >= 1:
        m_mean, _ = GM.reference(tables, z, "swap_gamma")
        assert GM.ratio(got, m_mean, bound) >= 10.0
    # and within that bound plus the full posterior's own bound of gp(z)[0]
    full, _ = stack(z)
    ref_full = GR.reference(GR.stack_tables(stack), z)
    total = bound.astype(np.float64) + ref_full["mean_bound"] + GM.gamma_gap_bound(tables, z)
    assert np.all(np.abs(got - full) <= total)


def test_one_step_mean_independent_of_position_and_count():
    stack = _stack(3, (300, 70), seed=3)
    pm = stack.to_mean_function()
    z = _query(3, 1000, np.random.default_rng(1))
    full = pm(z)
    for lo, hi in ((0, 1), (5, 6), (0, 257), (123, 1000), (999, 1000)):
        assert np.array_equal(pm(z[lo:hi]), full[lo:hi])
    assert np.array_equal(pm(z[::-1])[::-1], full)
    assert pm(np.zeros((0, 3))).shape == (0, 2)


# ---------------------------------------------------------------- 2. rollouts, bit for bit
def _pendulum(M=60, seed=1):
    par = W.make_pendulum(num_points=8, M=M, seed=seed)
    _, dynamics = W._build(sl, par, "product")
    policy = sl.Saturation(sl.LinearSystem(-par["K"]), -1., 1.)
    return par, dynamics, policy


def _compose(cl, x, steps):
    """[n, d, steps + 1]: x and `steps` compositions of the one-step evaluation."""
    out = [dev.to_device(x)]
    for _ in range(steps):
        out.append(cl.evaluate_device(out[-1]))
    return torch.stack(out, dim=2).cpu().numpy()


@pytest.mark.parametrize("n", [1, 63, 64, 65, 257, 10001])
def test_roa_trajectories_equal_one_step_compositions(n):
    par, dynamics, policy = _pendulum()
    cl = sl.ClosedLoop(dynamics.to_mean_function(), policy)
    assert cl.fused
    x = np.random.default_rng(n).uniform(-1, 1, (n, 2))
    ref = _compose(cl, x, 99)
    for horizon in (1, 2, 32, 33, 34, 100):
        roa, traj = sl.compute_roa(x, cl, horizon, 0.1, no_traj=False)
        assert np.array_equal(traj, ref[:, :, :horizon])
        end = ref[:, :, horizon - 1]
        assert np.array_equal(roa, np.linalg.norm(end, 2, axis=1) <= 0.1)
        assert np.array_equal(sl.compute_roa(x, cl, horizon, 0.1), roa)


def test_roa_grid_starts_and_index_ranges():
    par, dynamics, policy = _pendulum()
    cl = sl.ClosedLoop(dynamics.to_mean_function(), policy)
    grid = sl.GridWorld(par["limits"], [37, 29])
    pts = grid.all_points
    ref = _compose(cl, pts, 40)
    roa, traj = sl.compute_roa(grid, cl, 41, 0.05, no_traj=False)
    assert np.array_equal(traj, ref)
    assert np.array_equal(roa, np.linalg.norm(ref[:, :, -1], 2, axis=1) <= 0.05)
    # an index range [lo, hi) of the grid through the C entry point
    lib = nat.load()
    cfg = sl.rollout._descriptor(grid, 2, cl)
    lo, hi = 300, 777
    n = hi - lo
    flags = dev.empty((n,), torch.uint8)
    ends = dev.empty((n, 2))
    work = dev.empty((int(lib.slb_rollout_workspace(cfg, n, 0)) // 8 + 1,))
    eq = np.zeros(2)
    nat.check(lib.slb_rollout_gp_mean(dev.stream(), cfg, None, lo, n, 41, eq.ctypes.data, 0.05,
                                      flags.data_ptr(), ends.data_ptr(), None, work.data_ptr()), "roll")
    assert np.array_equal(ends.cpu().numpy(), ref[lo:hi, :, -1])
    assert np.array_equal(flags.cpu().numpy().astype(bool), roa[lo:hi])


def _reward_loop(cl, rw, x, discount, horizon, tol):
    """examples/utilities.py:531-545 over device one-step evaluations."""
    sums = np.zeros(x.shape[0])
    cur = dev.to_device(x)
    for t in range(horizon):
        temp = (discount ** t) * rw.evaluate_device(cur).cpu().numpy().ravel()
        sums += temp
        if np.max(np.abs(temp)) < tol:
            return sums, t
        cur = cl.evaluate_device(cur)
    return sums, -1


@pytest.mark.parametrize("n, horizon, tol", [(1, 40, 1e-3), (65, 100, 1e-4), (257, 70, 0.0),
                                             (10001, 150, 1e-5)])
def test_reward_rollout_equals_the_stopping_loop(n, horizon, tol, capsys):
    par, dynamics, policy = _pendulum()
    cl = sl.ClosedLoop(dynamics.to_mean_function(), policy)
    rw = sl.ClosedLoop(sl.QuadraticFunction(-np.diag([1., 2., 1.2])), policy)
    x = np.random.default_rng(n).uniform(-1, 1, (n, 2))
    sums = sl.reward_rollout(x, cl, rw, 0.95, horizon, tol)
    ref, stop = _reward_loop(cl, rw, x, 0.95, horizon, tol)
    assert np.array_equal(sums, ref)
    out = capsys.readouterr().out
    assert ("after {} steps".format(stop + 1) in out) if stop >= 0 else ("did not converge" in out)


# ---------------------------------------------------------------- 4. M = 0: the prior mean
def test_empty_model_rolls_out_its_prior_mean():
    rng = np.random.default_rng(0)
    A = np.array([[1., 0.05], [-0.1, 0.98]])
    B = np.array([[0.0], [0.05]])
    rows = np.hstack((A, B))
    gps = [sl.GaussianProcess(sl.GPRCached(np.zeros((0, 3)), np.zeros((0, 1)), sl.RBF(3),
                                           mean_function=sl.LinearSystem(rows[[j]]), noise_variance=1e-2))
           for j in range(2)]
    policy = sl.Saturation(sl.LinearSystem(-np.array([[0.5, 0.8]])), -1., 1.)
    cl_gp = sl.ClosedLoop(sl.FunctionStack(gps).to_mean_function(), policy)
    cl_lin = sl.ClosedLoop(sl.LinearSystem((A, B)), policy)
    x = rng.uniform(-1, 1, (500, 2))
    _, t_gp = sl.compute_roa(x, cl_gp, 50, 0.1, no_traj=False)
    _, t_lin = sl.compute_roa(x, cl_lin, 50, 0.1, no_traj=False)
    np.testing.assert_allclose(t_gp, t_lin, rtol=1e-12, atol=1e-14)


# ---------------------------------------------------------------- 5. PolicyIteration
def _rl(dynamics, policy, grid, value0):
    reward = sl.QuadraticFunction(-np.diag([1., 2., 1.2]))
    value = sl.Triangulation(grid, value0.copy(), project=True)
    return sl.PolicyIteration(policy, dynamics, reward, value, gamma=0.9)


def test_policy_iteration_with_the_mean_equals_the_gp():
    par, dynamics, policy = _pendulum(M=80)
    grid = sl.GridWorld(par["limits"], 21)
    v0 = -np.random.default_rng(2).random((grid.nindex, 1))
    rl_gp = _rl(dynamics, policy, grid, v0)
    rl_pm = _rl(dynamics.to_mean_function(), policy, grid, v0)
    for _ in range(3):
        expect = rl_pm.future_values(rl_pm.state_space)
        a = rl_gp.value_iteration()
        b = rl_pm.value_iteration()
        assert a == b
        table = rl_pm.value_function.parameters[0]
        assert np.array_equal(rl_gp.value_function.parameters[0], table)
        assert np.array_equal(table, expect)          # the mean model: the sweep is future_values
    # greedy policies, both paths of the argmax
    actions = np.linspace(-1, 1, 9)[:, None]
    for factor in (True, False):
        pols = []
        for dyn in (dynamics, dynamics.to_mean_function()):
            rl = sl.PolicyIteration(sl.Triangulation(grid, np.zeros((grid.nindex, 1))), dyn,
                                    sl.QuadraticFunction(-np.diag([1., 2., 1.2])),
                                    sl.Triangulation(grid, v0.copy(), project=True), gamma=0.9)
            rl.factor_actions = factor
            pols.append(rl.discrete_policy_optimization(actions).cpu().numpy())
        assert np.array_equal(pols[0], pols[1])
    # exact policy evaluation
    vals = []
    for dyn in (dynamics, dynamics.to_mean_function()):
        rl = _rl(dyn, policy, grid, v0)
        vals.append(rl.optimize_value_function())
    assert np.array_equal(vals[0], vals[1])


# ---------------------------------------------------------------- 6. autograd
def test_torch_node_forward_backward():
    stack = _stack(3, (120, 90), seed=7)
    pm = stack.to_mean_function()
    z = dev.to_device(_query(3, 64, np.random.default_rng(3)))
    zr = z.clone().requires_grad_(True)
    out = pm.torch(zr)
    assert torch.equal(out.detach(), pm.evaluate_device(z))
    cot = dev.to_device(np.random.default_rng(4).standard_normal((64, 2)))
    (g_pm,) = torch.autograd.grad(out, zr, cot)
    zg = z.clone().requires_grad_(True)
    mean, _ = stack.torch(zg)
    (g_gp,) = torch.autograd.grad(mean, zg, cot)
    assert torch.equal(g_pm, g_gp)
    # central differences of the mean form itself
    h = 1e-6
    zn = z.cpu().numpy()
    fd = np.zeros_like(zn)
    for c in range(3):
        e = np.zeros(3)
        e[c] = h
        fd[:, c] = ((pm(zn + e) - pm(zn - e)) / (2 * h) * cot.cpu().numpy()).sum(axis=1)
    np.testing.assert_allclose(g_pm.cpu().numpy(), fd, rtol=1e-6, atol=1e-7)
    jac = pm.jacobian_device(z).cpu().numpy()
    np.testing.assert_allclose(np.einsum("no,noi->ni", cot.cpu().numpy(), jac), g_pm.cpu().numpy(),
                               rtol=1e-13, atol=1e-15)


def test_future_values_differentiates_with_mean_dynamics():
    par, dynamics, policy = _pendulum(M=80)
    grid = sl.GridWorld(par["limits"], 15)
    v0 = -np.random.default_rng(2).random((grid.nindex, 1))
    rl = _rl(dynamics.to_mean_function(), policy, grid, v0)
    lyap = sl.Lyapunov(grid, sl.QuadraticFunction(par["P"]), dynamics.to_mean_function(), par["L_dyn"],
                       sl.AbsFunction(sl.LinearSystem((2 * par["P"],))), par["tau"], policy,
                       initial_set=None)
    states = dev.to_device(np.random.default_rng(5).uniform(-0.8, 0.8, (50, 2)))
    actions = dev.to_device(np.random.default_rng(6).uniform(-1, 1, (50, 1))).requires_grad_(True)
    out = rl.future_values(states, actions=actions)
    ref = rl.future_values(states.cpu().numpy(), actions=actions.detach().cpu().numpy())
    assert np.array_equal(out.detach().cpu().numpy(), ref)
    out = rl.future_values(states, actions=actions, lyapunov=lyap)
    (g,) = torch.autograd.grad(out.sum(), actions)
    # each point's value depends on its own action only: central differences of the forward, all points
    # at once (V and the decrease are smooth here; a kink of the value Triangulation inside +-h is unlikely)
    h = 1e-6
    a = actions.detach()
    up = rl.future_values(states, actions=a + h, lyapunov=lyap).detach()
    down = rl.future_values(states, actions=a - h, lyapunov=lyap).detach()
    fd = ((up - down) / (2 * h)).cpu().numpy()
    np.testing.assert_allclose(g.cpu().numpy(), fd, rtol=1e-5, atol=1e-7)


# ---------------------------------------------------------------- 7. Lyapunov
def test_lyapunov_with_mean_dynamics_equals_the_oracle():
    """The composed path with the mean on the device against the numpy oracle's Lyapunov (the reference's
    host loop, deterministic dynamics) fed the same one-step means: no decision may lie within a relative
    margin of its threshold (counted and reported), then the safe set is equal and c_max agrees to the
    rounding of V, evaluated on the GPU here and in numpy there."""
    par, dynamics, policy = _pendulum(M=80)
    grid = sl.GridWorld(par["limits"], 41)
    pm = dynamics.to_mean_function()
    init = np.linalg.norm(grid.all_points, 2, axis=1) <= 0.2
    lyap = sl.Lyapunov(grid, sl.QuadraticFunction(par["P"]), pm, par["L_dyn"],
                       sl.AbsFunction(sl.LinearSystem((2 * par["P"],))), par["tau"], policy, initial_set=init)
    assert lyap._is_composed()
    o_policy = O.Saturation(O.LinearSystem((-par["K"],)), -1., 1.)
    oracle = O.Lyapunov(O.GridWorld(par["limits"], 41), O.QuadraticFunction(par["P"]),
                        lambda x, u: pm(x, u), par["L_dyn"], O.AbsFunction(O.LinearSystem((2 * par["P"],))),
                        par["tau"], o_policy, initial_set=init)
    decrease, threshold = oracle.decrease_and_threshold(grid.all_points)
    near = np.abs(decrease - threshold) <= 1e-10 * (np.abs(decrease) + np.abs(threshold))
    print("decisions within the margin: %d" % near.sum())
    assert near.sum() == 0
    lyap.update_safe_set()
    oracle.update_safe_set()
    assert 0 < oracle.safe_set.sum() < grid.nindex
    assert np.array_equal(lyap.safe_set, oracle.safe_set)
    np.testing.assert_allclose(lyap.feed_dict[lyap.c_max], oracle.c_max, rtol=1e-13)


# ---------------------------------------------------------------- 8. compute_trajectory
def test_compute_trajectory_reference_test():
    """tests/test_utilities.py:94-113 of the reference."""
    A = np.array([[1., 0.1], [0., 1.]])
    B = np.array([[0.01], [0.1]])
    dynamics = sl.LinearSystem((A, B))
    K, _ = sl.utilities.dlqr(A, B, np.diag([1., 0.01]), np.array([[0.01]]))
    policy = sl.LinearSystem([-K])
    x0 = np.array([[0.1, 0.]])
    states, actions = sl.compute_trajectory(dynamics, policy, x0, num_steps=20)
    np.testing.assert_allclose(states[[0], :], x0)
    np.testing.assert_allclose(states[-1, :], np.array([0., 0.]), atol=0.01)
    np.testing.assert_allclose(actions, states[:-1].dot(-K.T))


@pytest.mark.parametrize("num_steps", [1, 2, 33, 100])
def test_compute_trajectory_fused_equals_host_loop(num_steps):
    par, dynamics, policy = _pendulum()
    pm = dynamics.to_mean_function()
    x0 = np.array([0.3, -0.2])
    states, actions = sl.compute_trajectory(pm, policy, x0, num_steps)
    h_states, h_actions = sl.compute_trajectory(lambda x, u: pm(x, u), _Wrap(policy), x0, num_steps)
    assert states.shape == (num_steps, 2) and actions.shape == (num_steps - 1, 1)
    assert np.array_equal(states, h_states) and np.array_equal(actions, h_actions)
    if num_steps > 1:
        assert np.array_equal(states[1], pm(states[:1], policy(states[:1]))[0])


class _Wrap(object):
    def __init__(self, fun):
        self.fun, self.output_dim = fun, fun.output_dim

    def __call__(self, *a):
        return self.fun(*a)


# ---------------------------------------------------------------- 9. data and bad states
def test_rollout_after_add_data_point_equals_a_fresh_model():
    """A PosteriorMean made before add_data_point rolls out the updated model: its rollouts equal those
    of one made afterwards, and differ from the rollouts before the update."""
    par, dynamics, policy = _pendulum(M=40)
    pm = dynamics.to_mean_function()
    cl = sl.ClosedLoop(pm, policy)
    x = np.random.default_rng(0).uniform(-1, 1, (300, 2))
    before = sl.compute_roa(x, cl, 30, 0.1, no_traj=False)[1]
    v0 = pm.version
    dynamics.add_data_point(np.array([[0.1, -0.2, 0.05]]), np.array([[0.09, -0.21]]))
    assert pm.version != v0
    after = sl.compute_roa(x, cl, 30, 0.1, no_traj=False)[1]
    fresh = sl.ClosedLoop(dynamics.to_mean_function(), policy)
    assert np.array_equal(after, sl.compute_roa(x, fresh, 30, 0.1, no_traj=False)[1])
    assert not np.array_equal(before, after)


def test_non_finite_starts_give_nan_trajectories():
    par, dynamics, policy = _pendulum()
    cl = sl.ClosedLoop(dynamics.to_mean_function(), policy)
    x = np.array([[np.nan, 0.1], [0.2, np.inf], [-np.inf, 0.], [0.01, 0.02]])
    roa, traj = sl.compute_roa(x, cl, 40, 0.5, no_traj=False)
    assert np.all(np.isnan(traj[:3, :, 1:]))
    assert not roa[:3].any()
    assert np.all(np.isfinite(traj[3]))


# ---------------------------------------------------------------- 3. the reference
GOLDEN = os.path.join(HERE, "golden", "gp_mean.npz")
TOL_MARGIN = 1e-6          # flags are compared where |reference end distance - tol| > TOL_MARGIN * tol
FIXTURE_KEYS = ("X", "Y", "variances", "lengthscales", "noise_variance", "beta", "scale", "prior_rows", "K",
                "limits")


def _golden_model(g, tag):
    """The product's model and policy from the fixture's parameters (the same samples and hypers)."""
    par = {k: g[tag + "_" + k] for k in FIXTURE_KEYS}
    par["variances"] = [float(v) for v in par["variances"]]
    par["lengthscales"] = [list(map(float, ls)) for ls in par["lengthscales"]]
    for k in ("noise_variance", "beta", "scale"):
        par[k] = float(par[k])
    par["num_points"] = [2, 2]                       # the builder's grid, unused here
    _, dynamics = W._build(sl, par, "product")
    policy = sl.Saturation(sl.LinearSystem(-par["K"]), -1., 1.)
    return par, dynamics, policy


@pytest.mark.parametrize("tag", ["s1", "s2"])
def test_against_the_reference(tag, capsys):
    """tests/golden/make_golden_gp_mean.py: the unmodified reference's compute_roa / reward_rollout on
    GaussianProcess(...).to_mean_function() (scale 1 and 2, linear prior mean).  One-step means within the
    one-step bound (the gamma form's, plus the full posterior's twice: once for the reference's own fp64
    evaluation of the a . alpha form, plus the rounding of gamma itself); end states, trajectories and
    sums within 1e-9 relative (many steps: the one-step bound does not carry over); flags equal at every
    start outside the margin, and no start inside it; the stop step equal."""
    g = np.load(GOLDEN)
    par, dynamics, policy = _golden_model(g, tag)
    pm = dynamics.to_mean_function()
    pts = g[tag + "_points"]
    got = pm(pts)
    bound = GM.reference(GM.staged_tables(dynamics), pts)[1].astype(np.float64)
    full = GR.reference(GR.stack_tables(dynamics), pts)["mean_bound"]
    tol1 = bound + 2 * full + GM.gamma_gap_bound(GM.staged_tables(dynamics), pts)
    assert np.all(np.abs(got - g[tag + "_mean"]) <= tol1)
    cl = sl.ClosedLoop(pm, policy)
    rw = sl.ClosedLoop(sl.QuadraticFunction(g["reward"]), policy)
    starts = {"grid": sl.GridWorld(par["limits"], g[tag + "_grid_num_points"]),
              "states": g[tag + "_states"], "inner": g[tag + "_inner"]}
    inside = 0
    for name, start in starts.items():
        for horizon in (40, 120):
            key = "%s_%s_h%d" % (tag, name, horizon)
            tol = float(g[key + "_tol"])
            roa, traj = sl.compute_roa(start, cl, horizon, tol, no_traj=False)
            end_ref = g[key + "_end"]
            np.testing.assert_allclose(traj[:, :, -1], end_ref, rtol=1e-9, atol=1e-12)
            np.testing.assert_allclose(traj[g[key + "_traj_index"]], g[key + "_traj"], rtol=1e-9, atol=1e-12)
            dist = np.linalg.norm(end_ref, 2, axis=1)
            clear = np.abs(dist - tol) > TOL_MARGIN * tol
            inside += int((~clear).sum())
            assert np.array_equal(roa[clear], g[key + "_roa"][clear])
        for horizon in (60, 400):
            key = "%s_%s_r%d" % (tag, name, horizon)
            sums = sl.reward_rollout(start, cl, rw, float(g[key + "_discount"]), horizon, float(g[key + "_tol"]))
            np.testing.assert_allclose(sums, g[key + "_sums"], rtol=1e-9, atol=1e-12)
            stop = int(g[key + "_stop"])
            out = capsys.readouterr().out
            assert ("after {} steps".format(stop + 1) in out) if stop >= 0 else ("did not converge" in out)
    print("starts within the margin of tol: %d" % inside)
    assert inside == 0
