"""GPU tests of ``PiecewiseConstant`` (``SLB_FN_PIECEWISE_CONSTANT``): evaluation, VJP and
``parameter_derivative`` against the reference-generated fixture and the numpy restatement; the table as V,
policy and closed-loop policy of the fused sweeps and rollouts against the composed path / host loop; and
tabular dynamic programming (value iteration, greedy policy, exact policy evaluation) against the numpy
oracle."""
import os
import sys

import numpy as np
import pytest
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
sys.path.insert(0, os.path.dirname(HERE))

import bench_workloads as W  # noqa: E402
import piecewise_constant_oracle as P  # noqa: E402

pytestmark = pytest.mark.gpu

GOLDEN = np.load(os.path.join(HERE, "golden", "piecewise_constant.npz"))
GRIDS = ("g1", "g2", "g2m", "g3")
GROUPS = ("inside", "vertices", "ties", "outside", "inf")


@pytest.fixture(scope="module")
def sl():
    import safe_learning_b200 as sl
    from safe_learning_b200 import _native
    _native.require_device()
    return sl


def _grid(tag):
    return GOLDEN[tag + "_limits"], GOLDEN[tag + "_num"]


def _pwc(sl, tag, ncol):
    limits, num = _grid(tag)
    return sl.PiecewiseConstant(sl.GridWorld(limits, num), GOLDEN["%s_c%d_table" % (tag, ncol)])


# ---------------------------------------------------------------- evaluation
@pytest.mark.parametrize("tag", GRIDS)
@pytest.mark.parametrize("ncol", [1, 2])
def test_evaluation_matches_reference(sl, tag, ncol):
    pwc = _pwc(sl, tag, ncol)
    for group in GROUPS:
        k = "%s_c%d_%s" % (tag, ncol, group)
        got = pwc(GOLDEN[k + "_points"])
        assert np.array_equal(got, GOLDEN[k + "_values"]), (k, np.flatnonzero((got != GOLDEN[k + "_values"]).any(1)))


def test_nan_rows_and_post_ops(sl):
    pwc = _pwc(sl, "g3", 2)
    limits, num = _grid("g3")
    table = GOLDEN["g3_c2_table"]
    pts = np.concatenate([GOLDEN["g3_c2_inside_points"], GOLDEN["g3_c2_ties_points"][:50]])
    pts[::7, 1] = np.nan
    want = P.evaluate(limits, num, table, pts)
    assert np.isnan(want[::7]).all()
    assert np.array_equal(pwc(pts), want, equal_nan=True)
    # the post-ops apply as for every kind: Saturation and MaxAbs take fmin / fmax, which (like np.fmin /
    # np.fmax) return the other operand of a NaN
    cases = ((sl.Saturation(pwc, -0.5, 0.25), np.fmin(np.fmax(want, -0.5), 0.25)),
             (-pwc, -want),
             (2.5 * pwc, want * 2.5),
             (abs(pwc), np.abs(want)),
             (sl.Norm1Function(pwc), np.abs(want[:, :1]) + np.abs(want[:, 1:])),
             (sl.MaxAbsFunction(pwc), np.fmax(np.abs(want[:, :1]), np.abs(want[:, 1:]))))
    for fn, ref in cases:
        assert np.array_equal(fn(pts), ref, equal_nan=True), type(fn).__name__
    with pytest.raises(sl.DimensionError):
        pwc(np.zeros((3, 2)))


def test_parameter_derivative_matches_reference(sl):
    for tag in GRIDS:
        pwc = _pwc(sl, tag, 1)
        for group in GROUPS:
            k = "%s_c1_%s" % (tag, group)
            m = pwc.parameter_derivative(GOLDEN[k + "_points"])
            assert np.array_equal(m.row, GOLDEN[k + "_pd_row"]) and np.array_equal(m.col, GOLDEN[k + "_pd_col"])
            assert np.array_equal(m.data, GOLDEN[k + "_pd_data"]) and m.shape == (len(m.row), pwc.nindex)
    g = GOLDEN
    pwc = sl.PiecewiseConstant(sl.GridWorld([[-1, 1], [-1, 1]], 3), g["t_eval_values"])
    np.testing.assert_allclose(pwc.parameter_derivative(g["t_eval_points"]).toarray().dot(g["t_eval_values"]),
                               g["t_eval_constraint"])
    with pytest.raises(ValueError):
        pwc.parameter_derivative(np.array([[0.0, np.nan]]))


# ---------------------------------------------------------------- VJP
@pytest.mark.parametrize("case", ["random", "one_vertex", "nan"])
def test_vjp_is_np_add_at(sl, case):
    tag, ncol = "g2m", 2
    limits, num = _grid(tag)
    rng = np.random.default_rng(5)
    pts = np.concatenate([GOLDEN["%s_c2_%s_points" % (tag, g)] for g in GROUPS])
    if case == "one_vertex":
        pts = np.tile([[10.0, 10.0]], (3000, 1))          # every point clips to the last vertex
    if case == "nan":
        pts = pts.copy()
        pts[::5, 0] = np.nan
    gout = rng.standard_normal((len(pts), ncol))
    want = P.table_vjp(limits, num, pts, gout, ncol)
    pwc = _pwc(sl, tag, ncol)
    leaf = pwc.vertex_values
    grads = []
    for _ in range(2):
        x = torch.tensor(pts, device=leaf.device, requires_grad=True)
        y = pwc.torch(x)
        y.backward(torch.tensor(gout, device=leaf.device))
        grads.append(leaf.grad.cpu().numpy().copy())
        assert not x.grad.abs().sum().item()
        leaf.grad = None
    assert np.array_equal(grads[0], want) and np.array_equal(grads[1], want)


def test_sgd_step_on_vertex_values(sl):
    limits, num = _grid("g2")
    pwc = _pwc(sl, "g2", 1)
    table = GOLDEN["g2_c1_table"].copy()
    pts = GOLDEN["g2_c1_inside_points"]
    target = np.sin(pts[:, :1])
    leaf = pwc.vertex_values
    for _ in range(3):
        leaf.grad = None
        x = torch.tensor(pts, device=leaf.device)
        loss = ((pwc.torch(x) - torch.tensor(target, device=x.device)) ** 2).sum()
        loss.backward()
        with torch.no_grad():                 # p <- p - lr g, one rounding per operation as in numpy
            leaf -= 0.1 * leaf.grad
        res = P.evaluate(limits, num, table, pts) - target
        table = table - 0.1 * P.table_vjp(limits, num, pts, 2.0 * res, 1)
    assert np.array_equal(pwc.parameters, table)
    assert np.array_equal(pwc(pts), P.evaluate(limits, num, table, pts))


# ---------------------------------------------------------------- sweeps and rollouts
def _pendulum(sl, par, deterministic, table_v, table_policy):
    grid = sl.GridWorld(par["limits"], par["num_points"])
    if deterministic:
        pl = par["plant"]
        dyn = sl.InvertedPendulum(normalization=[pl["state_norm"], pl["action_norm"]], **pl["true"])
    else:
        _, dyn = W._build(sl, par, "product")
    vgrid = sl.GridWorld(par["limits"], [33, 29])
    pts = vgrid.all_points
    vtab = np.sum(pts.dot(par["P"]) * pts, axis=1, keepdims=True)
    ptab = np.clip(pts.dot(-par["K"].T), -1, 1)
    fused = {"V": sl.PiecewiseConstant(vgrid, vtab) if table_v else sl.QuadraticFunction(par["P"]),
             "pi": sl.PiecewiseConstant(vgrid, ptab) if table_policy else sl.Saturation(
                 sl.LinearSystem(-par["K"]), -1., 1.)}
    composed = dict(fused)
    if table_v:
        composed["V"] = lambda x: P.evaluate(vgrid.limits, vgrid.num_points, vtab, x)
    if table_policy:
        composed["pi"] = lambda x: P.evaluate(vgrid.limits, vgrid.num_points, ptab, x)
    out = []
    for fns in (fused, composed):
        out.append(sl.Lyapunov(grid, fns["V"], dyn, par["L_dyn"], 2.0, par["tau"], fns["pi"],
                               initial_set=par["initial"]))
    return out


@pytest.mark.parametrize("deterministic", [True, False])
@pytest.mark.parametrize("which", ["V", "policy"])
def test_update_safe_set_fused_equals_composed(sl, deterministic, which):
    par = W.make_pendulum(num_points=96, M=64, tau_scale=1.0 / 16)
    fused, composed = _pendulum(sl, par, deterministic, which == "V", which == "policy")
    assert composed._is_composed() and not fused._is_composed()
    fused.update_safe_set()
    composed.update_safe_set()
    assert np.array_equal(fused.values, composed.values)
    assert np.array_equal(fused.safe_set, composed.safe_set)
    assert fused.feed_dict[fused.c_max] == composed.feed_dict[composed.c_max]


def test_rollouts_with_a_table_policy(sl):
    """The fused rollouts against the host loop of the same closed loop with the restatement as the
    policy (a Python callable, so ClosedLoop steps on the host)."""
    par = W.make_pendulum(num_points=8, M=16)
    pl = par["plant"]
    plant = sl.InvertedPendulum(normalization=[pl["state_norm"], pl["action_norm"]], **pl["true"])
    vgrid = sl.GridWorld(par["limits"], [41, 41])
    ptab = np.clip(vgrid.all_points.dot(-par["K"].T), -1, 1)
    table = sl.PiecewiseConstant(vgrid, ptab)
    host_policy = lambda x: P.evaluate(vgrid.limits, vgrid.num_points, ptab, x)  # noqa: E731
    fused, host = sl.ClosedLoop(plant, table), sl.ClosedLoop(plant, host_policy)
    assert fused.fused and not host.fused
    grid = sl.GridWorld(par["limits"], [31, 31])
    roa_f, traj_f = sl.compute_roa(grid, fused, horizon=60, tol=0.05, no_traj=False)
    roa_h, traj_h = sl.compute_roa(grid, host, horizon=60, tol=0.05, no_traj=False)
    assert np.array_equal(traj_f, traj_h, equal_nan=True) and np.array_equal(roa_f, roa_h)
    assert 0 < roa_f.sum() < roa_f.size
    reward = sl.QuadraticFunction(-np.eye(3))
    sums_f = sl.reward_rollout(grid, fused, sl.ClosedLoop(reward, table), 0.9, horizon=40, tol=0.0)
    sums_h = sl.reward_rollout(grid, host, sl.ClosedLoop(reward, host_policy), 0.9, horizon=40, tol=0.0)
    assert np.array_equal(sums_f, sums_h)


# ---------------------------------------------------------------- tabular dynamic programming
def _tabular(sl, n=(40, 36), gp=False, seed=0, v0=None, policy0=None):
    par = W.make_pendulum(num_points=8, M=100)
    grid = sl.GridWorld(par["limits"], list(n))
    if gp:
        _, dyn = W._build(sl, par, "product")
    else:
        pl = par["plant"]
        dyn = sl.InvertedPendulum(normalization=[pl["state_norm"], pl["action_norm"]], **pl["true"])
    reward = sl.QuadraticFunction(-np.diag([1., 2., 1.2]))
    rng = np.random.default_rng(seed)
    v0 = -np.sum(grid.all_points ** 2, axis=1, keepdims=True) - 0.01 * rng.random((grid.nindex, 1)) \
        if v0 is None else v0
    value = sl.PiecewiseConstant(grid, v0)
    policy = sl.PiecewiseConstant(grid, np.zeros((grid.nindex, 1)) if policy0 is None else policy0)
    return sl.PolicyIteration(policy, dyn, reward, value, gamma=0.9), grid, dyn, reward


def _states(grid):
    """The grid points as the kernels form them (ijk * unit_maxes + offset)."""
    return grid.index_to_state(np.arange(grid.nindex))


def _transitions(grid, dyn, reward, actions):
    x = _states(grid)
    out = []
    for a in actions:
        u = np.broadcast_to(a, (len(x), len(a))).copy()
        nxt = dyn(x, u)
        nxt = nxt[0] if isinstance(nxt, tuple) else nxt
        out.append((nxt, reward(x, u)[:, 0]))
    return out


def test_value_iteration_equals_the_oracle(sl):
    rl, grid, dyn, reward = _tabular(sl)
    policy_tab = np.clip(np.random.default_rng(1).standard_normal((grid.nindex, 1)), -1, 1)
    rl.policy.parameters = policy_tab
    x = _states(grid)
    nxt = dyn(x, policy_tab)
    rew = reward(x, policy_tab)[:, 0]
    v = rl.value_function.parameters[:, 0].copy()
    for _ in range(5):
        delta = rl.value_iteration()
        want = P.bellman_sweep(grid.limits, grid.num_points, v, nxt, rew, rl.gamma)
        assert np.array_equal(rl.value_function.parameters[:, 0], want)
        assert delta == np.max(np.abs(want - v))
        v = want
    # -V (the table stores the un-scaled values)
    rl.value_function = -rl.value_function
    rl.value_iteration()
    want = -P.bellman_sweep(grid.limits, grid.num_points, -v, nxt, rew, rl.gamma)
    assert np.array_equal(rl.value_function.fun.parameters[:, 0], want)


def test_value_iteration_nan_next_states(sl):
    rl, grid, dyn, reward = _tabular(sl)
    rl.policy.parameters = np.where(np.arange(grid.nindex)[:, None] % 11 == 0, np.nan, 0.3)
    v = rl.value_function.parameters[:, 0].copy()
    rl.value_iteration()
    x = _states(grid)
    u = rl.policy.parameters
    want = P.bellman_sweep(grid.limits, grid.num_points, v, dyn(x, u), reward(x, u)[:, 0], rl.gamma)
    got = rl.value_function.parameters[:, 0]
    assert np.isnan(got[::11]).all()
    assert np.array_equal(got, want, equal_nan=True)


@pytest.mark.parametrize("gp", [False, True])
def test_discrete_policy_optimization_equals_the_oracle(sl, gp):
    rl, grid, dyn, reward = _tabular(sl, gp=gp)
    actions = np.linspace(-1, 1, 21)[:, None]
    v = rl.value_function.parameters[:, 0]
    trans = _transitions(grid, dyn, reward, actions)
    best, q = P.greedy(grid.limits, grid.num_points, v, [t[0] for t in trans], [t[1] for t in trans], rl.gamma)
    results = {}
    for factored in (True, False):
        rl.factor_actions = factored
        rl.discrete_policy_optimization(actions)
        results[factored] = rl.policy.parameters[:, 0].copy()
        assert isinstance(rl.policy.parameters, np.ndarray) and rl.policy.parameters.shape == (grid.nindex, 1)
    if not gp:
        assert np.array_equal(results[True], actions[best, 0])
        assert np.array_equal(results[False], actions[best, 0])
        return
    # GP: the Bellman kernels' means round differently from slb_gp_predict's, and a next state within
    # rounding of a half-cell boundary looks up the neighbouring vertex; both paths agree with each other
    # and with the oracle everywhere else
    assert np.mean(results[True] == results[False]) > 0.99
    for got in results.values():
        assert np.mean(got == actions[best, 0]) > 0.97


def test_greedy_ties_take_the_first_action(sl):
    """Constant V and an action-independent reward: every action ties, np.argmax takes the first."""
    rl, grid, dyn, reward = _tabular(sl, v0=np.ones((40 * 36, 1)))
    rl.reward_function = sl.QuadraticFunction(-np.diag([1., 2., 0.]))
    actions = np.array([[0.5], [-0.25], [0.75]])
    rl.discrete_policy_optimization(actions)
    assert np.all(rl.policy.parameters == 0.5)


def test_policy_must_share_the_value_grid(sl):
    rl, grid, dyn, reward = _tabular(sl)
    rl.policy = sl.PiecewiseConstant(sl.GridWorld(grid.limits, [10, 10]), np.zeros((100, 1)))
    with pytest.raises(NotImplementedError):
        rl.discrete_policy_optimization(np.array([[0.0], [1.0]]))


@pytest.mark.parametrize("gp", [False, True])
def test_optimize_value_function_within_its_bound(sl, gp):
    rl, grid, dyn, reward = _tabular(sl, gp=gp, n=(30, 30))
    policy_tab = np.clip(_states(grid).dot(np.array([[-0.6], [-0.3]])), -1, 1)
    rl.policy.parameters = policy_tab
    got = rl.optimize_value_function()
    x = _states(grid)
    nxt = dyn(x, policy_tab)
    nxt = nxt[0] if isinstance(nxt, tuple) else nxt
    exact = P.evaluate_policy(grid.limits, grid.num_points, nxt, reward(x, policy_tab)[:, 0], rl.gamma)
    info = rl.last_solve
    # one-hot rows, stored as (vertex, 1) and (vertex, 0): rho = 1, smallest weight 0
    assert info["rho"] == 1.0 and info["min_weight"] == 0.0 and info["repaired_rows"] == 0
    if gp:       # a next state within rounding of a half-cell boundary may pick the other vertex
        assert np.mean(np.abs(got[:, 0] - exact) <= info["bound"] * 1.01 + 1e-12) > 0.99
    else:
        assert np.max(np.abs(got[:, 0] - exact)) <= info["bound"] * 1.01 + 1e-12
    assert np.array_equal(rl.value_function.parameters, got)
    # a NaN next state is reported, not iterated on
    rl.policy.parameters = np.where(np.arange(grid.nindex)[:, None] == 7, np.nan, policy_tab)
    with pytest.raises(sl.OptimizationError, match="NaN"):
        rl.optimize_value_function()


def test_future_values_torch_reaches_the_table(sl):
    rl, grid, dyn, reward = _tabular(sl)
    x = torch.tensor(grid.all_points[::17], device="cuda")
    leaf = rl.value_function.vertex_values
    out = rl.future_values(x, actions=torch.zeros((1, 1), device="cuda", dtype=torch.float64))
    want = rl.future_values(grid.all_points[::17], actions=np.zeros((1, 1)))
    assert np.array_equal(out.detach().cpu().numpy(), want)
    out.sum().backward()
    nxt = dyn(grid.all_points[::17], np.zeros((len(x), 1)))
    g = P.table_vjp(grid.limits, grid.num_points, nxt, np.full((len(x), 1), rl.gamma), 1)
    assert np.array_equal(leaf.grad.cpu().numpy(), g)
