"""GPU tests of exact policy evaluation (``PolicyIteration.optimize_value_function``,
``csrc/value_opt.cu``) against the numpy restatement (``tests/value_opt_oracle.py``), scipy's
``spsolve``, the fixture's LP values and one ``value_iteration`` sweep.

The operator parity tests compare with the restatement of the LIBRARY's simplex lookup
(``lookup="library"``).  It differs from the reference's ``parameter_derivative`` (Qhull's walk) only
on the repaired grid-line rows and where both pick different simplices that contain the point (a tie
on a shared face); ``tests/test_value_opt_host.py`` pins both against the reference fixture."""
import os
import subprocess
import sys

import numpy as np
import pytest
import scipy.sparse as sp
import scipy.sparse.linalg as spla

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
sys.path.insert(0, HERE)

import oracle as O  # noqa: E402
import value_opt_oracle as V  # noqa: E402

pytestmark = pytest.mark.gpu
EPS = np.finfo(np.float64).eps
A = np.array([[1., .05], [-.2, .97]])
B = np.array([[0.], [.05]])
K = np.array([[.8, 1.1]])
REWARD = np.diag([-1., -1., -0.1])
GOLDEN = os.path.join(HERE, "golden", "value_optimization.npz")


@pytest.fixture(scope="module")
def sl():
    import safe_learning_b200 as mod
    return mod


def _lqr(ns, num_points, project=True, gamma=0.98, v0=None):
    grid = ns.GridWorld([[-1., 1.], [-1., 1.]], list(num_points))
    v0 = np.zeros((grid.nindex, 1)) if v0 is None else v0
    value = ns.Triangulation(grid, v0, project=project)
    policy = ns.Saturation(ns.LinearSystem((-K,)), -1., 1.)
    return ns.PolicyIteration(policy, ns.LinearSystem((A, B)), ns.QuadraticFunction(REWARD), value,
                              gamma=gamma), grid


def _oracle_operator(num_points, project=True):
    rl, grid = _lqr(O, num_points, project)
    states = grid.all_points
    actions = rl.policy(states)
    nxt = rl.dynamics(states, actions)
    rewards = rl.reward_function(states, actions).ravel()
    cols, w, q6 = V.operator(rl.value_function, nxt, lookup="library")
    return cols, w, rewards, q6, nxt


def _device_operator(sl, rl, n, d):
    """The fused assembly of `rl` on the device: (cols, weights, rewards, stats) on the host."""
    import torch
    from safe_learning_b200 import _device as dev, _native as nat
    lib = nat.load()
    cols = dev.empty((n, d + 1), torch.int32)
    w = dev.empty((n, d + 1))
    r = dev.empty((n,))
    stats = dev.zeros((nat.VALUE_STATS,), torch.int64)
    nat.check(lib.slb_value_operator(dev.stream(), rl.bellman_descriptor(), 0, n, cols.data_ptr(),
                                     w.data_ptr(), r.data_ptr(), stats.data_ptr()), "operator")
    return cols.cpu().numpy(), w.cpu().numpy(), r.cpu().numpy(), stats.cpu().numpy()


@pytest.mark.parametrize("num_points", [(24, 20), (25, 21)])
def test_operator_bit_parity(sl, num_points):
    rl, grid = _lqr(sl, num_points)
    cols, w, r, stats = _device_operator(sl, rl, grid.nindex, 2)
    oc, ow, orew, q6, _ = _oracle_operator(num_points)
    assert np.array_equal(cols, oc)
    assert np.array_equal(w, ow)
    assert np.array_equal(r, orew)
    assert stats[2] == q6.sum() == (9 if num_points == (25, 21) else 0)


def test_one_iteration_is_one_value_iteration_sweep(sl):
    rng = np.random.default_rng(1)
    v0 = -rng.random((24 * 20, 1))
    rl, grid = _lqr(sl, (24, 20), v0=v0)
    values, info = rl._evaluate_policy(1e-10, 1)
    assert info["iterations"] == 1
    rl.value_iteration()
    assert np.array_equal(values, rl.value_function.parameters[0])


@pytest.mark.parametrize("num_points", [(24, 20), (25, 21), (512, 512)])
def test_solve_equals_restated_iteration_and_spsolve(sl, num_points):
    """Values and iteration count bit for bit; within the certified bound of spsolve; the one-CTA
    tier below 12288 vertices, the cooperative tier for the 512^2 grid (C3)."""
    rl, grid = _lqr(sl, num_points)
    got = rl.optimize_value_function()
    info = rl.last_solve
    assert info["tier"] == (2 if grid.nindex > 12288 else 1)
    cols, w, rewards, q6, _ = _oracle_operator(num_points)
    v, iters, _, bound = V.solve(cols, w, rewards, 0.98, np.zeros(grid.nindex))
    assert info["iterations"] == iters
    assert info["repaired_rows"] == q6.sum()
    assert np.array_equal(got.ravel(), v)
    assert np.array_equal(rl.value_function.parameters[0].ravel(), v)
    n = grid.nindex
    T = sp.csr_matrix((w.ravel(), (np.repeat(np.arange(n), 3), cols.ravel())), shape=(n, n))
    exact = spla.spsolve((sp.identity(n) - 0.98 * T).tocsc(), rewards)
    assert np.max(np.abs(got.ravel() - exact)) <= info["bound"] + 10 * EPS * np.max(np.abs(exact)) / 0.02
    if num_points == (24, 20):
        lp = np.load(GOLDEN)["lqr24_values"].ravel()
        assert np.max(np.abs(got.ravel() - lp)) <= 1e-8 * np.max(np.abs(lp))


def test_warm_start(sl):
    rl, grid = _lqr(sl, (25, 21))
    first = rl.optimize_value_function(solver="SCS", verbose=False)
    n1 = rl.last_solve["iterations"]
    second = rl.optimize_value_function()
    n2 = rl.last_solve["iterations"]
    assert n2 < n1 / 5
    assert np.max(np.abs(first - second)) <= 2 * rl.last_solve["bound"] + 1e-9


def test_errors(sl):
    from safe_learning_b200 import OptimizationError
    # next states leaving the unprojected grid: the rows extrapolate
    rl, _ = _lqr(sl, (9, 7), project=False)
    rl.dynamics = sl.LinearSystem((2.0 * A, B))
    with pytest.raises(OptimizationError, match="unbounded"):
        rl.optimize_value_function()
    rl, _ = _lqr(sl, (9, 7), gamma=1.0)
    with pytest.raises(OptimizationError, match="contraction"):
        rl.optimize_value_function()
    rl, grid = _lqr(sl, (9, 7))
    rl.reward_function = lambda x, u: np.where(x[:, :1] > 0.5, np.nan, 0.0)
    with pytest.raises(OptimizationError, match="NaN"):
        rl.optimize_value_function()
    v0 = np.zeros((63, 1))
    v0[10] = np.nan                      # a NaN start value is named, not iterated on max_iters times
    rl, _ = _lqr(sl, (9, 7), v0=v0)
    with pytest.raises(OptimizationError, match="NaN"):
        rl.optimize_value_function()
    assert rl.last_solve["iterations"] == 0
    rl, _ = _lqr(sl, (9, 7))
    with pytest.raises(OptimizationError, match="iterations"):
        rl.optimize_value_function(max_iters=3)
    rl, grid = _lqr(sl, (9, 7))
    rl.value_function = 2.0 * rl.value_function
    with pytest.raises(TypeError):
        rl.optimize_value_function()


def test_composed_path_with_numpy_callables(sl):
    """Plain callables (mountain-car style): next states and rewards from the host, the operator
    and the solve on the device, bit for bit against the restatement on the same next states."""
    grid = sl.GridWorld([[-1.2, 0.6], [-0.07, 0.07]], [20, 20])
    value = sl.Triangulation(grid, np.zeros((grid.nindex, 1)), project=True)

    def policy(x):
        return np.where(x[:, 1:2] >= 0, 1.0, -1.0)

    def dynamics(x, u):
        v = np.clip(x[:, 1] + 0.001 * u[:, 0] - 0.0025 * np.cos(3 * x[:, 0]), -0.07, 0.07)
        p = np.clip(x[:, 0] + v, -1.2, 0.6)
        return np.stack((p, np.where(p <= -1.2, 0.0, v)), axis=1)

    def reward(x, u):
        return np.where(x[:, :1] >= 0.5, 0.0, -1.0)

    rl = sl.PolicyIteration(policy, dynamics, reward, value, gamma=0.99)
    got = rl.optimize_value_function()
    ov = O.Triangulation(O.GridWorld(grid.limits, [20, 20]), np.zeros(grid.nindex), project=True)
    states = grid.all_points
    nxt = dynamics(states, policy(states))
    cols, w, _ = V.operator(ov, nxt, lookup="library")
    v, iters, _, _ = V.solve(cols, w, reward(states, None).ravel(), 0.99, np.zeros(grid.nindex))
    assert rl.last_solve["iterations"] == iters
    assert np.array_equal(got.ravel(), v)


def test_one_dimensional_policy_iteration_loop(sl):
    """The 1d_example loop (cell 15): optimize_value_function, then discrete_policy_optimization,
    three rounds, against the restatement + the oracle's greedy step."""
    limits, n = [[-1., 1.]], 51
    actions = np.linspace(-0.5, 0.5, 11)[:, None]
    dyn = np.array([[1.0, 0.1]])
    rew = np.diag([-1.0, -0.2])
    rl_g = sl.PolicyIteration(sl.Triangulation(sl.GridWorld(limits, n), np.zeros((n, 1))),
                              sl.LinearSystem((dyn,)), sl.QuadraticFunction(rew),
                              sl.Triangulation(sl.GridWorld(limits, n), np.zeros((n, 1)), project=True))
    grid_c = O.GridWorld(limits, n)
    rl_c = O.PolicyIteration(O.Triangulation(grid_c, np.zeros((n, 1))), O.LinearSystem((dyn,)),
                             O.QuadraticFunction(rew), O.Triangulation(grid_c, np.zeros((n, 1)), project=True))
    for _ in range(3):
        got = rl_g.optimize_value_function()
        states = grid_c.all_points
        u = rl_c.policy(states)
        cols, w, _ = V.operator(rl_c.value_function, rl_c.dynamics(states, u), lookup="library")
        v, _, _, _ = V.solve(cols, w, rl_c.reward_function(states, u).ravel(), rl_c.gamma,
                             rl_c.value_function.parameters.ravel())
        assert np.array_equal(got.ravel(), v)
        rl_c.value_function.parameters = v
        best_g = rl_g.discrete_policy_optimization(actions)
        best_c = rl_c.discrete_policy_optimization(actions)
        assert np.array_equal(best_g.cpu().numpy(), best_c)


# ---------------------------------------------------------------- GP-mean dynamics
def _tp_agree(cols_a, w_a, cols_b, w_b, n, rtol=1e-8):
    """T_a p == T_b p within rtol (relative to max |T p|) for seeded random vertex vectors p."""
    Ta = sp.csr_matrix((w_a.ravel(), (np.repeat(np.arange(n), cols_a.shape[1]), cols_a.ravel())),
                       shape=(n, n))
    Tb = sp.csr_matrix((w_b.ravel(), (np.repeat(np.arange(n), cols_b.shape[1]), cols_b.ravel())),
                       shape=(n, n))
    rng = np.random.default_rng(5)
    for _ in range(4):
        p = rng.standard_normal(n)
        a, b = Ta @ p, Tb @ p
        assert np.max(np.abs(a - b)) <= rtol * np.max(np.abs(b))


def test_gp55_operator_and_solve(sl):
    """Notebook-kernel GP pendulum (55 x 55, Linear + Matern32 x Linear): the fused GP-mean
    assembly's T p and rewards against the oracle's, and the solve against the reference's LP."""
    rl, grid = V.gp55_objects(sl, "product")
    n = grid.nindex
    cols, w, r, stats = _device_operator(sl, rl, n, 2)
    rl_c, _ = V.gp55_objects(O, "oracle")
    _, ocols, ow, orew = V.evaluate(rl_c)
    _tp_agree(cols, w, ocols, ow, n)
    assert np.array_equal(r, orew)                          # reward: policy + quadratic, exact
    got = rl.optimize_value_function().ravel()
    assert rl.last_solve["tier"] == 1
    lp = np.load(GOLDEN)["gp55_values"].ravel()
    assert np.max(np.abs(got - lp)) <= 1e-8 * np.max(np.abs(lp))


def test_gp1d_policy_iteration_loop(sl):
    """1d_example cell 15 with a GP model (Matern32 x Linear, 10 data points, 51 vertices):
    optimize_value_function -> discrete_policy_optimization, three rounds, against the values and
    greedy policies the unmodified reference produced."""
    z = np.load(GOLDEN)
    rl, grid = V.gp1d_objects(sl, z, "product")
    rl_c, _ = V.gp1d_objects(O, z, "oracle")
    _, ocols, ow, _ = V.evaluate(rl_c)
    cols, w, _, _ = _device_operator(sl, rl, grid.nindex, 1)
    _tp_agree(cols, w, ocols, ow, grid.nindex)
    for k in range(3):
        got = rl.optimize_value_function().ravel()
        ref = z["gp1d_values"][k].ravel()
        assert np.max(np.abs(got - ref)) <= 1e-8 * max(1.0, np.max(np.abs(ref)))
        best = rl.discrete_policy_optimization(V.GP1D_ACTIONS)
        assert np.array_equal(best.cpu().numpy().reshape(-1, 1), z["gp1d_policies"][k].reshape(-1, 1))


def test_ranks_hold_identical_tables():
    """torch.distributed: every rank solves the whole system (no collective); the tables are
    identical on all ranks (needs 2 GPUs)."""
    import torch
    if torch.cuda.device_count() < 2:
        pytest.skip("needs 2 GPUs")
    import __graft_entry__
    __graft_entry__.build()
    cmd = [sys.executable, "-m", "torch.distributed.run", "--nnodes=1", "--nproc-per-node", "2",
           "--master-addr", "127.0.0.1", "--master-port", "29631",
           os.path.join(ROOT, "tests", "_dist_value_opt_worker.py")]
    proc = subprocess.run(cmd, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True,
                          timeout=900)
    assert proc.returncode == 0, proc.stdout[-4000:]
    assert "value_opt dist worker ok" in proc.stdout
